"""Ed25519 on the H100: the device arithmetic (sbv_debug_ed25519) against Python integers, the production SHA-512 kernel
against hashlib, and sbv_ed25519_verify_batch bit-exact against the OpenSSL oracle on seeded corpora with every
corruption class — large batches, empty and 10 KiB messages, pinned and pageable input, concurrent callers, the ECDSA
path around the first Ed25519 call, the fault convention and a two-device engine."""
import ctypes as C
import threading

import numpy as np
import pytest

import ed25519_cases as cases
import oracle
import oracle_ed25519 as oe
from oracle import corpus as ecorpus
from oracle_ed25519 import corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _runner(eng):
    def run(op, inp):
        inp = np.ascontiguousarray(inp, np.uint32)
        out = np.zeros_like(inp)
        rc = eng._lib.sbv_debug_ed25519(eng._h, C.c_int(op), C.c_size_t(inp.shape[0]), _p(inp), _p(out))
        assert rc == 0
        return out
    return run


def test_field_ops(eng):
    assert cases.check_field(_runner(eng), np.random.default_rng(1)) > 400


def test_sqrt_ratio(eng):
    cases.check_sqrt_ratio(_runner(eng), np.random.default_rng(2))


def test_decode_every_edge_key(eng):
    cases.check_decode(_runner(eng), np.random.default_rng(3))


def test_reduce_mod_L(eng):
    cases.check_reduce(_runner(eng), np.random.default_rng(4))


def test_sha512_of_R_A_M(eng):
    msgs, off, sig, pub = cases.ragged_batch(np.random.default_rng(5))
    n = off.size - 1
    dig = np.zeros((n, 64), np.uint8)
    k = np.zeros((n, 8), np.uint32)
    rc = eng._lib.sbv_debug_ed25519_sha512(eng._h, C.c_size_t(n), _p(msgs), _p(off), _p(sig), _p(pub), _p(dig), _p(k))
    assert rc == 0
    want = cases.expected_digests(msgs, off, sig, pub)
    for i in range(n):
        assert bytes(dig[i]) == want[i], i
        assert sum(int(k[i, w]) << (32 * w) for w in range(8)) == int.from_bytes(want[i], "little") % cases.L


def _check(eng, c):
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    got = eng.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]
    return want


def test_corpus_65536_every_class(eng):
    c = corpus.make_corpus(65536, seed=21, n_keys=1024)
    want = _check(eng, c)
    for k, name in enumerate(corpus.CLASS_NAMES):
        m = c["cls"] == k
        assert m.sum() > 0, name
    for k in (corpus.SMALL_ORDER, corpus.MIXED_ORDER, corpus.R_NONCANON):
        m = c["cls"] == k
        assert 0 < want[m].sum() < m.sum(), corpus.CLASS_NAMES[k]


def test_corpus_262144(eng):
    _check(eng, corpus.make_corpus(262144, seed=22, n_keys=4096))


def test_empty_and_10k_messages_pageable_and_pinned(eng):
    import consensus_b200 as sbv
    for fixed in (0, 10240):
        c = corpus.make_corpus(3000, seed=23 + fixed, fixed_len=fixed, crafted_max=32)
        want = _check(eng, c)
        if fixed == 0:  # every message empty: msgs may be NULL
            got = np.zeros_like(want)
            eng.ed25519_verify_batch_ptr(want.size, 0, c["off"].ctypes.data, c["sig"].ctypes.data, c["pub"].ctypes.data, got.ctypes.data)
            assert np.array_equal(got, want)
        lib = sbv.load_library()
        lib.sbv_host_alloc.restype = C.c_void_p
        bufs = []

        def pinned(a):
            a = np.ascontiguousarray(a)
            ptr = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
            assert ptr
            bufs.append(ptr)
            view = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(ptr))
            view[:] = a.view(np.uint8).reshape(-1)
            return ptr
        try:
            m, o, s, pb, ok = (pinned(c["msgs"]), pinned(c["off"]), pinned(c["sig"]), pinned(c["pub"]),
                               pinned(np.zeros(want.size, np.uint8)))
            eng.ed25519_verify_batch_ptr(want.size, m, o, s, pb, ok)
            got = np.ctypeslib.as_array((C.c_uint8 * want.size).from_address(ok)).copy()
            assert np.array_equal(got, want)
        finally:
            for ptr in bufs:
                lib.sbv_host_free(C.c_void_p(ptr))


def test_six_threads_at_once(eng):
    cs = [corpus.make_corpus(8192, seed=40 + t, crafted_max=32) for t in range(6)]
    wants = [oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]) for c in cs]
    gots, errs = [None] * 6, []

    def work(t):
        try:
            c = cs[t]
            for _ in range(3):
                gots[t] = eng.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=work, args=(t,)) for t in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for g, w in zip(gots, wants):
        assert np.array_equal(g, w)


def test_ecdsa_before_and_after_the_first_ed25519_call():
    import consensus_b200 as sbv
    b = ecorpus.make_batch(oracle.P256, n=4096, K=64, seed=9, corrupt_rate=4)
    want = oracle.verify_batch(oracle.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    c = corpus.make_corpus(2048, seed=24, crafted_max=32)
    with sbv.Engine(devices=[0]) as e:
        before = e.verify_batch(sbv.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
        _check(e, c)
        after = e.verify_batch(sbv.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert np.array_equal(before, want) and np.array_equal(after, want)


def test_fault_convention(eng):
    c = corpus.make_corpus(64, seed=25, crafted_max=4)
    n = 64
    msgs, off, sig, pub = c["msgs"], c["off"], c["sig"], c["pub"]
    lib, h = eng._lib, eng._h
    ok = np.full(n, 7, np.uint8)

    def call(nn, m, o, s, pb):
        return lib.sbv_ed25519_verify_batch(h, C.c_size_t(nn), m, o, s, pb, _p(ok))
    assert call(n, None, _p(off), _p(sig), _p(pub)) < 0      # messages present, msgs NULL
    assert call(n, _p(msgs), None, _p(sig), _p(pub)) < 0
    assert call(n, _p(msgs), _p(off), None, _p(pub)) < 0
    assert call(n, _p(msgs), _p(off), _p(sig), None) < 0
    assert lib.sbv_ed25519_verify_batch(h, C.c_size_t(n), _p(msgs), _p(off), _p(sig), _p(pub), None) < 0
    bad = off.copy()
    bad[10], bad[11] = bad[11], bad[10]
    assert call(n, _p(msgs), _p(bad), _p(sig), _p(pub)) < 0  # non-monotonic offsets
    assert call(2**31, _p(msgs), _p(off), _p(sig), _p(pub)) < 0
    assert (ok == 7).all()
    assert b"" != lib.sbv_last_error(h)
    # the engine still works afterwards
    _check(eng, c)


def test_two_devices():
    import torch
    import consensus_b200 as sbv
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    c = corpus.make_corpus(20000, seed=26, crafted_max=64)
    with sbv.Engine(devices=[0, 1]) as e:
        _check(e, c)
