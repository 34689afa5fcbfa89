"""Registered Ed25519 keys on the H100: sbv_ed25519_set_keys / sbv_ed25519_verify_registered bit-exact against OpenSSL
and sbv_ed25519_verify_batch on corpora with every class, the registry's semantics, the device's per-key tables against
the model (sbv_debug_ed25519_ktab), the edge sets of tests/ed25519_registered.py (crafted k through
sbv_debug_ed25519_verify_registered_k), batch shapes, pinned and pageable input, concurrent callers, the fault convention
and a two-device engine.  tests/test_hostsim_ed25519_registered.py runs the same sets on the CPU simulation."""
import ctypes as C
import threading

import numpy as np
import pytest

import ed25519_edges as edges
import ed25519_registered as reg
import oracle
import oracle_ed25519 as oe
from oracle import corpus as ecorpus
from oracle_ed25519 import corpus, ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _verify(eng):
    def run(a, slot):
        return eng.ed25519_verify_registered(a["msgs"], a["off"], slot, a["sig"])
    return run


def _verify_k(eng):
    def run(a, slot):
        n = a["off"].size - 1
        slot = np.ascontiguousarray(slot, np.uint32)
        ok = np.full(n, 7, np.uint8)
        assert eng._lib.sbv_debug_ed25519_verify_registered_k(eng._h, C.c_size_t(n), _p(slot), _p(a["sig"]), _p(a["k"]), _p(ok)) == 0
        return ok
    return run


def _ktab(eng, slot, first=0, count=32 * 128):
    out = np.zeros((count, 24), np.uint32)
    rc = eng._lib.sbv_debug_ed25519_ktab(eng._h, C.c_uint32(slot), C.c_size_t(first), C.c_size_t(count), _p(out))
    return out if rc == 0 else None


def _check(eng, c):
    pub, slot = reg.corpus_registry(c)
    eng.ed25519_set_keys(pub)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    got = eng.ed25519_verify_registered(c["msgs"], c["off"], slot, c["sig"])
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]
    per_item = eng.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(per_item, want)
    return want


def test_corpus_65536_every_class(eng):
    c = reg.merge(corpus.make_corpus(65536, seed=21, n_keys=1024), reg.class_rows())
    want = _check(eng, c)
    cls = np.array([reg.key_class(bytes(A)) for A in c["pub"]])
    for name in ("y>=p", "-0", "small order", "mixed order"):
        assert 0 < want[cls == name].sum() < (cls == name).sum(), name
    assert (cls == "off-curve").any() and not want[cls == "off-curve"].any()
    for k in (corpus.SMALL_ORDER, corpus.MIXED_ORDER, corpus.R_NONCANON):
        m = c["cls"] == k
        assert 0 < want[m].sum() < m.sum(), corpus.CLASS_NAMES[k]


def test_corpus_262144_4096_keys(eng):
    c = reg.merge(corpus.make_corpus(262144, seed=22, n_keys=4096), reg.class_rows())
    _check(eng, c)
    assert reg.corpus_registry(c)[0].shape[0] > 4096


def test_table_of_the_encoding_of_B_is_the_table_of_B(eng):
    eng.ed25519_set_keys(np.frombuffer(ref.encode(ref.B), np.uint8))
    b = np.zeros((32 * 128, 24), np.uint32)
    assert eng._lib.sbv_debug_ed25519_btab(eng._h, C.c_size_t(0), C.c_size_t(32 * 128), _p(b)) == 0
    assert np.array_equal(_ktab(eng, 0), b)


def test_every_entry_of_every_kind_of_key(eng):
    keys = reg.table_keys()
    bad = corpus.off_curve_encodings(np.random.default_rng(5), 1)[0]
    eng.ed25519_set_keys(np.frombuffer(b"".join(keys[:2] + [bad] + keys[2:]), np.uint8))
    for slot, A in zip((0, 1, 3, 4), keys):
        assert np.array_equal(_ktab(eng, slot).reshape(32, 128, 24), reg.ktab_words(A)), reg.key_class(A)
    assert np.array_equal(_ktab(eng, 4, 17 * 128 + 99, 5), reg.ktab_words(keys[3])[17, 99:104])
    assert _ktab(eng, 2) is None and _ktab(eng, 5) is None and _ktab(eng, 0, 4095, 2) is None


def test_unknown_slots_reject_in_the_kernel(eng):
    """Rows that accept under slot 0's key with their k reject by slot n and 2^32 - 1, and in an empty registry: the
    kernel's own slot check, with no gather involved."""
    A0, rows = reg.slot0_rows()
    a, n = rows.arrays(), len(rows)
    others = reg.table_keys()[1:]
    eng.ed25519_set_keys(np.frombuffer(b"".join([A0] + others), np.uint8))
    verify_k = _verify_k(eng)
    assert verify_k(a, np.zeros(n, np.uint32)).all()
    for bad in (len(others) + 1, 2**32 - 1):
        assert not verify_k(a, np.full(n, bad, np.uint32)).any(), bad
    eng.ed25519_set_keys(np.zeros(0, np.uint8))
    assert not verify_k(a, np.zeros(n, np.uint32)).any()


def test_S_boundary(eng):
    acc, n = reg.check(edges.s_boundary(), eng.ed25519_set_keys, verify=_verify(eng), seed=1)
    assert 0 < acc < n


def test_every_B_loop_digit(eng):
    acc, n = reg.check(edges.digit_sweep(), eng.ed25519_set_keys, verify=_verify(eng), seed=2)
    assert acc == 7954


def test_small_order_R(eng):
    acc, n = reg.check(edges.small_order_r(), eng.ed25519_set_keys, verify=_verify(eng), seed=3)
    assert 0 < acc < n


def test_every_key_loop_digit(eng):
    acc, n = reg.check(reg.k_sweep(), eng.ed25519_set_keys, verify_k=_verify_k(eng), seed=4)
    assert acc == len(reg.k_sweep_ks())


def test_collisions(eng):
    acc, n = reg.check(reg.collisions(), eng.ed25519_set_keys, verify_k=_verify_k(eng), seed=5)
    assert 0 < acc < n


def test_verify_k_rejects_k_at_least_L(eng):
    rows = edges._subset(reg.k_sweep(), range(4))
    pub, slot = reg.registry(rows.A)
    eng.ed25519_set_keys(pub)
    a = rows.arrays()
    for bad in (edges.L, 2**256 - 1):
        a["k"][2] = np.frombuffer(bad.to_bytes(32, "little"), "<u4")
        ok = np.full(4, 7, np.uint8)
        assert eng._lib.sbv_debug_ed25519_verify_registered_k(eng._h, C.c_size_t(4), _p(slot), _p(a["sig"]), _p(a["k"]), _p(ok)) < 0
        assert (ok == 7).all()


def test_registry_semantics(eng):
    c = corpus.make_corpus(3000, seed=32, n_keys=64, crafted_max=0)
    pub, slot = reg.corpus_registry(c)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    verify = _verify(eng)
    eng.ed25519_set_keys(pub)
    for bad in (pub.shape[0], 2**32 - 1):
        s2 = slot.copy()
        s2[::3] = bad
        got = verify(c, s2)
        assert not got[::3].any() and np.array_equal(np.delete(got, np.s_[::3]), np.delete(want, np.s_[::3]))
    eng.ed25519_set_keys(np.zeros(0, np.uint8))
    assert not verify(c, slot).any()
    eng.ed25519_set_keys(np.concatenate([pub, pub]))
    assert np.array_equal(verify(c, slot + pub.shape[0]), want) and np.array_equal(verify(c, slot), want)
    new = pub[::-1].copy()
    eng.ed25519_set_keys(new)
    assert np.array_equal(verify(c, pub.shape[0] - 1 - slot), want)
    want_new = oe.verify_batch(c["msgs"], c["off"], c["sig"], new[slot])
    assert np.array_equal(verify(c, slot), want_new) and want_new.sum() < want.sum() // 2


def test_ecdsa_and_ed25519_registries_are_independent():
    import consensus_b200 as sbv
    b = ecorpus.make_batch(oracle.P256, n=4096, K=64, seed=9, corrupt_rate=4)
    ewant = oracle.verify_batch(oracle.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    qxy = np.concatenate([b["qx"].reshape(-1, 32), b["qy"].reshape(-1, 32)], axis=1)
    keys, kslot = np.unique(qxy, axis=0, return_inverse=True)
    kslot = kslot.reshape(-1).astype(np.uint32)
    c = corpus.make_corpus(4096, seed=33, n_keys=64, crafted_max=32)
    pub, slot = reg.corpus_registry(c)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    with sbv.Engine(devices=[0]) as e:
        def ecdsa():
            return e.verify_registered(sbv.P256, kslot, b["r"], b["s"], b["digest"])
        e.set_keys(np.zeros(keys.shape[0], np.uint8), keys.reshape(-1, 2, 32))
        before = ecdsa()
        e.ed25519_set_keys(pub)
        after = ecdsa()
        assert np.array_equal(e.ed25519_verify_registered(c["msgs"], c["off"], slot, c["sig"]), want)
        e.set_keys(np.zeros(keys.shape[0], np.uint8), keys.reshape(-1, 2, 32))  # ECDSA registry replaced
        assert np.array_equal(e.ed25519_verify_registered(c["msgs"], c["off"], slot, c["sig"]), want)
        e.ed25519_set_keys(np.zeros(0, np.uint8))
        assert np.array_equal(ecdsa(), ewant)
    assert np.array_equal(before, ewant) and np.array_equal(after, ewant)


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049])
def test_batch_shapes(eng, n):
    """EDK_BLOCK = 128, the gather's 256 threads (two per item), SHA-512's 128 and the length sort from 2048 items on."""
    c = corpus.make_corpus(n, seed=300 + n, n_keys=16, crafted_max=16)
    pub, slot = reg.corpus_registry(c)
    eng.ed25519_set_keys(pub)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(_verify(eng)(c, slot), want)


def test_empty_and_10k_messages_pageable_and_pinned(eng):
    import consensus_b200 as sbv
    for fixed in (0, 10240):
        c = corpus.make_corpus(3000, seed=23 + fixed, fixed_len=fixed, crafted_max=32)
        want = _check(eng, c)
        pub, slot = reg.corpus_registry(c)
        if fixed == 0:  # every message empty: msgs may be NULL
            got = np.zeros_like(want)
            eng.ed25519_verify_registered_ptr(want.size, 0, c["off"].ctypes.data, slot.ctypes.data, c["sig"].ctypes.data, got.ctypes.data)
            assert np.array_equal(got, want)
        lib = sbv.load_library()
        lib.sbv_host_alloc.restype = C.c_void_p
        bufs = []

        def pinned(a):
            a = np.ascontiguousarray(a)
            ptr = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
            assert ptr
            bufs.append(ptr)
            np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(ptr))[:] = a.view(np.uint8).reshape(-1)
            return ptr
        try:
            m, o, sl, s, ok = (pinned(c["msgs"]), pinned(c["off"]), pinned(slot), pinned(c["sig"]), pinned(np.zeros(want.size, np.uint8)))
            eng.ed25519_verify_registered_ptr(want.size, m, o, sl, s, ok)
            assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * want.size).from_address(ok)), want)
        finally:
            for ptr in bufs:
                lib.sbv_host_free(C.c_void_p(ptr))


def test_six_threads_at_once(eng):
    cs = [corpus.make_corpus(8192, seed=40 + t, n_keys=32, crafted_max=32) for t in range(6)]
    allpub = np.unique(np.concatenate([c["pub"] for c in cs]), axis=0)
    index = {bytes(A): i for i, A in enumerate(allpub)}
    slots = [np.array([index[bytes(A)] for A in c["pub"]], np.uint32) for c in cs]
    wants = [oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]) for c in cs]
    eng.ed25519_set_keys(allpub)
    gots, errs = [None] * 6, []

    def work(t):
        try:
            for _ in range(3):
                gots[t] = eng.ed25519_verify_registered(cs[t]["msgs"], cs[t]["off"], slots[t], cs[t]["sig"])
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


def test_fault_convention(eng):
    c = corpus.make_corpus(64, seed=25, crafted_max=4)
    pub, slot = reg.corpus_registry(c)
    eng.ed25519_set_keys(pub)
    n = 64
    msgs, off, sig = c["msgs"], c["off"], c["sig"]
    lib, h = eng._lib, eng._h
    ok = np.full(n, 7, np.uint8)

    def call(nn, m, o, sl, s):
        return lib.sbv_ed25519_verify_registered(h, C.c_size_t(nn), m, o, sl, s, _p(ok))
    assert call(n, None, _p(off), _p(slot), _p(sig)) < 0      # messages present, msgs NULL
    assert call(n, _p(msgs), None, _p(slot), _p(sig)) < 0
    assert call(n, _p(msgs), _p(off), None, _p(sig)) < 0
    assert call(n, _p(msgs), _p(off), _p(slot), None) < 0
    assert lib.sbv_ed25519_verify_registered(h, C.c_size_t(n), _p(msgs), _p(off), _p(slot), _p(sig), None) < 0
    bad = off.copy()
    bad[10], bad[11] = bad[11], bad[10]
    assert call(n, _p(msgs), _p(bad), _p(slot), _p(sig)) < 0  # non-monotonic offsets
    assert call(2**31, _p(msgs), _p(off), _p(slot), _p(sig)) < 0
    assert (ok == 7).all()
    assert lib.sbv_ed25519_set_keys(h, C.c_size_t(3), None) < 0
    assert lib.sbv_ed25519_set_keys(h, C.c_size_t(2**31), _p(pub)) < 0
    assert b"" != lib.sbv_last_error(h)
    # the engine and its registry still work afterwards
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(eng.ed25519_verify_registered(msgs, off, slot, sig), want)


def test_two_devices():
    import torch
    import consensus_b200 as sbv
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    c = corpus.make_corpus(20000, seed=26, crafted_max=64)
    with sbv.Engine(devices=[0, 1]) as e:
        _check(e, c)
