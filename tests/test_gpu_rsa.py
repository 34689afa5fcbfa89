"""RSA PKCS #1 v1.5 on the device: sbv_rsa_verify_batch, sbv_rsa_hash_verify_batch and sbv_sha512_batch (the CPU twin of the
kernels is test_hostsim_rsa.py).

Every class of tests/rsa_cases.py, for every modulus size and hash, through both calls, bit-exact against oracle_rsa.ref;
the fused call item for item against the digest call on host-computed digests; digests against hashlib; pinned and
pageable buffers; six concurrent callers; every argument fault; item counts off the group and block sizes; two devices."""
import ctypes as C
import hashlib
import threading

import numpy as np
import pytest

import rsa_cases as rc
from oracle_rsa import ref

pytestmark = pytest.mark.gpu

P8, P32, P64 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    with sbv.Engine(n_devices=1) as e:
        yield e


def _hashes(c):
    return np.stack([np.frombuffer(ref.HASHLIB[c["hash"]](c["msgs"][int(c["off"][i]):int(c["off"][i + 1])].tobytes()).digest(), np.uint8)
                     for i in range(c["n"])])


@pytest.mark.parametrize("k", rc.SIZES)
@pytest.mark.parametrize("hash", rc.HASHES)
def test_every_class_both_calls(eng, k, hash):
    c = rc.make_cases(k, hash)
    got = eng.rsa_verify_batch(hash, c["digest"], c["sig"], c["mod"], c["exp"])
    bad = [(cl, int(g), int(w)) for cl, g, w in zip(c["cls"], got, c["want"]) if g != w]
    assert not bad, bad
    fused, dig = eng.rsa_hash_verify_batch(hash, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"], want_digest=True)
    assert np.array_equal(fused, got), "the fused call differs from the digest call on host-computed digests"
    assert np.array_equal(dig, _hashes(c))
    assert np.array_equal(fused, eng.rsa_hash_verify_batch(hash, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]))
    assert 0 < int(c["want"].sum()) < c["n"]


def _tiled(c, n):
    """n items cycled from the corpus c (messages included)."""
    idx = np.arange(n) % c["n"]
    parts = [c["msgs"][int(c["off"][i]):int(c["off"][i + 1])] for i in idx]
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint64)
    msgs = np.concatenate(parts) if off[-1] else np.zeros(0, np.uint8)
    return dict(k=c["k"], hash=c["hash"], n=n, msgs=msgs, off=off, digest=c["digest"][idx].copy(), sig=c["sig"][idx].copy(), mod=c["mod"][idx].copy(),
                exp=c["exp"][idx].copy(), want=c["want"][idx].copy())


@pytest.mark.parametrize("n", [1, 2, 17, 4097])
def test_item_counts_off_the_group_and_block(eng, n):
    c = _tiled(rc.make_cases(256, ref.SHA256), n)
    assert np.array_equal(eng.rsa_verify_batch(ref.SHA256, c["digest"], c["sig"], c["mod"], c["exp"]), c["want"])
    assert np.array_equal(eng.rsa_hash_verify_batch(ref.SHA256, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]), c["want"])


def test_sha512_batch_ragged_and_empty(eng):
    rng = np.random.default_rng(5)
    lens = [0, 0, 1, 111, 112, 127, 128, 129, 239, 240, 3000, 0] + list(rng.integers(0, 700, 3000))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    got = eng.sha512_batch(msgs, off)
    for i in range(len(lens)):
        assert got[i].tobytes() == hashlib.sha512(msgs[int(off[i]):int(off[i + 1])].tobytes()).digest(), i
    # every message empty: msgs may be NULL
    empty = np.zeros(5, np.uint64)
    out = np.zeros((4, 64), np.uint8)
    assert eng._lib.sbv_sha512_batch(eng._h, C.c_size_t(4), None, empty.ctypes.data_as(P64), out.ctypes.data_as(P8)) == 0
    assert all(o.tobytes() == hashlib.sha512(b"").digest() for o in out)


def test_pinned_and_pageable_buffers(eng):
    c = rc.make_cases(384, ref.SHA384)
    lib = eng._lib
    lib.sbv_host_alloc.restype = C.c_void_p
    n, k = c["n"], c["k"]
    arrays = [c["msgs"], c["off"], c["sig"], c["mod"], c["exp"], np.zeros(48 * n, np.uint8), np.zeros(n, np.uint8), c["digest"]]
    ptrs = []
    try:
        views = []
        for a in arrays:
            p = lib.sbv_host_alloc(C.c_size_t(max(a.nbytes, 1)))
            assert p
            ptrs.append(p)
            v = np.ctypeslib.as_array((C.c_uint8 * max(a.nbytes, 1)).from_address(p))
            v[:a.nbytes] = a.view(np.uint8).reshape(-1)
            views.append(v)
        eng.rsa_hash_verify_batch_ptr(k, ref.SHA384, n, *ptrs[:7])
        assert np.array_equal(views[6], c["want"])
        assert np.array_equal(views[5].reshape(n, 48), c["digest"])
        views[6][:] = 7
        eng.rsa_verify_batch_ptr(k, ref.SHA384, n, ptrs[7], ptrs[2], ptrs[3], ptrs[4], ptrs[6])
        assert np.array_equal(views[6], c["want"])
        ok = np.zeros(n, np.uint8)
        eng.rsa_verify_batch_ptr(k, ref.SHA384, n, c["digest"].ctypes.data, c["sig"].ctypes.data, c["mod"].ctypes.data, c["exp"].ctypes.data,
                                 ok.ctypes.data)
        assert np.array_equal(ok, c["want"])
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_six_concurrent_callers(eng):
    cases = [_tiled(rc.make_cases(k, h), 600) for k, h in [(256, 0), (384, 1), (512, 2), (256, 2), (384, 0), (512, 1)]]
    serial = [eng.rsa_hash_verify_batch(c["hash"], c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]) for c in cases]
    got, errs = [None] * 6, []

    def run(i):
        try:
            c = cases[i]
            for _ in range(3):
                got[i] = eng.rsa_hash_verify_batch(c["hash"], c["msgs"], c["off"], c["sig"], c["mod"], c["exp"])
                assert np.array_equal(got[i], serial[i])
                assert np.array_equal(eng.rsa_verify_batch(c["hash"], c["digest"], c["sig"], c["mod"], c["exp"]), serial[i])
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(6)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    for c, s in zip(cases, serial):
        assert np.array_equal(s, c["want"])


FAULTS = ["mod_bytes", "hash", "null_sig", "null_mod", "null_exp", "null_ok", "null_digest", "decreasing", "null_off", "null_msgs"]


@pytest.mark.parametrize("name,fault", [("sbv_rsa_verify_batch", f) for f in FAULTS[:7]]
                         + [("sbv_rsa_hash_verify_batch", f) for f in FAULTS if f != "null_digest"]
                         + [("sbv_sha512_batch", f) for f in ("decreasing", "null_off", "null_msgs", "null_ok")])
def test_argument_faults(eng, name, fault):
    """SBV_ERR_ARG before anything is written or launched, with ok (and the digests) untouched; then the same call with
    n >= 2^31."""
    n, k = 4, 256
    msgs = np.arange(64, dtype=np.uint8)
    off = np.array([0, 5, 3, 9, 20] if fault == "decreasing" else [0, 5, 9, 9, 20], np.uint64)
    sig, mod, dig = np.ones(k * n, np.uint8), np.full(k * n, 0xff, np.uint8), np.ones(64 * n, np.uint8)
    exp = np.full(n, 65537, np.uint32)
    ok, out = np.full(n, 0x5A, np.uint8), np.full(64 * n, 0x5A, np.uint8)
    nul = lambda f, a, t=P8: None if fault == f else a.ctypes.data_as(t)  # noqa: E731
    mb = C.c_uint32(300 if fault == "mod_bytes" else k)
    hs = C.c_uint8(3 if fault == "hash" else 0)
    args = {
        "sbv_rsa_verify_batch": (mb, hs, C.c_size_t(n), nul("null_digest", dig), nul("null_sig", sig), nul("null_mod", mod), nul("null_exp", exp, P32),
                                 nul("null_ok", ok)),
        "sbv_rsa_hash_verify_batch": (mb, hs, C.c_size_t(n), nul("null_msgs", msgs), nul("null_off", off, P64), nul("null_sig", sig), nul("null_mod", mod),
                                      nul("null_exp", exp, P32), out.ctypes.data_as(P8), nul("null_ok", ok)),
        "sbv_sha512_batch": (C.c_size_t(n), nul("null_msgs", msgs), nul("null_off", off, P64), None if fault == "null_ok" else out.ctypes.data_as(P8)),
    }[name]
    before = eng.kernel_launches
    assert getattr(eng._lib, name)(eng._h, *args) == -1
    assert (ok == 0x5A).all() and (out == 0x5A).all(), "a rejected call must not write its outputs"
    assert eng.kernel_launches == before
    big = list(args)
    big[0 if name == "sbv_sha512_batch" else 2] = C.c_size_t(1 << 31)
    assert getattr(eng._lib, name)(eng._h, *big) == -1
    assert (ok == 0x5A).all() and eng.kernel_launches == before


@pytest.mark.parametrize("name", ["sbv_rsa_verify_batch", "sbv_rsa_hash_verify_batch", "sbv_sha512_batch"])
def test_n_of_2_pow_31_with_valid_buffers(eng, name):
    """n = 2^31 is refused on its own: every other argument valid and non-null.  The buffers hold one item; the call must
    not read past them, write anything or launch."""
    k = 256
    msgs = np.arange(64, dtype=np.uint8)
    off = np.array([0, 5], np.uint64)
    sig, mod, dig = np.ones(k, np.uint8), np.full(k, 0xff, np.uint8), np.ones(64, np.uint8)
    exp = np.full(1, 65537, np.uint32)
    ok, out = np.full(1, 0x5A, np.uint8), np.full(64, 0x5A, np.uint8)
    n = C.c_size_t(1 << 31)
    p8 = lambda a: a.ctypes.data_as(P8)  # noqa: E731
    args = {
        "sbv_rsa_verify_batch": (C.c_uint32(k), C.c_uint8(0), n, p8(dig), p8(sig), p8(mod), exp.ctypes.data_as(P32), p8(ok)),
        "sbv_rsa_hash_verify_batch": (C.c_uint32(k), C.c_uint8(0), n, p8(msgs), off.ctypes.data_as(P64), p8(sig), p8(mod), exp.ctypes.data_as(P32),
                                      p8(out), p8(ok)),
        "sbv_sha512_batch": (n, p8(msgs), off.ctypes.data_as(P64), p8(out)),
    }[name]
    before = eng.kernel_launches
    assert getattr(eng._lib, name)(eng._h, *args) == -1
    assert ok[0] == 0x5A and (out == 0x5A).all() and eng.kernel_launches == before


def test_every_mod_bytes_and_hash_is_refused_outside_the_set(eng):
    for mb in (0, 128, 255, 257, 1024):
        ok = np.full(1, 0x5A, np.uint8)
        z = np.zeros(1024, np.uint8)
        e = np.full(1, 65537, np.uint32)
        assert eng._lib.sbv_rsa_verify_batch(eng._h, C.c_uint32(mb), C.c_uint8(0), C.c_size_t(1), z.ctypes.data_as(P8), z.ctypes.data_as(P8),
                                             z.ctypes.data_as(P8), e.ctypes.data_as(P32), ok.ctypes.data_as(P8)) == -1
        assert ok[0] == 0x5A


def test_multi_device_sharding():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {torch.cuda.device_count()}")
    import consensus_b200 as sbv
    c = _tiled(rc.make_cases(256, ref.SHA256), 301)
    with sbv.Engine(n_devices=2) as e2:
        assert np.array_equal(e2.rsa_verify_batch(0, c["digest"], c["sig"], c["mod"], c["exp"]), c["want"])
        ok, dig = e2.rsa_hash_verify_batch(0, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"], want_digest=True)
        assert np.array_equal(ok, c["want"]) and np.array_equal(dig, c["digest"])
        d512 = e2.sha512_batch(c["msgs"], c["off"])
        assert all(d512[i].tobytes() == hashlib.sha512(c["msgs"][int(c["off"][i]):int(c["off"][i + 1])].tobytes()).digest() for i in range(301))
