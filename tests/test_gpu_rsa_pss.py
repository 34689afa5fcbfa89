"""RSA-PSS on the device: sbv_rsa_pss_verify_batch and sbv_rsa_pss_hash_verify_batch (the CPU twin of the kernels is
test_hostsim_rsa_pss.py).

Every class of tests/rsa_pss_cases.py, for every modulus size and hash and every salt mode of the corpus, through both
calls, bit-exact against oracle_rsa.ref; the fused call item for item against the digest call, digests against hashlib;
a PSS signature refused by the PKCS #1 v1.5 call; item counts off the group and block sizes; pinned and pageable buffers;
six concurrent callers; every argument fault; two devices."""
import ctypes as C
import threading

import numpy as np
import pytest

import rsa_pss_cases as pc
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


@pytest.mark.parametrize("k", pc.SIZES)
@pytest.mark.parametrize("hash", pc.HASHES)
def test_every_class_every_salt_mode_both_calls(eng, k, hash):
    c = pc.make_cases(k, hash)
    dig_checked = False
    for sl in pc.salt_lens(c):
        want = pc.want(c, sl)
        got = eng.rsa_pss_verify_batch(hash, sl, c["digest"], c["sig"], c["mod"], c["exp"])
        bad = [(cl, int(g), int(w)) for cl, g, w in zip(c["cls"], got, want) if g != w]
        assert not bad, (sl, bad)
        if not dig_checked:
            fused, dig = eng.rsa_pss_hash_verify_batch(hash, sl, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"], want_digest=True)
            assert np.array_equal(dig, _hashes(c))
            dig_checked = True
        else:
            fused = eng.rsa_pss_hash_verify_batch(hash, sl, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"])
        assert np.array_equal(fused, got), ("the fused call differs from the digest call on host-computed digests", sl)
        if sl in (ref.SALT_AUTO, ref.SALT_EQUALS_HASH):
            assert 0 < int(want.sum()) < c["n"]
    # cross-padding: no PSS signature passes the PKCS #1 v1.5 call, and the v1.5 one in the corpus fails under PSS
    v15 = eng.rsa_verify_batch(hash, c["digest"], c["sig"], c["mod"], c["exp"])
    assert np.array_equal(v15, ref.verify_batch(k, hash, c["digest"], c["sig"], c["mod"], c["exp"])) and v15.sum() == 1
    assert c["cls"][int(np.flatnonzero(v15)[0])] == "cross_pkcs1"


def _tiled(c, n):
    idx = np.arange(n) % c["n"]
    parts = [c["msgs"][int(c["off"][i]):int(c["off"][i + 1])] for i in idx]
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint64)
    msgs = np.concatenate(parts) if off[-1] else np.zeros(0, np.uint8)
    return dict(k=c["k"], hash=c["hash"], n=n, msgs=msgs, off=off, digest=c["digest"][idx].copy(), sig=c["sig"][idx].copy(), mod=c["mod"][idx].copy(),
                exp=c["exp"][idx].copy(), want=pc.want(c, ref.SALT_AUTO)[idx].copy())


@pytest.mark.parametrize("n", [1, 2, 17, 4097])
def test_item_counts_off_the_group_and_block(eng, n):
    c = _tiled(pc.make_cases(256, ref.SHA256), n)
    assert np.array_equal(eng.rsa_pss_verify_batch(ref.SHA256, ref.SALT_AUTO, c["digest"], c["sig"], c["mod"], c["exp"]), c["want"])
    assert np.array_equal(eng.rsa_pss_hash_verify_batch(ref.SHA256, ref.SALT_AUTO, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]), c["want"])


def test_pinned_and_pageable_buffers(eng):
    c = pc.make_cases(384, ref.SHA384)
    want = pc.want(c, ref.SALT_EQUALS_HASH)
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
        eng.rsa_pss_hash_verify_batch_ptr(k, ref.SHA384, ref.SALT_EQUALS_HASH, n, *ptrs[:7])
        assert np.array_equal(views[6], want)
        assert np.array_equal(views[5].reshape(n, 48), c["digest"])
        assert np.array_equal(views[2], c["sig"].reshape(-1)), "the host signatures are never written"
        views[6][:] = 7
        eng.rsa_pss_verify_batch_ptr(k, ref.SHA384, ref.SALT_EQUALS_HASH, n, ptrs[7], ptrs[2], ptrs[3], ptrs[4], ptrs[6])
        assert np.array_equal(views[6], want)
        ok = np.zeros(n, np.uint8)
        eng.rsa_pss_verify_batch_ptr(k, ref.SHA384, ref.SALT_EQUALS_HASH, n, c["digest"].ctypes.data, c["sig"].ctypes.data, c["mod"].ctypes.data,
                                     c["exp"].ctypes.data, ok.ctypes.data)
        assert np.array_equal(ok, want)
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_six_concurrent_callers(eng):
    cases = [_tiled(pc.make_cases(k, h), 600) for k, h in [(256, 0), (384, 1), (512, 2), (256, 2), (384, 0), (512, 1)]]
    serial = [eng.rsa_pss_hash_verify_batch(c["hash"], ref.SALT_AUTO, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]) for c in cases]
    got, errs = [None] * 6, []

    def run(i):
        try:
            c = cases[i]
            for _ in range(3):
                got[i] = eng.rsa_pss_hash_verify_batch(c["hash"], ref.SALT_AUTO, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"])
                assert np.array_equal(got[i], serial[i])
                assert np.array_equal(eng.rsa_pss_verify_batch(c["hash"], ref.SALT_AUTO, c["digest"], c["sig"], c["mod"], c["exp"]), serial[i])
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


FAULTS = ["mod_bytes", "hash", "salt_-2", "salt_int32_min", "null_sig", "null_mod", "null_exp", "null_ok", "null_digest", "decreasing", "null_off",
          "null_msgs"]


@pytest.mark.parametrize("name,fault", [("sbv_rsa_pss_verify_batch", f) for f in FAULTS[:9]]
                         + [("sbv_rsa_pss_hash_verify_batch", f) for f in FAULTS if f != "null_digest"])
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
    sl = C.c_int32({"salt_-2": -2, "salt_int32_min": -2**31}.get(fault, 0))
    args = {
        "sbv_rsa_pss_verify_batch": (mb, hs, sl, C.c_size_t(n), nul("null_digest", dig), nul("null_sig", sig), nul("null_mod", mod),
                                     nul("null_exp", exp, P32), nul("null_ok", ok)),
        "sbv_rsa_pss_hash_verify_batch": (mb, hs, sl, C.c_size_t(n), nul("null_msgs", msgs), nul("null_off", off, P64), nul("null_sig", sig),
                                          nul("null_mod", mod), nul("null_exp", exp, P32), out.ctypes.data_as(P8), nul("null_ok", ok)),
    }[name]
    before = eng.kernel_launches
    assert getattr(eng._lib, name)(eng._h, *args) == -1
    assert (ok == 0x5A).all() and (out == 0x5A).all(), "a rejected call must not write its outputs"
    assert eng.kernel_launches == before
    big = list(args)
    big[3] = C.c_size_t(1 << 31)
    assert getattr(eng._lib, name)(eng._h, *big) == -1
    assert (ok == 0x5A).all() and eng.kernel_launches == before


def test_salt_len_at_the_int32_ends(eng):
    """salt_len = 2^31 - 1 is a valid argument that rejects every item; -1 and 0 are the two named modes."""
    c = pc.make_cases(256, ref.SHA256)
    assert not eng.rsa_pss_verify_batch(ref.SHA256, 2**31 - 1, c["digest"], c["sig"], c["mod"], c["exp"]).any()
    before = eng.kernel_launches
    eng.rsa_pss_verify_batch(ref.SHA256, ref.SALT_EQUALS_HASH, c["digest"], c["sig"], c["mod"], c["exp"])
    assert eng.kernel_launches == before + 2  # k_rsa_em and k_rsa_pss


def test_multi_device_sharding():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {torch.cuda.device_count()}")
    import consensus_b200 as sbv
    c = _tiled(pc.make_cases(256, ref.SHA256), 301)
    with sbv.Engine(n_devices=2) as e2:
        assert np.array_equal(e2.rsa_pss_verify_batch(0, ref.SALT_AUTO, c["digest"], c["sig"], c["mod"], c["exp"]), c["want"])
        ok, dig = e2.rsa_pss_hash_verify_batch(0, ref.SALT_AUTO, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"], want_digest=True)
        assert np.array_equal(ok, c["want"]) and np.array_equal(dig, c["digest"])
