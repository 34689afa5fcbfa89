"""SHA-384 on the device for ECDSA: sbv_sha384_batch, sbv_hash384_verify_batch and sbv_hash384_verify_registered (the CPU
twin of the kernel is test_hostsim_sha384.py).

The corpus is signed over SHA-384 digests with the OpenSSL oracle's signer.  Every valid item has rejecting twins (a
flipped message byte, r or s = 0 and = n, a key off the curve), and some items are signed over SHA-256 and must reject.
Verdicts must equal, byte for byte, the OpenSSL oracle on SHA-384(M) and the digest calls (sbv_verify_batch /
sbv_verify_registered with the 48-byte digests); returned digests must equal hashlib.  Crafted-digest cases such as
R.x >= n cannot be reached through a hash: the digest calls, which share the verify kernels, cover them.  Settings read at
sbv_create (SBV_GROUP_THRESHOLD, SBV_CHUNK_ITEMS) get an engine of their own."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import oracle
from oracle import corpus
from oracle.ecdsa_ref import CURVES

pytestmark = pytest.mark.gpu

P256, P384, ED25519 = 0, 1, 2
FB = {P256: 32, P384: 48}
P8, P32, P64 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
TWINS = 7  # per valid item: itself, flipped message byte, r = 0, s = 0, r = n, s = n, key off the curve


def _engine(**env):
    import consensus_b200 as sbv
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return sbv.Engine(n_devices=1)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _sha384(msgs, off):
    n = off.size - 1
    return np.frombuffer(b"".join(hashlib.sha384(msgs[int(off[i]):int(off[i + 1])].tobytes()).digest() for i in range(n)),
                         np.uint8).reshape(n, 48).copy()


def _sha256(msgs, off):
    n = off.size - 1
    return np.frombuffer(b"".join(hashlib.sha256(msgs[int(off[i]):int(off[i + 1])].tobytes()).digest() for i in range(n)),
                         np.uint8).reshape(n, 32).copy()


def make_corpus(curve, n_valid, K, seed, sha256_every=9):
    """n_valid signed items, each followed by its TWINS - 1 rejecting twins; every `sha256_every`-th valid item is signed over
    SHA-256 instead (so it and its twins reject).  Returns a dict with msgs, off, r, s, qx, qy, key_idx and the signing keys."""
    L, nn = FB[curve], CURVES[curve].n
    d, kxy = corpus.make_keys(curve, K, seed=seed)
    msgs, off = corpus.make_requests(n_valid, seed=seed + 1, fixed_len=None, lo=1, hi=700)
    key_idx = (np.arange(n_valid) * 7 % K).astype(np.uint32)
    k = corpus._blocks(seed + 2, n_valid, L, b"k")
    r, s = oracle.sign_batch(curve, d, key_idx, _sha384(msgs, off), k)
    old = np.arange(0, n_valid, sha256_every)
    r[old], s[old] = oracle.sign_batch(curve, d, key_idx[old], _sha256(msgs, off)[old], k[old])
    n = n_valid * TWINS
    src = np.repeat(np.arange(n_valid), TWINS)
    kind = np.tile(np.arange(TWINS), n_valid)
    lens = np.diff(off.astype(np.int64))[src]
    o = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    m = np.concatenate([msgs[int(off[i]):int(off[i + 1])] for i in src])
    R, S, KI = r[src].copy(), s[src].copy(), key_idx[src].copy()
    QX, QY = kxy[KI, :L].copy(), kxy[KI, L:].copy()
    rng = np.random.default_rng(seed + 3)
    for j in np.nonzero(kind == 1)[0]:
        m[int(o[j]) + int(rng.integers(lens[j]))] ^= 1 << int(rng.integers(8))
    nb = nn.to_bytes(L, "big")
    R[kind == 2] = 0
    S[kind == 3] = 0
    R[kind == 4] = np.frombuffer(nb, np.uint8)
    S[kind == 5] = np.frombuffer(nb, np.uint8)
    QY[kind == 6, L - 1] ^= 1
    return dict(curve=curve, n=n, msgs=m, off=o, r=R, s=S, qx=QX, qy=QY, key_idx=KI, kind=kind, src=src, old=np.isin(src, old), kxy=kxy, K=K)


def check_batch(e, c):
    """hash384_verify_batch against the oracle, the digest call and hashlib; returns the verdicts."""
    curve = c["curve"]
    dig = _sha384(c["msgs"], c["off"])
    want = oracle.verify_batch(curve, c["r"], c["s"], c["qx"], c["qy"], dig)
    got, gdig = e.hash384_verify_batch(curve, c["msgs"], c["off"], c["r"], c["s"], c["qx"], c["qy"], want_digest=True)
    assert np.array_equal(gdig, dig)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (bad[:10], c["kind"][bad[:10]])
    assert np.array_equal(got, e.verify_batch(curve, c["r"], c["s"], c["qx"], c["qy"], dig))
    # the corpus is what it claims to be: exactly the SHA-384-signed originals accept
    assert np.array_equal(want.astype(bool), (c["kind"] == 0) & ~c["old"])
    assert np.array_equal(e.hash384_verify_batch(curve, c["msgs"], c["off"], c["r"], c["s"], c["qx"], c["qy"]), got)
    return got


# ------------------------------------------------------------------------------------------------ sbv_sha384_batch
def test_sha384_batch_ragged_with_empty_messages(eng):
    lens = [0, 3, 0, 111, 112, 127, 128, 129, 0, 239, 240, 1000, 0] + list(range(0, 300, 13))
    rng = np.random.default_rng(1)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    assert np.array_equal(eng.sha384_batch(msgs, off), _sha384(msgs, off))
    assert bytes(eng.sha384_batch(msgs, off)[0]).hex() == hashlib.sha384(b"").hexdigest()
    # caller offsets starting past 0: the bytes before off[0] are not hashed
    lead = 1_000_003
    buf = np.concatenate([rng.integers(0, 256, lead, dtype=np.uint8), msgs])
    assert np.array_equal(eng.sha384_batch(buf, off + np.uint64(lead)), _sha384(msgs, off))


def test_sha384_batch_length_sorted_and_null_msgs(eng):
    """Above 2,048 items the launch sorts by block count first; msgs = NULL is allowed when every message is empty."""
    msgs, off = corpus.make_requests(5000, seed=3, fixed_len=None, lo=1, hi=2000)
    assert np.array_equal(eng.sha384_batch(msgs, off), _sha384(msgs, off))
    n = 40
    off0 = np.full(n + 1, 77, np.uint64)
    out = np.zeros((n, 48), np.uint8)
    assert eng._lib.sbv_sha384_batch(eng._h, C.c_size_t(n), None, off0.ctypes.data_as(P64), out.ctypes.data_as(P8)) == 0
    assert all(bytes(d) == hashlib.sha384(b"").digest() for d in out)


def test_pinned_and_pageable_buffers(eng):
    """The same call with every buffer pinned (sbv_host_alloc) and every buffer pageable."""
    c = make_corpus(P384, 120, 5, seed=31)
    want = oracle.verify_batch(P384, c["r"], c["s"], c["qx"], c["qy"], _sha384(c["msgs"], c["off"]))
    lib = eng._lib
    lib.sbv_host_alloc.restype = C.c_void_p
    n = c["n"]
    arrays = [c["msgs"], c["off"], c["r"], c["s"], c["qx"], c["qy"], np.zeros(48 * n, np.uint8), np.zeros(n, np.uint8)]
    ptrs, views = [], []
    try:
        for a in arrays:
            p = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
            assert p
            ptrs.append(p)
            v = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(p))
            v[:] = a.view(np.uint8).reshape(-1)
            views.append(v)
        eng.hash384_verify_batch_ptr(P384, n, *ptrs)
        assert np.array_equal(views[7], want)
        assert np.array_equal(views[6].reshape(n, 48), _sha384(c["msgs"], c["off"]))
        dig = np.zeros(48 * n, np.uint8)
        ok = np.zeros(n, np.uint8)
        eng.hash384_verify_batch_ptr(P384, n, *(a.ctypes.data for a in arrays[:6]), dig.ctypes.data, ok.ctypes.data)
        assert np.array_equal(ok, want) and np.array_equal(dig.reshape(n, 48), views[6].reshape(n, 48))
        out = np.ctypeslib.as_array((C.c_uint8 * (48 * n)).from_address(ptrs[6]))
        out[:] = 0
        assert lib.sbv_sha384_batch(eng._h, C.c_size_t(n), C.c_void_p(ptrs[0]), C.c_void_p(ptrs[1]), C.c_void_p(ptrs[6])) == 0
        assert np.array_equal(out.reshape(n, 48), _sha384(c["msgs"], c["off"]))
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


# ------------------------------------------------------------------------------------------------ keys per item
@pytest.mark.parametrize("curve", [P384, P256])
@pytest.mark.parametrize("grouped", [True, False])
def test_hash384_verify_batch(curve, grouped):
    """Grouped: 6 keys over about 2,100 items, each far above SBV_GROUP_THRESHOLD.  Generic: grouping off."""
    e = _engine() if grouped else _engine(SBV_GROUP_THRESHOLD="0")
    try:
        c = make_corpus(curve, 300, 6, seed=40 + curve)
        got = check_batch(e, c)
        assert 0 < got.sum() < c["n"]
        # small batches: a single item, and the first twins
        for lo, cnt in [(0, 1), (7, 7), (0, 64)]:
            sl = slice(lo, lo + cnt)
            o = c["off"][lo:lo + cnt + 1]
            sub = e.hash384_verify_batch(curve, c["msgs"], o, c["r"][sl], c["s"][sl], c["qx"][sl], c["qy"][sl])
            assert np.array_equal(sub, got[sl]), (lo, cnt)
    finally:
        e.close()


def test_chunked_upload_matches_unchunked(eng):
    """SBV_CHUNK_ITEMS = 256: a shard of 2,800 items arrives in 10 chunks.  The digests of every chunk must land at their
    items (48 bytes apart), so verdicts and digests equal the unchunked call's."""
    c = make_corpus(P384, 400, 8, seed=50)
    want, wdig = eng.hash384_verify_batch(P384, c["msgs"], c["off"], c["r"], c["s"], c["qx"], c["qy"], want_digest=True)
    e = _engine(SBV_CHUNK_ITEMS="256")
    try:
        got, gdig = e.hash384_verify_batch(P384, c["msgs"], c["off"], c["r"], c["s"], c["qx"], c["qy"], want_digest=True)
        assert np.array_equal(gdig, wdig)
        assert np.array_equal(got, want)
        check_batch(e, c)
        c2 = make_corpus(P256, 400, 8, seed=51)   # P-256 reads the leftmost 32 of the 48 bytes of each chunk's digests
        check_batch(e, c2)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------ registered keys
@pytest.mark.parametrize("curve", [P384, P256])
def test_hash384_verify_registered(eng, curve):
    """Against sbv_verify_registered with the 48-byte digests and against the oracle: unknown slots, slots of the other
    curve and an off-curve registered key reject.  Also the one-signature-per-warp kernel of small batches."""
    L, K = FB[curve], 6
    c = make_corpus(curve, 300, K, seed=60 + curve)
    other = corpus.make_keys(1 - curve, 1, seed=9)[1].reshape(2, FB[1 - curve])
    xy = np.zeros((K + 2, 2, 48), np.uint8)
    xy[:K, :, 48 - L:] = c["kxy"].reshape(K, 2, L)
    xy[K, :, 48 - L:] = xy[0, :, 48 - L:]
    xy[K, 1, 47] ^= 1                                   # slot K: the key of slot 0 off the curve
    xy[K + 1, :, 48 - FB[1 - curve]:] = other           # slot K + 1: a key of the other curve
    curves = np.full(K + 2, curve, np.uint8)
    curves[K + 1] = 1 - curve
    eng.set_keys(curves, xy)
    slot = c["key_idx"].copy()
    slot[c["kind"] == 6] = K                            # the off-curve twin: its registered key is off the curve too
    sel = np.arange(c["n"])
    slot[sel % 29 == 3] = K + 1
    slot[sel % 31 == 4] = K + 9
    dig = _sha384(c["msgs"], c["off"])
    want = oracle.verify_batch(curve, c["r"], c["s"], c["qx"], c["qy"], dig)
    want[np.isin(slot, [K + 1, K + 9])] = 0
    got = eng.hash384_verify_registered(curve, c["msgs"], c["off"], slot, c["r"], c["s"])
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (bad[:10], c["kind"][bad[:10]], slot[bad[:10]])
    assert np.array_equal(got, eng.verify_registered(curve, slot, c["r"], c["s"], dig))
    assert 0 < got.sum() < c["n"]
    for lo, cnt in [(0, 1), (5, 40)]:
        sl = slice(lo, lo + cnt)
        sub = eng.hash384_verify_registered(curve, c["msgs"], c["off"][lo:lo + cnt + 1], slot[sl], c["r"][sl], c["s"][sl])
        assert np.array_equal(sub, got[sl]), (lo, cnt)


# ------------------------------------------------------------------------------------------------ argument faults
FAULTS = ["decreasing", "null_off", "null_msgs", "null_out"]


@pytest.mark.parametrize("name,fault", [("sbv_sha384_batch", f) for f in FAULTS]
                         + [(c, f) for c in ("sbv_hash384_verify_batch", "sbv_hash384_verify_registered") for f in ["ed25519"] + FAULTS])
def test_argument_faults(eng, name, fault):
    """SBV_ERR_ARG before anything is written or launched: curve = SBV_ED25519 (the calls that take a curve), decreasing
    offsets, null offsets, null messages that are not all empty, a null output."""
    n = 4
    msgs = np.arange(64, dtype=np.uint8)
    off = np.array([0, 5, 9, 9, 20], np.uint64)
    if fault == "decreasing":
        off = np.array([0, 5, 3, 9, 20], np.uint64)
    field = np.ones(48 * n, np.uint8)
    slots = np.zeros(n, np.uint32)
    out = np.full(48 * n, 0x5A, np.uint8)
    ok = np.full(n, 0x5A, np.uint8)
    mp = None if fault == "null_msgs" else msgs.ctypes.data_as(P8)
    op = None if fault == "null_off" else off.ctypes.data_as(P64)
    fp = field.ctypes.data_as(P8)
    okp = None if fault == "null_out" else ok.ctypes.data_as(P8)
    curve = C.c_uint8(ED25519 if fault == "ed25519" else P384)
    args = {
        "sbv_sha384_batch": (C.c_size_t(n), mp, op, None if fault == "null_out" else out.ctypes.data_as(P8)),
        "sbv_hash384_verify_batch": (curve, C.c_size_t(n), mp, op, fp, fp, fp, fp, out.ctypes.data_as(P8), okp),
        "sbv_hash384_verify_registered": (curve, C.c_size_t(n), mp, op, slots.ctypes.data_as(P32), fp, fp, okp),
    }[name]
    before = eng.kernel_launches
    assert getattr(eng._lib, name)(eng._h, *args) == -1
    assert (ok == 0x5A).all() and (out == 0x5A).all(), "a rejected call must not write its outputs"
    assert eng.kernel_launches == before
    # the same call with n >= 2^31 is refused before msg_off[n] is read
    big = list(args)
    big[0 if name == "sbv_sha384_batch" else 1] = C.c_size_t(1 << 31)
    assert getattr(eng._lib, name)(eng._h, *big) == -1


# ------------------------------------------------------------------------------------------------ several devices
def test_multi_device_sharding():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {torch.cuda.device_count()}")
    import consensus_b200 as sbv
    c = make_corpus(P384, 300, 6, seed=70)
    with sbv.Engine(n_devices=2) as e2:
        check_batch(e2, c)
        assert np.array_equal(e2.sha384_batch(c["msgs"], c["off"]), _sha384(c["msgs"], c["off"]))
        K, L = c["K"], 48
        e2.set_keys(np.full(K, P384, np.uint8), c["kxy"].reshape(K, 2, L))
        dig = _sha384(c["msgs"], c["off"])
        got = e2.hash384_verify_registered(P384, c["msgs"], c["off"], c["key_idx"], c["r"], c["s"])
        assert np.array_equal(got, e2.verify_registered(P384, c["key_idx"], c["r"], c["s"], dig))
