"""The ECDSA per-key tables on the device, every entry against the Python models of tests/ecdsa_keys.py, and the
inputs that reach every part of them:

  - registered tables (sbv_set_keys, 8-bit windows, read back with sbv_debug_key_table) and the tables of keys grouped
    in a launch (P-256 comb, P-384 5-bit windows, read back with sbv_debug_grouped_key_table) at the key counts around
    the build kernels' block sizes and at the benchmark's shape;
  - digit sweeps: u2 that takes every reachable (window, digit) pair of each window kernel and every (block, column,
    mask) triple of the comb, on the kernel that reads it;
  - key encodings at the range edges on every path, keys that collide in the half of the words the grouping hash once
    read, and partial sums of the warp kernel's shuffle tree that are equal or opposite."""
import ctypes as C

import numpy as np
import pytest

import ecdsa_keys as ek
import oracle
from oracle import P256, P384, corpus
from oracle import ecdsa_ref as ref
from test_gpu_edges import WARP_LIMIT, _every_path, _registered
from test_gpu_round2 import _engine

pytestmark = pytest.mark.gpu

ERR_ARG = -1


@pytest.fixture(scope="module")
def engines():
    es = {"generic": _engine(SBV_GROUP_THRESHOLD=0), "grouped": _engine(SBV_GROUP_THRESHOLD=1),
          "grouped2": _engine(SBV_GROUP_THRESHOLD=2), "default": _engine(SBV_GROUP_THRESHOLD=16)}
    yield es
    for e in es.values():
        e.close()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _key_table(eng, curve, slot, first, count):
    N = ref.CURVES[curve].size // 4
    out = np.zeros((min(count, 8000) + 1) * 2 * N, np.uint32)      # a range the call must refuse gets a small buffer
    rc = eng._lib.sbv_debug_key_table(eng._h, C.c_uint8(curve), C.c_uint32(slot), C.c_size_t(first), C.c_size_t(count), _p(out))
    return rc, out[: min(count, 8000) * 2 * N]


def _grouped_tables(eng, curve, qx, qy, items):
    qx, qy = np.ascontiguousarray(qx, np.uint8), np.ascontiguousarray(qy, np.uint8)
    items = np.ascontiguousarray(items, np.uint32)
    words = 512 * 16 if curve == P256 else ek.windows(P384, 5) * 16 * 24    # CombTab<P256> / KeyTab<384, 5>: entries x 2N
    status = np.full(items.size, -1, np.int32)
    out = np.zeros((items.size, words), np.uint32)
    rc = eng._lib.sbv_debug_grouped_key_table(eng._h, C.c_uint8(curve), C.c_size_t(qx.shape[0]), _p(qx), _p(qy), C.c_size_t(items.size),
                                             _p(items), _p(status), _p(out))
    assert rc == 0
    return status, out


_MODELS = {}


def _model(curve, W, Q):
    key = (curve, W, Q)
    if key not in _MODELS:
        _MODELS[key] = ek.comb_table(Q) if W is None else ek.window_table(curve, W, Q)
    return _MODELS[key]


def _assert_table(got, want, what):
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{what}: {bad.size} words differ, first words {bad[:8].tolist()}"


# ---------------------------------------------------------------- registered tables
def _registry_keys(curve):
    c = ref.CURVES[curve]
    G = (c.gx, c.gy)
    return [("G", G), ("-G", (c.gx, c.p - c.gy)), ("2G", ref._add(c, G, G)), ("random", ek._point(curve, 0x5EED + 77 * curve)),
            ("small x", ek.small_x_point(curve)), ("small y", ek.small_y_point(curve))]


@pytest.mark.parametrize("curve", [P256, P384])
def test_every_entry_of_registered_tables(engines, curve):
    """Every entry of the 8-bit window tables of G, -G, 2G, a random key and the keys with a small coordinate equals the
    model; partial reads return their slice; a slot past the registry, a key without a table (off the curve, x >= p),
    a key of the other curve and a range outside the table return SBV_ERR_ARG."""
    eng = engines["generic"]
    c = ref.CURVES[curve]
    L = c.size
    keys = _registry_keys(curve)
    other = ek._point(1 - curve, 12345)
    xy = np.zeros((len(keys) + 3, 2, 48), np.uint8)
    for i, (_, Q) in enumerate(keys):
        xy[i, 0, 48 - L:], xy[i, 1, 48 - L:] = ek._be(Q[0], L), ek._be(Q[1], L)
    off, big, oth = len(keys), len(keys) + 1, len(keys) + 2
    xy[off] = xy[3]
    xy[off, 1, 47] ^= 1                                                      # off the curve
    xy[big, 0, 48 - L:], xy[big, 1, 48 - L:] = ek._be(keys[4][1][0] + c.p, L), ek._be(keys[4][1][1], L)   # x + p
    Lo = ref.CURVES[1 - curve].size
    xy[oth, 0, 48 - Lo:], xy[oth, 1, 48 - Lo:] = ek._be(other[0], Lo), ek._be(other[1], Lo)
    curves = np.array([curve] * (len(keys) + 2) + [1 - curve], np.uint8)
    eng.set_keys(curves, xy.reshape(-1, 96))
    entries = ek.windows(curve, 8) * 128
    for slot, (label, Q) in enumerate(keys):
        rc, got = _key_table(eng, curve, slot, 0, entries)
        assert rc == 0, label
        _assert_table(got, _model(curve, 8, Q), label)
        want = _model(curve, 8, Q)
        for first, count in ((0, 1), (129, 77), (entries - 1, 1), (entries // 2, entries - entries // 2), (5, 0)):
            rc, part = _key_table(eng, curve, slot, first, count)
            assert rc == 0 and np.array_equal(part, want[first * 2 * (L // 4):(first + count) * 2 * (L // 4)]), (label, first, count)
    for slot, first, count in ((off, 0, 1), (big, 0, 1), (oth, 0, 1), (len(keys) + 3, 0, 1), (2 ** 31, 0, 1), (0, entries, 1),
                               (0, 0, entries + 1), (0, entries + 1, 0), (0, 1, 2 ** 64 - 1)):
        assert _key_table(eng, curve, slot, first, count)[0] == ERR_ARG, (slot, first, count)
    assert _key_table(eng, curve, 0, entries, 0)[0] == 0


# ---------------------------------------------------------------- tables of keys grouped in a launch
_COUNTS = (1, 15, 16, 17, 31, 32, 33, 63, 64, 65)


def _keys(curve, count, seed):
    rng = np.random.default_rng(seed)
    return [ek._point(curve, ek._rand(rng, ref.CURVES[curve])) for _ in range(count)]


def _grouped_model(curve, Q):
    return _model(curve, None if curve == P256 else 5, Q)


@pytest.mark.parametrize("T", [1, 2])
@pytest.mark.parametrize("curve", [P256, P384])
def test_every_entry_of_grouped_tables(engines, curve, T):
    """Every entry of the table of every key of a launch of K keys, T items each (interleaved), K around the 64- and
    128-thread blocks of the build kernels (which index t % nkeys and t / nkeys), equals the model; the last key is off
    the curve when K > 1 and reports status 2 (a table slot, no table)."""
    eng = engines["grouped" if T == 1 else "grouped2"]
    L = ref.CURVES[curve].size
    pool = _keys(curve, max(_COUNTS), seed=90 + curve)
    for K in _COUNTS:
        Qs = pool[:K]
        kx = np.stack([ek._be(Q[0], L) for Q in Qs])
        ky = np.stack([ek._be(Q[1], L) for Q in Qs])
        good = K if K == 1 else K - 1
        ky[good:, L - 1] ^= 1                                                       # off the curve
        idx = np.tile(np.arange(K), T)
        items = (T - 1) * K + np.arange(K)                                          # the last item of every key
        status, out = _grouped_tables(eng, curve, kx[idx], ky[idx], items)
        assert status.tolist() == [0] * good + [2] * (K - good), (K, status.tolist())
        for k in range(good):
            _assert_table(out[k], _grouped_model(curve, Qs[k]), f"K={K}, key {k}")


def test_grouped_tables_at_the_benchmark_shape(engines):
    """65,536 P-256 items over 1,024 keys at the default threshold (16): 8 sampled keys' comb tables equal the model."""
    _, kxy = corpus.make_keys(P256, 1024, seed=1)
    idx = np.arange(65536) % 1024
    rng = np.random.default_rng(3)
    sample = np.sort(rng.choice(1024, 8, replace=False))
    status, out = _grouped_tables(engines["default"], P256, kxy[idx, :32], kxy[idx, 32:], 65536 - 1024 + sample)
    assert status.tolist() == [0] * 8
    for q, k in enumerate(sample):
        Q = (int.from_bytes(kxy[k, :32].tobytes(), "big"), int.from_bytes(kxy[k, 32:].tobytes(), "big"))
        _assert_table(out[q], ek.comb_table(Q), f"key {k}")


@pytest.mark.parametrize("curve", [P256, P384])
def test_grouped_tables_when_the_slots_run_out(curve):
    """SBV_GROUP_MAX_KEYS = 8 with 20 keys of 2 items at threshold 2: the key count is clamped to the 8 slots; the keys
    that got one have exact tables, the other 12 report no table."""
    L = ref.CURVES[curve].size
    Qs = _keys(curve, 20, seed=70 + curve)
    kx, ky = np.stack([ek._be(Q[0], L) for Q in Qs]), np.stack([ek._be(Q[1], L) for Q in Qs])
    idx = np.tile(np.arange(20), 2)
    e = _engine(SBV_GROUP_THRESHOLD=2, SBV_GROUP_MAX_KEYS=8)
    try:
        status, out = _grouped_tables(e, curve, kx[idx], ky[idx], np.arange(20))
    finally:
        e.close()
    assert sorted(status.tolist()) == [0] * 8 + [1] * 12
    for k in np.nonzero(status == 0)[0]:
        _assert_table(out[k], _grouped_model(curve, Qs[k]), f"key {k}")


# ---------------------------------------------------------------- digit sweeps
def _check(got, want, what):
    assert np.array_equal(got, want), (what, np.nonzero(got != want)[0][:10])


def _oracle(curve, b):
    return oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])


@pytest.mark.parametrize("curve", [P256, P384])
def test_registered_digit_sweep(engines, curve):
    """u2 takes every reachable (window, digit) pair of the 8-bit windows: the warp kernel (one batch of a few hundred
    rows) and the thread kernel (the rows repeated past the warp limit) give the verdicts of the construction."""
    b, want = ek.sweep_batch(curve, ek.window_sweep_u2(curve, 8, seed=8 + curve), seed=20 + curve)
    _check(_oracle(curve, b), want, "oracle")
    eng = engines["generic"]
    _check(_registered(eng, curve, b), want, "registered warp")
    _check(_registered(eng, curve, b, n_min=WARP_LIMIT), want, "registered thread")


@pytest.mark.parametrize("curve", [P256, P384])
def test_grouped_digit_sweep(engines, curve):
    """Every key with a table (threshold 1): P-256 u2 takes every (block, column, mask) triple of the comb
    (k_verify_comb), P-384 u2 every reachable (window, digit) pair of the 5-bit windows (k_verify_kt)."""
    u2s = ek.comb_sweep_u2(seed=1) if curve == P256 else ek.window_sweep_u2(P384, 5, seed=5)
    b, want = ek.sweep_batch(curve, u2s, seed=30 + curve)
    _check(_oracle(curve, b), want, "oracle")
    args = (b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    _check(engines["grouped"].verify_batch(curve, *args), want, "grouped")


@pytest.mark.parametrize("curve", [P256, P384])
def test_generic_digit_sweep(engines, curve):
    """Grouping off: u2 takes every reachable (window, digit) pair of k_verify_coz's 4-bit windows."""
    b, want = ek.sweep_batch(curve, ek.window_sweep_u2(curve, 4, seed=4 + curve), seed=40 + curve)
    _check(_oracle(curve, b), want, "oracle")
    _check(engines["generic"].verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"]), want, "generic")


# ---------------------------------------------------------------- key encodings
def _slots48(b, curve):
    L = ref.CURVES[curve].size
    pad = lambda a: np.concatenate([np.zeros((a.shape[0], 48 - a.shape[1]), np.uint8), a], axis=1)
    return pad(b["qx"]), pad(b["qy"]), pad(b["r"]), pad(b["s"]), L


@pytest.mark.parametrize("curve", [P256, P384])
def test_key_encodings_on_every_path(engines, curve):
    """(x + p, y), (x, y + p) of valid points, x = p, y = p, (0, 0) and all-ones coordinates reject and their canonical
    twins accept: generic, grouped (thresholds 1, 2), DER signatures, registered keys on the warp and the thread kernel."""
    b, want, labels = ek.encoding_batch(curve, seed=11 + curve)
    _check(_oracle(curve, b), want, "oracle")
    args = (b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    for name in ("generic", "grouped", "grouped2"):
        _check(engines[name].verify_batch(curve, *args), want, name)
    # T = 2: every key twice, so the edge keys get a table slot too
    two = {k: np.concatenate([v, v]) for k, v in b.items()}
    _check(engines["grouped2"].verify_batch(curve, *(two[k] for k in ("r", "s", "qx", "qy", "digest"))), np.concatenate([want, want]), "grouped2 x2")
    der = [ref.der_encode(int.from_bytes(r.tobytes(), "big"), int.from_bytes(s.tobytes(), "big")) for r, s in zip(b["r"], b["s"])]
    off = np.concatenate([[0], np.cumsum([len(d) for d in der])]).astype(np.uint32)
    sigs = np.frombuffer(b"".join(der), np.uint8)
    qxy = np.concatenate([b["qx"], b["qy"]], axis=1)
    _check(engines["generic"].verify_batch_der(curve, sigs, off, qxy, b["digest"]), want, "der generic")
    _check(engines["grouped"].verify_batch_der(curve, sigs, off, qxy, b["digest"]), want, "der grouped")
    eng = engines["generic"]
    _check(_registered(eng, curve, b), want, "registered warp")
    _check(_registered(eng, curve, b, n_min=WARP_LIMIT), want, "registered thread")


def test_key_encodings_in_48_byte_slots(engines):
    """sbv_verify_mixed (both curves in one call, 32-byte digests) and registered keys in 48-byte slots: the edge
    encodings reject, their twins accept, and P-256 keys with a nonzero byte above the low 32 of a slot reject."""
    parts = []
    for curve in (P256, P384):
        b, want, _ = ek.encoding_batch(curve, seed=50 + curve, u1_zero=True)
        qx, qy, r, s, L = _slots48(b, curve)
        parts.append((curve, qx, qy, r, s, b["digest"], want))
    curve, qx, qy, r, s, dig, want = parts[0]
    ok_rows = np.nonzero(want == 1)[0]
    hx, hy = qx[ok_rows].copy(), qy[ok_rows].copy()
    hx[:, 15] = 1
    hy[:, 0] = 0x80
    high = (np.concatenate([hx, qx[ok_rows]]), np.concatenate([qy[ok_rows], hy]))
    parts.append((P256, high[0], high[1], np.concatenate([r[ok_rows]] * 2), np.concatenate([s[ok_rows]] * 2), np.concatenate([dig[ok_rows]] * 2),
                  np.zeros(2 * ok_rows.size, np.uint8)))
    tag = np.concatenate([np.full(p[1].shape[0], p[0], np.uint8) for p in parts])
    cat = lambda j: np.ascontiguousarray(np.concatenate([p[j] for p in parts]))
    want = cat(6)
    for name in ("generic", "grouped"):
        _check(engines[name].verify_mixed(tag, cat(3), cat(4), cat(1), cat(2), cat(5)), want, f"mixed {name}")
    # registered: one slot per distinct 48-byte key, both curves in one registry
    eng = engines["generic"]
    xy = np.concatenate([cat(1), cat(2)], axis=1)
    keys, slot = np.unique(np.concatenate([tag[:, None], xy], axis=1), axis=0, return_inverse=True)
    slot = slot.reshape(-1).astype(np.uint32)
    eng.set_keys(keys[:, 0].copy(), np.ascontiguousarray(keys[:, 1:]))
    for c in (P256, P384):
        rows = np.nonzero(tag == c)[0]
        L = ref.CURVES[c].size
        for reps in (1, WARP_LIMIT // rows.size + 1):                       # the warp kernel, then the thread kernel
            t = lambda a: np.ascontiguousarray(np.concatenate([a[rows]] * reps))
            got = eng.verify_registered(c, t(slot), t(cat(3))[:, 48 - L:], t(cat(4))[:, 48 - L:], t(cat(5)))
            _check(got[:rows.size], want[rows], (c, reps))


# ---------------------------------------------------------------- keys that collide in the old grouping hash
@pytest.mark.parametrize("T", [1, 2])
@pytest.mark.parametrize("curve", [P256, P384])
def test_colliding_keys(curve, T):
    """4,096 signatures under a valid key interleaved with 4,096 items under off-curve keys equal to it in every word
    the grouping hash once read (4,096 / T keys, T items each): every off-curve item rejects, the valid key's items
    give the oracle's verdicts (one in eight corrupted)."""
    c = ref.CURVES[curve]
    L, n = c.size, 4096
    d = 0xA11CE + curve
    Q = ek._point(curve, d)
    rng = np.random.default_rng(60 + curve)
    dig = np.frombuffer(rng.bytes(n * L), np.uint8).reshape(n, L)
    k = np.stack([ek._be(ek._rand(rng, c), L) for _ in range(n)])
    r, s = oracle.sign_batch(curve, ek._be(d, L)[None, :], np.zeros(n, np.uint32), dig, k)
    r[::8, L - 1] ^= 1
    cx, cy = ek.colliding_keys(curve, Q, n // T)
    cx, cy = np.tile(cx, (T, 1)), np.tile(cy, (T, 1))
    b = {"r": np.repeat(r, 2, axis=0), "s": np.repeat(s, 2, axis=0), "digest": np.repeat(dig, 2, axis=0)}
    b["qx"] = np.empty((2 * n, L), np.uint8)
    b["qy"] = np.empty((2 * n, L), np.uint8)
    b["qx"][0::2], b["qy"][0::2] = ek._be(Q[0], L), ek._be(Q[1], L)
    b["qx"][1::2], b["qy"][1::2] = cx, cy
    want = _oracle(curve, b)
    assert not want[1::2].any() and 0 < int(want[0::2].sum()) < n
    e = _engine(SBV_GROUP_THRESHOLD=T)
    try:
        got = e.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    finally:
        e.close()
    _check(got, want, ("colliding", curve, T))


@pytest.mark.parametrize("T", [1, 2])
@pytest.mark.parametrize("curve", [P256, P384])
def test_colliding_key_meets_the_valid_key(curve, T):
    """96 launches of one valid item and one item under a colliding off-curve key (T items each): with 2T items in a
    hash table of 4T slots, the two keys start at the same slot in about one launch in 4T, so kg_same_key has to tell
    them apart there.  The off-curve item rejects every time."""
    c = ref.CURVES[curve]
    L = c.size
    d = 0xB0B + curve
    Q = ek._point(curve, d)
    rng = np.random.default_rng(80 + curve)
    dig = np.frombuffer(rng.bytes(L), np.uint8).reshape(1, L)
    r, s = oracle.sign_batch(curve, ek._be(d, L)[None, :], np.zeros(1, np.uint32), dig, ek._be(ek._rand(rng, c), L)[None, :])
    cx, cy = ek.colliding_keys(curve, Q, 96)
    vx, vy = ek._be(Q[0], L), ek._be(Q[1], L)
    e = _engine(SBV_GROUP_THRESHOLD=T)
    try:
        for i in range(96):
            qx = np.ascontiguousarray(np.tile(np.stack([vx, cx[i]]), (T, 1)))
            qy = np.ascontiguousarray(np.tile(np.stack([vy, cy[i]]), (T, 1)))
            rep = lambda a: np.ascontiguousarray(np.repeat(a, 2 * T, axis=0))
            got = e.verify_batch(curve, rep(r), rep(s), qx, qy, rep(dig))
            assert got.tolist() == [1, 0] * T, (i, got.tolist())
    finally:
        e.close()


# ---------------------------------------------------------------- the shuffle tree of k_verify_kt_warp
@pytest.mark.parametrize("curve", [P256, P384])
def test_warp_tree_exceptional_sums(engines, curve):
    """Partial sums of k_verify_kt_warp's shuffle tree that are equal (the general addition doubles) or opposite (an
    infinity the levels above carry, as the shuffled operand where the lane moves up, up to R = infinity at the last
    level), at every level: the warp kernel and the thread kernel of registered keys, the generic and the grouped
    path give the verdicts of the construction and of the oracle."""
    b, want, events = ek.warp_tree_batch(curve, seed=300 + curve)
    assert {e[0] for e in events} == set(ek.TREE)
    _every_path(engines, curve, b, want=want)
