"""Edge cases of the verification kernels on the device, through the C ABI, every verdict against the oracle (and, for
the crafted sets, against the verdict the construction implies): R.x in [n, p) (final_check's comparison with
(r + n) * Z^2), e >= n and digests of other lengths (load_digest, nmul of an unreduced e in k_prep), scalars crafted for
the fixed-base kernels' order of operations, and every entry of the fixed-base table of G (k_gtable_init).

Each set runs on every path: the generic kernel (SBV_GROUP_THRESHOLD=0), per-key tables for every key (threshold 1;
P-256: comb, P-384: 5-bit windows), registered keys (sbv_set_keys) on the thread kernel (a batch larger than the warp
limit) and on the warp kernel (at most SBV_KEYED_WARP_LIMIT = 2,048 items)."""
import ctypes as C
import hashlib
import time

import numpy as np
import pytest

import edges
import oracle
from oracle import P256, P384
from oracle import ecdsa_ref as ref
from test_gpu_round2 import _engine

pytestmark = pytest.mark.gpu

WARP_LIMIT = 2048


@pytest.fixture(scope="module")
def engines():
    es = {"generic": _engine(SBV_GROUP_THRESHOLD=0), "grouped": _engine(SBV_GROUP_THRESHOLD=1),
          "grouped2": _engine(SBV_GROUP_THRESHOLD=2)}
    yield es
    for e in es.values():
        e.close()


def _registered(eng, curve, b, n_min=0):
    """b's rows through sbv_verify_registered, one slot per distinct key; the rows are repeated until there are more
    than n_min of them.  Returns the verdicts of the first copy."""
    L = b["qx"].shape[1]
    kxy = np.concatenate([b["qx"], b["qy"]], axis=1)
    keys, slot = np.unique(kxy, axis=0, return_inverse=True)
    slot = slot.reshape(-1).astype(np.uint32)
    eng.set_keys(np.full(len(keys), curve, np.uint8), keys.reshape(-1, 2, L))
    n = slot.size
    reps = n_min // n + 1
    t = lambda a: np.ascontiguousarray(np.concatenate([a] * reps))
    got = eng.verify_registered(curve, t(slot), t(b["r"]), t(b["s"]), t(b["digest"]))
    assert (got.reshape(reps, n) == got[:n]).all()
    return got[:n]


def _every_path(engines, curve, b, want=None, thresholds=("grouped",)):
    """the oracle's verdicts (== want, if given) on the generic kernel, the grouped paths and both registered kernels"""
    ref_ok = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    if want is not None:
        assert np.array_equal(ref_ok, want)
    assert 0 < int(ref_ok.sum()) < ref_ok.size                    # accepts and rejects both present
    args = (b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    for name in ("generic",) + tuple(thresholds):
        got = engines[name].verify_batch(curve, *args)
        assert np.array_equal(got, ref_ok), (name, np.nonzero(got != ref_ok)[0][:10])
    n = ref_ok.size
    assert n <= WARP_LIMIT
    eng = engines["generic"]
    got = _registered(eng, curve, b)                              # warp kernel
    assert np.array_equal(got, ref_ok), ("registered warp", np.nonzero(got != ref_ok)[0][:10])
    got = _registered(eng, curve, b, n_min=WARP_LIMIT)            # thread kernel
    assert np.array_equal(got, ref_ok), ("registered thread", np.nonzero(got != ref_ok)[0][:10])
    return ref_ok


def _ecdsa_ref(curve, b):
    rows = zip(*(b[k] for k in ("r", "s", "qx", "qy", "digest")))
    return np.array([ref.verify_bytes(curve, *(bytes(v) for v in row)) for row in rows], np.uint8)


@pytest.mark.parametrize("curve", [P256, P384])
def test_R_x_at_least_n(engines, curve):
    """R.x in [n, p): r = R.x - n accepts (final_check: X == (r + n) * Z^2, only reached when r < p - n), r = R.x is out of
    range and r + 1 does not match; r = R'.x + p - n with a small R'.x rejects (r + n is R'.x mod p, but r >= p - n).
    Random signatures get there with probability ~2^-128 (P-256) / 2^-190 (P-384)."""
    b = edges.big_x_signatures(curve, 24, seed=100 + curve)
    n = ref.CURVES[curve].n
    assert sum(x >= n for x in b["rx"]) == 3 * 24 and b["want"].sum() == 24
    small = {k: b[k][:9] for k in ("r", "s", "qx", "qy", "digest")}
    assert np.array_equal(_ecdsa_ref(curve, small), b["want"][:9])
    _every_path(engines, curve, b, want=b["want"])


@pytest.mark.parametrize("curve", [P256, P384])
def test_s_with_only_its_top_limb_set(engines, curve):
    """s = t * 2^(32(N-1)): k_prep's s != 0 check reads every limb — valid signatures accept, their e + 1 rows reject."""
    b = edges.sparse_s_signatures(curve, 8, seed=300 + curve)
    _every_path(engines, curve, b, want=b["want"])


@pytest.mark.parametrize("curve", [P256, P384])
def test_s_plus_n_rejects_where_s_1_accepts(engines, curve):
    """(r, 1) valid and (r, n + 1): k_prep computes the flagged second row with s = 1, so every kernel must read the flag."""
    b = edges.s_plus_n_signatures(curve, 8, seed=310 + curve)
    _every_path(engines, curve, b, want=b["want"])


@pytest.mark.parametrize("thr", [0, 1])
@pytest.mark.parametrize("curve", [P256, P384])
def test_R_x_at_least_n_chunked_hash_and_verify(curve, thr):
    """The same edge through sbv_hash_verify_batch, with e the SHA-256 of a message, uploaded and verified in several
    chunks (SBV_CHUNK_ITEMS=40), on the generic kernel (threshold 0) or with a table for every key (threshold 1)."""
    count = 30
    rng = np.random.default_rng(7 + curve)
    lens = rng.integers(0, 300, count)
    msgs = [rng.integers(0, 256, int(k), dtype=np.uint8).tobytes() for k in lens]
    digs = np.stack([np.frombuffer(hashlib.sha256(m).digest(), np.uint8) for m in msgs])
    b = edges.big_x_signatures(curve, count, seed=200 + curve, digests=digs)
    rows = [msgs[i // 4] for i in range(4 * count)]
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(m) for m in rows])
    blob = np.frombuffer(b"".join(rows) + b"\0", np.uint8)
    want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert np.array_equal(want, b["want"])
    e = _engine(SBV_CHUNK_ITEMS=40, SBV_GROUP_THRESHOLD=thr)
    try:
        got, dig = e.hash_verify_batch(curve, blob, off, b["r"], b["s"], b["qx"], b["qy"], want_digest=True)
    finally:
        e.close()
    assert np.array_equal(dig, b["digest"])
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]


@pytest.mark.parametrize("dlen", [4, 20, 28, 32, 48, 64])
@pytest.mark.parametrize("curve", [P256, P384])
def test_digest_at_least_n_and_other_lengths(engines, curve, dlen):
    """e = the leftmost min(dlen, BYTES) bytes: e >= n (k_prep multiplies it unreduced), e mod n written below n gives
    the same verdict, a bit flipped beyond the first BYTES bytes changes nothing, one flipped inside them rejects."""
    c = ref.CURVES[curve]
    b = edges.wide_digest_signatures(curve, dlen, 6, seed=300 + dlen + curve)
    if dlen >= c.size:
        assert sum(e >= c.n for e in b["e"]) >= 3
    assert np.array_equal(_ecdsa_ref(curve, b), b["want"])
    _every_path(engines, curve, b, want=b["want"])


@pytest.mark.parametrize("curve", [P256, P384])
def test_crafted_scalars_for_the_fixed_base_kernels(engines, curve):
    """The comb-order cases (u1*G = +-u2*Q, u1*G + u2*Q one G entry, u2's comb masks all ones or all zero) and the
    fixed-base exceptional cases (the running sum meets the next entry, its negative, or ends at infinity), at
    thresholds 1 and 2 and on the registered kernels."""
    b = edges.crafted(curve, edges.comb_cases(curve) + edges.fixed_base_cases(curve))
    _every_path(engines, curve, b, thresholds=("grouped", "grouped2"))


@pytest.mark.parametrize("curve", [P256, P384])
def test_u1_comb_digit_sweeps(engines, curve):
    """u1 whose 16-bit comb digits of G are 0x0000 (u1 = 0: the G part is infinity), 0x0001, 0x8000, 0xFFFF in every
    column, or mixed from those; each row also with r + 1 (same u1, must reject)."""
    b = edges.with_bumped_r(edges.crafted(curve, edges.u1_digit_cases(curve, seed=curve)))
    _every_path(engines, curve, b)


def _gtable_expected(curve):
    """T[i][b] = b * 2^(16 i) * G in affine Montgomery form, b = 0 as zeros, as the bytes of the device table: limbs are
    little-endian words, so an entry is x*R mod p then y*R mod p, each as 4N little-endian bytes.  Every column is walked
    by affine additions of its base (one doubling for b = 2), all columns in step, so one inversion (Montgomery's batch
    trick) serves a whole row of the table.  No exceptional case: b * base = +-base needs b = +-1 mod n."""
    c = ref.CURVES[curve]
    p, L = c.p, c.size
    Rm = (1 << (8 * L)) % p
    cols = 8 * L // 16
    bases = [(c.gx, c.gy)]
    for _ in range(cols - 1):
        P = bases[-1]
        for _ in range(16):
            P = ref._add(c, P, P)
        bases.append(P)
    ent = lambda P: (P[0] * Rm % p).to_bytes(L, "little") + (P[1] * Rm % p).to_bytes(L, "little")
    out = [[bytes(2 * L), ent(B)] for B in bases]
    cur = list(bases)
    pref = [0] * cols
    for bb in range(2, 1 << 16):
        dens = [2 * B[1] % p for B in bases] if bb == 2 else [(P[0] - B[0]) % p for P, B in zip(cur, bases)]
        acc = 1
        for i, d in enumerate(dens):
            pref[i] = acc
            acc = acc * d % p
        inv = pow(acc, -1, p)
        for i in range(cols - 1, -1, -1):
            di = inv * pref[i] % p
            inv = inv * dens[i] % p
            (x1, y1), (x2, y2) = cur[i], bases[i]
            lam = (3 * x2 * x2 - 3) * di % p if bb == 2 else (y1 - y2) * di % p
            x3 = (lam * lam - x1 - x2) % p
            cur[i] = (x3, (lam * (x2 - x3) - y2) % p)
            out[i].append(ent(cur[i]))
    return b"".join(b"".join(col) for col in out)


@pytest.mark.parametrize("curve", [P256, P384])
def test_every_entry_of_the_G_table(engines, curve):
    """All 16 x 65,536 (P-256) / 24 x 65,536 (P-384) entries of the table k_gtable_init builds, against Python integers."""
    eng = engines["generic"]
    L = ref.CURVES[curve].size
    entries = (8 * L // 16) << 16
    t0 = time.time()
    want = _gtable_expected(curve)
    t1 = time.time()
    got = np.zeros(entries * 2 * L // 4, np.uint32)
    rc = eng._lib.sbv_debug_gtable(eng._h, C.c_uint8(curve), C.c_size_t(0), C.c_size_t(entries), got.ctypes.data_as(C.POINTER(C.c_uint32)))
    assert rc == 0
    gb = got.tobytes()
    assert len(gb) == len(want)
    if gb != want:
        g, w = np.frombuffer(gb, np.uint8).reshape(entries, -1), np.frombuffer(want, np.uint8).reshape(entries, -1)
        bad = np.nonzero((g != w).any(axis=1))[0]
        raise AssertionError(f"{bad.size} entries differ, first (column, b): {[(int(i) >> 16, int(i) & 0xFFFF) for i in bad[:8]]}")
    print(f"G table curve {curve}: expected bytes in {t1 - t0:.1f} s, comparison in {time.time() - t1:.1f} s")
