"""CPU simulation of the DEVICE code (tools/hostsim: mp.cuh / curve.cuh / kernels.cuh / keygroup.cuh / sha256.cuh / quorum.cuh
compiled with g++, PTX carry-flag primitives emulated; thread-per-item kernels one simulated thread at a time,
warp-cooperative kernels in lockstep with one OS thread per lane) against Python big integers, hashlib and the oracle.

This is how limb-level arithmetic and the kernels' control flow are checked without a GPU; the `-m gpu` tests run the
same checks on the real thing.  The simulation is test infrastructure — libsbv.so has no CPU path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import edges
import oracle
from oracle import corpus
from oracle import ecdsa_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _limbs(vals, N):
    out = np.zeros((len(vals), 2 * N), np.uint32)
    for i, pair in enumerate(vals):
        for h, v in enumerate(pair):
            for k in range(N):
                out[i, h * N + k] = (v >> (32 * k)) & 0xFFFFFFFF
    return out


def _ints(arr, N):
    return [tuple(sum(int(row[h * N + k]) << (32 * k) for k in range(N)) for h in range(2)) for row in arr]


def _run(hs, curve, op, a, b):
    N = 8 if curve == 0 else 12
    A, B = _limbs(a, N), _limbs(b, N)
    out = np.zeros_like(A)
    p32 = lambda x: x.ctypes.data_as(C.POINTER(C.c_uint32))
    assert hs.hs_debug_op(C.c_int(curve), C.c_int(op), C.c_size_t(len(a)), p32(A), p32(B), p32(out)) == 0
    return _ints(out, N)


@pytest.mark.parametrize("curve", [0, 1])
def test_field_ops(hs, curve):
    """Montgomery products (out of line and, with edges.INL, inlined as Inl<C> runs them), field additions and the
    inverses against Python integers: edge values, operands on both sides of each reduction's final subtraction, and
    operands in [m, R)."""
    c = ref.CURVES[curve]
    N = c.size // 4
    R = 1 << (32 * N)
    rng = np.random.default_rng(curve + 11)
    for label, op, xs, ys, want in edges.montgomery_cases(curve, rng, 1500):
        a = [(x, 0) for x in xs]; b = [(y, 0) for y in ys]
        for flag in (0, edges.INL):
            assert [g[0] for g in _run(hs, curve, op | flag, a, b)] == want, (label, op | flag)
    xs = [v for v in edges.edge_values(c.p, rng, 10) if v]
    got = _run(hs, curve, 4, [(x * R % c.p, 0) for x in xs], [(0, 0)] * len(xs))
    assert [g[0] for g in got] == [pow(x, -1, c.p) * R % c.p for x in xs]
    # binary-GCD inverses, with the residues that need the most passes (32N - 1, edges.longest_inverse_inputs)
    xs = [v for v in edges.edge_values(c.p, rng, 300) if v] + [pow(2, k, c.p) for k in (1, 31, 32, 33, 64, 96, 128, 224, 255, 256, 300)]
    xs += [a * pow(R, -1, c.p) % c.p for a in edges.longest_inverse_inputs(c.p, N)]
    got = _run(hs, curve, 10, [(x * R % c.p, 0) for x in xs], [(0, 0)] * len(xs))
    assert [g[0] for g in got] == [pow(x, -1, c.p) * R % c.p for x in xs]
    xs = [v for v in edges.edge_values(c.n, rng, 200) if v]
    xs += [pow(2, k, c.n) for k in (1, 31, 32, 33, 63, 64, 65, 96, 128, 255, 256, 300, 383)]
    xs += [a * pow(R, -1, c.n) % c.n for a in edges.longest_inverse_inputs(c.n, N)]
    got = _run(hs, curve, 8, [(x * R % c.n, 0) for x in xs], [(0, 0)] * len(xs))
    assert [g[0] for g in got] == [pow(x, -1, c.n) * R % c.n for x in xs]


@pytest.mark.parametrize("curve", [0, 1])
def test_group_law(hs, curve):
    """Doubling, mixed and general addition (with neg / skip, from an accumulator at infinity), out of line and inlined."""
    c = ref.CURVES[curve]
    ks = [1, 2, 3, 4, 5, 7, 8, 255, c.n - 1, c.n - 2, 2**100 + 3]
    for op, a, b, want in edges.group_cases(curve, ks):
        for flag in (0, edges.INL):
            assert _run(hs, curve, op | flag, a, b) == want, op | flag


def _p8(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def _verify(hs, curve, b, grouped=None):
    n = b["r"].shape[0]
    ok = np.full(n, 7, np.uint8)
    f = [np.ascontiguousarray(b[k]) for k in ("r", "s", "qx", "qy", "digest")]
    dlen = f[4].size // n
    if grouped is None:
        assert hs.hs_verify(C.c_int(curve), C.c_size_t(n), *map(_p8, f), C.c_uint32(dlen), _p8(ok)) == 0
        return ok
    thr, maxk = grouped
    stats = np.zeros(3, np.uint32)
    assert hs.hs_verify_grouped(C.c_int(curve), C.c_size_t(n), *map(_p8, f), C.c_uint32(dlen), C.c_uint32(thr), C.c_uint32(maxk), _p8(ok),
                                stats.ctypes.data_as(C.POINTER(C.c_uint32))) == 0
    return ok, stats


def test_verify_generic_kernel_p256(hs):
    """k_prep + k_verify_coz (the kernels of the product, simulated) on a corrupted corpus: every class of the
    corpus, bit-exact with the oracle."""
    b = corpus.make_batch(oracle.P256, n=192, K=8, seed=21, corrupt_rate=3)
    want = oracle.verify_batch(oracle.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert 0 < int(want.sum()) < want.size
    assert np.array_equal(_verify(hs, 0, b), want)


def test_verify_generic_kernel_p384(hs):
    b = corpus.make_batch(oracle.P384, n=48, K=4, seed=22, corrupt_rate=3)
    want = oracle.verify_batch(oracle.P384, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert np.array_equal(_verify(hs, 1, b), want)


@pytest.mark.parametrize("thr,maxk", [(4, 64), (1, 64), (4, 3), (1000, 64)])
def test_verify_grouped_p256(hs, thr, maxk):
    """Key grouping + on-the-fly per-key tables + fixed-base kernel, with the generic kernel for the rest: same
    verdicts as the oracle whatever the threshold / table capacity (all keys grouped, capacity exhausted, nothing
    grouped)."""
    b = corpus.make_batch(oracle.P256, n=256, K=8, seed=23, corrupt_rate=3)
    want = oracle.verify_batch(oracle.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    got, stats = _verify(hs, 0, b, grouped=(thr, maxk))
    assert np.array_equal(got, want)
    assert int(stats[1]) + int(stats[2]) == 256
    if thr == 1000:
        assert int(stats[1]) == 0
    if thr == 1 and maxk == 64:
        assert int(stats[2]) == 0          # every key (also the corrupted, off-curve ones) got a slot; invalid ones reject by flag
    if maxk == 3:
        assert int(stats[0]) >= 3 and int(stats[2]) > 0


def test_verify_grouped_p384(hs):
    b = corpus.make_batch(oracle.P384, n=64, K=3, seed=24, corrupt_rate=3)
    want = oracle.verify_batch(oracle.P384, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    got, stats = _verify(hs, 1, b, grouped=(4, 16))
    assert np.array_equal(got, want)
    assert int(stats[1]) > 0


@pytest.mark.parametrize("curve,n,K,thr,chunk", [(0, 250, 8, 4, 96), (0, 250, 8, 3, 37), (1, 60, 3, 4, 25)])
def test_verify_chunked_second_half(hs, curve, n, K, thr, chunk):
    """The second half of the pipeline run chunk by chunk (what a chunked host-buffer call enqueues, csrc/pipeline.cu:
    sbv_launch_verify_chunk): shared grouping and key tables, per-chunk routing with chunk-local indices, every per-item
    array addressed as the contiguous slice of the chunk — same verdicts and the same split between the two paths as
    the launch of one chunk, for chunk sizes that do not divide the batch, with odd and even thresholds."""
    cv = oracle.P256 if curve == 0 else oracle.P384
    b = corpus.make_batch(cv, n=n, K=K, seed=25 + chunk, corrupt_rate=3)
    want = oracle.verify_batch(cv, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    whole, st_whole = _verify(hs, curve, b, grouped=(thr, 64))
    ok = np.full(n, 7, np.uint8)
    f = [np.ascontiguousarray(b[k]) for k in ("r", "s", "qx", "qy", "digest")]
    stats = np.zeros(3, np.uint32)
    assert hs.hs_verify_chunked(C.c_int(curve), C.c_size_t(n), *map(_p8, f), C.c_uint32(f[4].size // n), C.c_uint32(thr), C.c_uint32(64),
                                C.c_uint32(chunk), _p8(ok), stats.ctypes.data_as(C.POINTER(C.c_uint32))) == 0
    assert np.array_equal(ok, want)
    assert np.array_equal(whole, want)
    assert list(stats) == list(st_whole) and int(stats[1]) > 0


@pytest.mark.parametrize("curve,thr", [(0, 1), (0, 2), (1, 2)])
def test_exceptional_points_on_the_fixed_base_path(hs, curve, thr):
    """Every key gets a table (threshold 1 / 2) and the scalars are chosen so that the running sum meets the next table
    entry (doubling inside a mixed addition), its negative (infinity in the middle), or ends at infinity (must reject).
    u1*G comes from k_gpart: where it meets the accumulator, that is the closing general addition of k_verify_comb (P-256)
    or the first window addition of k_verify_kt (P-384)."""
    b = edges.crafted(curve, edges.fixed_base_cases(curve))
    want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert 0 < int(want.sum()) < want.size
    got, stats = _verify(hs, curve, b, grouped=(thr, 64))
    assert int(stats[2]) == 0                                   # nothing on the generic path
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]


def _registered(hs, curve, b, warp):
    """b's rows through hs_verify_registered: one slot per distinct key"""
    L = b["qx"].shape[1]
    kxy = np.concatenate([b["qx"], b["qy"]], axis=1)
    keys, slot = np.unique(kxy, axis=0, return_inverse=True)
    slot = np.ascontiguousarray(slot.reshape(-1), dtype=np.uint32)
    kx, ky = np.ascontiguousarray(keys[:, :L]), np.ascontiguousarray(keys[:, L:])
    n = slot.size
    f = [np.ascontiguousarray(b[k]) for k in ("r", "s", "digest")]
    ok = np.full(n, 7, np.uint8)
    assert hs.hs_verify_registered(C.c_int(curve), C.c_size_t(n), C.c_size_t(len(keys)), _p8(kx), _p8(ky), slot.ctypes.data_as(C.POINTER(C.c_uint32)),
                                   _p8(f[0]), _p8(f[1]), _p8(f[2]), C.c_uint32(f[2].size // n), C.c_int(warp), _p8(ok)) == 0
    return ok


def _every_simulated_path(hs, curve, b):
    want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert np.array_equal(want, b["want"])
    assert np.array_equal(_verify(hs, curve, b), want), "generic"
    got, stats = _verify(hs, curve, b, grouped=(1, 64))
    assert int(stats[2]) == 0 and np.array_equal(got, want), "grouped"
    for warp in (0, 1):
        assert np.array_equal(_registered(hs, curve, b, warp), want), ("registered", warp)


@pytest.mark.parametrize("curve", [0, 1])
def test_r_plus_n_accepts_when_R_x_is_at_least_n(hs, curve):
    """R.x in [n, p): r = R.x - n must be accepted (final_check compares X with (r + n) * Z^2), r = R.x (out of range) and
    r + 1 rejected, and r = R'.x + p - n for a small R'.x rejected (final_check's r < p - n condition) — on the generic,
    grouped and registered thread / warp kernels."""
    c = ref.CURVES[curve]
    b = edges.big_x_signatures(curve, 3, seed=7 + curve)
    assert [x >= c.n for x in b["rx"]] == [True, True, True, False] * 3 and b["want"].sum() == 3
    assert all(int.from_bytes(bytes(r), "big") >= c.p - c.n for r in b["r"][3::4])
    _every_simulated_path(hs, curve, b)


@pytest.mark.parametrize("curve", [0, 1])
def test_s_with_only_its_top_limb_set(hs, curve):
    """s = t * 2^(32(N-1)): k_prep's s != 0 check must read every limb — valid signatures accept and their e + 1 rows
    reject on every simulated path."""
    _every_simulated_path(hs, curve, edges.sparse_s_signatures(curve, 4, seed=30 + curve))


@pytest.mark.parametrize("curve", [0, 1])
def test_s_plus_n_rejects_where_s_1_accepts(hs, curve):
    """(r, 1) valid and (r, n + 1): k_prep flags the second row and computes it with s = 1, so every kernel must read
    that flag — on every simulated path."""
    _every_simulated_path(hs, curve, edges.s_plus_n_signatures(curve, 4, seed=40 + curve))


@pytest.mark.parametrize("curve", [0, 1])
def test_key_encodings_at_the_range_edges(hs, curve):
    """ecdsa_keys.encoding_cases on every simulated path: (x + p, y), (x, y + p), x = p, y = p, (0, 0), all ones — each
    signature accepts under its canonical key and rejects under the edge encoding (load_key's range checks)."""
    import ecdsa_keys
    b, want, _ = ecdsa_keys.encoding_batch(curve, seed=50 + curve)
    b["want"] = want
    _every_simulated_path(hs, curve, b)


@pytest.mark.parametrize("curve", [0, 1])
def test_grouping_keys_that_differ_in_one_word_of_y(hs, curve):
    """A valid key Q and an off-curve key Q' equal to Q but in the last 32-bit word of y, chosen so that both start at the
    same hash-table slot (kg_hash under the simulation's seed): Q' must get its own group, so its items — Q's valid
    signatures — reject, while Q's accept (kg_same_key compares every word of x and y)."""
    import ecdsa_keys
    c = ref.CURVES[curve]
    L, m = c.size, 8
    rng = np.random.default_rng(60 + curve)
    d = int.from_bytes(rng.bytes(L + 8), "big") % (c.n - 1) + 1
    Q = ref.pubkey(curve, d)
    hsize = 1
    while hsize < 2 * 2 * m:
        hsize <<= 1
    hs.hs_kg_hash.restype = C.c_int

    def probe(qx, qy):
        out = np.zeros(1, np.uint32)
        assert hs.hs_kg_hash(C.c_int(curve), C.c_size_t(1), _p8(qx), _p8(qy), C.c_uint32(0x1234567), out.ctypes.data_as(C.POINTER(C.c_uint32))) == 0
        return int(out[0]) & (hsize - 1)

    qx, qy = edges._be(Q[0], L).copy(), edges._be(Q[1], L).copy()
    start = probe(qx, qy)
    y2 = qy.copy()
    for v in range(1, 100000):
        y2[L - 4:] = np.frombuffer(((int.from_bytes(qy[L - 4:].tobytes(), "big") ^ v) & 0xFFFFFFFF).to_bytes(4, "big"), np.uint8)
        if probe(qx, y2) == start:
            break
    else:
        raise AssertionError("no colliding probe start")
    Qy2 = int.from_bytes(y2.tobytes(), "big")
    assert not ref.on_curve(c, Q[0], Qy2)
    rows, want = [], []
    for i in range(m):
        r, s, e = ecdsa_keys.signature_for(curve, Q, *(int.from_bytes(rng.bytes(L + 8), "big") % (c.n - 1) + 1 for _ in range(2)))
        rows += [(r, s, Q[0], Q[1], e), (r, s, Q[0], Qy2, e)] if i % 2 else [(r, s, Q[0], Qy2, e), (r, s, Q[0], Q[1], e)]
        want += [1, 0] if i % 2 else [0, 1]
    b = edges._rows(rows, L)
    want = np.array(want, np.uint8)
    assert np.array_equal(oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"]), want)
    got, stats = _verify(hs, curve, b, grouped=(1, 64))
    assert int(stats[0]) == 2 and int(stats[2]) == 0
    assert np.array_equal(got, want), np.nonzero(got != want)[0]


@pytest.mark.parametrize("curve,dlen", [(0, 32), (0, 48), (0, 20), (1, 64), (1, 48), (1, 28)])
def test_digests_at_least_n_and_of_other_lengths(hs, curve, dlen):
    """e from the leftmost min(dlen, BYTES) digest bytes, also when that is >= n or the digest is longer than the field:
    the same verdicts on every simulated path, and a bit flipped past the first BYTES bytes changes nothing."""
    b = edges.wide_digest_signatures(curve, dlen, 4, seed=dlen + curve)
    c = ref.CURVES[curve]
    assert (dlen < c.size) or any(e >= c.n for e in b["e"])
    assert 0 < b["want"].sum() < b["want"].size
    _every_simulated_path(hs, curve, b)


def _tables(hs, curve, w8, kxy, four):
    L = 32 if curve == 0 else 48
    n = kxy.shape[0]
    qx, qy = np.ascontiguousarray(kxy[:, :L]), np.ascontiguousarray(kxy[:, L:])
    hs.hs_ktab_words.restype = C.c_size_t
    words = hs.hs_ktab_words(C.c_int(curve), C.c_int(w8), C.c_size_t(n))
    kt, fl = np.zeros(words, np.uint32), np.zeros(n, np.uint8)
    assert hs.hs_tables(C.c_int(curve), C.c_int(w8), C.c_size_t(n), _p8(qx), _p8(qy), C.c_int(four), kt.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(fl)) == 0
    return kt, fl


@pytest.mark.parametrize("curve,w8,nkeys", [(0, 0, 6), (0, 1, 3), (1, 0, 3)])
def test_four_lane_doubling_chain_in_lockstep(hs, curve, w8, nkeys):
    """k_kt_bases4 — four lanes per key, the independent multiplications of a doubling on different lanes, quad shuffles —
    simulated with one OS thread per lane meeting at every shuffle: the tables it leads to are bit-identical to those of the
    one-thread-per-key kernel, the validity flags too (an off-curve key and a coordinate >= p among the keys), and every
    entry of a table is e * 2^(W*w) * Q in affine Montgomery form."""
    cv = oracle.P256 if curve == 0 else oracle.P384
    c = ref.CURVES[cv]
    L, N, W = c.size, c.size // 4, 8 if w8 else 5
    d, kxy = corpus.make_keys(cv, nkeys, seed=3 + curve)
    kxy = kxy.copy()
    kxy[1, L + 8] ^= 1                                            # off the curve
    if nkeys > 3:
        kxy[4, :L] = np.frombuffer(int(c.p + 2).to_bytes(L, "big"), np.uint8)   # x >= p
    a, fa = _tables(hs, curve, w8, kxy, four=0)
    b, fb = _tables(hs, curve, w8, kxy, four=1)
    assert fa.tolist() == fb.tolist() and fa[0] == 1 and fa[1] == 0 and (nkeys <= 3 or fa[4] == 0)
    assert np.array_equal(a, b)
    # key 0 against Python integers
    nwin = (8 * L + 1 + W - 1) // W
    ent = 1 << (W - 1)
    tab = b[: nwin * ent * 2 * N].reshape(nwin, ent, 2, N)
    Q = (int.from_bytes(kxy[0, :L].tobytes(), "big"), int.from_bytes(kxy[0, L:].tobytes(), "big"))
    Rm = 1 << (8 * L)
    val = lambda w: sum(int(x) << (32 * i) for i, x in enumerate(w))
    for win in sorted({0, 1, nwin // 2, nwin - 1}):
        for e in (1, 2, 3, ent - 1, ent):
            if win == nwin - 1 and (e << (W * win)) >= c.n:
                continue
            P = ref.scalar_mult(c, (e << (W * win)) % c.n, Q)
            assert val(tab[win, e - 1, 0]) == P[0] * Rm % c.p and val(tab[win, e - 1, 1]) == P[1] * Rm % c.p, (win, e)


@pytest.mark.parametrize("curve,n", [(0, 40), (1, 12)])
def test_registered_keys_thread_and_warp_kernels(hs, curve, n):
    """sbv_set_keys / sbv_verify_registered on the CPU: 8-bit-window tables, keys taken by slot, the thread-per-signature
    kernel and the ONE-SIGNATURE-PER-WARP kernel (32 OS threads per signature, shuffle-tree reduction in lockstep):
    both equal the oracle, including an invalid registered key and an out-of-range slot."""
    cv = oracle.P256 if curve == 0 else oracle.P384
    c = ref.CURVES[cv]
    L, K = c.size, 4
    b = corpus.make_batch(cv, n=n, K=K - 1, seed=60 + curve, corrupt_rate=4)
    d, kxy = corpus.make_keys(cv, K, seed=70 + curve)
    key_idx = (np.arange(n) % K).astype(np.uint32)
    r, s = oracle.sign_batch(cv, d, key_idx, b["digest"], corpus._blocks(71, n, L, b"k"))
    s[::5, L // 2] ^= 4                                          # bad signatures
    kxy = kxy.copy()
    kxy[3, L + 3] ^= 8                                           # registered key 3 is not on the curve
    slot = key_idx.copy()
    slot[7] = 99                                                 # no such slot
    slot[8] = K                                                  # one past the last slot (item 8 is signed by key 0)
    qx, qy = np.ascontiguousarray(kxy[key_idx, :L]), np.ascontiguousarray(kxy[key_idx, L:])
    want = oracle.verify_batch(cv, r, s, qx, qy, b["digest"])
    want[7] = want[8] = 0
    assert want[key_idx == 3].sum() == 0 and 0 < want.sum() < n
    kx, ky = np.ascontiguousarray(kxy[:, :L]), np.ascontiguousarray(kxy[:, L:])
    dig = np.ascontiguousarray(b["digest"])
    for warp in (0, 1):
        ok = np.full(n, 7, np.uint8)
        assert hs.hs_verify_registered(C.c_int(curve), C.c_size_t(n), C.c_size_t(K), _p8(kx), _p8(ky), slot.ctypes.data_as(C.POINTER(C.c_uint32)),
                                       _p8(r), _p8(s), _p8(dig), C.c_uint32(dig.size // n), C.c_int(warp), _p8(ok)) == 0
        assert np.array_equal(ok, want), (warp, np.nonzero(ok != want)[0])


def test_sha256_kernel_on_a_ragged_batch(hs):
    """k_sha256 (aligned 32-bit loads re-aligned with PRMT, padding built in registers) against hashlib: every length
    0..200 plus block boundaries, at arbitrary byte offsets, in input order and in a permuted processing order."""
    import hashlib
    rng = np.random.default_rng(5)
    lens = list(range(0, 200)) + [247, 248, 255, 256, 257, 1000, 4095, 4096] + rng.integers(0, 1500, 60).tolist()
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    lead = 3                                                    # the batch does not start on a word boundary
    off += np.uint64(lead)
    buf = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    n = len(lens)
    want = np.stack([np.frombuffer(hashlib.sha256(buf[int(off[i]):int(off[i + 1])].tobytes()).digest(), np.uint8) for i in range(n)])
    for perm in (None, rng.permutation(n).astype(np.uint32)):
        out = np.zeros((n, 32), np.uint8)
        assert hs.hs_sha256(C.c_size_t(n), _p8(buf), off.ctypes.data_as(C.POINTER(C.c_uint64)), C.c_uint64(0),
                            None if perm is None else perm.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(out)) == 0
        assert np.array_equal(out, want)


def test_quorum_and_pack_kernels(hs):
    """k_quorum_count / k_quorum_reached against the oracle's restatement of processCommits (view.go:519-551, util.go:130-143)
    on a Byzantine vote stream — whole, and as the two shards of a two-device engine (instances split, instance base
    subtracted) — and k_pack_bits (a warp ballot per 32 verdicts, in lockstep) against the host-side packing."""
    from consensus_b200 import sharding
    rng = np.random.default_rng(11)
    I, NV = 37, 7
    inst = np.repeat(np.arange(I, dtype=np.uint32), NV)
    nv = inst.size
    sender = (np.tile(np.arange(NV), I) + 1).astype(np.uint16)
    dup = rng.random(nv) < 0.15
    sender[dup] = np.roll(sender, 1)[dup]                       # duplicate senders: the later vote must not count
    signer = sender.copy()
    wrong = rng.random(nv) < 0.1
    signer[wrong] = (signer[wrong] % NV) + 1                     # signer != sender: never registered (and burns nothing)
    dm = (rng.random(nv) > 0.1).astype(np.uint8)
    ok = (rng.random(nv) > 0.2).astype(np.uint8)
    self_id = (rng.integers(0, NV, I) + 1).astype(np.uint16)     # the counting node's own id per instance
    thr = 4
    want_cnt, want_rch = ref.count_commit_votes_batch(inst, sender, signer, dm, ok, I, thr, self_id)
    p16, p32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint16)), lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))

    def run(vlo, vhi, ilo, ihi, with_ok=True):
        cnt, rch = np.zeros(ihi - ilo, np.uint32), np.zeros(ihi - ilo, np.uint8)
        a = [np.ascontiguousarray(x[vlo:vhi]) for x in (inst, sender, signer, dm, ok)]
        sid = np.ascontiguousarray(self_id[ilo:ihi])
        assert hs.hs_quorum(C.c_size_t(vhi - vlo), p32(a[0]), p16(a[1]), p16(a[2]), _p8(a[3]), _p8(a[4]) if with_ok else None, p16(sid),
                            C.c_uint32(ilo), C.c_size_t(ihi - ilo), C.c_uint32(thr), p32(cnt), _p8(rch)) == 0
        return cnt, rch
    cnt, rch = run(0, nv, 0, I)
    assert np.array_equal(cnt, want_cnt) and np.array_equal(rch, want_rch) and 0 < rch.sum() < I
    parts = []
    for g in range(2):                                           # sharded by instance, as sbv_verify_quorum does on two devices
        ilo, ihi = sharding.shard_range(I, g, 2)
        vlo, vhi = int(np.searchsorted(inst, ilo)), int(np.searchsorted(inst, ihi))
        parts.append(run(vlo, vhi, ilo, ihi))
    assert np.array_equal(np.concatenate([p[0] for p in parts]), want_cnt)
    # prepares carry no signature (ok == NULL): every registered vote with a matching digest counts
    cnt_p, _ = run(0, nv, 0, I, with_ok=False)
    want_p, _ = ref.count_commit_votes_batch(inst, sender, signer, dm, np.ones(nv, np.uint8), I, thr, self_id)
    assert np.array_equal(cnt_p, want_p)
    # verdict bytes -> bitmask
    for n in (1, 31, 32, 33, 1000):
        v = (rng.random(n) > 0.4).astype(np.uint8)
        words = np.zeros((n + 31) // 32, np.uint32)
        assert hs.hs_pack_bits(C.c_size_t(n), _p8(v), p32(words)) == 0
        assert np.array_equal(words, sharding.pack_bits(v, words.size)), n
