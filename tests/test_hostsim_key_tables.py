"""The ECDSA per-key tables and the key-grouping hash in the CPU simulation of the device code (tools/hostsim): the
Python models of tests/ecdsa_keys.py against the construction kernels (hs_tables) for one key of each kind, the coverage
of the digit sweeps, kg_hash on keys that agree with a valid key in half of their words, and the exceptional sums of
k_verify_kt_warp's shuffle tree."""
import ctypes as C

import numpy as np
import pytest

import ecdsa_keys as ek
import oracle
from oracle import ecdsa_ref as ref
from test_hostsim import _p8, hs  # noqa: F401  (hs: the simulation library fixture)

W5, W8, COMB = 0, 1, 2  # hs_tables / hs_ktab_words: table kinds


def _tables(hs, curve, kind, Q):
    L = ref.CURVES[curve].size
    qx, qy = ek._be(Q[0], L).copy(), ek._be(Q[1], L).copy()
    hs.hs_ktab_words.restype = C.c_size_t
    words = hs.hs_ktab_words(C.c_int(curve), C.c_int(kind), C.c_size_t(1))
    kt, fl = np.zeros(words, np.uint32), np.zeros(1, np.uint8)
    assert hs.hs_tables(C.c_int(curve), C.c_int(kind), C.c_size_t(1), _p8(qx), _p8(qy), C.c_int(1), kt.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(fl)) == 0
    assert fl[0] == 1
    return kt


@pytest.mark.parametrize("curve,kind,W", [(0, COMB, None), (1, W5, 5), (0, W8, 8), (1, W8, 8)])
def test_models_equal_the_construction_kernels(hs, curve, kind, W):
    """Every entry of the table the construction kernels build (four-lane doubling chain, as the product runs it) for a
    random key equals the model: the layout (window / chain, entry, slot order) and the values."""
    c = ref.CURVES[curve]
    Q = ek._point(curve, 0x1234567890ABCDEF1234567 + curve)
    got = _tables(hs, curve, kind, Q)
    want = ek.comb_table(Q) if kind == COMB else ek.window_table(curve, W, Q)
    assert got.size == want.size
    bad = np.nonzero((got != want).reshape(-1, c.size // 2).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} entries differ, first {bad[:8].tolist()}"


@pytest.mark.parametrize("curve,W", [(0, 8), (1, 8), (1, 5), (0, 4), (1, 4)])
def test_window_sweeps_cover_every_reachable_digit(curve, W):
    """The sweep of each window kernel (registered: W = 8; P-384 grouped: W = 5; generic: W = 4) takes every digit
    -2^(W-1)..2^(W-1) in every window where some u2 < n can take it, in a few hundred rows; the windows below the top
    take all 2^W + 1 of them."""
    u2s = ek.window_sweep_u2(curve, W, seed=W + curve)
    reach = ek.reachable_digits(curve, W)
    nwin, half = ek.windows(curve, W), 1 << (W - 1)
    assert nwin == {(0, 8): 33, (1, 8): 49, (1, 5): 77, (0, 4): 65, (1, 4): 97}[(curve, W)]
    for win in range(1, nwin - 2):
        assert {d for w, d in reach if w == win} == set(range(-half, half + 1)), win
    assert {d for w, d in reach if w == 0} == set(range(-half, half))      # bit -1 is zero: no +2^(W-1) at the bottom
    assert len(u2s) <= 4 * half + 16


def test_comb_sweep_covers_every_mask():
    u2s = ek.comb_sweep_u2(seed=1)
    assert len(u2s) == 255


@pytest.mark.parametrize("curve", [0, 1])
def test_encoding_cases(curve):
    """The edge encodings have a small coordinate where the case needs one, and each carries a signature that accepts
    under the canonical key and rejects under the encoding (the reference verifier)."""
    b, want, labels = ek.encoding_batch(curve, seed=5)
    assert len(labels) >= 16
    rows = zip(*(b[k] for k in ("r", "s", "qx", "qy", "digest")))
    got = np.array([ref.verify_bytes(curve, *(bytes(v) for v in row)) for row in rows], np.uint8)
    assert np.array_equal(got, want)


def _kg_hash(hs, curve, qx, qy, seed):
    out = np.zeros(qx.shape[0], np.uint32)
    assert hs.hs_kg_hash(C.c_int(curve), C.c_size_t(qx.shape[0]), _p8(qx), _p8(qy), C.c_uint32(seed), out.ctypes.data_as(C.POINTER(C.c_uint32))) == 0
    return out


@pytest.mark.parametrize("curve", [0, 1])
def test_kg_hash_reads_every_word(hs, curve):
    """kg_hash gives keys that differ from a valid key only in x's odd words (which it once skipped: every such key
    shared one probe start for every seed, and k_kg_insert took O(n^2) probes), the same keys with x and y swapped, and
    keys that differ in bit 31 of one word of x and of the same word of y (a difference one multiplication passes
    unchanged, so the next word could cancel it) distinct values, and spreads their probe starts, for every seed tried."""
    c = ref.CURVES[curve]
    L = c.size
    Q = ek._point(curve, 0xC0FFEE + curve)
    qx, qy = ek.colliding_keys(curve, Q, 4096)
    sets = [(qx, qy), (qy.copy(), qx.copy())]                                # the same words of y (in x's place)
    tx, ty = np.tile(ek._be(Q[0], L), (L // 4, 1)), np.tile(ek._be(Q[1], L), (L // 4, 1))
    for w in range(L // 4):                                                  # bit 31 of word w of x and of y
        tx[w, 4 * w] ^= 0x80
        ty[w, 4 * w] ^= 0x80
    sets.append((tx, ty))
    for seed in (0x9E3779B9, 1, 0xDEADBEEF):
        for sx, sy in sets:
            h = _kg_hash(hs, curve, np.ascontiguousarray(sx), np.ascontiguousarray(sy), seed)
            assert np.unique(h).size >= sx.shape[0] * 0.99, (seed, np.unique(h).size)
            assert np.unique(h & 8191).size >= min(sx.shape[0], 8192) * 0.5        # the probe starts spread too


@pytest.mark.parametrize("curve", [0, 1])
def test_warp_tree_exceptional_sums(hs, curve):
    """Partial sums of k_verify_kt_warp's shuffle tree that are equal (the general addition doubles) or opposite (an
    infinity the levels above carry, up to R = infinity at the last level), at every level: the simulated warp kernel
    (32 lanes in lockstep) and thread kernel give the verdicts of the construction and of the oracle.  The simulation
    builds P-384's table of G with 8-bit windows, so its lane sums are modelled with GW = 8."""
    from test_hostsim import _registered
    b, want, events = ek.warp_tree_batch(curve, seed=200 + curve, GW=16 if curve == 0 else 8)
    assert {e[0] for e in events} == set(ek.TREE) and want.sum() and not want.all()
    assert np.array_equal(oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"]), want)
    for warp in (1, 0):
        got = _registered(hs, curve, b, warp)
        assert np.array_equal(got, want), (warp, [events[i] for i in np.nonzero(got != want)[0][:6]])
