"""The per-key comb tables of the key-grouped P-256 path (CombTab, k_comb_affine / k_comb_fill, k_verify_comb) in the CPU
simulation of the device code (tools/hostsim): table entries against Python integers, and verdicts against the oracle
on scalars crafted for the comb's order of additions and doublings."""
import ctypes as C

import numpy as np
import pytest

import edges
import oracle
from oracle import corpus
from oracle import ecdsa_ref as ref
from test_hostsim import _p8, _verify, hs  # noqa: F401  (hs: the simulation library fixture)

COMB = 2  # hs_tables / hs_ktab_words: table kind of the comb


def _comb_tables(hs, curve, kxy, four):
    L = 32 if curve == 0 else 48
    n = kxy.shape[0]
    qx, qy = np.ascontiguousarray(kxy[:, :L]), np.ascontiguousarray(kxy[:, L:])
    hs.hs_ktab_words.restype = C.c_size_t
    words = hs.hs_ktab_words(C.c_int(curve), C.c_int(COMB), C.c_size_t(n))
    kt, fl = np.zeros(words, np.uint32), np.zeros(n, np.uint8)
    assert hs.hs_tables(C.c_int(curve), C.c_int(COMB), C.c_size_t(n), _p8(qx), _p8(qy), C.c_int(four), kt.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(fl)) == 0
    return kt, fl


@pytest.mark.parametrize("curve", [0])
def test_comb_entries_match_python_integers(hs, curve):
    """Every entry T_b[m] = sum over the set bits t of m of 2^(SPACING*(8b+t)) * Q, affine Montgomery form, at its slot
    (chain (b, m >> 4), Gray-code position of m & 15); the bases by the four-lane and the one-thread doubling chain give
    bit-identical tables; an off-curve key and a key with x >= p get no table."""
    cv = oracle.P256 if curve == 0 else oracle.P384
    c = ref.CURVES[cv]
    L, N = c.size, c.size // 4
    spacing = 8 * L // 16
    _, kxy = corpus.make_keys(cv, 5, seed=40 + curve)
    kxy = kxy.copy()
    kxy[1, L + 8] ^= 1                                                       # off the curve
    kxy[4, :L] = np.frombuffer(int(c.p + 2).to_bytes(L, "big"), np.uint8)    # x >= p
    a, fa = _comb_tables(hs, curve, kxy, four=0)
    b, fb = _comb_tables(hs, curve, kxy, four=1)
    assert fa.tolist() == fb.tolist() == [1, 0, 1, 1, 0]
    assert np.array_equal(a, b)
    Rm = 1 << (8 * L)
    val = lambda w: sum(int(x) << (32 * i) for i, x in enumerate(w))
    tabs = b.reshape(5, 2, 16, 16, 2, N)                                     # key, block, high nibble, Gray position, x/y
    for key in (0, 3):
        Q = (int.from_bytes(kxy[key, :L].tobytes(), "big"), int.from_bytes(kxy[key, L:].tobytes(), "big"))
        bases = [Q]
        for _ in range(15):
            bases.append(ref.scalar_mult(c, 1 << spacing, bases[-1]))
        for blk in range(2):
            for m in range(1, 256) if key == 0 else (1, 15, 16, 0xA5, 255):
                P = None
                for t in range(8):
                    if (m >> t) & 1:
                        P = ref._add(c, P, bases[8 * blk + t])
                g, k = m & 15, 0
                while (k ^ (k >> 1)) != g:
                    k += 1
                e = tabs[key, blk, m >> 4, k]
                assert (val(e[0]), val(e[1])) == (P[0] * Rm % c.p, P[1] * Rm % c.p), (key, blk, m)


@pytest.mark.parametrize("curve,thr", [(0, 1), (0, 2)])
def test_comb_order_exceptional_points(hs, curve, thr):
    """Every key gets a comb table (threshold 1 / 2) and k_gpart's point closes with one general addition: the oracle's
    verdicts when u1*G = +-u2*Q (the closing addition doubles or reaches infinity) or u1*G + u2*Q is one G comb entry,
    and when u2's masks are all ones or all zero."""
    b = edges.crafted(curve, edges.comb_cases(curve))
    want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert 0 < int(want.sum()) < want.size
    got, stats = _verify(hs, curve, b, grouped=(thr, 64))
    assert int(stats[2]) == 0                                   # nothing on the generic path
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]
