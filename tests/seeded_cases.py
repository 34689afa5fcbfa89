"""Scalars for the first addition of each fixed-base pass, which the kernels load instead of add because the accumulator
starts at infinity: k_gpart seeds from u1's comb digit 0 of G, k_verify_comb from the mask of its step 0 (block 0, top
column of u2's comb), and the registered-key k_verify_kt from u2's Booth digit 0 (8-bit windows).  A digit or mask of 0
must leave the accumulator at infinity, and a negative Booth digit must seed the negated entry."""
import numpy as np

import edges
from oracle import ecdsa_ref as ref


def comb_mask(curve, u2, b, j):
    """the mask of column j, block b of u2's comb (CombTab: 16 rows of SPACING bits, 8 teeth per block)"""
    sp = 8 * ref.CURVES[curve].size // 16
    return sum(((u2 >> (sp * (8 * b + t) + j)) & 1) << t for t in range(8))


def first_comb_bits(curve, b):
    """the bits of u2 that make the first mask of block b (column SPACING - 1)"""
    sp = 8 * ref.CURVES[curve].size // 16
    return sum(1 << (sp * (8 * b + t) + sp - 1) for t in range(8))


def booth_digit0(u2, w=8):
    """u2's Booth digit 0 for w-bit signed windows (bit -1 is 0)"""
    v = (u2 << 1) & ((2 << w) - 1)
    d = (((2 << w) - 1 - v) if v >> w else v) + 1 >> 1
    return -d if v >> w else d


def seeded_cases(curve, seed):
    """(u1, u2, k) for Q = k*G:
    - u1 with comb digit 0 of G equal to 0, and u1 = 0 and n - 1;
    - u2 with the first comb mask of block 0 (step 0, seeded), of block 1 (step 1, the first one added) or of both equal
      to 0, and u2 = 1 and n - 1 (u2 = 0 has no signature: s = r / u2);
    - u2 with Booth digit 0 equal to 0, to the most negative digit, to -1 and to positive digits;
    - a key whose first comb entry is the first G entry u1*G starts from: Q = d*G, u2's step-0 mask 1, u1's digit 0 = d."""
    c = ref.CURVES[curve]
    n, L = c.n, c.size
    rng = np.random.default_rng(seed)
    rand = lambda: int.from_bytes(rng.bytes(L + 8), "big") % (n - 1) + 1
    key = lambda: int.from_bytes(rng.bytes(12), "big") + 2
    lo16 = (1 << 16) - 1
    cases = []
    for u1 in (rand() & ~lo16, (rand() & ~lo16) | (1 << 16), 0, n - 1):
        cases.append((u1, rand(), key()))
    m0, m1 = first_comb_bits(curve, 0), first_comb_bits(curve, 1)
    for clear in (m0, m1, m0 | m1):
        for u1 in (rand(), rand() & ~lo16):
            cases.append((u1, rand() & ~clear or 1, key()))
    for u2 in (1, n - 1):
        cases.append((rand(), u2, key()))
        cases.append((0, u2, key()))
    for low in (0x00, 0x80, 0xFF, 0x7F, 0x01, 0x40):
        cases.append((rand(), (rand() & ~0xFF) | low, key()))
    for d in (5, 0xFFFF):
        u2 = (rand() & ~m0) | (1 << (8 * L // 16 - 1))               # step 0: mask 1, the entry is Q itself
        cases.append(((rand() & ~lo16) | d, u2, d))
        cases.append((d, u2, d))
    assert all(0 <= u1 < n and 0 < u2 < n for u1, u2, _ in cases)
    return cases


def seeded_batch(curve, seed):
    """the cases as signatures, each followed (as a second half) by a copy with r + 1 that must reject"""
    return edges.with_bumped_r(edges.crafted(curve, seeded_cases(curve, seed)))
