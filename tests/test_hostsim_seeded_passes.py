"""The first addition of each fixed-base pass is a load (pt_seed), in the CPU simulation of the device code (tools/hostsim):
k_gpart seeds from u1's comb digit 0 of G, k_verify_comb from the mask of its step 0, the registered-key k_verify_kt from
u2's Booth digit 0.  Verdicts against the oracle on scalars that make those digits and masks 0, negative or equal to the
other pass's first entry, on every simulated path."""
import numpy as np
import pytest

import oracle
import seeded_cases
from oracle import ecdsa_ref as ref
from test_hostsim import _registered, _verify, hs  # noqa: F401  (hs: the simulation library fixture)


def test_the_cases_reach_what_they_are_named_for():
    """the crafted scalars do make the seeded digits and masks 0, negative and positive, for both block parities"""
    c = ref.CURVES[0]
    cases = seeded_cases.seeded_cases(0, seed=5)
    sp = 8 * c.size // 16
    assert any(u1 & 0xFFFF == 0 and u1 for u1, _, _ in cases)
    assert {0, c.n - 1} <= {u1 for u1, _, _ in cases} and {1, c.n - 1} <= {u2 for _, u2, _ in cases}
    masks = [(seeded_cases.comb_mask(0, u2, 0, sp - 1), seeded_cases.comb_mask(0, u2, 1, sp - 1)) for _, u2, _ in cases]
    assert (0, 0) in masks and any(a == 0 and b for a, b in masks) and any(a and b == 0 for a, b in masks)
    digits = {seeded_cases.booth_digit0(u2) for _, u2, _ in cases}
    assert {0, -128, -1, 1, 127} <= digits
    # Q = d*G with step 0's mask 1: the first comb entry is Q = d*G, u1's first G entry d*G
    assert any(k == u1 & 0xFFFF and seeded_cases.comb_mask(0, u2, 0, sp - 1) == 1 for u1, u2, k in cases)


@pytest.mark.parametrize("curve,seed", [(0, 5), (0, 6), (1, 7)])
def test_seeded_passes_match_the_oracle(hs, curve, seed):
    """The signatures accept and their copies with r + 1 reject, on the generic kernel, with a table for every key
    (threshold 1 and 2: k_gpart, then k_verify_comb for P-256 or k_verify_kt from k_gpart's point for P-384), and on the
    registered-key thread and warp kernels."""
    b = seeded_cases.seeded_batch(curve, seed)
    want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    m = want.size // 2
    assert want[:m].all() and not want[m:].any()
    assert np.array_equal(_verify(hs, curve, b), want), "generic"
    for thr in (1, 2):
        got, stats = _verify(hs, curve, b, grouped=(thr, 64))
        assert int(stats[2]) == 0
        assert np.array_equal(got, want), ("grouped", thr, np.nonzero(got != want)[0][:10])
    for warp in (0, 1):
        got = _registered(hs, curve, b, warp)
        assert np.array_equal(got, want), ("registered", warp, np.nonzero(got != want)[0][:10])
