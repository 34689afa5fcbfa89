"""Proofs, run with exact integers, that the mutants tools/mutants.py marks `equivalent` cannot change a result: the
code they alter is dead or unreachable for every input the kernels can receive.  CPU only, no build needed."""
import random

import edges
from oracle import ecdsa_ref as ref

W32 = 1 << 32


def test_p256_redc_chains_a_and_b_never_carry_out():
    """P256::redc keeps V = T + M*2^96 + M*2^192 + M*2^256 - M*2^224 - M in 16 limbs plus t16.  Its inputs are products of
    a residue < p and a value < 2^256 (every fmul / fsqr call site), so T < p*2^256, and M < 2^256.  Then the partial sums
    after chain A (T + M*2^96) and after chain B (+ M*2^192) stay below 2^512: neither chain carries out of limb 15, and
    their carry captures (t16 = addc(0, 0), the first t16 = addc(t16, 0)) always read 0.  Only the + M*2^256 chain and
    the - M*2^224 chain move t16."""
    p = ref.CURVES[0].p
    T_max, M_max = p * 2**256 - 1, 2**256 - 1
    after_a = T_max + M_max * 2**96
    after_b = after_a + M_max * 2**192
    assert after_a < 2**512 and after_b < 2**512
    assert 2**512 - after_b > 2**478                     # not a near miss
    # and the two carries that do move: chain M*2^256 can carry out, chain C can borrow
    assert after_b + M_max * 2**256 >= 2**512


def test_mp_mul_row_carries_above_the_partial_product_are_zero():
    """mp_mul accumulates a*b row by row in E (limb k has weight 2^(32k)) and O (weight 2^(32(k+1))).  After row j each
    accumulator holds part of a * (b mod 2^(32(j+1))) < 2^(32(N+j+1)), so it has no bit at weight 2^(32(N+j+1)) or above.
    The carry of an even row's O chain lands in O[j+N] (weight 2^(32(N+j+1))) and that of an odd row's E chain in
    E[j+N+1] (the same weight): both are always 0, so dropping either addc changes nothing.  The carries one weight lower
    (E[j+N] of even rows, O[j+N-1] of odd rows) are live, and the model shows them set."""
    for N in (8, 12):
        for j in range(N):
            bound = 32 * (N + j + 1)                     # every accumulated value of rows 0..j is < 2^bound
            if j % 2 == 0:
                assert 32 * ((j + N) + 1) >= bound      # O[j+N]
            elif j + N + 1 < 2 * N:
                assert 32 * (j + N + 1) >= bound        # E[j+N+1]
        top = (1 << (32 * N)) - 1
        rng = random.Random(N)
        seen = {("E", 0): 0, ("O", 1): 0}
        for a, b in [(top, top)] + [(rng.getrandbits(32 * N), rng.getrandbits(32 * N)) for _ in range(300)]:
            for (acc, j), c in edges.mp_mul_row_carries(a, b, N).items():
                if (acc, j % 2) in (("O", 0), ("E", 1)):
                    assert c == 0, (N, acc, j)
                else:
                    seen[(acc, j % 2)] |= c
        assert seen == {("E", 0): 1, ("O", 1): 1}


def test_mp_sqr_off_diagonal_sum_leaves_the_top_limb_empty():
    """mp_sqr adds its off-diagonal accumulators into T = sum over i < j of a_i a_j 2^(32(i+j)) before doubling it.  That
    sum is below 2^(32(2N-1)), so T's top limb is 0 and the carry into it (the addc of the merge) is always 0."""
    for N in (8, 12):
        off_max = (W32 - 1) ** 2 * sum(1 << (32 * (i + j)) for i in range(N) for j in range(i + 1, N))
        assert off_max < 1 << (32 * (2 * N - 1))


def test_binary_gcd_pass_bound_and_reduced_cofactors():
    """mod_inv (curve.cuh) on u = a < m, v = m, both odd after the first strip:
      * a pass replaces the larger of (u, v) by (larger - smaller) / 2^tz with tz >= 1, so u + v at least halves:
        (u - v)/2 + v = (u + v)/2.  It starts below 2m and ends at 2 (u = v = 1), so there are at most
        log2(m) < 32N passes.  The 64N + 8 cap is never reached, and neither is a cap of 32N.
      * a strip step maps a cofactor x < m to (x + k*m) / 2^tz with k < 2^tz, which is < 2^tz * m / 2^tz = m; the other
        cofactor updates (mod_sub, m - x of a non-zero x) keep [0, m) too.  So the cofactor is always reduced, and the
        conditional subtraction after the shift (mp_select on bw == 0) never fires.
    The model (edges.mod_inv_model) follows the limb code; on edges.longest_inverse_inputs it needs exactly 32N - 1
    passes, the bound, and it asserts at every step that the cofactor is below m."""
    for curve in (0, 1):
        c = ref.CURVES[curve]
        N = c.size // 4
        for m in (c.n, c.p):
            assert m < 1 << (32 * N) and (2 * m).bit_length() - 1 <= 32 * N
            for tz in range(1, 32):
                assert (m - 1) + ((1 << tz) - 1) * m < (1 << tz) * m
            worst = edges.longest_inverse_inputs(m, N)
            assert worst
            for a in worst:
                x, passes = edges.mod_inv_model(a, m, N)
                assert x == pow(a, -1, m) and passes == 32 * N - 1
            rng = random.Random(curve)
            for a in [rng.randrange(1, m) for _ in range(200)] + [1, 2, m - 1, m - 2]:
                x, passes = edges.mod_inv_model(a, m, N)
                assert x == pow(a, -1, m) and passes < 32 * N


def test_r_zero_or_n_accepts_only_at_a_discrete_log():
    """Without k_prep's r != 0 (or with r <= n in place of r < n), r = 0 (or n) reaches the kernels with u2 = r/s = 0 mod n,
    so R = u1*G, and final_check accepts iff R != infinity and R.x = 0 mod n.  Since p < 2n, that is R.x in {0, n}: x = 0
    and x = n are on both curves exactly when x^3 - 3x + b is a square, and such a case needs u1 = log_G of one of those
    points — a discrete logarithm.  Otherwise (R.x mod n != 0, or R = infinity) the verdict is the same reject, so no
    feasible input tells the mutants apart; the suite's r = 0 and r = n rows reject either way."""
    for curve in (0, 1):
        c = ref.CURVES[curve]
        assert c.n < c.p < 2 * c.n
        roots = [x for x in (0, c.n) if edges._sqrt((x ** 3 - 3 * x + c.b) % c.p, c.p) is not None]
        for x in roots:                                 # points that exist, of unknown discrete log
            y = edges._sqrt((x ** 3 - 3 * x + c.b) % c.p, c.p)
            assert (y * y - (x ** 3 - 3 * x + c.b)) % c.p == 0


def test_comb_accumulator_never_equals_its_next_entry():
    """k_verify_comb hands pt_add_m's acc == entry case to its doubling site (DEFER).  That case never arises: before the
    addition of column j, block b, the accumulator is A*Q where A holds u2's bits of the columns already added, bit
    16r + j' of u2 moved to 16r + (j' - j) (j' > j; j' = j for block 0 when b = 1), a sum of distinct powers of two no
    larger than u2 < n; the entry is E*Q, E = sum of 2^(16(8b + t)) over the mask's teeth, also < n.  A = E mod n would
    need A = E, but A has no bit at the entry's positions (offset 0 in the rows of block b), so only A = E = 0 — a
    skipped entry.  Checked here over every (column, block): the position sets are disjoint and E stays below n."""
    n = ref.CURVES[0].n
    SP, TEETH = 16, 8
    for j in range(SP):
        for b in (0, 1):
            entry = {SP * (TEETH * b + t) for t in range(TEETH)}
            acc = {SP * r + (jj - j) for r in range(2 * TEETH) for jj in range(j + 1, SP)}
            if b == 1:
                acc |= {SP * t for t in range(TEETH)}
            assert not entry & acc, (j, b)
            assert sum(1 << q for q in entry) < n and all(q < 256 for q in acc)


def test_sc_reduce512_ninth_limb_is_zero():
    """sc_reduce512 subtracts L from t = x - q3*L over nine limbs.  t < B*L with B < 1.2250 (the Barrett bound,
    ed25519_arith.barrett_bound), so t < 2^256 and its ninth limb is 0: the borrow out of that limb (0 - 0 - b) is the
    borrow b out of the eighth, and skipping the limb's subtraction changes nothing."""
    import ed25519_arith as arith
    L = 2**252 + 27742317777372353535851937790883648493
    B = arith.barrett_bound()
    assert B * L < 2**256
