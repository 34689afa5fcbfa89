#!/usr/bin/env python3
"""Mutation survey of the device code on the CPU simulation (tools/hostsim) — test infrastructure.

Each catalogue entry names one deliberate fault in a device header: an exact source snippet that occurs exactly once in
its file, its replacement, and the CPU-simulation test files that cover the file.  The runner copies the files git
tracks (`git ls-files`, plus untracked files that are not ignored, so that uncommitted tests take part) into a temporary
directory, applies one mutant there, builds libhostsim.so and runs `pytest -m "not gpu" -x` on the mapped files.  A
mutant is

    killed       a test failed (the row names the first one) or the simulation did not build
    survived     every mapped test passed: the suite is blind to this fault
    equivalent   the entry carries `equivalent: <reason>` and names the test that proves it; it is not run
    timeout      the build or the tests ran past the limit
    stale        the snippet no longer occurs exactly once (tests/test_mutant_catalogue.py checks this without building)

The checkout is never modified, and nothing here runs on a GPU: a mutated kernel may index out of bounds or not
terminate, so mutants only ever run in the CPU simulation.

Not covered, because the CPU simulation does not compile it: the PTX branch of the carry primitives in mp.cuh (the
simulation emulates the carry flag in C++) and every `#if defined(__CUDA_ARCH__)` block (warp-aggregated atomics of
k_kg_insert and k_kg_route), nor the re-check of key_cache_assoc.cuh's pin after a lost CAS, which only a concurrent
launch can reach (the simulation runs one warp at a time).

    python tools/mutants.py -j 8                 # the whole catalogue
    python tools/mutants.py --only final_check_pmn mod_inv_cap_32n
    python tools/mutants.py --list
"""
import argparse
import concurrent.futures as cf
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = "consensus_b200/csrc/"

# CPU-simulation test files by area, cheapest killers first (pytest -x stops at the first failure)
ECDSA = ["tests/test_hostsim.py", "tests/test_hostsim_key_tables.py", "tests/test_hostsim_comb.py"]
ED = ["tests/test_hostsim_ed25519_arith.py", "tests/test_hostsim_ed25519.py", "tests/test_hostsim_ed25519_edges.py",
      "tests/test_hostsim_ed25519_registered.py", "tests/test_hostsim_ed25519_grouped.py"]
MIXED = ["tests/test_hostsim_mixed.py"]
MIXED_KEYS = ["tests/test_hostsim_mixed_keys.py"]  # keys per item (k_mix_split<true>)
SHARDS = ["tests/test_hostsim_shards.py"]
WIDE = ["tests/test_hostsim_wide.py"]  # bit lengths, offsets and byte sums past 32 bits
SHA384 = ["tests/test_hostsim_sha384.py"]
KEY_CACHE = ["tests/test_hostsim_key_cache.py"]
KEY_CACHE_EVICT = ["tests/test_hostsim_key_cache_evict.py"]
SEEDED = ["tests/test_hostsim_seeded_passes.py"]
COMB_WARP = ["tests/test_hostsim_comb_warp.py"]  # the comb build a warp per key against the one-thread-per-chain reference  # the first entry of a pass loaded, not added (pt_seed)
TABLE_SHAPES = ["tests/test_hostsim_table_shapes.py"]
RSA = ["tests/test_hostsim_rsa.py"]  # rsa.cuh and k_sha512 (sha512_batch.cuh)
MIXED384 = ["tests/test_hostsim_mixed384.py"]  # k_mix_alg and k_sha2_sel (mixed_hash.cuh)  # every entry of the per-key tables at the key counts where the builds turn over


def M(id, file, find, repl, tests, equivalent=None, proof=None):
    return {"id": id, "file": CSRC + file, "find": find, "repl": repl, "tests": tests, "equivalent": equivalent, "proof": proof}


CATALOGUE = [
    # ---------------------------------------------------------------- mp.cuh: carries and borrows of the limb primitives
    M("mp_mul_even_row_carry", "mp.cuh", "E[j + N] = addc(E[j + N], 0);", "(void)0;", ECDSA + ED),
    M("mp_mul_even_row_odd_carry", "mp.cuh", "O[j + N] = addc(O[j + N], 0);", "(void)0;", ECDSA + ED,
      equivalent="after row j the odd accumulator is below 2^(32(N+j+1)), the weight of O[j+N]: the carry is always 0",
      proof="tests/test_mutant_proofs.py::test_mp_mul_row_carries_above_the_partial_product_are_zero"),
    M("mp_mul_odd_row_carry", "mp.cuh", "if (j + N + 1 < 2 * N) E[j + N + 1] = addc(E[j + N + 1], 0);", "(void)0;", ECDSA + ED,
      equivalent="after row j the even accumulator is below 2^(32(N+j+1)), the weight of E[j+N+1]: the carry is always 0",
      proof="tests/test_mutant_proofs.py::test_mp_mul_row_carries_above_the_partial_product_are_zero"),
    M("mp_mul_odd_row_odd_carry", "mp.cuh", "O[j + N - 1] = addc(O[j + N - 1], 0);", "(void)0;", ECDSA + ED),
    M("mp_mul_final_carry_in", "mp.cuh", "r[2 * N - 1] = addc(E[2 * N - 1], O[2 * N - 2]);", "r[2 * N - 1] = E[2 * N - 1] + O[2 * N - 2];", ECDSA + ED),
    M("mp_mul_mid_carry_chain", "mp.cuh", "for (int i = 2; i < 2 * N - 1; i++) r[i] = addc_cc(E[i], O[i - 1]);",
      "for (int i = 2; i < 2 * N - 1; i++) r[i] = add_cc(E[i], O[i - 1]);", ECDSA + ED),
    M("mp_sqr_even_row_carry", "mp.cuh", "if (i + jl + 2 < 2 * N) E[i + jl + 2] = addc(E[i + jl + 2], 0);", "(void)jl;", ECDSA + ED),
    M("mp_sqr_odd_row_carry", "mp.cuh", "if (i + jl + 1 < 2 * N) O[i + jl + 1] = addc(O[i + jl + 1], 0);", "(void)jl;", ECDSA + ED),
    M("mp_sqr_merge_carry", "mp.cuh", "T[2 * N - 1] = addc(E[2 * N - 1], O[2 * N - 2]);", "T[2 * N - 1] = E[2 * N - 1] + O[2 * N - 2];", ECDSA + ED,
      equivalent="the off-diagonal sum is below 2^(32(2N-1)): the top limb, and the carry into it, are always 0",
      proof="tests/test_mutant_proofs.py::test_mp_sqr_off_diagonal_sum_leaves_the_top_limb_empty"),
    M("mp_sqr_double_carry", "mp.cuh", "T[2 * N - 1] = addc(T[2 * N - 1], T[2 * N - 1]);", "T[2 * N - 1] = T[2 * N - 1] + T[2 * N - 1];", ECDSA + ED),
    M("mp_sqr_diagonal_carry", "mp.cuh", "for (int i = 1; i < N; i++) madc_wide_cc(T[2 * i], T[2 * i + 1], a[i], a[i]);",
      "for (int i = 1; i < N; i++) mad_wide_cc(T[2 * i], T[2 * i + 1], a[i], a[i]);", ECDSA + ED),
    M("mp_add_carry_out", "mp.cuh", "for (int i = 1; i < N; i++) r[i] = addc_cc(a[i], b[i]);\n    return addc(0, 0);",
      "for (int i = 1; i < N; i++) r[i] = addc_cc(a[i], b[i]);\n    return 0;", ECDSA + ED),
    M("mp_sub_borrow_out", "mp.cuh", "return subc(0, 0) & 1u;  // subc(0,0) = -borrow", "return 0;", ECDSA + ED),
    M("mp_sub_borrow_chain", "mp.cuh", "for (int i = 1; i < N; i++) r[i] = subc_cc(a[i], b[i]);",
      "for (int i = 1; i < N; i++) r[i] = sub_cc(a[i], b[i]);", ECDSA + ED),
    M("mp_lt_is_le", "mp.cuh", "return mp_sub<N>(t, a, b) != 0;", "return mp_sub<N>(t, b, a) == 0;", ECDSA + ED),
    M("mp_eq_low_limbs", "mp.cuh", "for (int i = 0; i < N; i++) o |= a[i] ^ b[i];", "for (int i = 0; i < N - 1; i++) o |= a[i] ^ b[i];", ECDSA + ED),
    M("mp_is_zero_low_limbs", "mp.cuh", "for (int i = 0; i < N; i++) o |= a[i];", "for (int i = 0; i < N - 1; i++) o |= a[i];", ECDSA + ED),
    M("mod_add_no_carry_term", "mp.cuh", "bool use_t = (c != 0) || (bw == 0);", "bool use_t = (bw == 0);", ECDSA),
    M("mod_add_no_compare", "mp.cuh", "bool use_t = (c != 0) || (bw == 0);", "bool use_t = (c != 0);", ECDSA),
    M("mod_sub_top_carry", "mp.cuh", "r[N - 1] = addc(d[N - 1], m[N - 1] & mask);", "r[N - 1] = d[N - 1] + (m[N - 1] & mask);", ECDSA),
    M("mod_sub_no_fix", "mp.cuh", "uint32_t mask = 0u - bw;", "uint32_t mask = 0u;", ECDSA),
    M("mp_mul_lo_top_carry", "mp.cuh", "r[N - 1] = addc(E[N - 1], O[N - 2]);", "r[N - 1] = E[N - 1] + O[N - 2];", ECDSA),
    M("mont_reduce_sos_carry_lo_1", "mp.cuh", "carry_lo = carry_lo ? 1u : 0u;", "carry_lo = 1u;", ECDSA),
    M("mont_reduce_sos_carry_lo_0", "mp.cuh", "carry_lo = carry_lo ? 1u : 0u;", "carry_lo = 0u;", ECDSA),
    M("mont_reduce_sos_top_carry", "mp.cuh", "top = addc(top, 0);", "(void)0;", ECDSA),
    M("mont_reduce_sos_no_top_term", "mp.cuh", "bool use_t = (top != 0) || (bw == 0);", "bool use_t = (bw == 0);", ECDSA),
    M("mont_reduce_sos_ge_is_gt", "mp.cuh", "uint32_t bw = mp_sub<N>(t, hi, m);\n    bool use_t",
      "uint32_t bw = mp_sub<N>(t, hi, m);\n    if (mp_eq<N>(hi, m)) bw = 1;\n    bool use_t", ECDSA),
    # ---------------------------------------------------------------- curve.cuh: P-256 / P-384 reductions, halving
    M("p256_redc_chain_a_carry", "curve.cuh", "t16 = addc(0, 0);", "t16 = 0;", ECDSA,
      equivalent="T < p*2^256 bounds the running sum after chain A below 2^512, so chain A never carries out",
      proof="tests/test_mutant_proofs.py::test_p256_redc_chains_a_and_b_never_carry_out"),
    M("p256_redc_chain_b_carry", "curve.cuh", "hi[7] = addc_cc(hi[7], 0);\n        t16 = addc(t16, 0);",
      "hi[7] = addc_cc(hi[7], 0);\n        t16 = t16;", ECDSA,
      equivalent="T < p*2^256 bounds the running sum after chain B below 2^512, so chain B never carries out",
      proof="tests/test_mutant_proofs.py::test_p256_redc_chains_a_and_b_never_carry_out"),
    M("p256_redc_m256_carry", "curve.cuh", "hi[7] = addc_cc(hi[7], m7);\n        t16 = addc(t16, 0);",
      "hi[7] = addc_cc(hi[7], m7);\n        t16 = t16;", ECDSA),
    M("p256_redc_chain_c_borrow", "curve.cuh", "t16 = subc(t16, 0);", "t16 = t16;", ECDSA),
    M("p256_redc_take_no_carry", "curve.cuh", "const uint32_t take = addc(t16, 0u);  // carry or t16 (never both)",
      "const uint32_t take = t16;", ECDSA),
    M("p256_redc_take_no_t16", "curve.cuh", "const uint32_t take = addc(t16, 0u);  // carry or t16 (never both)",
      "const uint32_t take = addc(0u, 0u);", ECDSA),
    M("p256_redc_m7_carry", "curve.cuh", "const uint32_t b7 = a7 + m1 + (m6 < m0 ? 1u : 0u);", "const uint32_t b7 = a7 + m1;", ECDSA),
    M("p256_redc_delta_limb6", "curve.cuh", "d[6] = addc_cc(hi[6], 0xfffffffeu);", "d[6] = addc_cc(hi[6], 0xffffffffu);", ECDSA),
    M("p256_fhalf_top_carry", "curve.cuh", "r[7] = __funnelshift_r(t[7], top, 1);", "r[7] = t[7] >> 1;", ECDSA),
    M("p384_fhalf_top_carry", "curve.cuh", "r[11] = __funnelshift_r(t[11], top, 1);", "r[11] = t[11] >> 1;", ECDSA),
    M("p384_redc_m11_term", "curve.cuh", "if (i == 0) acc += (int64_t)(uint64_t)m[11];", "(void)0;", ECDSA),
    M("p384_redc_m128_range", "curve.cuh", "if (k >= 4) acc -= (int64_t)(uint64_t)m[k - 4];", "if (k >= 5) acc -= (int64_t)(uint64_t)m[k - 4];", ECDSA),
    M("p384_redc_hi_m96_range", "curve.cuh", "if (i < 3) acc -= (int64_t)(uint64_t)m[9 + i];", "if (i < 2) acc -= (int64_t)(uint64_t)m[9 + i];", ECDSA),
    M("p384_redc_take_no_carry", "curve.cuh", "const uint32_t take = addc(t24, 0u);", "const uint32_t take = t24;", ECDSA),
    M("p384_redc_delta_limb4", "curve.cuh", "d[4] = addc_cc(hi[4], 1u);", "d[4] = addc_cc(hi[4], 0u);", ECDSA),
    # ---------------------------------------------------------------- curve.cuh: group law
    M("pt_double_no_halving", "curve.cuh", "C::fhalf(bb, t1);           // 8 Y^4", "mp_copy<N>(bb, t1);", ECDSA),
    M("pt_double_alpha_2x", "curve.cuh", "C::fadd(alpha, t1, alpha);  // 3 (X - delta)(X + delta)", "mp_copy<N>(alpha, t1);", ECDSA),
    M("pt_add_neg_select_swapped", "curve.cuh", "mp_select<N>(y2, neg, ny, y2_in);", "mp_select<N>(y2, neg, y2_in, ny);", ECDSA),
    M("pt_add_neg_dropped", "curve.cuh", "mp_select<N>(y2, neg, ny, y2_in);", "mp_copy<N>(y2, y2_in);", ECDSA),
    M("pt_add_doubling_without_r0", "curve.cuh", "if (h0 && r0 && !p_inf && !skip) {", "if (h0 && !p_inf && !skip) {", ECDSA),
    M("pt_add_no_doubling_branch", "curve.cuh", "if (h0 && r0 && !p_inf && !skip) {", "if (false) {", ECDSA),
    M("pt_add_inf_z_is_one", "curve.cuh", "az = MODE == 1 ? one[i] : z2[i];", "az = one[i];", ECDSA),
    M("pt_add_inf_ignores_neg", "curve.cuh", "uint32_t ax = x2[i], ay = y2[i]", "uint32_t ax = x2[i], ay = y2_in[i]", ECDSA),
    M("pt_add_skip_ignored_for_z", "curve.cuh", "P.Z[i] = skip ? P.Z[i] : nz;", "P.Z[i] = nz;", ECDSA),
    M("pt_add_mode2_no_z2", "curve.cuh", "if (MODE != 1) C::fmul(z3, z3, z2);", "if (MODE == 0) C::fmul(z3, z3, z2);", ECDSA),
    M("pt_madd_table_y_term", "curve.cuh", "C::fsub(P.Y, P.Y, t);\n    C::fmul(P.Z, P.Z, h);", "C::fmul(P.Z, P.Z, h);", ECDSA),
    # ---------------------------------------------------------------- curve.cuh: binary-GCD inverse
    M("mod_inv_cap_32n", "curve.cuh", "for (int pass = 0; pass < 64 * N + 8; pass++) {", "for (int pass = 0; pass < 32 * N; pass++) {", ECDSA,
      equivalent="u + v at least halves per pass, so no input needs more than 32N - 1 passes",
      proof="tests/test_mutant_proofs.py::test_binary_gcd_pass_bound_and_reduced_cofactors"),
    M("mod_inv_cap_short", "curve.cuh", "for (int pass = 0; pass < 64 * N + 8; pass++) {", "for (int pass = 0; pass < 32 * N - 2; pass++) {", ECDSA),
    M("mod_inv_strip_no_reduce", "curve.cuh", "mp_select<N>(x, bw == 0, d, x);", "(void)bw;", ECDSA,
      equivalent="a strip maps a cofactor below m to (x + k*m) / 2^tz < m (k < 2^tz): the subtraction never fires",
      proof="tests/test_mutant_proofs.py::test_binary_gcd_pass_bound_and_reduced_cofactors"),
    M("mod_inv_strip_top_word", "curve.cuh", "w[N] = (uint32_t)cy;", "w[N] = 0;", ECDSA),
    M("mod_inv_lt_swap_cofactor", "curve.cuh", "if (lt) { mp_sub<N>(t, M, xd); mp_copy<N>(xd, t); }  // x2 - x1", "(void)0;", ECDSA),
    M("mod_inv_initial_strip", "curve.cuh", "if ((u[0] & 1u) == 0u) strip(u, x1);", "(void)0;", ECDSA),
    M("f_inv_skip_top_bit", "curve.cuh", "for (int i = 32 * N - 1; i >= 0; i--) {", "for (int i = 32 * N - 2; i >= 0; i--) {", ECDSA),
    # ---------------------------------------------------------------- kernels.cuh
    M("final_check_pmn", "kernels.cuh", "if (!match && mp_lt<N>(r, pmn)) {", "if (!match) {", ECDSA),
    M("final_check_no_r_plus_n", "kernels.cuh", "if (!match && mp_lt<N>(r, pmn)) {", "if (false) {", ECDSA),
    M("load_digest_no_clamp", "kernels.cuh", "const int L = dlen < (uint32_t)C::BYTES ? (int)dlen : C::BYTES;", "const int L = (int)dlen;", ECDSA),
    M("load_digest_off_by_one", "kernels.cuh", "int pos = L - 1 - (4 * j + k);", "int pos = L - (4 * j + k);", ECDSA),
    M("comb_digit_u1_narrow", "kernels.cuh", "return (__ldg(uw + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & ((1u << C::GW) - 1u);",
      "return (__ldg(uw + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & ((1u << (C::GW - 1)) - 1u);", ECDSA),
    M("booth_digit_window0_top_bit", "kernels.cuh", "b = (__ldg(u2) << 1) & ((2u << W) - 1);", "b = (__ldg(u2) << 1) & ((1u << W) - 1);", ECDSA),
    M("booth_digit_no_high_word", "kernels.cuh", "const uint32_t hi = wd + 1 < N ?", "const uint32_t hi = wd + 1 < N - 1 ?", ECDSA),
    M("booth_digit_no_round", "kernels.cuh", "d = (d + 1) >> 1;", "d = d >> 1;", ECDSA),
    M("booth_digit_min_positive", "kernels.cuh", "return sign ? -(int)d : (int)d;", "return sign && d != (1u << (W - 1)) ? -(int)d : (int)d;", ECDSA),
    M("k_prep_r_zero", "kernels.cuh", "&& !mp_is_zero<N>(r) && mp_lt<N>(r, nmod);", "&& mp_lt<N>(r, nmod);", ECDSA,
      equivalent="with r = 0 the verifier accepts only if u1*G has x in {0, n}; building such a case is a discrete logarithm",
      proof="tests/test_mutant_proofs.py::test_r_zero_or_n_accepts_only_at_a_discrete_log"),
    M("k_prep_r_le_n", "kernels.cuh", "&& !mp_is_zero<N>(r) && mp_lt<N>(r, nmod);", "&& !mp_is_zero<N>(r) && !mp_lt<N>(nmod, r);", ECDSA,
      equivalent="with r = n the verifier accepts only if u1*G has x = n; building such a case is a discrete logarithm",
      proof="tests/test_mutant_proofs.py::test_r_zero_or_n_accepts_only_at_a_discrete_log"),
    M("k_prep_prefix_step", "kernels.cuh", "C::nmul(w, inv, pv);\n            C::nmul(inv, inv, m);", "C::nmul(w, inv, pv);", ECDSA),
    M("k_verify_coz_flags_ignored", "kernels.cuh", "&& flags[idx] != 0;\n        if (!good) { ok_out[idx] = 0; return; }\n        // forward",
      ";\n        if (!good) { ok_out[idx] = 0; return; }\n        // forward", ECDSA),
    M("k_verify_coz_entry1_y", "kernels.cuh", "y2[i] = e == 1 ? gy1 : sy;", "y2[i] = sy;", ECDSA),
    M("k_verify_coz_doublings", "kernels.cuh", "for (int k = 0; k < W; k++) pt_double<C>(acc);", "for (int k = 0; k < W - 1; k++) pt_double<C>(acc);", ECDSA),
    M("k_verify_coz_ratio_index", "kernels.cuh", "h[i] = SCR((5 + j + 1 - 2) * N + i);", "h[i] = SCR((5 + j - 2) * N + i);", ECDSA),
    M("load_key_no_y_range", "kernels.cuh", "bool good = mp_lt<N>(x, pmod) && mp_lt<N>(y, pmod);", "bool good = mp_lt<N>(x, pmod);", ECDSA),
    M("load_key_b_dropped", "kernels.cuh", "C::fadd(rhs, rhs, b);", "(void)b;", ECDSA),
    M("add_u1G_skip_ignored", "kernels.cuh", "pt_add<C, true>(acc, gx, gy, one, false, gb == 0);", "pt_add<C, true>(acc, gx, gy, one, false, false);", ECDSA),
    M("add_u1G_seed_zero_digit", "kernels.cuh", "pt_seed<C>(acc, sx, sy, false, sb == 0);", "pt_seed<C>(acc, sx, sy, false, false);", SEEDED + ECDSA),
    M("add_u1G_seed_window_added_again", "kernels.cuh", "constexpr int W0 = FROM_INF ? 1 : 0;", "constexpr int W0 = 0;", SEEDED + ECDSA),
    M("pt_seed_infinity_z", "curve.cuh", "P.Z[i] = skip ? 0u : one[i];", "P.Z[i] = one[i];", SEEDED + ECDSA),
    M("pt_seed_negation_ignored", "curve.cuh", "mp_select<N>(y, neg, ny, y_in);\n    }\n    C::get_one(one);", "mp_copy<N>(y, y_in);\n    }\n    C::get_one(one);",
      SEEDED + ECDSA),
    M("k_verify_kt_slot_range", "kernels.cuh", "kid = sl < n_slots ? kidmap[sl] : -1;", "kid = sl <= n_slots ? kidmap[sl] : -1;", ECDSA),
    M("k_verify_kt_entry_index", "kernels.cuh", "load_affine<C>(x, y, kt + ((size_t)w * KT::ENT + (e ? e - 1 : 0)) * EU4);",
      "load_affine<C>(x, y, kt + ((size_t)w * KT::ENT + (e > 1 ? e - 2 : 0)) * EU4);", ECDSA),
    M("comb_slot_gray", "kernels.cuh", "(g ^ (g >> 1) ^ (g >> 2) ^ (g >> 3));", "(g ^ (g >> 1));", ECDSA),
    M("comb_mask_tooth_stride", "kernels.cuh", "const int pos = CT::SPACING * (CT::TEETH * b + t) + j;", "const int pos = CT::SPACING * (CT::TEETH * b + t) + j + (t == 7);", ECDSA),
    M("k_verify_comb_defer_ignored", "kernels.cuh", "dbl = pt_add_m<A, 1, true>(acc, cx, cy, one, one, one, false, cskip) ? 1 : 0;",
      "dbl = 0; pt_add_m<A, 1, true>(acc, cx, cy, one, one, one, false, cskip);", ECDSA,
      equivalent="the comb accumulator and the entry it meets are distinct binary numbers below n: they never coincide",
      proof="tests/test_mutant_proofs.py::test_comb_accumulator_never_equals_its_next_entry"),
    M("k_verify_comb_seed_zero_mask", "kernels.cuh", "pt_seed<A>(acc, sx, sy, false, sskip);", "pt_seed<A>(acc, sx, sy, false, false);", SEEDED + ECDSA),
    M("k_verify_comb_loop_from_step_0", "kernels.cuh", "int s = 1, dbl = 0;", "int s = 0, dbl = 0;", SEEDED + ECDSA),
    M("k_verify_kt_seed_zero_digit", "kernels.cuh", "pt_seed<A>(acc, cx, cy, cneg, cskip);", "pt_seed<A>(acc, cx, cy, cneg, false);", SEEDED + ECDSA),
    M("k_verify_kt_seed_sign_ignored", "kernels.cuh", "pt_seed<A>(acc, cx, cy, cneg, cskip);", "pt_seed<A>(acc, cx, cy, false, cskip);", SEEDED + ECDSA),
    M("k_verify_kt_loop_from_window_0", "kernels.cuh", "        w0 = 1;\n", "        w0 = 0;\n", SEEDED + ECDSA),
    M("k_verify_comb_closing_skip", "kernels.cuh", "pt_add<C, false>(fin, g.X, g.Y, g.Z, false, mp_is_zero<N>(g.Z));",
      "pt_add<C, false>(fin, g.X, g.Y, g.Z, false, false);", ECDSA),
    M("k_verify_kt_warp_tree_flag", "kernels.cuh", "pt_add<C, false>(acc, x2, y2, z2, false, mp_is_zero<N>(z2));",
      "pt_add<C, false>(acc, x2, y2, z2, false, false);", ECDSA),
    M("k_verify_kt_warp_slot_range", "kernels.cuh", "int32_t local = sl < n_slots ? slot2local[sl] : -1;", "int32_t local = sl <= n_slots ? slot2local[sl] : -1;", ECDSA),
    # ---------------------------------------------------------------- keygroup.cuh: hash, assign, route, tables
    M("kg_hash_x_only", "keygroup.cuh", "h = kg_mix(h, __ldg(y + k));", "(void)y;", ECDSA),
    M("kg_same_key_x_only", "keygroup.cuh", "diff |= (__ldg(xi + k) ^ __ldg(xj + k)) | (__ldg(yi + k) ^ __ldg(yj + k));",
      "diff |= (__ldg(xi + k) ^ __ldg(xj + k));", ECDSA),
    M("kg_same_key_short", "keygroup.cuh", "for (int k = 0; k < C::N; k++) diff |=", "for (int k = 0; k < C::N - 1; k++) diff |=", ECDSA),
    M("kg_key32_same_short", "keygroup.cuh", "for (int k = 0; k < 8; k++) diff |= __ldg(xi + k) ^ __ldg(xj + k);",
      "for (int k = 0; k < 7; k++) diff |= __ldg(xi + k) ^ __ldg(xj + k);", ED),
    M("k_kg_insert_no_compare", "keygroup.cuh", "if (key.same(i, cur)) { r = cur; break; }", "if (true) { r = cur; break; }", ECDSA + ED),
    M("k_kg_assign_threshold_gt", "keygroup.cuh", "if (rep[i] == i && kcnt[i] >= threshold) {", "if (rep[i] == i && kcnt[i] > threshold) {", ECDSA + ED),
    M("k_kg_assign_le_max_keys", "keygroup.cuh", "if (k < max_keys) { id = (int32_t)k; keylist[k] = i; }", "if (k <= max_keys) { id = (int32_t)k; keylist[k] = i; }", ECDSA + ED),
    M("k_kg_assign_not_rep", "keygroup.cuh", "if (rep[i] == i && kcnt[i] >= threshold) {", "if (kcnt[rep[i]] >= threshold) {", ECDSA + ED),
    M("k_kg_route_own_id", "keygroup.cuh", "const int32_t kid = live ? keyid[rep[i]] : -1;", "const int32_t kid = live ? keyid[i] : -1;", ECDSA + ED),
    M("k_kt_bases4_level2_select", "keygroup.cuh", "mp_select<N>(a, role == 2, bb, a);", "mp_select<N>(a, role == 1, bb, a);", ECDSA),
    M("k_kt_fill_h2", "keygroup.cuh", "C::fadd(h, by, by);\n    pt_double<C>(P);", "mp_copy<N>(h, by);\n    pt_double<C>(P);", ECDSA),
    M("k_kt_fill_last_entry", "keygroup.cuh", "for (int e = 3; e <= KT::ENT; e++) {", "for (int e = 3; e < KT::ENT; e++) {", ECDSA),
    M("k_kt_inv_prefix", "keygroup.cuh", "C::fmul(zi, inv, pv);\n        C::fmul(inv, inv, z);\n#pragma unroll\n        for (int i = 0; i < N; i++) ztop[ZL::at(k, win, i, cap)] = zi[i];",
      "mp_copy<N>(zi, inv);\n        C::fmul(inv, inv, z);\n#pragma unroll\n        for (int i = 0; i < N; i++) ztop[ZL::at(k, win, i, cap)] = zi[i];", ECDSA),
    M("k_kt_final_ratio", "keygroup.cuh", "A::fmul(zi, zi, h);\n            mp_copy<N>(x, nx);", "mp_copy<N>(x, nx);", ECDSA),
    # k_comb_fill is the CPU simulation's reference for k_comb_fill_warp: the comparison of the two kills its mutants
    M("k_comb_fill_no_subtract", "keygroup.cuh", "sub = !(((kk ^ (kk >> 1)) >> tooth) & 1);", "sub = false;", COMB_WARP),
    M("k_comb_fill_high_teeth", "keygroup.cuh", "tooth = 4 + __ffs(rest) - 1;", "tooth = 3 + __ffs(rest) - 1;", COMB_WARP),
    M("k_comb_fill_warp_no_negate", "keygroup.cuh", "neg = !(((kk ^ (kk >> 1)) >> tooth) & 1);", "neg = false;", ECDSA + COMB_WARP),
    M("k_comb_fill_warp_high_teeth", "keygroup.cuh", "tooth = HT + __ffs(rest) - 1;", "tooth = HT - 1 + __ffs(rest) - 1;", ECDSA + COMB_WARP),
    M("k_comb_fill_warp_base_lane", "keygroup.cuh", "for (int i = 0; i < N; i++) pb[ch * N + i] = o[(size_t)i * cap];",
      "for (int i = 0; i < N; i++) pb[(ch ^ 1) * N + i] = o[(size_t)i * cap];", ECDSA + COMB_WARP),
    M("k_comb_fill_warp_ratio_slot", "keygroup.cuh", "for (int w = 0; w < Q; w++) h4[S::hs(k, slot, w) + ch] = quad<N>(h, w);",
      "for (int w = 0; w < Q; w++) h4[S::hs(k, slot, w) + ch] = quad<N>(x, w);", ECDSA + COMB_WARP),
    M("k_comb_final_ratio", "keygroup.cuh", "A::fmul(zi, zi, nh);", "(void)nh;", ECDSA + COMB_WARP),
    M("k_comb_final_transpose", "keygroup.cuh", "= stage[j * ROW + ch];", "= stage[ch * ROW + j];", ECDSA + COMB_WARP),
    # ---------------------------------------------------------------- sha256.cuh
    M("sha256_pad_rem", "sha256.cuh", "if (rem < 4) v = (v & (0xffffffffu << (8 * (4 - rem)))) | (0x80u << (8 * (3 - rem)));\n                } else if (p == len) {",
      "if (rem < 4) v = (v & (0xffffffffu << (8 * (4 - rem))));\n                } else if (p == len) {", ECDSA),
    M("sha256_pad_word", "sha256.cuh", "v = 0x80000000u;\n                }\n                w[j] = v;", "v = 0u;\n                }\n                w[j] = v;", ECDSA),
    M("sha256_nblocks", "sha256.cuh", "const uint64_t nblocks = (len + 9 + 63) / 64;", "const uint64_t nblocks = (len + 8 + 63) / 64;", ECDSA),
    M("sha256_length_bytes", "sha256.cuh", "const uint64_t bits = len * 8;", "const uint64_t bits = len;", ECDSA),
    M("sha256_aligned_tail_word", "sha256.cuh", "uint32_t next = (sh || j < 15) ? __ldg(words + blk * 16 + j + 1) : 0u;",
      "uint32_t next = (j < 15) ? __ldg(words + blk * 16 + j + 1) : 0u;", ECDSA),
    M("sha256_length_high_word", "sha256.cuh", "w[14] = (uint32_t)(bits >> 32);", "w[14] = 0u;", WIDE),
    M("sha256_bits_32", "sha256.cuh", "const uint64_t bits = len * 8;", "const uint64_t bits = (uint32_t)len * 8u;", WIDE),
    M("sha256_offset_32", "sha256.cuh", "const uint64_t o = off[idx] - base;", "const uint64_t o = (uint32_t)(off[idx] - base);", WIDE),
    # ---------------------------------------------------------------- sha512_core.cuh (SHA-512 and SHA-384)
    M("sha512_pad_rem", "sha512_core.cuh", "if (rem < 4) v = (v & (0xffffffffu << (8 * (4 - rem)))) | (0x80u << (8 * (3 - rem)));",
      "if (rem < 4) v = (v & (0xffffffffu << (8 * (4 - rem))));", SHA384 + ED),
    M("sha512_pad_word", "sha512_core.cuh", "v = 0x80000000u;", "v = 0u;", SHA384 + ED),
    M("sha512_aligned_tail_word", "sha512_core.cuh", "const uint32_t next = (sh || j < 15) ? __ldg(p + j + 1) : 0u;",
      "const uint32_t next = (j < 15) ? __ldg(p + j + 1) : 0u;", SHA384 + ED),
    # ---------------------------------------------------------------- sha384.cuh
    M("sha384_nblocks", "sha384.cuh", "const uint64_t nblocks = (len + 17 + 127) / 128;", "const uint64_t nblocks = (len + 16 + 127) / 128;", SHA384),
    M("sha384_second_half_offset", "sha384.cuh", "sha512_msg16(w32 + 16, blk * 128 + 64, len, words, sel, sh);",
      "sha512_msg16(w32 + 16, blk * 128 + 60, len, words, sel, sh);", SHA384),
    M("sha384_length_bytes", "sha384.cuh", "w[15] = len << 3;", "w[15] = len;", SHA384),
    M("sha384_bits_32", "sha384.cuh", "w[15] = len << 3;", "w[15] = (uint32_t)(len << 3);", SHA384),
    M("sha384_iv", "sha384.cuh", "0x47b5481dbefa4fa4ull", "0x5be0cd19137e2179ull", SHA384),
    # ---------------------------------------------------------------- sha512.cuh
    M("sha512_nblocks", "sha512.cuh", "const uint64_t nblocks = (total + 17 + 127) / 128;", "const uint64_t nblocks = (total + 16 + 127) / 128;", ED),
    M("sha512_length_bytes", "sha512.cuh", "if (blk == nblocks - 1) w[15] = total * 8;", "if (blk == nblocks - 1) w[15] = total;", ED),
    M("sha512_first_block_msg_offset", "sha512.cuh", "sha512_msg16(w32, blk * 128 - 64, len, words, sel, sh);", "sha512_msg16(w32, blk * 128 - 60, len, words, sel, sh);", ED),
    M("sha512_offset_32", "sha512.cuh", "const uint64_t o = off[idx] - base;", "const uint64_t o = (uint32_t)(off[idx] - base);", WIDE),
    M("sha512_total_32", "sha512.cuh", "const uint64_t total = 64 + len;  // bytes hashed", "const uint32_t total = 64 + len;  // bytes hashed", WIDE),
    # ---------------------------------------------------------------- ed25519.cuh
    M("fe_fold_second_fold", "ed25519.cuh", "r[0] = add_cc(r[0], (uint32_t)acc * 38u);", "r[0] = add_cc(r[0], 0u);", ED),
    M("fe_fold_wrap", "ed25519.cuh", "r[0] += 38u * c;  // after a wrap the value is < 38^2: no further carry", "(void)c;", ED),
    M("fe_add_wrap", "ed25519.cuh", "r[0] += 38u * addc(0, 0);", "(void)0;", ED),
    M("fe_add_carry", "ed25519.cuh", "r[0] = add_cc(r[0], 38u * c);", "r[0] = add_cc(r[0], 0u);", ED),
    M("fe_sub_wrap", "ed25519.cuh", "r[0] -= 38u * (subc(0, 0) & 1u);  // after a wrap the value is >= 2^256 - 38: no further borrow", "(void)0;", ED),
    M("fe_sub_borrow", "ed25519.cuh", "r[0] = sub_cc(r[0], 38u * bw);", "r[0] = sub_cc(r[0], 0u);", ED),
    M("fe_canon_bit255", "ed25519.cuh", "t[0] = add_cc(a[0], 19u * (a[7] >> 31));", "t[0] = add_cc(a[0], 0u);", ED),
    M("fe_canon_ge_p_minus_1", "ed25519.cuh", "u[0] = add_cc(t[0], 19u);  // t >= p  <=>  t + 19 >= 2^255", "u[0] = add_cc(t[0], 20u);", ED),
    M("fe_canon_ge_p_plus_1", "ed25519.cuh", "u[0] = add_cc(t[0], 19u);  // t >= p  <=>  t + 19 >= 2^255", "u[0] = add_cc(t[0], 18u);", ED),
    M("fe_sqrt_ratio_flipped_i", "ed25519.cuh", "if (flipped || flipped_i) mp_copy<8>(r, t);", "if (flipped) mp_copy<8>(r, t);", ED),
    M("fe_sqrt_ratio_even_root", "ed25519.cuh", "if (r[0] & 1u) mp_copy<8>(r, t);", "(void)0;", ED),
    M("fe_sqrt_ratio_ok_flipped_i", "ed25519.cuh", "return correct || flipped;", "return correct || flipped || flipped_i;", ED),
    M("ed_decode_y_high_bit", "ed25519.cuh", "y[7] &= 0x7fffffffu;\n    ed_one(one);", "ed_one(one);", ED),
    M("ed_decode_sign", "ed25519.cuh", "if (enc[7] >> 31) fe_neg(x, x);", "(void)0;", ED),
    M("ed_add_neg_no_swap", "ed25519.cuh", "fe_mul(A, s, neg ? ypx : ymx);", "fe_mul(A, s, ymx);", ED),
    M("ed_add_neg_no_fg_swap", "ed25519.cuh", "if (neg) { mp_copy<8>(F, G); mp_copy<8>(G, s); } else { mp_copy<8>(F, s); }", "mp_copy<8>(F, s);", ED),
    M("ed_double_c2", "ed25519.cuh", "fe_sqr(C, P.Z);\n    fe_add(C, C, C);", "fe_sqr(C, P.Z);", ED),
    M("ed_encode_parity", "ed25519.cuh", "enc[7] |= (x[0] & 1u) << 31;", "(void)x;", ED),
    M("sc_reduce512_final_sub", "ed25519.cuh", "for (int i = 0; i < 8; i++) r[i] = lt ? t[i] : u[i];", "for (int i = 0; i < 8; i++) r[i] = t[i];", ED),
    M("sc_reduce512_u8_borrow", "ed25519.cuh", "u[8] = subc_cc(t[8], 0);", "u[8] = t[8];", ED,
      equivalent="t < 1.225 L < 2^256, so the ninth limb is 0 and its borrow is the eighth limb's",
      proof="tests/test_mutant_proofs.py::test_sc_reduce512_ninth_limb_is_zero"),
    M("sc_lt_order_le", "ed25519.cuh", "return mp_lt<8>(s, Lm);", "return !mp_lt<8>(Lm, s);", ED),
    M("ed_digit4_no_carry_in", "ed25519.cuh", "return (int)(w & 7u) - (int)(w & 8u) + (int)prev;", "return (int)(w & 7u) - (int)(w & 8u);", ED),
    M("ed_digit8_no_carry_in", "ed25519.cuh", "const uint32_t prev = win ? (uint32_t)(__ldg(s + win - 1) >> 7) : 0u;", "const uint32_t prev = 0u;", ED),
    M("ed_digit8w_prev_bit", "ed25519.cuh", "const int pos = 8 * win - 1;", "const int pos = 8 * win - 2;", ED),
    M("ed_digit8w_sign", "ed25519.cuh", "const uint32_t w = (__ldg(k + (size_t)(win >> 2) * n + idx) >> (8 * (win & 3))) & 255u;\n    const int pos = 8 * win - 1;\n    const uint32_t prev = win ? (__ldg(k + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & 1u : 0u;\n    return (int)(w & 127u) - (int)(w & 128u) + (int)prev;",
      "const uint32_t w = (__ldg(k + (size_t)(win >> 2) * n + idx) >> (8 * (win & 3))) & 255u;\n    const int pos = 8 * win - 1;\n    const uint32_t prev = win ? (__ldg(k + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & 1u : 0u;\n    return (int)(w & 127u) + (int)prev;", ED),
    # ---------------------------------------------------------------- ed25519_verify.cuh / _keyed.cuh / _comb.cuh
    M("k_ed_verify_s_range", "ed25519_verify.cuh", "if (!sc_lt_order(s)) { ok_out[idx] = 0; return; }", "(void)s;", ED),
    M("k_ed_verify_key_neg", "ed25519_verify.cuh", "ed_add<true, false>(acc, ypx, ymx, t2d, z2, d > 0);  // d > 0: subtract d*A",
      "ed_add<true, false>(acc, ypx, ymx, t2d, z2, d < 0);", ED),
    M("k_ed_verify_doublings", "ed25519_verify.cuh", "ed_double<false>(acc);\n            ed_double<false>(acc);\n            ed_double<false>(acc);",
      "ed_double<false>(acc);\n            ed_double<false>(acc);", ED),
    M("k_ed_verify_b_neg", "ed25519_verify.cuh", "ed_add<true, true>(acc, ypx, ymx, t2d, ypx, d < 0);", "ed_add<true, true>(acc, ypx, ymx, t2d, ypx, false);", ED),
    M("k_ed_btab_top_bit", "ed25519_verify.cuh", "for (int b = top - 1; b >= 0; b--) {", "for (int b = top - 2; b >= 0; b--) {", ED),
    M("k_ed_verify_keyed_slot_range", "ed25519_keyed.cuh", "const int32_t loc = slot < n_slots ? __ldg(slot2local + slot) : -1;",
      "const int32_t loc = slot <= n_slots ? __ldg(slot2local + slot) : -1;", ED),
    M("k_ed_verify_keyed_neg", "ed25519_keyed.cuh", "const bool neg = key ? d > 0 : d < 0;", "const bool neg = d < 0;", ED),
    M("k_ed_verify_keyed_s_range", "ed25519_keyed.cuh", "if (!sc_lt_order(s)) { ok_out[idx] = 0; return; }", "(void)s;", ED),
    M("k_ed_ktab_first_entry", "ed25519_keyed.cuh", "if (j) ed_add<true, false>(P, base.ypx, base.ymx, base.t2d, base.z2, false);",
      "ed_add<true, false>(P, base.ypx, base.ymx, base.t2d, base.z2, false);", ED),
    M("edc_fill_subtract", "ed25519_comb.cuh", "add_base(EDC_TEETH * b + tooth, !((g >> tooth) & 1));  // the bit goes off: subtract",
      "add_base(EDC_TEETH * b + tooth, false);", ED),
    M("edc_fill_high_teeth", "ed25519_comb.cuh", "if ((hi >> i) & 1) add_base(EDC_TEETH * b + 4 + i, false);", "if ((hi >> i) & 1) add_base(EDC_TEETH * b + 3 + i, false);", ED),
    M("edc_final_first_slot", "ed25519_comb.cuh", "for (int s = EDC_CHAIN - 1; s >= (hi ? 0 : 1); s--) {", "for (int s = EDC_CHAIN - 1; s >= 1; s--) {", ED),
    M("edc_mask_high_row", "ed25519_comb.cuh", "m |= ((v >> (16 + j)) & 1u) << (2 * w + 1);", "(void)0;", ED),
    M("edc_verify_s_range", "ed25519_comb.cuh", "if (!sc_lt_order(s)) { ok_out[idx] = 0; return; }", "(void)s;", ED),
    M("edc_verify_doubling_step", "ed25519_comb.cuh", "if (key && step && (step & 1) == 0) ed_double<true>(acc);", "if (key && step && (step & 3) == 0) ed_double<true>(acc);", ED),
    # the grids and the [...][cap] scratch of the per-key builds: faults that damage only the keys past a block or a
    # chunk, or only a launch whose capacity is not its key count (test_hostsim_table_shapes.py runs those shapes).
    # The Ed25519 files alone kill each of these as well, through verdicts and the tables of a few keys
    # (test_hostsim_ed25519_grouped.py: the threshold test's launch of 4 slots for 3 keys, the crafted-k and pipeline
    # runs; test_hostsim_ed25519_registered.py: the tables of 4 keys and the chunked build)
    M("edc_bases_block_index", "ed25519_comb.cuh",
      "const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;\n    uint32_t nkeys = __ldg(nkeys_ptr);\n    if (nkeys > cap) nkeys = cap;\n    if (q >= nkeys) return;",
      "const uint32_t q = threadIdx.x;\n    uint32_t nkeys = __ldg(nkeys_ptr);\n    if (nkeys > cap) nkeys = cap;\n    if (q >= nkeys) return;", TABLE_SHAPES + ED),
    M("edc_inv_block_index", "ed25519_comb.cuh",
      "const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;\n    uint32_t nkeys = __ldg(nkeys_ptr);\n    if (nkeys > cap) nkeys = cap;\n    if (q >= nkeys || !keyflags[q]) return;",
      "const uint32_t q = threadIdx.x;\n    uint32_t nkeys = __ldg(nkeys_ptr);\n    if (nkeys > cap) nkeys = cap;\n    if (q >= nkeys || !keyflags[q]) return;", TABLE_SHAPES + ED),
    M("edc_fill_split_by_cap", "ed25519_comb.cuh", "const uint32_t q = t % nkeys, ch = t / nkeys;\n    if (!keyflags[q]) return;\n    const int b = (int)(ch >> 4), hi = (int)(ch & 15);\n    uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    EdP P;",
      "const uint32_t q = t % cap, ch = t / cap;\n    if (!keyflags[q]) return;\n    const int b = (int)(ch >> 4), hi = (int)(ch & 15);\n    uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    EdP P;", TABLE_SHAPES + ED),
    M("edc_final_split_by_cap", "ed25519_comb.cuh", "const uint32_t q = t % nkeys, ch = t / nkeys;\n    if (!keyflags[q]) return;\n    const int b = (int)(ch >> 4), hi = (int)(ch & 15);\n    uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    uint32_t inv[8], d2[8];",
      "const uint32_t q = t % cap, ch = t / cap;\n    if (!keyflags[q]) return;\n    const int b = (int)(ch >> 4), hi = (int)(ch & 15);\n    uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    uint32_t inv[8], d2[8];", TABLE_SHAPES + ED),
    M("edc_fill_table_mod_32", "ed25519_comb.cuh", "uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    EdP P;",
      "uint32_t *tab = ctab + (size_t)(q % 32) * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    EdP P;", TABLE_SHAPES + ED),
    M("edc_final_table_mod_32", "ed25519_comb.cuh", "uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    uint32_t inv[8], d2[8];",
      "uint32_t *tab = ctab + (size_t)(q % 32) * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;\n    uint32_t inv[8], d2[8];", TABLE_SHAPES + ED),
    M("edc_bases_stride_nkeys", "ed25519_comb.cuh", "        }\n        uint32_t *o = bases + (size_t)c * 32 * cap + q;",
      "        }\n        uint32_t *o = bases + (size_t)c * 32 * nkeys + q;", TABLE_SHAPES + ED),
    M("edc_hs_stride_nkeys", "ed25519_comb.cuh", "uint32_t *hp = hs + ((size_t)ch * EDC_CHAIN + s) * 8 * cap + q;\n#pragma unroll\n        for (int i = 0; i < 8; i++) { o[i] = P.X[i];",
      "uint32_t *hp = hs + ((size_t)ch * EDC_CHAIN + s) * 8 * nkeys + q;\n#pragma unroll\n        for (int i = 0; i < 8; i++) { o[i] = P.X[i];", TABLE_SHAPES + ED),
    M("edc_ztop_stride_nkeys", "ed25519_comb.cuh", "uint32_t *zp = ztop + (size_t)ch * 8 * cap + q;\n#pragma unroll\n    for (int i = 0; i < 8; i++) zp[(size_t)i * cap] = run[i];",
      "uint32_t *zp = ztop + (size_t)ch * 8 * nkeys + q;\n#pragma unroll\n    for (int i = 0; i < 8; i++) zp[(size_t)i * cap] = run[i];", TABLE_SHAPES + ED),
    M("edc_pref_stride_nkeys", "ed25519_comb.cuh", "uint32_t *pp = pref + (size_t)ch * 8 * cap + q;\n#pragma unroll\n        for (int i = 0; i < 8; i++) { z[i] = zp[(size_t)i * cap]; pp[(size_t)i * cap] = run[i]; }",
      "uint32_t *pp = pref + (size_t)ch * 8 * nkeys + q;\n#pragma unroll\n        for (int i = 0; i < 8; i++) { z[i] = zp[(size_t)i * cap]; pp[(size_t)i * cap] = run[i]; }", TABLE_SHAPES + ED),
    M("ed_ktab_key_split", "ed25519_keyed.cuh", "const uint32_t q = t % nkeys;", "const uint32_t q = t / ED_BWINS;", TABLE_SHAPES + ED),
    M("ed_ktab_window_major_tables", "ed25519_keyed.cuh", "uint32_t *out = tab + ((size_t)q * ED_BWINS + win) * ED_BENT * ED_BWORDS;",
      "uint32_t *out = tab + ((size_t)win * nkeys + q) * ED_BENT * ED_BWORDS;", TABLE_SHAPES + ED),
    M("ed_ktab_slots_contiguous", "ed25519_keyed.cuh", "const uint32_t *src = xy + (size_t)__ldg(slot_of + q) * 16;",
      "const uint32_t *src = xy + (size_t)(__ldg(slot_of) + q) * 16;", TABLE_SHAPES + ED),
    M("ed_ktab_grid_guard", "ed25519_keyed.cuh", "if (t >= T) return;\n    const uint32_t q = t % nkeys;", "if (t > T) return;\n    const uint32_t q = t % nkeys;", TABLE_SHAPES + ED),
    # ---------------------------------------------------------------- quorum.cuh
    M("quorum_ignores_signer", "quorum.cuh", "if (signer[v] != snd) return;", "(void)signer;", ECDSA),
    M("quorum_counts_self", "quorum.cuh", "if (self_id && self_id[inst] == snd) return;", "(void)self_id;", ECDSA),
    M("quorum_ignores_ok", "quorum.cuh", "if (!(digest_match[v] && (!ok || ok[v]))) return;", "if (!digest_match[v]) return;", ECDSA),
    M("quorum_ignores_digest", "quorum.cuh", "if (!(digest_match[v] && (!ok || ok[v]))) return;", "if (!(!ok || ok[v])) return;", ECDSA),
    M("quorum_burn_needs_signer", "quorum.cuh", "if (sender[j] == snd && signer[j] == snd) return;", "if (sender[j] == snd) return;", ECDSA),
    M("quorum_scan_other_instance", "quorum.cuh", "if (instance[j] - inst_base != inst) break;", "(void)0;", ECDSA),
    M("quorum_reached_gt", "quorum.cuh", "reached[i] = valid_count[i] >= threshold ? 1 : 0;", "reached[i] = valid_count[i] > threshold ? 1 : 0;", ECDSA),
    M("pack_bits_tail", "quorum.cuh", "const uint32_t bit = (i < n && ok[i]) ? 1u : 0u;", "const uint32_t bit = ok[i] ? 1u : 0u;", ECDSA),
    # ---------------------------------------------------------------- rsa.cuh: carries, final subtraction, range, encoding, exponent
    M("rsa_lazy_word_dropped", "rsa.cuh", "    if (g.l == 0) c = 0;", "    c = 0;", RSA),
    M("rsa_carry_propagate_ignored", "rsa.cuh", "const uint32_t cin = ((gen << 1) + prop) ^ prop;", "const uint32_t cin = gen << 1;", RSA),
    M("rsa_carry_out_of_top_dropped", "rsa.cuh", "const uint32_t top = ((cin >> 16) & 1) + rsa_from(g, czl, RSA_GROUP - 1);",
      "const uint32_t top = rsa_from(g, czl, RSA_GROUP - 1);", RSA),
    M("rsa_final_sub_ignores_top", "rsa.cuh", "if (top || !borrow) {", "if (!borrow) {", RSA),
    M("rsa_final_sub_ignores_borrow", "rsa.cuh", "if (top || !borrow) {", "if (top) {", RSA),
    M("rsa_borrow_propagate_ignored", "rsa.cuh", "const uint32_t bin = ((gen << 1) + prop) ^ prop;", "const uint32_t bin = gen << 1;", RSA),
    M("rsa_key_leading_byte_dropped", "rsa.cuh", "if (!(n0 & 1) || (ntop >> 24) == 0 || e < 2 || e > 0x7fffffffu) return false;",
      "if (!(n0 & 1) || e < 2 || e > 0x7fffffffu) return false;", RSA),
    M("rsa_key_e_lower_bound", "rsa.cuh", "if (!(n0 & 1) || (ntop >> 24) == 0 || e < 2 || e > 0x7fffffffu) return false;",
      "if (!(n0 & 1) || (ntop >> 24) == 0 || e < 1 || e > 0x7fffffffu) return false;", RSA),
    M("rsa_key_e_upper_bound", "rsa.cuh", "if (!(n0 & 1) || (ntop >> 24) == 0 || e < 2 || e > 0x7fffffffu) return false;",
      "if (!(n0 & 1) || (ntop >> 24) == 0 || e < 2) return false;", RSA),
    M("rsa_range_check_dropped", "rsa.cuh", "if (!rsa_sub(g, x, s, n)) return false;", "rsa_sub(g, x, s, n);", RSA),
    M("rsa_ff_run_short", "rsa.cuh", "else if (r < k - 2) v = 0xff;", "else if (r < k - 3) v = 0xff;", RSA),
    M("rsa_separator_byte", "rsa.cuh", "else if (r == tl) v = 0x00;", "else if (r == tl) v = 0xff;", RSA),
    M("rsa_digest_info_of_sha256", "rsa.cuh", "v = RSA_DIGEST_INFO[hash][tl - 1 - r];", "v = RSA_DIGEST_INFO[0][tl - 1 - r];", RSA),
    M("rsa_block_type_byte", "rsa.cuh", "else if (r == k - 2) v = 0x01;", "else if (r == k - 2) v = 0x02;", RSA),
    M("rsa_compare_lane_local", "rsa.cuh", "return rsa_bits(g, bad != 0) == 0;", "return bad == 0;", RSA),
    M("rsa_exp_multiply_bit", "rsa.cuh", "else if ((e >> i) & 1) mul = true;", "else if ((e >> i) & 2) mul = true;", RSA),
    M("rsa_exp_top_bit", "rsa.cuh", "int i = 30 - __clz((int)e);", "int i = 31 - __clz((int)e);", RSA),
    M("rsa_exp_square_skipped", "rsa.cuh", "if (mul) { mul = false; i--; }", "if (mul) { mul = false; i -= 2; }", RSA),
    M("rsa_r2_doublings", "rsa.cuh", "for (int i = 0; i < 33 * K - b + 1; i++) {", "for (int i = 0; i < 33 * K - b; i++) {", RSA),
    M("rsa_quotient_digit", "rsa.cuh", "const uint32_t q = rsa_from(g, t[0], 0) * ninv;", "const uint32_t q = t[0] * ninv;", RSA),
    # the bit length of N in rsa_r2 taken as 32K: wrong for every modulus whose top bit is clear
    M("rsa_r2_bit_length_32k", "rsa.cuh", "const int b = 32 * K - __clz((int)ntop);", "const int b = 32 * K;", RSA),
    M("rsa_resolve_lazy_word_lane", "rsa.cuh", "uint32_t c = rsa_from(g, czl, g.l ? g.l - 1 : 0)", "uint32_t c = rsa_from(g, czl, g.l > 1 ? g.l - 2 : 0)", RSA),
    # a byte-index slip confined to SHA-384 at 4096 bits: the whole verifications of test_hostsim_rsa.py skip that pair, the
    # edge classes run it
    M("rsa_encoding_byte_index_sha384_4096", "rsa.cuh", "const uint32_t r = 4 * (g.l * NL + j) + q;",
      "const uint32_t r = 4 * (g.l * NL + j) + (hash == 1 && NL == 8 ? q ^ 1 : q);", RSA),
    # an exponent whose bit 0 is clear ends on a squaring: only the even exponents of the edge classes reach it
    M("rsa_exp_last_square_dropped", "rsa.cuh", "while (i >= 0) {", "while (i > 0 || (i == 0 && (mul || (e & 1)))) {", RSA),
    # ---------------------------------------------------------------- sha512_batch.cuh
    M("sha512_batch_length_bytes", "sha512_batch.cuh", "w[15] = len << 3;", "w[15] = len;", RSA),
    M("sha512_batch_iv", "sha512_batch.cuh", "0x5be0cd19137e2179ull", "0x47b5481dbefa4fa4ull", RSA),
    # ---------------------------------------------------------------- mixed_hash.cuh
    M("mix_alg_tag_map", "mixed_hash.cuh", "tag[i] = (uint8_t)(wide ? t - MIX_TAG_SHA384 : t);", "tag[i] = (uint8_t)t;", MIXED384),
    M("mix_alg_flag", "mixed_hash.cuh", "sha384[i] = wide ? 1 : 0;", "sha384[i] = 0;", MIXED384),
    M("mix_alg_threshold", "mixed_hash.cuh", "const bool wide = t >= MIX_TAG_SHA384;", "const bool wide = t > MIX_TAG_SHA384;", MIXED384),
    M("sha2_sel_flag_by_shard_index", "mixed_hash.cuh", "if (sha384[idx[j]]) {", "if (sha384[j]) {", MIXED384),
    M("sha2_sel_p384_sha256_offset", "mixed_hash.cuh", "if (dlen == 48) *out++ = make_uint4(0u, 0u, 0u, 0u);", "if (dlen == 48) *out = make_uint4(0u, 0u, 0u, 0u);",
      MIXED384),
    M("sha2_sel_p384_sha256_zeros", "mixed_hash.cuh", "if (dlen == 48) *out++ = make_uint4(0u, 0u, 0u, 0u);", "if (dlen == 48) out++;", MIXED384),
    M("sha2_sel_p256_truncation", "mixed_hash.cuh", "if (dlen == 48)\n            out[2] =", "if (dlen >= 32)\n            out[2] =", MIXED384),
    M("sha2_sel_slot_width", "mixed_hash.cuh", "digest_out + (size_t)j * dlen);", "digest_out + (size_t)j * 48);", MIXED384),
    # ---------------------------------------------------------------- mixed.cuh
    M("mix_count_tile_end", "mixed.cuh", "const uint32_t lo = t * MIX_TILE, hi = n - lo < MIX_TILE ? n : lo + MIX_TILE;\n    for (uint32_t i = lo; i < hi; i++) {\n        const uint32_t f = tag[i];\n        const uint64_t len",
      "const uint32_t lo = t * MIX_TILE, hi = n - lo <= MIX_TILE ? n - 1 : lo + MIX_TILE;\n    for (uint32_t i = lo; i < hi; i++) {\n        const uint32_t f = tag[i];\n        const uint64_t len", MIXED),
    M("mix_scan_slack", "mixed.cuh", "start[1] = mix_align16(sb[0][T - 1] + 16);", "start[1] = mix_align16(sb[0][T - 1]);", MIXED),
    M("mix_scan_exclusive", "mixed.cuh", "uint32_t rc = sc[k][tid] - c[k];", "uint32_t rc = sc[k][tid];", MIXED),
    M("mix_scan_close_offsets", "mixed.cuh", "if (tid == 0) p.f[k].off[sc[k][T - 1]] = start[k] + sb[k][T - 1];", "(void)0;", MIXED),
    M("mix_split_rank_family", "mixed.cuh", "const uint32_t j = f == 0 ? rank[0] : f == 1 ? rank[1] : rank[2];", "const uint32_t j = f == 0 ? rank[0] : rank[1];", MIXED),
    M("mix_split_p384_width", "mixed.cuh", "mix_copy16(F.s + (size_t)j * 48, row + 48, 3);", "mix_copy16(F.s + (size_t)j * 48, row + 32, 3);", MIXED),
    M("mix_split_p384_qy_offset", "mixed.cuh", "mix_copy16(k.qy[1] + (size_t)j * 48, key96 + (size_t)i * 96 + 48, 3);",
      "mix_copy16(k.qy[1] + (size_t)j * 48, key96 + (size_t)i * 96 + 32, 3);", MIXED_KEYS),
    M("mix_split_p384_qy_width", "mixed.cuh", "mix_copy16(k.qy[1] + (size_t)j * 48, key96 + (size_t)i * 96 + 48, 3);",
      "mix_copy16(k.qy[1] + (size_t)j * 48, key96 + (size_t)i * 96 + 48, 2);", MIXED_KEYS),
    M("mix_split_ed_pub_width", "mixed.cuh", "mix_copy16(k.pub + (size_t)j * 32, key96 + (size_t)i * 96, 2);",
      "mix_copy16(k.pub + (size_t)j * 32, key96 + (size_t)i * 96, 1);", MIXED_KEYS),
    M("mix_compact_edge_bytes", "mixed.cuh", "const uint64_t a = lo > d ? lo : d, b = lo + 16 < d + len ? lo + 16 : d + len;",
      "const uint64_t a = lo > d ? lo : d, b = lo + 16 < d + len ? lo + 15 : d + len;", MIXED),
    M("mix_compact_family_bounds", "mixed.cuh", "const uint32_t f = g < m0 ? 0 : g < m0 + m1 ? 1 : 2, j = g - (f == 0 ? 0 : f == 1 ? m0 : m0 + m1);\n    const MixFamily F = mix_family(p, f);\n    const uint32_t i = F.idx[j];",
      "const uint32_t f = g < m0 ? 0 : g <= m0 + m1 ? 1 : 2, j = g - (f == 0 ? 0 : f == 1 ? m0 : m0 + m1);\n    const MixFamily F = mix_family(p, f);\n    const uint32_t i = F.idx[j];", MIXED),
    M("mix_ok_family_bounds", "mixed.cuh", "const uint32_t f = g < m0 ? 0 : g < m0 + m1 ? 1 : 2, j = g - (f == 0 ? 0 : f == 1 ? m0 : m0 + m1);\n    const MixFamily F = mix_family(p, f);\n    ok[F.idx[j]]",
      "const uint32_t f = g < m0 ? 0 : g < m0 + m1 ? 1 : 2, j = g - (f == 0 ? 0 : f == 1 ? m0 : m0);\n    const MixFamily F = mix_family(p, f);\n    ok[F.idx[j]]", MIXED),
    M("mix_count_bytes_32", "mixed.cuh", "uint64_t b[MIX_FAMILIES] = {0, 0, 0};\n    const uint32_t lo = t * MIX_TILE", "uint32_t b[MIX_FAMILIES] = {0, 0, 0};\n    const uint32_t lo = t * MIX_TILE", WIDE),
    M("mix_scan_bytes_32", "mixed.cuh", "uint64_t b[MIX_FAMILIES] = {0, 0, 0};\n    for (uint32_t t = lo; t < hi; t++)", "uint32_t b[MIX_FAMILIES] = {0, 0, 0};\n    for (uint32_t t = lo; t < hi; t++)", WIDE),
    M("mix_split_pos_32", "mixed.cuh", "uint64_t pos[MIX_FAMILIES];", "uint32_t pos[MIX_FAMILIES];", WIDE),
    M("mix_split_at_32", "mixed.cuh", "const uint64_t at = f == 0 ? pos[0]", "const uint32_t at = f == 0 ? pos[0]", WIDE),
    M("mix_compact_src_32", "mixed.cuh", "const uint64_t s = off[i] - base, len", "const uint64_t s = (uint32_t)(off[i] - base), len", WIDE),
    M("mix_compact_dst_32", "mixed.cuh", "d = F.off[j];", "d = (uint32_t)F.off[j];", WIDE),
    # ---------------------------------------------------------------- shards.h
    M("shard_range_hi", "shards.h", "const size_t lo = n * g / G, hi = n * (g + 1) / G;", "const size_t lo = n * g / G, hi = (n * (g + 1) + G - 1) / G;", SHARDS),
    M("batch_shards_words", "shards.h", "s.wv = std::max(s.wv, (s.vr[g].n + 31) / 32);\n    }\n    return s;\n}\n\n// Commit",
      "s.wv = std::max(s.wv, s.vr[g].n / 32);\n    }\n    return s;\n}\n\n// Commit", SHARDS),
    M("quorum_shards_trailing_votes", "shards.h", "const uint32_t *b = g == G - 1 ? instance + n_votes :", "const uint32_t *b = false ? instance + n_votes :", SHARDS),
    M("quorum_shards_instance_words", "shards.h", "s.wi = std::max(s.wi, (ir.n + 31) / 32);", "s.wi = std::max(s.wi, ir.n / 32);", SHARDS),
    M("unpack_reached_offset", "shards.h", "reached[s.ir[g].lo + i] = bit(w + s.wv, i);", "reached[s.ir[g].lo + i] = bit(w + s.wi, i);", SHARDS),
    # ---------------------------------------------------------------- key_cache.cuh
    M("kc_find_busy_hits", "key_cache.cuh", "if (s == ready && kc_same<W>(c, h, w)) return (int32_t)h;",
      "if ((s & ~3u) == (ready & ~3u) && kc_same<W>(c, h, w)) return (int32_t)h;", KEY_CACHE),
    M("kc_same_half_key", "key_cache.cuh", "for (int k = 0; k < W; k++) diff |= kc_ld(s + k) ^ w[k];", "for (int k = 0; k < W / 2; k++) diff |= kc_ld(s + k) ^ w[k];",
      KEY_CACHE),
    M("kc_lookup_no_clamp", "key_cache.cuh", "if (nk > kcap) nk = kcap;", "(void)0;", KEY_CACHE),
    M("kc_lookup_miss_id", "key_cache.cuh", "id = (int32_t)atomicAdd(lk + 0, 1u);", "id = (int32_t)atomicAdd(lk + 1, 1u);", KEY_CACHE),
    M("kc_lookup_hit_id", "key_cache.cuh", "id = (int32_t)(nk - 1 - atomicAdd(lk + 1, 1u));", "id = (int32_t)(nk - atomicAdd(lk + 1, 1u));", KEY_CACHE),
    M("kc_lookup_hit_flag", "key_cache.cuh", "keyflags[id] = 1;", "(void)0;", KEY_CACHE),
    M("kc_lookup_hit_count", "key_cache.cuh", "atomicAdd(c.stats + 2, 1ull);", "(void)0;", KEY_CACHE),
    M("kc_lookup_keylist", "key_cache.cuh", "lk[2 + id] = item;", "lk[2 + k] = item;", KEY_CACHE),
    M("kc_lookup_keyid", "key_cache.cuh", "keyid[item] = id;", "(void)0;", KEY_CACHE),
    M("kc_lookup_copy_stride", "key_cache.cuh", "for (uint32_t i = lane; i < tw4; i += 32) dst[i] = kc_ld(src + i);",
      "for (uint32_t i = lane; i < tw4; i += 64) dst[i] = kc_ld(src + i);", KEY_CACHE),
    M("kc_insert_invalid", "key_cache.cuh", "if (k >= m || !keyflags[k]) return;", "if (k >= m) return;", KEY_CACHE),
    M("kc_insert_miss_count", "key_cache.cuh", "atomicAdd(c.stats + 3, 1ull);", "(void)0;", KEY_CACHE),
    M("kc_claim_past_busy", "key_cache.cuh", "if ((s & 3u) == KC_BUSY) return -1;", "if ((s & 3u) == KC_BUSY) continue;", KEY_CACHE),
    M("kc_claim_other_fingerprint", "key_cache.cuh", "if ((s & ~3u) != fp) continue;", "(void)0;", KEY_CACHE),
    M("kc_claim_same_key", "key_cache.cuh", "if (kc_same<W>(c, h, w)) return -1;", "(void)0;", KEY_CACHE),
    M("kc_claim_full_pool", "key_cache.cuh", "if (*(const volatile unsigned long long *)c.stats >= c.cap) return -1;", "(void)0;", KEY_CACHE),
    M("kc_insert_pidx", "key_cache.cuh", "c.pidx[slot] = (uint32_t)at;", "c.pidx[slot] = 0;", KEY_CACHE),
    M("kc_insert_key_words", "key_cache.cuh", "for (int i = 0; i < KV::W; i++) kw[i] = w[i];", "for (int i = 1; i < KV::W; i++) kw[i] = w[i];", KEY_CACHE),
    M("kc_insert_pool_entry", "key_cache.cuh", "uint4 *dst = reinterpret_cast<uint4 *>(c.pool) + (size_t)at * tw4;",
      "uint4 *dst = reinterpret_cast<uint4 *>(c.pool) + (size_t)at;", KEY_CACHE),
    M("kc_insert_publish", "key_cache.cuh", "kc_store_release(c.state + slot, kc_fp<KV::W>(w, c.seed) | KC_READY);",
      "kc_store_release(c.state + slot, kc_fp<KV::W>(w, c.seed) | KC_BUSY);", KEY_CACHE),
    M("kc_insert_resident_count", "key_cache.cuh", "atomicAdd(c.stats + 1, 1ull);", "(void)0;", KEY_CACHE),
    # ---------------------------------------------------------------- key_cache_assoc.cuh
    M("kca_lookup_busy_candidate", "key_cache_assoc.cuh", "lane < KCA_WAYS && (s & ~KCA_PINS) == (fp | KC_READY));",
      "lane < KCA_WAYS && (s >> 32) == (fp >> 32));", KEY_CACHE_EVICT,
      equivalent="kca_pin re-reads the state word and pins only a READY word with the fingerprint: a BUSY candidate is a miss either way",
      proof="tests/test_hostsim_key_cache_evict.py::test_busy_way_is_a_miss_and_blocks_an_insert_of_its_fingerprint"),
    M("kca_pin_no_compare", "key_cache_assoc.cuh", "if (kca_same<W>(c, way, w)) return (int32_t)way;", "return (int32_t)way;", KEY_CACHE_EVICT),
    M("kca_pin_mismatch_kept", "key_cache_assoc.cuh", "atomicAdd(c.state + way, 0ull - KCA_PIN);  // refilled", "(void)0;  // refilled", KEY_CACHE_EVICT),
    M("kca_same_half_key", "key_cache_assoc.cuh", "for (int k = 0; k < W; k++) diff |= kc_ld(s + k) ^ w[k];",
      "for (int k = 0; k < W / 2; k++) diff |= kc_ld(s + k) ^ w[k];", KEY_CACHE_EVICT),
    M("kca_lookup_no_clamp", "key_cache_assoc.cuh", "if (nk > kcap) nk = kcap;", "(void)0;", KEY_CACHE_EVICT),
    M("kca_lookup_hit_id", "key_cache_assoc.cuh", "id = (int32_t)(nk - 1 - atomicAdd(lk + 1, 1u));", "id = (int32_t)(nk - atomicAdd(lk + 1, 1u));",
      KEY_CACHE_EVICT),
    M("kca_lookup_hit_flag", "key_cache_assoc.cuh", "keyflags[id] = 1;", "(void)0;", KEY_CACHE_EVICT),
    M("kca_lookup_no_stamp", "key_cache_assoc.cuh", "atomicMax(c.stamp + way, now);", "(void)0;", KEY_CACHE_EVICT),
    M("kca_lookup_hit_count", "key_cache_assoc.cuh", "atomicAdd(c.stats + 2, 1ull);", "(void)0;", KEY_CACHE_EVICT),
    M("kca_lookup_no_unpin", "key_cache_assoc.cuh", "        __threadfence();\n        atomicAdd(c.state + way, 0ull - KCA_PIN);\n    }",
      "        __threadfence();\n    }", KEY_CACHE_EVICT),
    M("kca_lookup_copy_stride", "key_cache_assoc.cuh", "for (uint32_t i = lane; i < tw4; i += 32) dst[i] = kc_ld(src + i);",
      "for (uint32_t i = lane; i < tw4; i += 64) dst[i] = kc_ld(src + i);", KEY_CACHE_EVICT),
    M("kca_insert_invalid", "key_cache_assoc.cuh", "if (k >= m || !keyflags[k]) return;", "if (k >= m) return;", KEY_CACHE_EVICT),
    M("kca_insert_miss_count", "key_cache_assoc.cuh", "if (lane == 0) atomicAdd(c.stats + 3, 1ull);", "(void)0;", KEY_CACHE_EVICT),
    M("kca_insert_past_busy", "key_cache_assoc.cuh", "(st == KC_BUSY || (st == KC_READY && kca_same<KV::W>(c, base + lane, w)));",
      "(st == KC_READY && kca_same<KV::W>(c, base + lane, w));", KEY_CACHE_EVICT),
    M("kca_insert_duplicate", "key_cache_assoc.cuh", "(st == KC_BUSY || (st == KC_READY && kca_same<KV::W>(c, base + lane, w)));",
      "(st == KC_BUSY);", KEY_CACHE_EVICT),
    M("kca_insert_evict_pinned", "key_cache_assoc.cuh", "if (lane < KCA_WAYS && st == KC_READY && (s & KCA_PINS) == 0) {",
      "if (lane < KCA_WAYS && st == KC_READY) {", KEY_CACHE_EVICT),
    M("kca_insert_evict_current", "key_cache_assoc.cuh", "if (a < now) age = a;", "age = a;", KEY_CACHE_EVICT),
    M("kca_insert_not_lru", "key_cache_assoc.cuh", "lo = o < lo ? o : lo;", "lo = o > lo && o != ~0ull ? o : lo;", KEY_CACHE_EVICT),
    M("kca_insert_evict_before_empty", "key_cache_assoc.cuh", "const unsigned pick = empty ? empty : __ballot_sync(",
      "const unsigned pick = !empty ? empty : __ballot_sync(", KEY_CACHE_EVICT),
    M("kca_insert_no_stamp", "key_cache_assoc.cuh", "c.stamp[way] = now;", "(void)0;", KEY_CACHE_EVICT),
    M("kca_insert_key_words", "key_cache_assoc.cuh", "for (int i = 0; i < KV::W; i++) kw[i] = w[i];", "for (int i = 1; i < KV::W; i++) kw[i] = w[i];",
      KEY_CACHE_EVICT),
    M("kca_insert_pool_entry", "key_cache_assoc.cuh", "uint4 *dst = reinterpret_cast<uint4 *>(c.pool) + (size_t)way * tw4;",
      "uint4 *dst = reinterpret_cast<uint4 *>(c.pool) + (size_t)way;", KEY_CACHE_EVICT),
    M("kca_insert_publish", "key_cache_assoc.cuh", "kca_store_release(c.state + way, fp | KC_READY);", "kca_store_release(c.state + way, fp | KC_BUSY);",
      KEY_CACHE_EVICT),
    M("kca_insert_counter", "key_cache_assoc.cuh", "atomicAdd(c.stats + (evict ? 4 : 1), 1ull);", "atomicAdd(c.stats + 1, 1ull);", KEY_CACHE_EVICT),
    M("kca_insert_give_up_count", "key_cache_assoc.cuh", "if (lane == 0 && !there) atomicAdd(c.stats + 5, 1ull);", "(void)0;", KEY_CACHE_EVICT),
    M("kca_set_index", "key_cache_assoc.cuh", "return __umulhi(kc_hash<W>(w, c.seed), c.sets) * KCA_WAYS;", "return 0;", KEY_CACHE_EVICT),
]


def tracked_files():
    out = subprocess.run(["git", "ls-files", "-z", "--cached", "--others", "--exclude-standard"], cwd=ROOT, check=True, capture_output=True).stdout
    return [f for f in out.decode().split("\0") if f]


def snippet_count(entry, root=ROOT):
    with open(os.path.join(root, entry["file"])) as f:
        return f.read().count(entry["find"])


def _copy_tree(dst):
    for rel in tracked_files():
        src = os.path.join(ROOT, rel)
        if not os.path.isfile(src):
            continue
        os.makedirs(os.path.dirname(os.path.join(dst, rel)), exist_ok=True)
        shutil.copy2(src, os.path.join(dst, rel))
    # the OpenSSL oracles are built from files no mutant touches: reuse them when they are already built
    for rel in ("oracle/liboracle.so", "oracle_ed25519/liboracle_ed25519.so"):
        if os.path.exists(os.path.join(ROOT, rel)):
            shutil.copy2(os.path.join(ROOT, rel), os.path.join(dst, rel))


def _first_failure(text):
    m = re.search(r"^(?:FAILED|ERROR) (\S+)", text, re.M)
    return m.group(1) if m else "pytest exit status"


def run_one(entry, timeout):
    if entry["equivalent"]:
        return "equivalent", entry["proof"], 0.0
    t0 = time.time()
    with tempfile.TemporaryDirectory(prefix="sbv-mutant-") as tmp:
        _copy_tree(tmp)
        path = os.path.join(tmp, entry["file"])
        with open(path) as f:
            src = f.read()
        if src.count(entry["find"]) != 1:
            return "stale", f"snippet occurs {src.count(entry['find'])} times", 0.0
        with open(path, "w") as f:
            f.write(src.replace(entry["find"], entry["repl"]))
        env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
        try:
            b = subprocess.run(["make", "-s", "-C", os.path.join(tmp, "tools", "hostsim"), "libhostsim.so"], capture_output=True, text=True,
                               timeout=timeout, env=env)
            if b.returncode != 0:
                return "killed", "build: " + (b.stderr.strip().splitlines() or ["make failed"])[0][:120], time.time() - t0
            left = max(1.0, timeout - (time.time() - t0))
            p = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "not gpu", "-p", "no:cacheprovider", *entry["tests"]],
                               cwd=tmp, capture_output=True, text=True, timeout=left, env=env)
        except subprocess.TimeoutExpired:
            return "timeout", f"> {timeout:.0f} s", time.time() - t0
        if p.returncode == 0:
            return "survived", "", time.time() - t0
        return "killed", _first_failure(p.stdout + p.stderr), time.time() - t0


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-j", type=int, default=os.cpu_count() or 1, help="mutants run in parallel")
    ap.add_argument("--timeout", type=float, default=900.0, help="seconds per mutant (build and tests)")
    ap.add_argument("--only", nargs="*", help="run these ids only")
    ap.add_argument("--list", action="store_true", help="print the catalogue and exit")
    a = ap.parse_args(argv)
    entries = CATALOGUE
    if a.only:
        unknown = set(a.only) - {e["id"] for e in CATALOGUE}
        if unknown:
            ap.error("unknown ids: " + " ".join(sorted(unknown)))
        entries = [e for e in CATALOGUE if e["id"] in a.only]
    if a.list:
        for e in entries:
            print(f"{e['id']:36s} {e['file'][len(CSRC):]:20s} {'equivalent' if e['equivalent'] else ' '.join(os.path.basename(t) for t in e['tests'])}")
        return 0
    t0 = time.time()
    results = {}
    with cf.ThreadPoolExecutor(max_workers=max(1, a.j)) as ex:
        futs = {ex.submit(run_one, e, a.timeout): e for e in entries}
        for fut in cf.as_completed(futs):
            e = futs[fut]
            results[e["id"]] = fut.result()
            status, detail, secs = results[e["id"]]
            print(f"{e['id']:36s} {e['file'][len(CSRC):]:20s} {status:10s} {secs:6.0f} s  {detail}", flush=True)
    counts = {}
    for e in entries:
        key = (e["file"][len(CSRC):], results[e["id"]][0])
        counts[key] = counts.get(key, 0) + 1
    print(f"\n{len(entries)} mutants in {time.time() - t0:.0f} s")
    for f in sorted({k[0] for k in counts}):
        print(f"  {f:20s} " + ", ".join(f"{s} {counts[(f, s)]}" for s in ("killed", "equivalent", "survived", "timeout", "stale") if (f, s) in counts))
    bad = [i for i, r in results.items() if r[0] in ("survived", "stale", "timeout")]
    if bad:
        print("not killed: " + " ".join(sorted(bad)))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
