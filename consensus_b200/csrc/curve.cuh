// curve.cuh — NIST prime curves (a = -3) in Montgomery form: field policies and Jacobian group law.
//
// A curve policy C provides: N (limbs), field ops fmul/fsqr/fadd/fsub on canonical residues in
// [0,p) (Montgomery form, R = 2^(32N)), scalar-field Montgomery product nmul, and constants.
// Everything is thread-private and register resident; callers choose where points live.
#pragma once
#include "curve_constants.h"
#include "mp.cuh"

namespace sbv {

// -------------------------------------------------------------------------------------------------
// P-256: p = 2^256 - 2^224 + 2^192 + 2^96 - 1.  -p^-1 mod 2^64 = 1, so Montgomery reduction needs
// no multiplications: per 64-bit step the quotient digit is the low limb pair itself and
// q*p = q*2^256 - q*2^224 + q*2^192 + q*2^96 - q is four shifted adds.
// -------------------------------------------------------------------------------------------------
struct Fe8 { uint32_t v[8]; };
static __device__ __noinline__ Fe8 p256_fmul_call(Fe8 a, Fe8 b);
static __device__ __noinline__ Fe8 p256_fsqr_call(Fe8 a);
static __device__ __noinline__ Fe8 p256_nmul_call(Fe8 a, Fe8 b);

struct P256 {
    static constexpr int N = 8;
    static constexpr int BYTES = 32;
    static constexpr int GW = 16;              // fixed-base comb window of G: 16 windows x 65536 entries (64 MB; H100's 50 MB L2 holds most of it)
    static constexpr int GWINS = 256 / GW;
    static constexpr uint32_t NINV = SBV_P256_NINV;
    static constexpr uint32_t PINV = SBV_P256_PINV;

    SBV_DEV static void get_p(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_P; mp_copy<8>(r, c); }
    SBV_DEV static void get_n(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_N; mp_copy<8>(r, c); }
    SBV_DEV static void get_one(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_ONE_P; mp_copy<8>(r, c); }
    SBV_DEV static void get_rr_p(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_RR_P; mp_copy<8>(r, c); }
    SBV_DEV static void get_b(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_B_MONT; mp_copy<8>(r, c); }
    SBV_DEV static void get_gx(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_GX_MONT; mp_copy<8>(r, c); }
    SBV_DEV static void get_gy(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_GY_MONT; mp_copy<8>(r, c); }
    SBV_DEV static void get_rr_n(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_RR_N; mp_copy<8>(r, c); }
    SBV_DEV static void get_one_n(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_ONE_N; mp_copy<8>(r, c); }
    SBV_DEV static void get_rrr_n(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_RRR_N; mp_copy<8>(r, c); }
    SBV_DEV static void get_rrr_p(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_RRR_P; mp_copy<8>(r, c); }
    SBV_DEV static void get_p_minus_n(uint32_t (&r)[8]) { const uint32_t c[8] = SBV_P256_P_MINUS_N; mp_copy<8>(r, c); }
    SBV_DEV static uint32_t p_minus_2_limb(int i) { const uint32_t c[8] = SBV_P256_P_MINUS_2; return c[i]; }
    SBV_DEV static uint32_t n_minus_2_limb(int i) { const uint32_t c[8] = SBV_P256_N_MINUS_2; return c[i]; }

    // T (16 limbs, < p*2^256) -> r = T * 2^-256 mod p, canonical.
    //
    // U = T + M*p must vanish mod 2^256.  With p = 2^256 - 2^224 + 2^192 + 2^96 - 1 write
    //   V = T + M*2^96 + M*2^192 - M*2^224,   U = V - M + M*2^256,
    // so the condition is M = V mod 2^256: limb k of M is limb k of V, and V's limb k only involves limbs < k of
    // M (the shifts are >= 3 limbs).  Limbs 0..2 of M are T's; the rest fall out of the low ends of the three
    // shifted chains.  The result is floor(V / 2^256) + M: four term-wise chains over the high half (49
    // instructions) instead of four digit-wise steps that each ripple to the top limb (72).
    SBV_DEV static void redc(uint32_t (&r)[8], uint32_t (&T)[16]) {
        const uint32_t m0 = T[0], m1 = T[1], m2 = T[2];
        uint32_t hi[8], t16;
        // chain A: + M*2^96 over limbs 3..10, ripple to the top
        const uint32_t m3 = add_cc(T[3], m0);
        const uint32_t m4 = addc_cc(T[4], m1);
        const uint32_t m5 = addc_cc(T[5], m2);
        const uint32_t a6 = addc_cc(T[6], m3);
        const uint32_t a7 = addc_cc(T[7], m4);
        hi[0] = addc_cc(T[8], m5);
        // limbs 6 and 7 of M also take the low ends of chains B and C; computed here with flag-free arithmetic
        // (the carry flag of chain A stays live), chains B and C redo those two limbs for their carries
        const uint32_t m6 = a6 + m0;
        const uint32_t b7 = a7 + m1 + (m6 < m0 ? 1u : 0u);
        const uint32_t m7 = b7 - m0;
        hi[1] = addc_cc(T[9], m6);
        hi[2] = addc_cc(T[10], m7);
#pragma unroll
        for (int i = 3; i < 8; i++) hi[i] = addc_cc(T[8 + i], 0);
        // chains A and B never carry out (T < p*2^256: tests/test_mutant_proofs.py), so these two captures read 0; they
        // stay because ptxas allocates registers differently without them (k_verify_kt 168 -> 155, k_comb_affine 120 -> 122)
        t16 = addc(0, 0);
        // chain B: + M*2^192 over limbs 6..13
        (void)add_cc(a6, m0);
        (void)addc_cc(a7, m1);
        hi[0] = addc_cc(hi[0], m2);
        hi[1] = addc_cc(hi[1], m3);
        hi[2] = addc_cc(hi[2], m4);
        hi[3] = addc_cc(hi[3], m5);
        hi[4] = addc_cc(hi[4], m6);
        hi[5] = addc_cc(hi[5], m7);
        hi[6] = addc_cc(hi[6], 0);
        hi[7] = addc_cc(hi[7], 0);
        t16 = addc(t16, 0);
        // + M*2^256
        hi[0] = add_cc(hi[0], m0);
        hi[1] = addc_cc(hi[1], m1);
        hi[2] = addc_cc(hi[2], m2);
        hi[3] = addc_cc(hi[3], m3);
        hi[4] = addc_cc(hi[4], m4);
        hi[5] = addc_cc(hi[5], m5);
        hi[6] = addc_cc(hi[6], m6);
        hi[7] = addc_cc(hi[7], m7);
        t16 = addc(t16, 0);
        // chain C: - M*2^224 over limbs 7..14
        (void)sub_cc(b7, m0);
        hi[0] = subc_cc(hi[0], m1);
        hi[1] = subc_cc(hi[1], m2);
        hi[2] = subc_cc(hi[2], m3);
        hi[3] = subc_cc(hi[3], m4);
        hi[4] = subc_cc(hi[4], m5);
        hi[5] = subc_cc(hi[5], m6);
        hi[6] = subc_cc(hi[6], m7);
        hi[7] = subc_cc(hi[7], 0);
        t16 = subc(t16, 0);
        // result = hi + t16*2^256 < 2p: subtract p iff it is >= p.  With delta = 2^256 - p = (1, 0, 0, F, F, F, E, 0) (limb 0
        // first; F = 2^32-1, E = F-1): hi + delta carries out of 256 bits exactly when hi >= p, and its low 256 bits are the
        // difference in both cases (t16 = 1: 2^256 + hi - p = hi + delta, which cannot carry because the result is < p).
        uint32_t d[8];
        d[0] = add_cc(hi[0], 1u);
        d[1] = addc_cc(hi[1], 0u);
        d[2] = addc_cc(hi[2], 0u);
        d[3] = addc_cc(hi[3], 0xffffffffu);
        d[4] = addc_cc(hi[4], 0xffffffffu);
        d[5] = addc_cc(hi[5], 0xffffffffu);
        d[6] = addc_cc(hi[6], 0xfffffffeu);
        d[7] = addc_cc(hi[7], 0u);
        const uint32_t take = addc(t16, 0u);  // carry or t16 (never both)
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = take ? d[i] : hi[i];
    }
    SBV_DEV static void fmul_inline(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
        uint32_t T[16];
        mp_mul<8>(T, a, b);
        redc(r, T);
    }
    SBV_DEV static void fsqr_inline(uint32_t (&r)[8], const uint32_t (&a)[8]) {
        uint32_t T[16];
        mp_sqr<8>(T, a);
        redc(r, T);
    }
    // Out of line on purpose: the whole verify loop then fits the instruction cache.  Operands and
    // result travel in registers (by-value struct ABI), so a call costs moves, not memory traffic.
    SBV_DEV static void fmul(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
        Fe8 x, y;
        mp_copy<8>(x.v, a); mp_copy<8>(y.v, b);
        Fe8 z = p256_fmul_call(x, y);
        mp_copy<8>(r, z.v);
    }
    SBV_DEV static void fsqr(uint32_t (&r)[8], const uint32_t (&a)[8]) {
        Fe8 x;
        mp_copy<8>(x.v, a);
        Fe8 z = p256_fsqr_call(x);
        mp_copy<8>(r, z.v);
    }
    // r = a/2 mod p
    SBV_DEV static void fhalf(uint32_t (&r)[8], const uint32_t (&a)[8]) {
        const uint32_t p[8] = SBV_P256_P;
        const uint32_t mask = 0u - (a[0] & 1u);
        uint32_t t[8];
        t[0] = add_cc(a[0], p[0] & mask);
#pragma unroll
        for (int i = 1; i < 8; i++) t[i] = addc_cc(a[i], p[i] & mask);
        const uint32_t top = addc(0, 0);
#pragma unroll
        for (int i = 0; i < 7; i++) r[i] = __funnelshift_r(t[i], t[i + 1], 1);
        r[7] = __funnelshift_r(t[7], top, 1);
    }
    SBV_DEV static void fadd(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
        const uint32_t p[8] = SBV_P256_P;
        mod_add<8>(r, a, b, p);
    }
    SBV_DEV static void fsub(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
        const uint32_t p[8] = SBV_P256_P;
        mod_sub<8>(r, a, b, p);
    }
    SBV_DEV static void nmul_inline(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
        const uint32_t n[8] = SBV_P256_N;
        const uint32_t ni[8] = SBV_P256_NINV_FULL;
        mont_mul_sos<8>(r, a, b, n, ni);
    }
    // out of line: k_prep is latency-bound, and with its scalar multiplications inlined it overflowed
    // the instruction cache (ncu: no_instruction was its top stall)
    SBV_DEV static void nmul(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
        Fe8 x, y;
        mp_copy<8>(x.v, a); mp_copy<8>(y.v, b);
        Fe8 z = p256_nmul_call(x, y);
        mp_copy<8>(r, z.v);
    }
};

static __device__ __noinline__ Fe8 p256_fmul_call(Fe8 a, Fe8 b) {
    Fe8 r;
    P256::fmul_inline(r.v, a.v, b.v);
    return r;
}
static __device__ __noinline__ Fe8 p256_fsqr_call(Fe8 a) {
    Fe8 r;
    P256::fsqr_inline(r.v, a.v);
    return r;
}
static __device__ __noinline__ Fe8 p256_nmul_call(Fe8 a, Fe8 b) {
    Fe8 r;
    P256::nmul_inline(r.v, a.v, b.v);
    return r;
}

// -------------------------------------------------------------------------------------------------
// P-384: generic word-serial Montgomery for both fields (12 limbs).
// -------------------------------------------------------------------------------------------------
struct Fe12 { uint32_t v[12]; };
struct Fe24 { uint32_t v[24]; };
static __device__ __noinline__ Fe12 p384_redc_call(Fe24 t);
static __device__ __noinline__ Fe12 p384_fmul_call(Fe12 a, Fe12 b);
static __device__ __noinline__ Fe12 p384_fsqr_call(Fe12 a);
static __device__ __noinline__ Fe12 p384_nmul_call(Fe12 a, Fe12 b);

struct P384 {
    static constexpr int N = 12;
    static constexpr int BYTES = 48;
#ifndef SBV_P384_GW
#define SBV_P384_GW 16
#endif
    // fixed-base comb of G: 24 windows x 65,536 entries = 151 MB, mostly in HBM (three times the L2, but the
    // gather of the next entry is in flight during the current addition and a P-384 addition takes microseconds);
    // 24 additions per verify instead of the 48 of an 8-bit comb.  The CPU simulation of tests/ builds an 8-bit one.
    static constexpr int GW = SBV_P384_GW;
    static constexpr int GWINS = 384 / GW;

    SBV_DEV static void get_p(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_P; mp_copy<12>(r, c); }
    SBV_DEV static void get_n(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_N; mp_copy<12>(r, c); }
    SBV_DEV static void get_one(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_ONE_P; mp_copy<12>(r, c); }
    SBV_DEV static void get_rr_p(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_RR_P; mp_copy<12>(r, c); }
    SBV_DEV static void get_b(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_B_MONT; mp_copy<12>(r, c); }
    SBV_DEV static void get_gx(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_GX_MONT; mp_copy<12>(r, c); }
    SBV_DEV static void get_gy(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_GY_MONT; mp_copy<12>(r, c); }
    SBV_DEV static void get_rr_n(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_RR_N; mp_copy<12>(r, c); }
    SBV_DEV static void get_one_n(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_ONE_N; mp_copy<12>(r, c); }
    SBV_DEV static void get_rrr_n(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_RRR_N; mp_copy<12>(r, c); }
    SBV_DEV static void get_rrr_p(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_RRR_P; mp_copy<12>(r, c); }
    static constexpr uint32_t NINV = SBV_P384_NINV;
    static constexpr uint32_t PINV = SBV_P384_PINV;
    SBV_DEV static void get_p_minus_n(uint32_t (&r)[12]) { const uint32_t c[12] = SBV_P384_P_MINUS_N; mp_copy<12>(r, c); }
    SBV_DEV static uint32_t p_minus_2_limb(int i) { const uint32_t c[12] = SBV_P384_P_MINUS_2; return c[i]; }
    SBV_DEV static uint32_t n_minus_2_limb(int i) { const uint32_t c[12] = SBV_P384_N_MINUS_2; return c[i]; }

    // p = 2^384 - 2^128 - 2^96 + 2^32 - 1 and -p^-1 = 1 mod 2^32.  U = T + M*p must vanish mod 2^384; with
    //   V = T + M*2^32 - M*2^96 - M*2^128,   U = V - M + M*2^384
    // that is M = V mod 2^384: limb k of M is limb k of V, which only involves limbs k-1, k-3, k-4 of M.  So the low half is
    // one pass over the limbs with a signed carry (each limb: T_k + m_{k-1} - m_{k-3} - m_{k-4} + carry — ptxas turns the
    // 64-bit sums into 3-input IADD3 with two carry predicates, ~5 instructions per limb), and the result is
    // floor(V / 2^384) + M, a second pass of the same shape.  No multiplications, ~130 instructions (the digit-serial form,
    // six 64-bit steps each rippling three chains to the top limb, took ~370).
    SBV_DEV static void redc(uint32_t (&r)[12], uint32_t (&T)[24]) {
        uint32_t m[12], hi[12];
        int64_t c = 0;
        m[0] = T[0];
#pragma unroll
        for (int k = 1; k < 12; k++) {
            int64_t acc = c + (int64_t)(uint64_t)T[k] + (int64_t)(uint64_t)m[k - 1];
            if (k >= 3) acc -= (int64_t)(uint64_t)m[k - 3];
            if (k >= 4) acc -= (int64_t)(uint64_t)m[k - 4];
            m[k] = (uint32_t)acc;
            c = acc >> 32;
        }
#pragma unroll
        for (int i = 0; i < 12; i++) {
            int64_t acc = c + (int64_t)(uint64_t)T[12 + i] + (int64_t)(uint64_t)m[i];
            if (i == 0) acc += (int64_t)(uint64_t)m[11];        // top limb of M*2^32
            if (i < 3) acc -= (int64_t)(uint64_t)m[9 + i];       // top limbs of M*2^96
            if (i < 4) acc -= (int64_t)(uint64_t)m[8 + i];       // top limbs of M*2^128
            hi[i] = (uint32_t)acc;
            c = acc >> 32;
        }
        const uint32_t t24 = (uint32_t)c;  // 0 or 1: the result is < 2p
        // subtract p iff the result is >= p: hi + delta carries out exactly then, delta = 2^384 - p = (1, F, F, 0, 1, 0, ...)
        uint32_t d[12];
        d[0] = add_cc(hi[0], 1u);
        d[1] = addc_cc(hi[1], 0xffffffffu);
        d[2] = addc_cc(hi[2], 0xffffffffu);
        d[3] = addc_cc(hi[3], 0u);
        d[4] = addc_cc(hi[4], 1u);
#pragma unroll
        for (int i = 5; i < 12; i++) d[i] = addc_cc(hi[i], 0u);
        const uint32_t take = addc(t24, 0u);
#pragma unroll
        for (int i = 0; i < 12; i++) r[i] = take ? d[i] : hi[i];
    }
    // The reduction is kept out of line behind the product: scheduled into the product's twelve carry chains, its
    // two-predicate additions overflow the predicate file and ptxas spills predicates through LOP3/P2R (+400 instructions).
    SBV_DEV static void redc_ool(uint32_t (&r)[12], const uint32_t (&T)[24]) {
        Fe24 t;
        mp_copy<24>(t.v, T);
        Fe12 z = p384_redc_call(t);
        mp_copy<12>(r, z.v);
    }
    SBV_DEV static void fmul_inline(uint32_t (&r)[12], const uint32_t (&a)[12], const uint32_t (&b)[12]) {
        uint32_t T[24];
        mp_mul<12>(T, a, b);
        redc_ool(r, T);
    }
    SBV_DEV static void fsqr_inline(uint32_t (&r)[12], const uint32_t (&a)[12]) {
        uint32_t T[24];
        mp_sqr<12>(T, a);
        redc_ool(r, T);
    }
    // out of line, operands in registers — same reason as P256::fmul
    SBV_DEV static void fmul(uint32_t (&r)[12], const uint32_t (&a)[12], const uint32_t (&b)[12]) {
        Fe12 x, y;
        mp_copy<12>(x.v, a); mp_copy<12>(y.v, b);
        Fe12 z = p384_fmul_call(x, y);
        mp_copy<12>(r, z.v);
    }
    SBV_DEV static void fsqr(uint32_t (&r)[12], const uint32_t (&a)[12]) {
        Fe12 x;
        mp_copy<12>(x.v, a);
        Fe12 z = p384_fsqr_call(x);
        mp_copy<12>(r, z.v);
    }
    SBV_DEV static void fhalf(uint32_t (&r)[12], const uint32_t (&a)[12]) {
        const uint32_t p[12] = SBV_P384_P;
        const uint32_t mask = 0u - (a[0] & 1u);
        uint32_t t[12];
        t[0] = add_cc(a[0], p[0] & mask);
#pragma unroll
        for (int i = 1; i < 12; i++) t[i] = addc_cc(a[i], p[i] & mask);
        const uint32_t top = addc(0, 0);
#pragma unroll
        for (int i = 0; i < 11; i++) r[i] = __funnelshift_r(t[i], t[i + 1], 1);
        r[11] = __funnelshift_r(t[11], top, 1);
    }
    SBV_DEV static void fadd(uint32_t (&r)[12], const uint32_t (&a)[12], const uint32_t (&b)[12]) {
        const uint32_t p[12] = SBV_P384_P;
        mod_add<12>(r, a, b, p);
    }
    SBV_DEV static void fsub(uint32_t (&r)[12], const uint32_t (&a)[12], const uint32_t (&b)[12]) {
        const uint32_t p[12] = SBV_P384_P;
        mod_sub<12>(r, a, b, p);
    }
    SBV_DEV static void nmul_inline(uint32_t (&r)[12], const uint32_t (&a)[12], const uint32_t (&b)[12]) {
        const uint32_t n[12] = SBV_P384_N;
        const uint32_t ni[12] = SBV_P384_NINV_FULL;
        mont_mul_sos<12>(r, a, b, n, ni);
    }
    SBV_DEV static void nmul(uint32_t (&r)[12], const uint32_t (&a)[12], const uint32_t (&b)[12]) {
        Fe12 x, y;
        mp_copy<12>(x.v, a); mp_copy<12>(y.v, b);
        Fe12 z = p384_nmul_call(x, y);
        mp_copy<12>(r, z.v);
    }
};

static __device__ __noinline__ Fe12 p384_redc_call(Fe24 t) {
    Fe12 r;
    P384::redc(r.v, t.v);
    return r;
}
static __device__ __noinline__ Fe12 p384_fmul_call(Fe12 a, Fe12 b) {
    Fe12 r;
    P384::fmul_inline(r.v, a.v, b.v);
    return r;
}
static __device__ __noinline__ Fe12 p384_fsqr_call(Fe12 a) {
    Fe12 r;
    P384::fsqr_inline(r.v, a.v);
    return r;
}
static __device__ __noinline__ Fe12 p384_nmul_call(Fe12 a, Fe12 b) {
    Fe12 r;
    P384::nmul_inline(r.v, a.v, b.v);
    return r;
}

// -------------------------------------------------------------------------------------------------
// Jacobian points (X, Y, Z) ~ (X/Z^2, Y/Z^3); Z == 0 is the point at infinity.
// -------------------------------------------------------------------------------------------------
template <class C>
struct Jac {
    uint32_t X[C::N], Y[C::N], Z[C::N];
};

// a = -3 doubling, 4M + 4S, 9 add/sub + 1 halving.  Infinity (Z = 0) maps to infinity; Y = 0
// cannot occur (odd group order).
//   S = 2Y, Z3 = S*Z, B = S^2 = 4Y^2, beta4 = X*B = 4XY^2, C = B^2/2 = 8Y^4,
//   alpha = 3(X - Z^2)(X + Z^2), X3 = alpha^2 - 2*beta4, Y3 = alpha*(beta4 - X3) - C
template <class C>
SBV_DEV void pt_double(Jac<C> &P) {
    constexpr int N = C::N;
    uint32_t delta[N], s[N], bb[N], beta4[N], alpha[N], t1[N], t2[N];
    C::fsqr(delta, P.Z);
    C::fadd(s, P.Y, P.Y);
    C::fmul(P.Z, s, P.Z);       // Z3 = 2 Y Z
    C::fsqr(bb, s);             // 4 Y^2
    C::fmul(beta4, P.X, bb);    // 4 X Y^2
    C::fsqr(t1, bb);            // 16 Y^4
    C::fhalf(bb, t1);           // 8 Y^4
    C::fsub(t1, P.X, delta);
    C::fadd(t2, P.X, delta);
    C::fmul(alpha, t1, t2);
    C::fadd(t1, alpha, alpha);
    C::fadd(alpha, t1, alpha);  // 3 (X - delta)(X + delta)
    C::fsqr(t1, alpha);
    C::fadd(t2, beta4, beta4);
    C::fsub(P.X, t1, t2);       // X3
    C::fsub(t1, beta4, P.X);
    C::fmul(t2, alpha, t1);
    C::fsub(P.Y, t2, bb);       // Y3
}

// P += (x2, y2[, z2]).  MODE 1: z2 == 1 (mixed add, 8M+3S).  MODE 0: general (12M+4S).
// MODE 2: z2 with its square and cube supplied (table points sharing one Z: 11M+3S).
// `skip` leaves P unchanged (digit 0).  `neg` adds the negated point.  Handles every exceptional
// case: P = inf -> result is the addend; P == addend -> doubling; P == -addend -> infinity (Z3 = 0).
// DEFER: P == addend leaves P unchanged and returns true — the caller doubles P at its own doubling site, so that a
// loop with one addition and one doubling does not carry a second inlined copy of the doubling.
template <class C, int MODE, bool DEFER = false>
SBV_DEV bool pt_add_m(Jac<C> &P, const uint32_t (&x2)[C::N], const uint32_t (&y2_in)[C::N], const uint32_t (&z2)[C::N],
                      const uint32_t (&z2sq)[C::N], const uint32_t (&z2cu)[C::N], bool neg, bool skip) {
    constexpr int N = C::N;
    uint32_t y2[N], zero[N];
#pragma unroll
    for (int i = 0; i < N; i++) zero[i] = 0;
    {
        uint32_t ny[N];
        C::fsub(ny, zero, y2_in);
        mp_select<N>(y2, neg, ny, y2_in);
    }
    const bool p_inf = mp_is_zero<N>(P.Z);
    uint32_t z1z1[N], u1[N], u2[N], s1[N], s2[N], h[N], r[N], t[N];
    C::fsqr(z1z1, P.Z);
    C::fmul(u2, x2, z1z1);
    C::fmul(t, P.Z, z1z1);
    C::fmul(s2, y2, t);
    if (MODE == 1) {
        mp_copy<N>(u1, P.X);
        mp_copy<N>(s1, P.Y);
    } else if (MODE == 2) {
        C::fmul(u1, P.X, z2sq);
        C::fmul(s1, P.Y, z2cu);
    } else {
        uint32_t z2z2[N];
        C::fsqr(z2z2, z2);
        C::fmul(u1, P.X, z2z2);
        C::fmul(t, z2, z2z2);
        C::fmul(s1, P.Y, t);
    }
    C::fsub(h, u2, u1);
    C::fsub(r, s2, s1);
    const bool h0 = mp_is_zero<N>(h), r0 = mp_is_zero<N>(r);
    if (h0 && r0 && !p_inf && !skip) {  // same point: rare, data dependent — take the doubling path
        if constexpr (!DEFER) pt_double<C>(P);
        return true;
    }
    uint32_t hh[N], hhh[N], v[N], x3[N], y3[N], z3[N];
    C::fsqr(hh, h);
    C::fmul(hhh, h, hh);
    C::fmul(v, u1, hh);
    C::fsqr(x3, r);
    C::fsub(x3, x3, hhh);
    C::fsub(x3, x3, v);
    C::fsub(x3, x3, v);
    C::fsub(t, v, x3);
    C::fmul(y3, r, t);
    C::fmul(t, s1, hhh);
    C::fsub(y3, y3, t);
    C::fmul(z3, P.Z, h);
    if (MODE != 1) C::fmul(z3, z3, z2);
    // select: skip -> P ; P inf -> addend ; else sum
    uint32_t one[N];
    C::get_one(one);
#pragma unroll
    for (int i = 0; i < N; i++) {
        uint32_t ax = x2[i], ay = y2[i], az = MODE == 1 ? one[i] : z2[i];
        uint32_t nx = p_inf ? ax : x3[i], ny = p_inf ? ay : y3[i], nz = p_inf ? az : z3[i];
        P.X[i] = skip ? P.X[i] : nx;
        P.Y[i] = skip ? P.Y[i] : ny;
        P.Z[i] = skip ? P.Z[i] : nz;
    }
    return false;
}
// P = the affine point (x, y_in), negated if `neg`, or the point at infinity (1, 1, 0) if `skip`: bit for bit what
// pt_add_m<C, 1> makes of the accumulators' starting value (1, 1, 0) and that point.  A pass whose accumulator starts at
// infinity loads its first entry with this instead of spending a complete addition on it.
template <class C>
SBV_DEV void pt_seed(Jac<C> &P, const uint32_t (&x)[C::N], const uint32_t (&y_in)[C::N], bool neg, bool skip) {
    constexpr int N = C::N;
    uint32_t y[N], zero[N], one[N];
#pragma unroll
    for (int i = 0; i < N; i++) zero[i] = 0;
    {
        uint32_t ny[N];
        C::fsub(ny, zero, y_in);
        mp_select<N>(y, neg, ny, y_in);
    }
    C::get_one(one);
#pragma unroll
    for (int i = 0; i < N; i++) {
        P.X[i] = skip ? one[i] : x[i];
        P.Y[i] = skip ? one[i] : y[i];
        P.Z[i] = skip ? 0u : one[i];
    }
}
template <class C, bool AFFINE>
SBV_DEV void pt_add(Jac<C> &P, const uint32_t (&x2)[C::N], const uint32_t (&y2)[C::N], const uint32_t (&z2)[C::N], bool neg, bool skip) {
    if (AFFINE) pt_add_m<C, 1>(P, x2, y2, z2, z2, z2, neg, skip);
    else pt_add_m<C, 0>(P, x2, y2, z2, z2, z2, neg, skip);
}

// Table construction step: P += (qx, qy) affine, with P = k*(qx, qy), k >= 2 (no exceptional case can
// occur: the group order is prime and huge).  Also returns H = Z3 / Z1, the factor the co-Z
// normalisation needs.
template <class C>
SBV_DEV void pt_madd_table(Jac<C> &P, const uint32_t (&qx)[C::N], const uint32_t (&qy)[C::N], uint32_t (&h)[C::N]) {
    constexpr int N = C::N;
    uint32_t z1z1[N], u2[N], s2[N], r[N], t[N], hh[N], hhh[N], v[N];
    C::fsqr(z1z1, P.Z);
    C::fmul(u2, qx, z1z1);
    C::fmul(t, P.Z, z1z1);
    C::fmul(s2, qy, t);
    C::fsub(h, u2, P.X);
    C::fsub(r, s2, P.Y);
    C::fsqr(hh, h);
    C::fmul(hhh, h, hh);
    C::fmul(v, P.X, hh);
    C::fmul(t, P.Y, hhh);   // Y1 * H^3
    C::fsqr(P.X, r);
    C::fsub(P.X, P.X, hhh);
    C::fsub(P.X, P.X, v);
    C::fsub(P.X, P.X, v);
    C::fsub(v, v, P.X);
    C::fmul(P.Y, r, v);
    C::fsub(P.Y, P.Y, t);
    C::fmul(P.Z, P.Z, h);
}

// r = a^(p-2) (field inverse, Montgomery in/out); a != 0.  Setup paths only.
template <class C>
__device__ __noinline__ void f_inv(uint32_t (&r)[C::N], const uint32_t (&a)[C::N]) {
    constexpr int N = C::N;
    uint32_t acc[N];
    C::get_one(acc);
    for (int i = 32 * N - 1; i >= 0; i--) {
        C::fsqr(acc, acc);
        if ((C::p_minus_2_limb(i >> 5) >> (i & 31)) & 1u) C::fmul(acc, acc, a);
    }
    mp_copy<N>(r, acc);
}
// r = a^-1 mod m for Montgomery-form a (= A*R), result in Montgomery form (A^-1 * R); m = the field prime p (FIELD) or
// the group order n.
// Binary extended GCD on the plain residue with batched trailing-zero stripping:
//   invariants  x1 * a == u,  x2 * a == v  (mod n), u and v odd;  each pass replaces the larger of
//   (u, v) by |u - v| (even), strips its tz <= 31 trailing zeros and fixes the cofactor with one
//   multiply-accumulate:  x = (x + k*n) >> tz,  k = x * (-n^-1) mod 2^tz.
// ~0.7 passes per bit of ~150 cheap instructions — about 4x fewer (and cheaper) instructions than the
// 4-bit-window Fermat chain, which is what the latency-bound scalar-preparation kernel needs.
// gcd(a, n) = 1 always holds here (n prime, a != 0); the pass count is capped defensively.
template <class C, bool FIELD>
__device__ __noinline__ void mod_inv(uint32_t (&r)[C::N], const uint32_t (&a)[C::N]) {
    constexpr int N = C::N;
    uint32_t M[N];
    if (FIELD) C::get_p(M); else C::get_n(M);
    constexpr uint32_t MINV = FIELD ? C::PINV : C::NINV;  // -m^-1 mod 2^32
    uint32_t u[N], v[N], x1[N], x2[N];
    mp_copy<N>(u, a);
    mp_copy<N>(v, M);
#pragma unroll
    for (int i = 0; i < N; i++) { x1[i] = (i == 0); x2[i] = 0; }
    // strip(t, x): t even and non-zero -> odd, cofactor adjusted
    auto strip = [&](uint32_t (&t)[N], uint32_t (&x)[N]) {
        while ((t[0] & 1u) == 0u) {
            const uint32_t tz = t[0] ? (uint32_t)(__ffs((int)t[0]) - 1) : 31u;  // 1..31
#pragma unroll
            for (int i = 0; i < N - 1; i++) t[i] = __funnelshift_r(t[i], t[i + 1], tz);
            t[N - 1] >>= tz;
            const uint32_t k = (x[0] * MINV) & ((1u << tz) - 1u);
            // x = (x + k*M) >> tz   (x + k*M < 2^tz * 2M fits N+1 limbs)
            uint32_t w[N + 1];
            uint64_t cy = 0;
#pragma unroll
            for (int i = 0; i < N; i++) {
                cy += (uint64_t)k * M[i] + x[i];
                w[i] = (uint32_t)cy;
                cy >>= 32;
            }
            w[N] = (uint32_t)cy;
#pragma unroll
            for (int i = 0; i < N; i++) x[i] = __funnelshift_r(w[i], w[i + 1], tz);
            uint32_t d[N];
            const uint32_t bw = mp_sub<N>(d, x, M);   // x < 2M: one conditional subtraction
            mp_select<N>(x, bw == 0, d, x);
        }
    };
    if ((u[0] & 1u) == 0u) strip(u, x1);
    for (int pass = 0; pass < 64 * N + 8; pass++) {
        if (mp_eq<N>(u, v)) break;
        uint32_t d[N], xd[N], t[N];
        const uint32_t lt = mp_sub<N>(d, u, v);        // borrow: u < v
        if (lt) {                                       // d = v - u
            uint32_t z[N];
#pragma unroll
            for (int i = 0; i < N; i++) z[i] = 0;
            mp_sub<N>(t, z, d);
            mp_copy<N>(d, t);
        }
        mod_sub<N>(xd, x1, x2, M);                      // x1 - x2 mod n (non-zero: u != v)
        if (lt) { mp_sub<N>(t, M, xd); mp_copy<N>(xd, t); }  // x2 - x1
        strip(d, xd);
        if (lt) { mp_copy<N>(v, d); mp_copy<N>(x2, xd); }
        else    { mp_copy<N>(u, d); mp_copy<N>(x1, xd); }
    }
    // u == v == 1: x1 = (A*R)^-1 ; times R^3 / R -> A^-1 * R
    uint32_t rrr[N];
    if (FIELD) { C::get_rrr_p(rrr); C::fmul(r, x1, rrr); }
    else { C::get_rrr_n(rrr); C::nmul(r, x1, rrr); }
}
template <class C>
SBV_DEV void n_inv(uint32_t (&r)[C::N], const uint32_t (&a)[C::N]) { mod_inv<C, false>(r, a); }
// field inverse by the same binary extended GCD (~3x shorter dependent chain than the Fermat ladder f_inv)
template <class C>
SBV_DEV void p_inv(uint32_t (&r)[C::N], const uint32_t (&a)[C::N]) { mod_inv<C, true>(r, a); }

// big-endian byte string (C::BYTES, 4-byte aligned) -> little-endian limbs
template <int N>
SBV_DEV void load_be(uint32_t (&r)[N], const uint8_t *src) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(src);
#pragma unroll
    for (int i = 0; i < N; i++) r[N - 1 - i] = __byte_perm(__ldg(w + i), 0, 0x0123);
}

}  // namespace sbv
