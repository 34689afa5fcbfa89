// mp.cuh — register-resident multiprecision primitives for sm_90a (32-bit limbs, little-endian).
//
// The multiply uses the even/odd column split: every a[i]*b[j] with i+j even is a 64-bit value at
// an even limb offset, so a row of them is one carry chain of IMAD.WIDE.U32.X instructions
// (ptxas fuses each mad.lo.cc/madc.hi.cc pair into a single wide MAD with a carry predicate);
// the odd columns go to a second accumulator that is added back shifted by one limb.
// N*N wide MADs + 2N carry words + one 2N-limb add per product.
#pragma once
#include <stdint.h>
#include "hostsim.h"

namespace sbv {

#define SBV_DEV __device__ __forceinline__

#if defined(SBV_HOSTSIM) && !defined(__CUDACC__)
// CPU emulation of the PTX carry-flag primitives (tests only, see hostsim.h): one thread-local CC.CF.
static thread_local uint32_t sbv_cc = 0;
SBV_DEV uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; sbv_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
SBV_DEV uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + sbv_cc; sbv_cc = (uint32_t)(t >> 32); return (uint32_t)t; }
SBV_DEV uint32_t addc(uint32_t a, uint32_t b) { return a + b + sbv_cc; }
SBV_DEV uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; sbv_cc = (uint32_t)(t >> 63); return (uint32_t)t; }
SBV_DEV uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - sbv_cc; sbv_cc = (uint32_t)(t >> 63); return (uint32_t)t; }
SBV_DEV uint32_t subc(uint32_t a, uint32_t b) { return a - b - sbv_cc; }
SBV_DEV void mad_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    const uint64_t p = (uint64_t)a * b;
    uint64_t t = (uint64_t)lo + (uint32_t)p; lo = (uint32_t)t;
    t = (uint64_t)hi + (uint32_t)(p >> 32) + (t >> 32); hi = (uint32_t)t; sbv_cc = (uint32_t)(t >> 32);
}
SBV_DEV void madc_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    const uint64_t p = (uint64_t)a * b;
    uint64_t t = (uint64_t)lo + (uint32_t)p + sbv_cc; lo = (uint32_t)t;
    t = (uint64_t)hi + (uint32_t)(p >> 32) + (t >> 32); hi = (uint32_t)t; sbv_cc = (uint32_t)(t >> 32);
}
#else
SBV_DEV uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SBV_DEV uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SBV_DEV uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SBV_DEV uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SBV_DEV uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SBV_DEV uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }

// (hi:lo) += a*b, carry-out to CC                 [first link of a chain]
SBV_DEV void mad_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
// (hi:lo) += a*b + CC, carry-out to CC            [inner link]
SBV_DEV void madc_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
#endif

// r[0..2N) = a[0..N) * b[0..N)
template <int N>
SBV_DEV void mp_mul(uint32_t (&r)[2 * N], const uint32_t (&a)[N], const uint32_t (&b)[N]) {
    static_assert(N % 2 == 0, "even limb count");
    uint32_t E[2 * N], O[2 * N];  // O[k] has weight 2^(32(k+1))
#pragma unroll
    for (int i = 0; i < 2 * N; i++) { E[i] = 0; O[i] = 0; }
#pragma unroll
    for (int j = 0; j < N; j++) {
        if ((j & 1) == 0) {
            // i even -> E at limb i+j ; i odd -> O at index i+j-1
            mad_wide_cc(E[j], E[j + 1], a[0], b[j]);
#pragma unroll
            for (int i = 2; i < N; i += 2) madc_wide_cc(E[i + j], E[i + j + 1], a[i], b[j]);
            E[j + N] = addc(E[j + N], 0);
            mad_wide_cc(O[j], O[j + 1], a[1], b[j]);
#pragma unroll
            for (int i = 3; i < N; i += 2) madc_wide_cc(O[i + j - 1], O[i + j], a[i], b[j]);
            O[j + N] = addc(O[j + N], 0);
        } else {
            // i odd -> E at limb i+j ; i even -> O at index i+j-1
            mad_wide_cc(E[j + 1], E[j + 2], a[1], b[j]);
#pragma unroll
            for (int i = 3; i < N; i += 2) madc_wide_cc(E[i + j], E[i + j + 1], a[i], b[j]);
            if (j + N + 1 < 2 * N) E[j + N + 1] = addc(E[j + N + 1], 0);
            mad_wide_cc(O[j - 1], O[j], a[0], b[j]);
#pragma unroll
            for (int i = 2; i < N; i += 2) madc_wide_cc(O[i + j - 1], O[i + j], a[i], b[j]);
            O[j + N - 1] = addc(O[j + N - 1], 0);
        }
    }
    r[0] = E[0];
    r[1] = add_cc(E[1], O[0]);
#pragma unroll
    for (int i = 2; i < 2 * N - 1; i++) r[i] = addc_cc(E[i], O[i - 1]);
    r[2 * N - 1] = addc(E[2 * N - 1], O[2 * N - 2]);
}

// r[0..2N) = a^2 : off-diagonal products once (even/odd split as in mp_mul), doubled, plus the diagonal.
// N(N-1)/2 + N wide MADs instead of N^2.
template <int N>
SBV_DEV void mp_sqr(uint32_t (&r)[2 * N], const uint32_t (&a)[N]) {
    static_assert(N % 2 == 0, "even limb count");
    uint32_t E[2 * N], O[2 * N];  // O[k] has weight 2^(32(k+1))
#pragma unroll
    for (int i = 0; i < 2 * N; i++) { E[i] = 0; O[i] = 0; }
#pragma unroll
    for (int i = 0; i < N - 1; i++) {
        // j > i, same parity as i  -> E at limb i+j
        if (i + 2 < N) {
            mad_wide_cc(E[2 * i + 2], E[2 * i + 3], a[i], a[i + 2]);
#pragma unroll
            for (int j = i + 4; j < N; j += 2) madc_wide_cc(E[i + j], E[i + j + 1], a[i], a[j]);
            // last j of this row: N-2 or N-1 (same parity as i)
            const int jl = ((N - 1 - i) % 2 == 0) ? N - 1 : N - 2;
            if (i + jl + 2 < 2 * N) E[i + jl + 2] = addc(E[i + jl + 2], 0);
        }
        // j > i, opposite parity -> O at index i+j-1
        mad_wide_cc(O[2 * i], O[2 * i + 1], a[i], a[i + 1]);
#pragma unroll
        for (int j = i + 3; j < N; j += 2) madc_wide_cc(O[i + j - 1], O[i + j], a[i], a[j]);
        {
            const int jl = ((N - 1 - i) % 2 == 1) ? N - 1 : N - 2;
            if (i + jl + 1 < 2 * N) O[i + jl + 1] = addc(O[i + jl + 1], 0);
        }
    }
    // T = E + (O << 32)
    uint32_t T[2 * N];
    T[0] = E[0];
    T[1] = add_cc(E[1], O[0]);
#pragma unroll
    for (int i = 2; i < 2 * N - 1; i++) T[i] = addc_cc(E[i], O[i - 1]);
    T[2 * N - 1] = addc(E[2 * N - 1], O[2 * N - 2]);
    // T = 2T
    T[0] = add_cc(T[0], T[0]);
#pragma unroll
    for (int i = 1; i < 2 * N - 1; i++) T[i] = addc_cc(T[i], T[i]);
    T[2 * N - 1] = addc(T[2 * N - 1], T[2 * N - 1]);
    // T += sum a_i^2 * 2^(64 i)
    mad_wide_cc(T[0], T[1], a[0], a[0]);
#pragma unroll
    for (int i = 1; i < N; i++) madc_wide_cc(T[2 * i], T[2 * i + 1], a[i], a[i]);
#pragma unroll
    for (int i = 0; i < 2 * N; i++) r[i] = T[i];
}

// r = a + b, returns carry-out
template <int N>
SBV_DEV uint32_t mp_add(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&b)[N]) {
    r[0] = add_cc(a[0], b[0]);
#pragma unroll
    for (int i = 1; i < N; i++) r[i] = addc_cc(a[i], b[i]);
    return addc(0, 0);
}
// r = a - b, returns borrow (1 if a < b)
template <int N>
SBV_DEV uint32_t mp_sub(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&b)[N]) {
    r[0] = sub_cc(a[0], b[0]);
#pragma unroll
    for (int i = 1; i < N; i++) r[i] = subc_cc(a[i], b[i]);
    return subc(0, 0) & 1u;  // subc(0,0) = -borrow
}
template <int N>
SBV_DEV bool mp_is_zero(const uint32_t (&a)[N]) {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < N; i++) o |= a[i];
    return o == 0;
}
template <int N>
SBV_DEV bool mp_eq(const uint32_t (&a)[N], const uint32_t (&b)[N]) {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < N; i++) o |= a[i] ^ b[i];
    return o == 0;
}
// a < b ?
template <int N>
SBV_DEV bool mp_lt(const uint32_t (&a)[N], const uint32_t (&b)[N]) {
    uint32_t t[N];
    return mp_sub<N>(t, a, b) != 0;
}
template <int N>
SBV_DEV void mp_copy(uint32_t (&r)[N], const uint32_t (&a)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = a[i];
}
// r = c ? a : b
template <int N>
SBV_DEV void mp_select(uint32_t (&r)[N], bool c, const uint32_t (&a)[N], const uint32_t (&b)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = c ? a[i] : b[i];
}

// ---- modular helpers for a modulus m (canonical residues in [0, m)) ----
template <int N>
SBV_DEV void mod_add(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&b)[N], const uint32_t (&m)[N]) {
    uint32_t s[N], t[N];
    uint32_t c = mp_add<N>(s, a, b);
    uint32_t bw = mp_sub<N>(t, s, m);
    bool use_t = (c != 0) || (bw == 0);
    mp_select<N>(r, use_t, t, s);
}
template <int N>
SBV_DEV void mod_sub(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&b)[N], const uint32_t (&m)[N]) {
    uint32_t d[N];
    uint32_t bw = mp_sub<N>(d, a, b);
    uint32_t mask = 0u - bw;
    r[0] = add_cc(d[0], m[0] & mask);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r[i] = addc_cc(d[i], m[i] & mask);
    r[N - 1] = addc(d[N - 1], m[N - 1] & mask);
}

// r[0..N) = (a * b) mod 2^(32N): the low half only (N(N+1)/2 wide MADs; the top product of each chain
// spills its high word into limb N, which is discarded).
template <int N>
SBV_DEV void mp_mul_lo(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&b)[N]) {
    static_assert(N % 2 == 0, "even limb count");
    uint32_t E[N + 2], O[N + 2];  // O[k] has weight 2^(32(k+1))
#pragma unroll
    for (int i = 0; i < N + 2; i++) { E[i] = 0; O[i] = 0; }
#pragma unroll
    for (int j = 0; j < N; j++) {
        if ((j & 1) == 0) {
            // i even -> E at limb i+j (needs i+j <= N-1) ; i odd -> O at index i+j-1
            mad_wide_cc(E[j], E[j + 1], a[0], b[j]);
#pragma unroll
            for (int i = 2; i + j < N; i += 2) madc_wide_cc(E[i + j], E[i + j + 1], a[i], b[j]);
            if (j + 1 < N) {
                mad_wide_cc(O[j], O[j + 1], a[1], b[j]);
#pragma unroll
                for (int i = 3; i + j < N; i += 2) madc_wide_cc(O[i + j - 1], O[i + j], a[i], b[j]);
            }
        } else {
            if (j + 1 < N) {
                mad_wide_cc(E[j + 1], E[j + 2], a[1], b[j]);
#pragma unroll
                for (int i = 3; i + j < N; i += 2) madc_wide_cc(E[i + j], E[i + j + 1], a[i], b[j]);
            }
            mad_wide_cc(O[j - 1], O[j], a[0], b[j]);
#pragma unroll
            for (int i = 2; i + j < N; i += 2) madc_wide_cc(O[i + j - 1], O[i + j], a[i], b[j]);
        }
    }
    r[0] = E[0];
    r[1] = add_cc(E[1], O[0]);
#pragma unroll
    for (int i = 2; i < N - 1; i++) r[i] = addc_cc(E[i], O[i - 1]);
    r[N - 1] = addc(E[N - 1], O[N - 2]);
}

// Montgomery reduction in separated-operand form: M = (T mod R) * minv_full mod R, r = (T + M*m) / R.
// Three independent-chain products instead of a word-serial carry walk: ~2x shorter dependency
// chain, which is what the latency-bound scalar-inversion kernel needs.  minv_full = -m^-1 mod R.
template <int N>
SBV_DEV void mont_reduce_sos(uint32_t (&r)[N], const uint32_t (&T)[2 * N], const uint32_t (&m)[N], const uint32_t (&minv_full)[N]) {
    uint32_t lo[N], M[N], U[2 * N];
#pragma unroll
    for (int i = 0; i < N; i++) lo[i] = T[i];
    mp_mul_lo<N>(M, lo, minv_full);
    mp_mul<N>(U, M, m);
    // (T + U) has zero low half; the carry out of the low half is 1 unless T_lo == 0
    uint32_t carry_lo = 0;
#pragma unroll
    for (int i = 0; i < N; i++) carry_lo |= T[i];
    carry_lo = carry_lo ? 1u : 0u;
    uint32_t hi[N];
    hi[0] = add_cc(T[N], carry_lo);
#pragma unroll
    for (int i = 1; i < N; i++) hi[i] = addc_cc(T[N + i], 0);
    uint32_t top = addc(0, 0);
    hi[0] = add_cc(hi[0], U[N]);
#pragma unroll
    for (int i = 1; i < N; i++) hi[i] = addc_cc(hi[i], U[N + i]);
    top = addc(top, 0);
    uint32_t t[N];
    uint32_t bw = mp_sub<N>(t, hi, m);
    bool use_t = (top != 0) || (bw == 0);
    mp_select<N>(r, use_t, t, hi);
}
template <int N>
SBV_DEV void mont_mul_sos(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&b)[N], const uint32_t (&m)[N], const uint32_t (&minv_full)[N]) {
    uint32_t T[2 * N];
    mp_mul<N>(T, a, b);
    mont_reduce_sos<N>(r, T, m, minv_full);
}
template <int N>
SBV_DEV void mont_sqr_sos(uint32_t (&r)[N], const uint32_t (&a)[N], const uint32_t (&m)[N], const uint32_t (&minv_full)[N]) {
    uint32_t T[2 * N];
    mp_sqr<N>(T, a);
    mont_reduce_sos<N>(r, T, m, minv_full);
}

}  // namespace sbv
