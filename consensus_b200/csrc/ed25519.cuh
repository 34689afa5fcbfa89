// ed25519.cuh — edwards25519 arithmetic for batched Ed25519 verification (RFC 8032 §5.1, with the accept set of Go's
// crypto/ed25519.Verify: see DESIGN.md §1).
//
// Field elements mod p = 2^255 - 19 are 8 little-endian 32-bit limbs holding ANY value in [0, 2^256): a product is
// reduced by folding its high half times 38 (2^256 = 38 mod p), sums and differences by folding their carry or borrow
// the same way.  Values are brought to [0, p) only where bytes are produced or compared (fe_canon).
// Points are extended twisted-Edwards coordinates (X:Y:Z:T), x = X/Z, y = Y/Z, xy = T/Z, on -x^2 + y^2 = 1 + d x^2 y^2.
// The addition and doubling formulas (RFC 8032 §5.1.4) are complete for this curve: no exceptional cases, small-order
// points included.
#pragma once
#include <stdint.h>

#include "mp.cuh"

namespace sbv {

struct EdFe { uint32_t v[8]; };
static __device__ __noinline__ EdFe ed_fmul_call(EdFe a, EdFe b);
static __device__ __noinline__ EdFe ed_fsqr_call(EdFe a);
struct EdRoot { EdFe r; uint32_t ok; };
static __device__ __noinline__ EdFe ed_inv_call(EdFe z);
static __device__ __noinline__ EdRoot ed_sqrt_ratio_call(EdFe u, EdFe v);

// ---- constants (little-endian limbs) ----
SBV_DEV void ed_set(uint32_t (&r)[8], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t a4, uint32_t a5, uint32_t a6,
                    uint32_t a7) {
    r[0] = a0; r[1] = a1; r[2] = a2; r[3] = a3; r[4] = a4; r[5] = a5; r[6] = a6; r[7] = a7;
}
SBV_DEV void ed_d(uint32_t (&r)[8]) {  // d = -121665/121666
    ed_set(r, 0x135978a3, 0x75eb4dca, 0x4141d8ab, 0x00700a4d, 0x7779e898, 0x8cc74079, 0x2b6ffe73, 0x52036cee);
}
SBV_DEV void ed_d2(uint32_t (&r)[8]) {  // 2d
    ed_set(r, 0x26b2f159, 0xebd69b94, 0x8283b156, 0x00e0149a, 0xeef3d130, 0x198e80f2, 0x56dffce7, 0x2406d9dc);
}
SBV_DEV void ed_sqrtm1(uint32_t (&r)[8]) {  // 2^((p-1)/4), a square root of -1
    ed_set(r, 0x4a0ea0b0, 0xc4ee1b27, 0xad2fe478, 0x2f431806, 0x3dfbd7a7, 0x2b4d0099, 0x4fc1df0b, 0x2b832480);
}
SBV_DEV void ed_bx(uint32_t (&r)[8]) {  // base point B (RFC 8032 §5.1)
    ed_set(r, 0x8f25d51a, 0xc9562d60, 0x9525a7b2, 0x692cc760, 0xfdd6dc5c, 0xc0a4e231, 0xcd6e53fe, 0x216936d3);
}
SBV_DEV void ed_by(uint32_t (&r)[8]) {
    ed_set(r, 0x66666658, 0x66666666, 0x66666666, 0x66666666, 0x66666666, 0x66666666, 0x66666666, 0x66666666);
}
SBV_DEV void ed_order(uint32_t (&r)[8]) {  // L = 2^252 + 27742317777372353535851937790883648493
    ed_set(r, 0x5cf5d3ed, 0x5812631a, 0xa2f79cd6, 0x14def9de, 0, 0, 0, 0x10000000);
}
SBV_DEV void ed_zero(uint32_t (&r)[8]) { ed_set(r, 0, 0, 0, 0, 0, 0, 0, 0); }
SBV_DEV void ed_one(uint32_t (&r)[8]) { ed_set(r, 1, 0, 0, 0, 0, 0, 0, 0); }

// ---- field arithmetic mod p ----
// r = T mod p, up to a multiple of p: T_lo + 38 * T_hi, whose carry limb (<= 38) is folded once more.
SBV_DEV void fe_fold(uint32_t (&r)[8], const uint32_t (&T)[16]) {
    uint64_t acc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        acc += (uint64_t)T[i] + (uint64_t)T[8 + i] * 38u;
        r[i] = (uint32_t)acc;
        acc >>= 32;
    }
    r[0] = add_cc(r[0], (uint32_t)acc * 38u);
#pragma unroll
    for (int i = 1; i < 8; i++) r[i] = addc_cc(r[i], 0);
    const uint32_t c = addc(0, 0);
    r[0] += 38u * c;  // after a wrap the value is < 38^2: no further carry
}
SBV_DEV void fe_mul_inline(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    uint32_t T[16];
    mp_mul<8>(T, a, b);
    fe_fold(r, T);
}
SBV_DEV void fe_sqr_inline(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    uint32_t T[16];
    mp_sqr<8>(T, a);
    fe_fold(r, T);
}
// Out of line, operands in registers, as P256::fmul: the verify loop then fits the instruction cache.
SBV_DEV void fe_mul(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    EdFe x, y;
    mp_copy<8>(x.v, a); mp_copy<8>(y.v, b);
    EdFe z = ed_fmul_call(x, y);
    mp_copy<8>(r, z.v);
}
SBV_DEV void fe_sqr(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    EdFe x;
    mp_copy<8>(x.v, a);
    EdFe z = ed_fsqr_call(x);
    mp_copy<8>(r, z.v);
}
SBV_DEV void fe_add(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t c = mp_add<8>(r, a, b);
    r[0] = add_cc(r[0], 38u * c);
#pragma unroll
    for (int i = 1; i < 8; i++) r[i] = addc_cc(r[i], 0);
    r[0] += 38u * addc(0, 0);
}
SBV_DEV void fe_sub(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t bw = mp_sub<8>(r, a, b);  // a - b + 2^256 * bw
    r[0] = sub_cc(r[0], 38u * bw);
#pragma unroll
    for (int i = 1; i < 8; i++) r[i] = subc_cc(r[i], 0);
    r[0] -= 38u * (subc(0, 0) & 1u);  // after a wrap the value is >= 2^256 - 38: no further borrow
}
SBV_DEV void fe_neg(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    uint32_t z[8];
    ed_zero(z);
    fe_sub(r, z, a);
}
// the canonical residue in [0, p)
SBV_DEV void fe_canon(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    uint32_t t[8], u[8];
    t[0] = add_cc(a[0], 19u * (a[7] >> 31));  // a mod 2^255 + 19 * bit 255: < 2^255 + 19
#pragma unroll
    for (int i = 1; i < 7; i++) t[i] = addc_cc(a[i], 0);
    t[7] = addc(a[7] & 0x7fffffffu, 0);
    u[0] = add_cc(t[0], 19u);  // t >= p  <=>  t + 19 >= 2^255
#pragma unroll
    for (int i = 1; i < 7; i++) u[i] = addc_cc(t[i], 0);
    u[7] = addc(t[7], 0);
    const bool ge = (u[7] >> 31) != 0;
    u[7] &= 0x7fffffffu;
    mp_select<8>(r, ge, u, t);
}
SBV_DEV bool fe_eq(const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    uint32_t d[8];
    fe_sub(d, a, b);
    fe_canon(d, d);
    return mp_is_zero<8>(d);
}
SBV_DEV void fe_sqr_n(uint32_t (&r)[8], const uint32_t (&a)[8], int n) {
    fe_sqr(r, a);
#pragma unroll 1
    for (int i = 1; i < n; i++) fe_sqr(r, r);
}
// z^(2^250 - 1), and z^11 on the side (the shared prefix of inversion and square root, ref10's chain)
SBV_DEV void fe_pow250(uint32_t (&r)[8], uint32_t (&z11)[8], const uint32_t (&z)[8]) {
    uint32_t t0[8], t1[8], t2[8];
    fe_sqr(t0, z);           // 2
    fe_sqr_n(t1, t0, 2);     // 8
    fe_mul(t1, t1, z);       // 9
    fe_mul(z11, t0, t1);     // 11
    fe_sqr(t0, z11);         // 22
    fe_mul(t0, t0, t1);      // 2^5 - 1
    fe_sqr_n(t1, t0, 5);
    fe_mul(t0, t1, t0);      // 2^10 - 1
    fe_sqr_n(t1, t0, 10);
    fe_mul(t1, t1, t0);      // 2^20 - 1
    fe_sqr_n(t2, t1, 20);
    fe_mul(t1, t2, t1);      // 2^40 - 1
    fe_sqr_n(t1, t1, 10);
    fe_mul(t0, t1, t0);      // 2^50 - 1
    fe_sqr_n(t1, t0, 50);
    fe_mul(t1, t1, t0);      // 2^100 - 1
    fe_sqr_n(t2, t1, 100);
    fe_mul(t1, t2, t1);      // 2^200 - 1
    fe_sqr_n(t1, t1, 50);
    fe_mul(r, t1, t0);       // 2^250 - 1
}
// r = z^(p-2) = 1/z (0 for z = 0)
SBV_DEV void fe_inv_inline(uint32_t (&r)[8], const uint32_t (&z)[8]) {
    uint32_t t[8], z11[8];
    fe_pow250(t, z11, z);
    fe_sqr_n(t, t, 5);       // 2^255 - 32
    fe_mul(r, t, z11);       // 2^255 - 21
}
SBV_DEV void fe_inv(uint32_t (&r)[8], const uint32_t (&z)[8]) {
    EdFe x;
    mp_copy<8>(x.v, z);
    EdFe y = ed_inv_call(x);
    mp_copy<8>(r, y.v);
}
// r = z^((p-5)/8) = z^(2^252 - 3)
SBV_DEV void fe_pow22523(uint32_t (&r)[8], const uint32_t (&z)[8]) {
    uint32_t t[8], z11[8];
    fe_pow250(t, z11, z);
    fe_sqr_n(t, t, 2);       // 2^252 - 4
    fe_mul(r, t, z);
}
// r = sqrt(u/v), Go edwards25519 field.Element.SqrtRatio: returns whether u/v is a square; r is the non-negative
// (even) root in [0, p) — when u/v is not a square, r is sqrt(i*u/v) — so callers test the flag.
SBV_DEV bool fe_sqrt_ratio_inline(uint32_t (&r)[8], const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    uint32_t v2[8], v3[8], v7[8], uv3[8], uv7[8], t[8], check[8], nu[8], nui[8], i[8];
    fe_sqr(v2, v);
    fe_mul(v3, v2, v);
    fe_mul(uv3, u, v3);
    fe_sqr(v7, v3);
    fe_mul(v7, v7, v);
    fe_mul(uv7, u, v7);
    fe_pow22523(t, uv7);
    fe_mul(r, uv3, t);       // (u v^3) (u v^7)^((p-5)/8)
    fe_sqr(check, r);
    fe_mul(check, check, v);
    fe_neg(nu, u);
    ed_sqrtm1(i);
    fe_mul(nui, nu, i);
    const bool correct = fe_eq(check, u), flipped = fe_eq(check, nu), flipped_i = fe_eq(check, nui);
    fe_mul(t, r, i);
    if (flipped || flipped_i) mp_copy<8>(r, t);
    fe_canon(r, r);
    fe_neg(t, r);
    fe_canon(t, t);
    if (r[0] & 1u) mp_copy<8>(r, t);
    return correct || flipped;
}
SBV_DEV bool fe_sqrt_ratio(uint32_t (&r)[8], const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    EdFe a, b;
    mp_copy<8>(a.v, u); mp_copy<8>(b.v, v);
    EdRoot t = ed_sqrt_ratio_call(a, b);
    mp_copy<8>(r, t.r.v);
    return t.ok != 0;
}

// ---- points ----
struct EdP { uint32_t X[8], Y[8], Z[8], T[8]; };         // extended
struct EdCached { uint32_t ypx[8], ymx[8], z2[8], t2d[8]; };  // (Y+X, Y-X, 2Z, 2dT)

// Decodes a 32-byte encoding (little-endian limbs) as Go's edwards25519 Point.SetBytes does: y = the low 255 bits,
// accepted even when >= p; x = sqrt((y^2-1)/(d y^2+1)), negated when bit 255 is set (x = 0 with the bit set is
// accepted); false when there is no square root.  No subgroup check.
SBV_DEV bool ed_decode(EdP &P, const uint32_t (&enc)[8]) {
    uint32_t y[8], y2[8], u[8], v[8], one[8], d[8], x[8];
    mp_copy<8>(y, enc);
    y[7] &= 0x7fffffffu;
    ed_one(one);
    ed_d(d);
    fe_sqr(y2, y);
    fe_sub(u, y2, one);
    fe_mul(v, y2, d);
    fe_add(v, v, one);
    const bool ok = fe_sqrt_ratio(x, u, v);
    if (enc[7] >> 31) fe_neg(x, x);
    mp_copy<8>(P.X, x);
    mp_copy<8>(P.Y, y);
    ed_one(P.Z);
    fe_mul(P.T, x, y);
    return ok;
}

SBV_DEV void ed_identity(EdP &P) {
    ed_zero(P.X); ed_one(P.Y); ed_one(P.Z); ed_zero(P.T);
}

// P = 2P (RFC 8032 §5.1.4: 4M + 4S, 3M + 4S without T)
template <bool WITH_T>
SBV_DEV void ed_double(EdP &P) {
    uint32_t A[8], B[8], C[8], H[8], E[8], G[8], F[8];
    fe_sqr(A, P.X);
    fe_sqr(B, P.Y);
    fe_sqr(C, P.Z);
    fe_add(C, C, C);
    fe_add(H, A, B);
    fe_add(E, P.X, P.Y);
    fe_sqr(E, E);
    fe_sub(E, H, E);
    fe_sub(G, A, B);
    fe_add(F, C, G);
    fe_mul(P.X, E, F);
    fe_mul(P.Y, G, H);
    if (WITH_T) fe_mul(P.T, E, H);
    fe_mul(P.Z, F, G);
}

// P += (neg ? -Q : Q) with Q given as (Y+X, Y-X, 2dT) and 2Z (AFFINE: Q.Z = 1, z2 is not read).
// -Q = (-X, Y, Z, -T) swaps Y+X and Y-X and negates 2dT.  8M (7M affine) + 1M for T.
template <bool WITH_T, bool AFFINE>
SBV_DEV void ed_add(EdP &P, const uint32_t (&ypx)[8], const uint32_t (&ymx)[8], const uint32_t (&t2d)[8], const uint32_t (&z2)[8], bool neg) {
    uint32_t A[8], B[8], C[8], D[8], E[8], F[8], G[8], H[8], s[8];
    fe_sub(s, P.Y, P.X);
    fe_mul(A, s, neg ? ypx : ymx);
    fe_add(s, P.Y, P.X);
    fe_mul(B, s, neg ? ymx : ypx);
    fe_mul(C, P.T, t2d);
    if (AFFINE) fe_add(D, P.Z, P.Z);
    else fe_mul(D, P.Z, z2);
    fe_sub(E, B, A);
    fe_add(H, B, A);
    fe_sub(s, D, C);
    fe_add(G, D, C);
    if (neg) { mp_copy<8>(F, G); mp_copy<8>(G, s); } else { mp_copy<8>(F, s); }
    fe_mul(P.X, E, F);
    fe_mul(P.Y, G, H);
    if (WITH_T) fe_mul(P.T, E, H);
    fe_mul(P.Z, F, G);
}

SBV_DEV void ed_to_cached(EdCached &c, const EdP &P) {
    uint32_t d2[8];
    ed_d2(d2);
    fe_add(c.ypx, P.Y, P.X);
    fe_sub(c.ymx, P.Y, P.X);
    fe_add(c.z2, P.Z, P.Z);
    fe_mul(c.t2d, P.T, d2);
}

// canonical 32-byte encoding as little-endian limbs: y with the parity of x in bit 255
SBV_DEV void ed_encode(uint32_t (&enc)[8], const EdP &P) {
    uint32_t zi[8], x[8], y[8];
    fe_inv(zi, P.Z);
    fe_mul(x, P.X, zi);
    fe_mul(y, P.Y, zi);
    fe_canon(x, x);
    fe_canon(enc, y);
    enc[7] |= (x[0] & 1u) << 31;
}

// ---- scalars mod L ----
// r = x mod L for a 512-bit x (16 little-endian limbs): Barrett reduction with b = 2^32, k = 8 (HAC 14.42),
// mu = floor(2^512 / L) (9 limbs); one final subtraction (HAC allows two; this L and mu never need the second).
SBV_DEV void sc_reduce512(uint32_t (&r)[8], const uint32_t (&x)[16]) {
    const uint32_t mu[9] = {0x0a2c131b, 0xed9ce5a3, 0x086329a7, 0x2106215d, 0xffffffeb, 0xffffffff, 0xffffffff, 0xffffffff, 0x0000000f};
    uint32_t Lm[8];
    ed_order(Lm);
    // q3 = floor(floor(x / b^7) * mu / b^9)
    uint32_t q2[18];
#pragma unroll
    for (int i = 0; i < 18; i++) q2[i] = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) {
        uint64_t c = 0;
#pragma unroll
        for (int j = 0; j < 9; j++) {
            c += (uint64_t)x[7 + i] * mu[j] + q2[i + j];
            q2[i + j] = (uint32_t)c;
            c >>= 32;
        }
        q2[i + 9] = (uint32_t)c;
    }
    // r = (x - q3 * L) mod b^9
    uint32_t q3L[9];
#pragma unroll
    for (int i = 0; i < 9; i++) q3L[i] = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) {
        uint64_t c = 0;
#pragma unroll
        for (int j = 0; i + j < 9; j++) {
            c += (uint64_t)q2[9 + i] * (j < 8 ? Lm[j] : 0u) + q3L[i + j];
            q3L[i + j] = (uint32_t)c;
            c >>= 32;
        }
    }
    uint32_t t[9], u[9];
    t[0] = sub_cc(x[0], q3L[0]);
#pragma unroll
    for (int i = 1; i < 9; i++) t[i] = subc_cc(x[i], q3L[i]);
    // t < 1.2250 L: q - q3 <= 1 for every x < 2^512 (mu = 2^512 / L - 0.2249..., tests/ed25519_arith.py:barrett_bound),
    // so one conditional subtraction ends in [0, L)
    u[0] = sub_cc(t[0], Lm[0]);
#pragma unroll
    for (int i = 1; i < 8; i++) u[i] = subc_cc(t[i], Lm[i]);
    u[8] = subc_cc(t[8], 0);
    const bool lt = (subc(0, 0) & 1u) != 0;
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = lt ? t[i] : u[i];
}
SBV_DEV bool sc_lt_order(const uint32_t (&s)[8]) {
    uint32_t Lm[8];
    ed_order(Lm);
    return mp_lt<8>(s, Lm);
}

// signed-digit recodings, read straight from memory (the loops that use them are not unrolled):
// 4-bit Booth digit `win` of k (word-major k[w * n + idx]), in [-8, 8]
SBV_DEV int ed_digit4(const uint32_t *__restrict__ k, uint32_t n, uint32_t idx, int win) {
    const int pos = 4 * win;
    const uint32_t w = (__ldg(k + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & 15u;
    const uint32_t prev = win ? (__ldg(k + (size_t)((pos - 1) >> 5) * n + idx) >> ((pos - 1) & 31)) & 1u : 0u;
    return (int)(w & 7u) - (int)(w & 8u) + (int)prev;
}
// 8-bit Booth digit `win` of a little-endian 32-byte scalar, in [-128, 128]
SBV_DEV int ed_digit8(const uint8_t *__restrict__ s, int win) {
    const uint32_t w = __ldg(s + win);
    const uint32_t prev = win ? (uint32_t)(__ldg(s + win - 1) >> 7) : 0u;
    return (int)(w & 127u) - (int)(w & 128u) + (int)prev;
}
// 8-bit Booth digit `win` of a word-major scalar k[w * n + idx] (k < L, so window 31 carries nothing out), in [-128, 128]
SBV_DEV int ed_digit8w(const uint32_t *__restrict__ k, uint32_t n, uint32_t idx, int win) {
    const uint32_t w = (__ldg(k + (size_t)(win >> 2) * n + idx) >> (8 * (win & 3))) & 255u;
    const int pos = 8 * win - 1;
    const uint32_t prev = win ? (__ldg(k + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & 1u : 0u;
    return (int)(w & 127u) - (int)(w & 128u) + (int)prev;
}

static __device__ __noinline__ EdFe ed_fmul_call(EdFe a, EdFe b) {
    EdFe r;
    fe_mul_inline(r.v, a.v, b.v);
    return r;
}
static __device__ __noinline__ EdFe ed_fsqr_call(EdFe a) {
    EdFe r;
    fe_sqr_inline(r.v, a.v);
    return r;
}
static __device__ __noinline__ EdFe ed_inv_call(EdFe z) {
    EdFe r;
    fe_inv_inline(r.v, z.v);
    return r;
}
static __device__ __noinline__ EdRoot ed_sqrt_ratio_call(EdFe u, EdFe v) {
    EdRoot t;
    t.ok = fe_sqrt_ratio_inline(t.r.v, u.v, v.v) ? 1u : 0u;
    return t;
}

}  // namespace sbv
