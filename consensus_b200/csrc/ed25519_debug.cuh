// ed25519_debug.cuh — test hooks of the Ed25519 arithmetic (debug.cu on the device, tools/hostsim on the CPU).
// Field and scalar ops: slots of ED_DEBUG_WORDS little-endian 32-bit words in and out; the operands are a = in[0..8),
// b = in[8..16).  Point ops: wider slots, see ed_point_dispatch.
#pragma once
#include "ed25519.cuh"

namespace sbv {

constexpr int ED_DEBUG_WORDS = 24;
enum EdDebugOp {
    ED_DBG_MUL = 0,      // out[0..8) = a * b, reduced by folding (any value < 2^256 that is right mod p)
    ED_DBG_SQR = 1,      // a^2, likewise
    ED_DBG_ADD = 2,      // a + b, likewise
    ED_DBG_SUB = 3,      // a - b, likewise
    ED_DBG_CANON = 4,    // a mod p in [0, p)
    ED_DBG_INV = 5,      // 1/a, canonical
    ED_DBG_SQRT = 6,     // sqrt_ratio(a, b): out[0..8) the root (canonical), out[8] = was square
    ED_DBG_DECODE = 7,   // decode the encoding a: out[0..8) = x, out[8..16) = y (canonical), out[16] = ok
    ED_DBG_REDUCE = 8,   // in[0..16) (512 bits) mod L
};

SBV_DEV void ed_debug_dispatch(int op, uint32_t i, const uint32_t *in_all, uint32_t *out_all) {
    const uint32_t *in = in_all + (size_t)i * ED_DEBUG_WORDS;
    uint32_t *out = out_all + (size_t)i * ED_DEBUG_WORDS;
    uint32_t a[8], b[8], r[8];
    for (int k = 0; k < 8; k++) { a[k] = in[k]; b[k] = in[8 + k]; }
    for (int k = 0; k < ED_DEBUG_WORDS; k++) out[k] = 0;
    switch (op) {
    case ED_DBG_MUL: fe_mul(r, a, b); break;
    case ED_DBG_SQR: fe_sqr(r, a); break;
    case ED_DBG_ADD: fe_add(r, a, b); break;
    case ED_DBG_SUB: fe_sub(r, a, b); break;
    case ED_DBG_CANON: fe_canon(r, a); break;
    case ED_DBG_INV: fe_inv(r, a); fe_canon(r, r); break;
    case ED_DBG_SQRT: out[8] = fe_sqrt_ratio(r, a, b) ? 1u : 0u; break;
    case ED_DBG_DECODE: {
        EdP P;
        out[16] = ed_decode(P, a) ? 1u : 0u;
        fe_canon(r, P.X);
        uint32_t y[8];
        fe_canon(y, P.Y);
        for (int k = 0; k < 8; k++) out[8 + k] = y[k];
        break;
    }
    case ED_DBG_REDUCE: {
        uint32_t x[16];
        for (int k = 0; k < 16; k++) x[k] = in[k];
        sc_reduce512(r, x);
        break;
    }
    default: return;
    }
    for (int k = 0; k < 8; k++) out[k] = r[k];
}

// Point ops: slots of ED_POINT_WORDS words, P = in[0..32) and Q = in[32..64) as extended points (X, Y, Z, T, 8 raw limbs
// each, any value < 2^256).  The low byte of op is the operation, ED_PT_* flags above it; out[0..32) is the result as the
// device holds it (not reduced), the rest zero.
constexpr int ED_POINT_WORDS = 64;
enum EdPointOp {
    ED_PT_DOUBLE = 0,  // ed_double<!NO_T>(P); without T, out's T is P.T (not written)
    ED_PT_ADD = 1,     // ed_add<!NO_T, AFFINE>(P, ed_to_cached(Q), NEG): P + Q or P - Q (AFFINE: Q.Z must be 1, 2Z not read)
    ED_PT_CACHED = 2,  // ed_to_cached(P): Y+X, Y-X, 2Z, 2dT
    ED_PT_ENCODE = 3,  // out[0..8) = ed_encode(P), canonical
};
constexpr int ED_PT_NO_T = 0x100, ED_PT_AFFINE = 0x200, ED_PT_NEG = 0x400;
// the ops the dispatch runs: flags only on the ops that take them
inline bool ed_point_op_ok(int op) {
    const int base = op & 0xff, flags = op & ~0xff;
    if (base == ED_PT_DOUBLE) return (flags & ~ED_PT_NO_T) == 0;
    if (base == ED_PT_ADD) return (flags & ~(ED_PT_NO_T | ED_PT_AFFINE | ED_PT_NEG)) == 0;
    return (base == ED_PT_CACHED || base == ED_PT_ENCODE) && flags == 0;
}

SBV_DEV void ed_point_dispatch(int op, uint32_t i, const uint32_t *in_all, uint32_t *out_all) {
    const uint32_t *in = in_all + (size_t)i * ED_POINT_WORDS;
    uint32_t *out = out_all + (size_t)i * ED_POINT_WORDS;
    EdP P, Q;
    for (int k = 0; k < 8; k++) {
        P.X[k] = in[k]; P.Y[k] = in[8 + k]; P.Z[k] = in[16 + k]; P.T[k] = in[24 + k];
        Q.X[k] = in[32 + k]; Q.Y[k] = in[40 + k]; Q.Z[k] = in[48 + k]; Q.T[k] = in[56 + k];
    }
    for (int k = 0; k < ED_POINT_WORDS; k++) out[k] = 0;
    const bool with_t = !(op & ED_PT_NO_T), affine = (op & ED_PT_AFFINE) != 0, neg = (op & ED_PT_NEG) != 0;
    switch (op & 0xff) {
    case ED_PT_DOUBLE:
        if (with_t) ed_double<true>(P);
        else ed_double<false>(P);
        break;
    case ED_PT_ADD: {
        EdCached c;
        ed_to_cached(c, Q);
        if (with_t && affine) ed_add<true, true>(P, c.ypx, c.ymx, c.t2d, c.z2, neg);
        else if (with_t) ed_add<true, false>(P, c.ypx, c.ymx, c.t2d, c.z2, neg);
        else if (affine) ed_add<false, true>(P, c.ypx, c.ymx, c.t2d, c.z2, neg);
        else ed_add<false, false>(P, c.ypx, c.ymx, c.t2d, c.z2, neg);
        break;
    }
    case ED_PT_CACHED: {
        EdCached c;
        ed_to_cached(c, P);
        mp_copy<8>(P.X, c.ypx); mp_copy<8>(P.Y, c.ymx); mp_copy<8>(P.Z, c.z2); mp_copy<8>(P.T, c.t2d);
        break;
    }
    case ED_PT_ENCODE: {
        uint32_t enc[8];
        ed_encode(enc, P);
        for (int k = 0; k < 8; k++) out[k] = enc[k];
        return;
    }
    default: return;
    }
    for (int k = 0; k < 8; k++) {
        out[k] = P.X[k]; out[8 + k] = P.Y[k]; out[16 + k] = P.Z[k]; out[24 + k] = P.T[k];
    }
}

}  // namespace sbv
