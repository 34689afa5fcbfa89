// ed25519_debug.cuh — test hooks of the Ed25519 arithmetic (debug.cu on the device, tools/hostsim on the CPU).
// Slots of ED_DEBUG_WORDS little-endian 32-bit words in and out; the operands are a = in[0..8), b = in[8..16).
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

}  // namespace sbv
