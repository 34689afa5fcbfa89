// ed25519_verify.cuh — the Ed25519 verification kernel and the fixed-base table of B it reads.
//
// Accept iff S < L, A decodes, and the canonical encoding of R' = [S]B - [k]A equals the 32 bytes of R (cofactorless;
// Go crypto/ed25519.Verify, DESIGN.md §1).  k comes from k_ed_sha512 (sha512.cuh).
#pragma once
#include <stdint.h>

#include "ed25519.cuh"

namespace sbv {

// Fixed-base table of B: entry (win, j - 1) = j * 256^win * B for win = 0..31, j = 1..128, in affine Niels form
// (y + x, y - x, 2dxy), canonical, 24 words.  32 x 128 x 96 B = 384 KiB per device.
constexpr int ED_BWINS = 32, ED_BENT = 128, ED_BWORDS = 24;
constexpr size_t ED_BTAB_WORDS = (size_t)ED_BWINS * ED_BENT * ED_BWORDS;

// One entry per thread, each computed on its own: 8 * win doublings of B, a double-and-add by j, one inversion.
// Runs once per device (the first Ed25519 call), so its cost does not matter.
__global__ void __launch_bounds__(64) k_ed_btab_init(uint32_t *__restrict__ tab) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ED_BWINS * ED_BENT) return;
    const int win = (int)(t / ED_BENT);
    const uint32_t j = t % ED_BENT + 1;
    EdP P;
    ed_bx(P.X); ed_by(P.Y); ed_one(P.Z);
    fe_mul(P.T, P.X, P.Y);
#pragma unroll 1
    for (int i = 0; i < 8 * win; i++) ed_double<true>(P);
    EdCached base;
    ed_to_cached(base, P);
    const int top = 31 - __clz((int)j);
#pragma unroll 1
    for (int b = top - 1; b >= 0; b--) {
        ed_double<true>(P);
        if ((j >> b) & 1u) ed_add<true, false>(P, base.ypx, base.ymx, base.t2d, base.z2, false);
    }
    uint32_t zi[8], x[8], y[8], xy[8], d2[8], o[8];
    fe_inv(zi, P.Z);
    fe_mul(x, P.X, zi);
    fe_mul(y, P.Y, zi);
    fe_mul(xy, x, y);
    ed_d2(d2);
    uint32_t *out = tab + (size_t)t * ED_BWORDS;
    fe_add(o, y, x);
    fe_canon(o, o);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = o[i];
    fe_sub(o, y, x);
    fe_canon(o, o);
#pragma unroll
    for (int i = 0; i < 8; i++) out[8 + i] = o[i];
    fe_mul(o, xy, d2);
    fe_canon(o, o);
#pragma unroll
    for (int i = 0; i < 8; i++) out[16 + i] = o[i];
}

// little-endian 32-byte value as 8 limbs (16-byte aligned)
SBV_DEV void ed_load32(uint32_t (&r)[8], const uint8_t *__restrict__ p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    const uint4 a = __ldg(q), b = __ldg(q + 1);
    r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}

// k_ed_verify — one signature per thread.  [k](-A) with 4-bit signed windows over 1A..8A (cached form, in shared memory
// with bank = lane: 1 KiB per thread), 252 doublings and 64 additions; then [S]B with 8-bit signed windows from the
// fixed-base table (32 additions, no doublings); one inversion to encode R'.
// sig: 64 bytes per item (R || S); pub: 32 bytes per item; k: word-major [8][n].
// list (optional): thread t verifies item list[t] for t < *count (the keys of a grouped launch that got no table);
// NULL: item t < n.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_ed_verify(uint32_t n, const uint8_t *__restrict__ sig, const uint8_t *__restrict__ pub,
                                                     const uint32_t *__restrict__ k, const uint4 *__restrict__ btab,
                                                     uint8_t *__restrict__ ok_out, const uint32_t *__restrict__ list,
                                                     const uint32_t *__restrict__ count) {
    extern __shared__ uint32_t tab[];  // [((e - 1) * 4 + coord) * 8 + limb][BLOCK], e = 1..8
    const uint32_t tid = threadIdx.x;
    const uint32_t t = blockIdx.x * BLOCK + tid;
    if (t >= (list ? __ldg(count) : n)) return;  // the table is thread-private: no block-wide barrier anywhere
    const uint32_t idx = list ? __ldg(list + t) : t;
#define TAB(e, c, w) tab[((((e) - 1) * 4 + (c)) * 8 + (w)) * BLOCK + tid]
    {
        uint32_t s[8];
        ed_load32(s, sig + (size_t)idx * 64 + 32);
        if (!sc_lt_order(s)) { ok_out[idx] = 0; return; }
    }
    EdP acc;
    {
        uint32_t enc[8];
        ed_load32(enc, pub + (size_t)idx * 32);
        if (!ed_decode(acc, enc)) { ok_out[idx] = 0; return; }
        // 1A..8A: 2A by doubling, then +A
        EdCached a1;
        ed_to_cached(a1, acc);
#pragma unroll 1
        for (int e = 1; e <= 8; e++) {
            if (e == 2) ed_double<true>(acc);
            else if (e > 2) ed_add<true, false>(acc, a1.ypx, a1.ymx, a1.t2d, a1.z2, false);
            EdCached c;
            ed_to_cached(c, acc);
#pragma unroll
            for (int i = 0; i < 8; i++) { TAB(e, 0, i) = c.ypx[i]; TAB(e, 1, i) = c.ymx[i]; TAB(e, 2, i) = c.z2[i]; TAB(e, 3, i) = c.t2d[i]; }
        }
    }
    ed_identity(acc);
#pragma unroll 1
    for (int win = 63; win >= 0; win--) {
        if (win != 63) {
            ed_double<false>(acc);
            ed_double<false>(acc);
            ed_double<false>(acc);
            ed_double<true>(acc);
        }
        const int d = ed_digit4(k, n, idx, win);
        if (d != 0) {
            const int e = d < 0 ? -d : d;
            uint32_t ypx[8], ymx[8], z2[8], t2d[8];
#pragma unroll
            for (int i = 0; i < 8; i++) { ypx[i] = TAB(e, 0, i); ymx[i] = TAB(e, 1, i); z2[i] = TAB(e, 2, i); t2d[i] = TAB(e, 3, i); }
            ed_add<true, false>(acc, ypx, ymx, t2d, z2, d > 0);  // d > 0: subtract d*A
        }
    }
    const uint8_t *s_bytes = sig + (size_t)idx * 64 + 32;
#pragma unroll 1
    for (int win = 0; win < ED_BWINS; win++) {
        const int d = ed_digit8(s_bytes, win);
        if (d == 0) continue;
        const int e = d < 0 ? -d : d;
        const uint4 *q = btab + ((size_t)win * ED_BENT + (e - 1)) * (ED_BWORDS / 4);
        uint32_t ypx[8], ymx[8], t2d[8];
        {
            const uint4 v0 = __ldg(q), v1 = __ldg(q + 1), v2 = __ldg(q + 2), v3 = __ldg(q + 3), v4 = __ldg(q + 4), v5 = __ldg(q + 5);
            ypx[0] = v0.x; ypx[1] = v0.y; ypx[2] = v0.z; ypx[3] = v0.w; ypx[4] = v1.x; ypx[5] = v1.y; ypx[6] = v1.z; ypx[7] = v1.w;
            ymx[0] = v2.x; ymx[1] = v2.y; ymx[2] = v2.z; ymx[3] = v2.w; ymx[4] = v3.x; ymx[5] = v3.y; ymx[6] = v3.z; ymx[7] = v3.w;
            t2d[0] = v4.x; t2d[1] = v4.y; t2d[2] = v4.z; t2d[3] = v4.w; t2d[4] = v5.x; t2d[5] = v5.y; t2d[6] = v5.z; t2d[7] = v5.w;
        }
        ed_add<true, true>(acc, ypx, ymx, t2d, ypx, d < 0);
    }
#undef TAB
    uint32_t enc[8], r[8];
    ed_encode(enc, acc);
    ed_load32(r, sig + (size_t)idx * 64);
    ok_out[idx] = mp_eq<8>(enc, r) ? 1 : 0;
}

}  // namespace sbv
