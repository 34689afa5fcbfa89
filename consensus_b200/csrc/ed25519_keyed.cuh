// ed25519_keyed.cuh — registered Ed25519 keys (sbv_ed25519_set_keys / sbv_ed25519_verify_registered): the per-key
// fixed-base tables, the gather of the registered key bytes that SHA-512 hashes, and the verification kernel that reads
// both fixed-base tables.
//
// With a table per key, [k](-A) is a fixed-base multiplication like [S]B: 32 affine additions instead of decoding A,
// building 1A..8A and 252 doublings.  The accept set is k_ed_verify's (ed25519_verify.cuh): S < L, A decodes, and the
// canonical encoding of [S]B - [k]A equals R.
#pragma once
#include <stdint.h>

#include "ed25519_verify.cuh"

namespace sbv {

// Table of a registered key A, laid out as the table of B: entry (win, j - 1) = j * 256^win * A for win = 0..31,
// j = 1..128, affine Niels (y + x, y - x, 2dxy), canonical, 24 words.  384 KiB per key.
constexpr size_t ED_KTAB_WORDS = ED_BTAB_WORDS;
constexpr uint32_t ED_KBUILD_MAX = 1024;  // keys per k_ed_ktab_build launch (bounds its prefix-product scratch)

// One thread per registry slot: decodes the slot's 32 bytes as ed_decode does; xy[16 * t ..] = x then y (8 limbs each,
// not necessarily canonical), flag[t] = 1 when the key decodes.
__global__ void __launch_bounds__(64) k_ed_kdecode(uint32_t n, const uint8_t *__restrict__ pub, uint32_t *__restrict__ xy,
                                                   uint8_t *__restrict__ flag) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t enc[8];
    ed_load32(enc, pub + (size_t)t * 32);
    EdP P;
    const bool ok = ed_decode(P, enc);
#pragma unroll
    for (int i = 0; i < 8; i++) { xy[(size_t)t * 16 + i] = P.X[i]; xy[(size_t)t * 16 + 8 + i] = P.Y[i]; }
    flag[t] = ok ? 1 : 0;
}

// One thread per (key, window), window-major so that the threads of a warp run doubling chains of one length.  8 * win
// doublings give 256^win A; 127 additions of it give j * 256^win A, whose (X, Y, Z) go straight into the entry's own table
// slot.  Montgomery's trick over the window's 128 Z's (prefix products in pref, word-major [128 * 8][threads]) needs one
// inversion; the backward pass rewrites each slot in place as canonical (y + x, y - x, 2dxy).
// key q of this launch is slot slot_of[q] of xy; tab = the tables of keys 0..nkeys-1 of this launch.
__global__ void __launch_bounds__(64) k_ed_ktab_build(uint32_t nkeys, const uint32_t *__restrict__ slot_of, const uint32_t *__restrict__ xy,
                                                      uint32_t *__restrict__ tab, uint32_t *__restrict__ pref) {
    const uint32_t T = nkeys * ED_BWINS;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t q = t % nkeys;
    const int win = (int)(t / nkeys);
    EdP P;
    const uint32_t *src = xy + (size_t)__ldg(slot_of + q) * 16;
#pragma unroll
    for (int i = 0; i < 8; i++) { P.X[i] = src[i]; P.Y[i] = src[8 + i]; }
    ed_one(P.Z);
    fe_mul(P.T, P.X, P.Y);
#pragma unroll 1
    for (int i = 0; i < 8 * win; i++) ed_double<true>(P);
    EdCached base;
    ed_to_cached(base, P);
    uint32_t *out = tab + ((size_t)q * ED_BWINS + win) * ED_BENT * ED_BWORDS;
    uint32_t run[8];
    ed_one(run);
#pragma unroll 1
    for (int j = 0; j < ED_BENT; j++) {
        if (j) ed_add<true, false>(P, base.ypx, base.ymx, base.t2d, base.z2, false);
        uint32_t *o = out + (size_t)j * ED_BWORDS;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            o[i] = P.X[i]; o[8 + i] = P.Y[i]; o[16 + i] = P.Z[i];
            pref[((size_t)j * 8 + i) * T + t] = run[i];
        }
        fe_mul(run, run, P.Z);
    }
    uint32_t inv[8], d2[8];
    fe_inv(inv, run);
    ed_d2(d2);
#pragma unroll 1
    for (int j = ED_BENT - 1; j >= 0; j--) {
        uint32_t *o = out + (size_t)j * ED_BWORDS;
        uint32_t X[8], Y[8], Z[8], pv[8], zi[8], x[8], y[8], r[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { X[i] = o[i]; Y[i] = o[8 + i]; Z[i] = o[16 + i]; pv[i] = pref[((size_t)j * 8 + i) * T + t]; }
        fe_mul(zi, inv, pv);   // 1 / Z_j
        fe_mul(inv, inv, Z);   // 1 / (Z_0 ... Z_{j-1})
        fe_mul(x, X, zi);
        fe_mul(y, Y, zi);
        fe_add(r, y, x);
        fe_canon(r, r);
#pragma unroll
        for (int i = 0; i < 8; i++) o[i] = r[i];
        fe_sub(r, y, x);
        fe_canon(r, r);
#pragma unroll
        for (int i = 0; i < 8; i++) o[8 + i] = r[i];
        fe_mul(r, x, y);
        fe_mul(r, r, d2);
        fe_canon(r, r);
#pragma unroll
        for (int i = 0; i < 8; i++) o[16 + i] = r[i];
    }
}

// pub_out[i] = the 32 bytes registered in slot key_slot[i], zeros for a slot >= n_slots: k_ed_sha512 then hashes exactly
// the bytes the caller registered.  Two 16-byte halves per item, one per thread.
__global__ void __launch_bounds__(256) k_ed_key_gather(uint32_t n, const uint32_t *__restrict__ key_slot, uint32_t n_slots,
                                                       const uint4 *__restrict__ kpub, uint4 *__restrict__ pub_out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * n) return;
    const uint32_t s = __ldg(key_slot + (t >> 1));
    pub_out[t] = s < n_slots ? __ldg(kpub + 2 * (size_t)s + (t & 1)) : make_uint4(0, 0, 0, 0);
}

// entry e - 1 of a fixed-base table row (6 x 16 bytes: y + x, y - x, 2dxy)
SBV_DEV void ed_load_niels(uint32_t (&ypx)[8], uint32_t (&ymx)[8], uint32_t (&t2d)[8], const uint4 *__restrict__ q) {
    const uint4 v0 = __ldg(q), v1 = __ldg(q + 1), v2 = __ldg(q + 2), v3 = __ldg(q + 3), v4 = __ldg(q + 4), v5 = __ldg(q + 5);
    ypx[0] = v0.x; ypx[1] = v0.y; ypx[2] = v0.z; ypx[3] = v0.w; ypx[4] = v1.x; ypx[5] = v1.y; ypx[6] = v1.z; ypx[7] = v1.w;
    ymx[0] = v2.x; ymx[1] = v2.y; ymx[2] = v2.z; ymx[3] = v2.w; ymx[4] = v3.x; ymx[5] = v3.y; ymx[6] = v3.z; ymx[7] = v3.w;
    t2d[0] = v4.x; t2d[1] = v4.y; t2d[2] = v4.z; t2d[3] = v4.w; t2d[4] = v5.x; t2d[5] = v5.y; t2d[6] = v5.z; t2d[7] = v5.w;
}

// k_ed_verify_keyed — one signature per thread, no shared memory.  S < L; slot -> table (reject for a slot >= n_slots or a
// key that does not decode: slot2local < 0); -[k]A in 32 affine additions from the key's table (8-bit signed digits of k,
// d > 0 subtracts d * 256^win * A); then [S]B in 32 from the table of B, as k_ed_verify; one inversion to encode R'.
// sig: 64 bytes per item (R || S); key_slot: one word per item; k: word-major [8][n].
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_ed_verify_keyed(uint32_t n, const uint8_t *__restrict__ sig, const uint32_t *__restrict__ key_slot,
                                                           uint32_t n_slots, const int32_t *__restrict__ slot2local, const uint4 *__restrict__ ktab,
                                                           const uint32_t *__restrict__ k, const uint4 *__restrict__ btab, uint8_t *__restrict__ ok_out) {
    const uint32_t idx = blockIdx.x * BLOCK + threadIdx.x;
    if (idx >= n) return;
    {
        uint32_t s[8];
        ed_load32(s, sig + (size_t)idx * 64 + 32);
        if (!sc_lt_order(s)) { ok_out[idx] = 0; return; }
    }
    const uint32_t slot = __ldg(key_slot + idx);
    const int32_t loc = slot < n_slots ? __ldg(slot2local + slot) : -1;
    if (loc < 0) { ok_out[idx] = 0; return; }
    const uint4 *kt = ktab + (size_t)loc * (ED_KTAB_WORDS / 4);
    const uint8_t *s_bytes = sig + (size_t)idx * 64 + 32;
    EdP acc;
    ed_identity(acc);
    // steps 0..31: the windows of k over the key's table; steps 32..63: the windows of S over the table of B
#pragma unroll 1
    for (int step = 0; step < 2 * ED_BWINS; step++) {
        const bool key = step < ED_BWINS;
        const int win = key ? step : step - ED_BWINS;
        const int d = key ? ed_digit8w(k, n, idx, win) : ed_digit8(s_bytes, win);
        if (d == 0) continue;
        const int e = d < 0 ? -d : d;
        uint32_t ypx[8], ymx[8], t2d[8], nt[8];
        ed_load_niels(ypx, ymx, t2d, (key ? kt : btab) + ((size_t)win * ED_BENT + (e - 1)) * (ED_BWORDS / 4));
        // -Q = (y - x, y + x, -2dxy), selected limb by limb: ed_add's own run-time sign would put the entry on the stack
        const bool neg = key ? d > 0 : d < 0;  // key: d > 0 subtracts d * 256^win * A
        fe_neg(nt, t2d);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const uint32_t a = ypx[i], b = ymx[i];
            ypx[i] = neg ? b : a;
            ymx[i] = neg ? a : b;
            t2d[i] = neg ? nt[i] : t2d[i];
        }
        ed_add<true, true>(acc, ypx, ymx, t2d, ypx, false);
    }
    uint32_t enc[8], r[8];
    ed_encode(enc, acc);
    ed_load32(r, sig + (size_t)idx * 64);
    ok_out[idx] = mp_eq<8>(enc, r) ? 1 : 0;
}

}  // namespace sbv
