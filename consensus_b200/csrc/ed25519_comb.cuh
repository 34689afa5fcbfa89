// ed25519_comb.cuh — Ed25519 keys that repeat inside a keys-per-item batch (sbv_ed25519_verify_batch): a comb table per
// key, built on the device during the launch, and the fixed-base verification kernel that reads it.
//
// The grouping is keygroup.cuh's: k_kg_insert over the 32 encoded bytes of each item's key (KgKey32), k_kg_assign and
// k_kg_route.  Grouping is by bytes, not by point: k hashes the item's own encoding, so a non-canonical encoding of a
// point (y >= p, "-0") is a key of its own.
//
// Comb (Lim–Lee, as CombTab for P-256): 16 bases A_c = 2^(16c) A in two blocks of eight teeth.  A scalar k < 2^256 is
// read as 16 rows of 16 bits (row c = bits [16c, 16c + 16)); column j of the rows of block b is the mask m of entry
// T_b[m] = sum of A_(8b+t) over the set bits t of m.  [k]A then takes 15 doublings and 32 additions.
//   k_edc_bases   one thread per key: A decoded as ed_decode does (the key's flag), the 16 bases by 240 doublings
//   k_edc_fill    one thread per (key, chain), chain = (block b, high nibble hi): the entries m = 16 hi + g along a
//                 Gray-code walk of the low nibble g, one addition per entry; each entry's X, Y, Z go into its own table
//                 slot, the prefix products of the chain's Z's into hs
//   k_edc_inv     one thread per key: ONE inversion for the 32 chains (Montgomery's trick over the chains' Z products)
//   k_edc_final   one thread per (key, chain): back-substitution, each entry to canonical affine Niels in place
// The edwards25519 formulas are complete: no exceptional case and no Z = 0 for any A that decodes (small-order and
// mixed-order keys and the identity included).
#pragma once
#include <stdint.h>

#include "ed25519_keyed.cuh"

namespace sbv {

constexpr int EDC_TEETH = 8, EDC_BLOCKS = 2, EDC_NBASE = EDC_TEETH * EDC_BLOCKS, EDC_SPACING = 16;
constexpr int EDC_ENT = 255;                      // entries per block: m = 1..255
constexpr int EDC_NCHAIN = EDC_BLOCKS * 16, EDC_CHAIN = 16;  // (block, high nibble) x low nibble
// Table of a key: entry (b, m) at b * 255 + m - 1, affine Niels (y + x, y - x, 2dxy), canonical, 24 words, as the table
// of B.  510 entries x 96 B = 47.8 KiB per key.
constexpr size_t EDC_TAB_WORDS = (size_t)EDC_BLOCKS * EDC_ENT * ED_BWORDS;
// construction scratch per key, word-major by key: bases [c][32][cap] (extended X, Y, Z, T), hs [chain][step][8][cap]
// (prefix products), ztop / pref [chain][8][cap]
constexpr size_t EDC_BASES_WORDS = (size_t)EDC_NBASE * 32, EDC_HS_WORDS = (size_t)EDC_NCHAIN * EDC_CHAIN * 8,
                 EDC_ZTOP_WORDS = (size_t)EDC_NCHAIN * 8;
static_assert(EDC_SPACING * EDC_NBASE == 256, "the rows cover the scalar exactly");

// nkeys_ptr: device counter (clamped to cap); key q is the 32 bytes of item keylist[q] of pub (keylist NULL: item q).
__global__ void __launch_bounds__(64) k_edc_bases(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ keylist,
                                                  const uint8_t *__restrict__ pub, uint32_t *__restrict__ bases,
                                                  uint8_t *__restrict__ keyflags) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (q >= nkeys) return;
    const uint32_t item = keylist ? keylist[q] : q;
    uint32_t enc[8];
    ed_load32(enc, pub + (size_t)item * 32);
    EdP P;
    const bool good = ed_decode(P, enc);
    keyflags[q] = good ? 1 : 0;
    if (!good) return;  // no table: every item of this key rejects (k_ed_verify_comb checks the flag)
#pragma unroll 1
    for (int c = 0; c < EDC_NBASE; c++) {
        if (c) {
#pragma unroll 1
            for (int i = 0; i < EDC_SPACING; i++) ed_double<true>(P);
        }
        uint32_t *o = bases + (size_t)c * 32 * cap + q;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            o[(size_t)i * cap] = P.X[i]; o[(size_t)(8 + i) * cap] = P.Y[i];
            o[(size_t)(16 + i) * cap] = P.Z[i]; o[(size_t)(24 + i) * cap] = P.T[i];
        }
    }
}

// Chain (b, hi) starts at the sum of the high teeth of hi (the identity for hi = 0, whose m = 0 is not an entry), then
// walks the 15 Gray codes of the low nibble: step s (1..15) adds or subtracts A_(8b+t), t = the bit gray(s - 1) ->
// gray(s) flips.  Step s of the walk (0: the start) records its prefix product at hs[chain][s].
__global__ void __launch_bounds__(64) k_edc_fill(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ bases,
                                                 const uint8_t *__restrict__ keyflags, uint32_t *__restrict__ hs, uint32_t *__restrict__ ztop,
                                                 uint32_t *__restrict__ ctab) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (t >= nkeys * EDC_NCHAIN) return;
    const uint32_t q = t % nkeys, ch = t / nkeys;
    if (!keyflags[q]) return;
    const int b = (int)(ch >> 4), hi = (int)(ch & 15);
    uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;
    EdP P;
    ed_identity(P);
    uint32_t run[8];
    ed_one(run);
    auto add_base = [&](int c, bool neg) {
        const uint32_t *o = bases + (size_t)c * 32 * cap + q;
        EdP A;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            A.X[i] = o[(size_t)i * cap]; A.Y[i] = o[(size_t)(8 + i) * cap];
            A.Z[i] = o[(size_t)(16 + i) * cap]; A.T[i] = o[(size_t)(24 + i) * cap];
        }
        EdCached Ac;
        ed_to_cached(Ac, A);
        uint32_t (&ypx)[8] = Ac.ypx, (&ymx)[8] = Ac.ymx, (&z2)[8] = Ac.z2, (&t2d)[8] = Ac.t2d, nt[8];
        // -Q = (Y - X, Y + X, 2Z, -2dT), selected limb by limb: ed_add's own run-time sign would put Q on the stack
        fe_neg(nt, t2d);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const uint32_t a = ypx[i], b2 = ymx[i];
            ypx[i] = neg ? b2 : a;
            ymx[i] = neg ? a : b2;
            t2d[i] = neg ? nt[i] : t2d[i];
        }
        ed_add<true, false>(P, ypx, ymx, t2d, z2, false);
    };
    auto record = [&](int s, int m) {
        uint32_t *o = tab + (size_t)(m - 1) * ED_BWORDS;
        uint32_t *hp = hs + ((size_t)ch * EDC_CHAIN + s) * 8 * cap + q;
#pragma unroll
        for (int i = 0; i < 8; i++) { o[i] = P.X[i]; o[8 + i] = P.Y[i]; o[16 + i] = P.Z[i]; hp[(size_t)i * cap] = run[i]; }
        fe_mul(run, run, P.Z);
    };
#pragma unroll 1
    for (int i = 0; i < 4; i++)
        if ((hi >> i) & 1) add_base(EDC_TEETH * b + 4 + i, false);
    if (hi) record(0, 16 * hi);
#pragma unroll 1
    for (int s = 1; s < EDC_CHAIN; s++) {
        const int tooth = __ffs(s) - 1, g = s ^ (s >> 1);
        add_base(EDC_TEETH * b + tooth, !((g >> tooth) & 1));  // the bit goes off: subtract
        record(s, 16 * hi + g);
    }
    uint32_t *zp = ztop + (size_t)ch * 8 * cap + q;
#pragma unroll
    for (int i = 0; i < 8; i++) zp[(size_t)i * cap] = run[i];
}

// ztop[chain] <- 1 / ztop[chain] for the 32 chains of a key with one inversion (pref: prefix products, [chain][8][cap])
__global__ void __launch_bounds__(64) k_edc_inv(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint8_t *__restrict__ keyflags,
                                                uint32_t *__restrict__ ztop, uint32_t *__restrict__ pref) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (q >= nkeys || !keyflags[q]) return;
    uint32_t run[8];
    ed_one(run);
#pragma unroll 1
    for (int ch = 0; ch < EDC_NCHAIN; ch++) {
        uint32_t z[8];
        const uint32_t *zp = ztop + (size_t)ch * 8 * cap + q;
        uint32_t *pp = pref + (size_t)ch * 8 * cap + q;
#pragma unroll
        for (int i = 0; i < 8; i++) { z[i] = zp[(size_t)i * cap]; pp[(size_t)i * cap] = run[i]; }
        fe_mul(run, run, z);
    }
    uint32_t inv[8];
    fe_inv(inv, run);
#pragma unroll 1
    for (int ch = EDC_NCHAIN - 1; ch >= 0; ch--) {
        uint32_t *zp = ztop + (size_t)ch * 8 * cap + q;
        const uint32_t *pp = pref + (size_t)ch * 8 * cap + q;
        uint32_t z[8], pv[8], zi[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { z[i] = zp[(size_t)i * cap]; pv[i] = pp[(size_t)i * cap]; }
        fe_mul(zi, inv, pv);
        fe_mul(inv, inv, z);
#pragma unroll
        for (int i = 0; i < 8; i++) zp[(size_t)i * cap] = zi[i];
    }
}

// Walks chain (b, hi) backwards from 1 / (product of its Z's): 1 / Z_s = that * prefix_s, then times Z_s for the step
// before; each entry becomes canonical (y + x, y - x, 2dxy) in place.
__global__ void __launch_bounds__(64) k_edc_final(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint8_t *__restrict__ keyflags,
                                                  const uint32_t *__restrict__ hs, const uint32_t *__restrict__ ztop, uint32_t *__restrict__ ctab) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (t >= nkeys * EDC_NCHAIN) return;
    const uint32_t q = t % nkeys, ch = t / nkeys;
    if (!keyflags[q]) return;
    const int b = (int)(ch >> 4), hi = (int)(ch & 15);
    uint32_t *tab = ctab + (size_t)q * EDC_TAB_WORDS + (size_t)b * EDC_ENT * ED_BWORDS;
    uint32_t inv[8], d2[8];
    {
        const uint32_t *zp = ztop + (size_t)ch * 8 * cap + q;
#pragma unroll
        for (int i = 0; i < 8; i++) inv[i] = zp[(size_t)i * cap];
    }
    ed_d2(d2);
#pragma unroll 1
    for (int s = EDC_CHAIN - 1; s >= (hi ? 0 : 1); s--) {
        uint32_t *o = tab + (size_t)(16 * hi + (s ^ (s >> 1)) - 1) * ED_BWORDS;
        const uint32_t *hp = hs + ((size_t)ch * EDC_CHAIN + s) * 8 * cap + q;
        uint32_t X[8], Y[8], Z[8], pv[8], zi[8], x[8], y[8], r[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { X[i] = o[i]; Y[i] = o[8 + i]; Z[i] = o[16 + i]; pv[i] = hp[(size_t)i * cap]; }
        fe_mul(zi, inv, pv);  // 1 / Z_s
        fe_mul(inv, inv, Z);  // 1 / (Z_0 ... Z_(s-1))
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

// column j of block b of k's comb: bit t = bit 16 (8b + t) + j of k, i.e. bit 16 (t & 1) + j of word 4b + t / 2
// (word-major k[w * n + idx])
SBV_DEV uint32_t edc_mask(const uint32_t *__restrict__ k, uint32_t n, uint32_t idx, int b, int j) {
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < 4; w++) {
        const uint32_t v = __ldg(k + (size_t)(4 * b + w) * n + idx);
        m |= ((v >> j) & 1u) << (2 * w);
        m |= ((v >> (16 + j)) & 1u) << (2 * w + 1);
    }
    return m;
}

// k_ed_verify_comb — one signature per thread, no shared memory; the sibling of k_ed_verify_keyed for keys grouped inside
// a launch.  S < L; the key's flag; [k](-A) column by column from the top of k's comb (a doubling before every column
// but the first, one table addition per block, entries negated in registers); then [S]B in 32 additions from the table
// of B, after the last doubling; one inversion to encode R'.
// The item of thread t is list[t] for t < *count (list NULL: item t < n); its key is kidmap[item] (>= 0 for every
// listed item), its table ctab + kid * EDC_TAB_WORDS.  sig: 64 bytes per item (R || S); k: word-major [8][n].
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_ed_verify_comb(uint32_t n, const uint8_t *__restrict__ sig, const int32_t *__restrict__ kidmap,
                                                          const uint8_t *__restrict__ keyflags, const uint4 *__restrict__ ctab,
                                                          const uint32_t *__restrict__ k, const uint4 *__restrict__ btab,
                                                          uint8_t *__restrict__ ok_out, const uint32_t *__restrict__ list,
                                                          const uint32_t *__restrict__ count) {
    const uint32_t t = blockIdx.x * BLOCK + threadIdx.x;
    if (t >= (list ? __ldg(count) : n)) return;
    const uint32_t idx = list ? __ldg(list + t) : t;
    {
        uint32_t s[8];
        ed_load32(s, sig + (size_t)idx * 64 + 32);
        if (!sc_lt_order(s)) { ok_out[idx] = 0; return; }
    }
    const int32_t kid = kidmap[idx];
    if (kid < 0 || !keyflags[kid]) { ok_out[idx] = 0; return; }
    const uint4 *kt = ctab + (size_t)kid * (EDC_TAB_WORDS / 4);
    const uint8_t *s_bytes = sig + (size_t)idx * 64 + 32;
    constexpr int KSTEPS = EDC_SPACING * EDC_BLOCKS;
    EdP acc;
    ed_identity(acc);
    // steps 0..31: column 15 - step / 2, block step % 2 of k's comb; steps 32..63: the windows of S over the table of B
#pragma unroll 1
    for (int step = 0; step < KSTEPS + ED_BWINS; step++) {
        const bool key = step < KSTEPS;
        if (key && step && (step & 1) == 0) ed_double<true>(acc);
        int e;
        bool neg;
        if (key) {
            const int b = step & 1;
            const uint32_t m = edc_mask(k, n, idx, b, EDC_SPACING - 1 - (step >> 1));
            if (m == 0) continue;
            e = b * EDC_ENT + (int)m - 1;
            neg = true;  // the sum is [k](-A)
        } else {
            const int win = step - KSTEPS;
            const int d = ed_digit8(s_bytes, win);
            if (d == 0) continue;
            e = win * ED_BENT + (d < 0 ? -d : d) - 1;
            neg = d < 0;
        }
        uint32_t ypx[8], ymx[8], t2d[8], nt[8];
        ed_load_niels(ypx, ymx, t2d, (key ? kt : btab) + (size_t)e * (ED_BWORDS / 4));
        // -Q = (y - x, y + x, -2dxy), selected limb by limb as in k_ed_verify_keyed
        fe_neg(nt, t2d);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const uint32_t a = ypx[i], c = ymx[i];
            ypx[i] = neg ? c : a;
            ymx[i] = neg ? a : c;
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
