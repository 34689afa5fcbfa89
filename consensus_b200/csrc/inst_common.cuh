// inst_common.cuh — launcher templates behind ops.h.  Each inst_*.cu instantiates one group for one curve.
#pragma once
#include "key_cache.cuh"
#include "key_cache_assoc.cuh"
#include "keygroup.cuh"
#include "ops.h"

namespace sbv {

// Blocks of 64 threads per SM (MINB) and inlined multiplications (INL) of each kernel, per curve.
template <class C> struct Cfg;
// P-256: the fixed-base kernels run with their multiplications inlined at 6 blocks per SM (window kernel 168 registers,
// comb kernel 152, no spills; the window kernel is equal or slightly ahead of the out-of-line build at 7 blocks, which
// spills); the generic kernel likewise at 6 blocks (no spills) now that it only sees the keys that do not repeat.
// COMB_INL also inlines the loops of the comb tables' build (k_kt_bases2, k_comb_fill_warp, k_comb_final: 71, 102 and 96
// registers, no spills; one site per multiplication of each loop).  k_gpart keeps its multiplications out of line (138
// registers): inlined (146 registers, no spills) it ran 14 % faster alone but did not raise the pipelined throughput
// (DESIGN.md §10).
template <> struct Cfg<P256> {
    static constexpr int COZ_MINB = 6, GPART_MINB = 6, KT_MINB = 6, COMB_MINB = 6;
    static constexpr bool KT_INL = true, COMB_INL = true;
};
template <> struct Cfg<P384> {
    static constexpr int COZ_MINB = 4, GPART_MINB = 3, KT_MINB = 4;
    static constexpr bool KT_INL = false;
};

template <class C>
cudaError_t op_gtable_init(uint32_t *gtab, cudaStream_t st) {
    const size_t entries = (size_t)C::GWINS << C::GW;
    k_gtable_init<C><<<(unsigned)((entries + 127) / 128), 128, 0, st>>>(gtab);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_prep(uint32_t n, const uint8_t *r, const uint8_t *s, const uint8_t *dig, uint32_t dlen, uint32_t *uw, uint8_t *flags,
                    cudaStream_t st) {
    return launch_prep<C, 8>(n, r, s, dig, dlen, uw, flags, st);
}

template <class C>
cudaError_t op_group(uint32_t n, const uint8_t *qx, const uint8_t *qy, uint32_t seed, uint32_t hmask, uint32_t *htab, uint32_t *rep,
                     uint32_t *kcnt, uint32_t threshold, uint32_t max_keys, int32_t *keyid, uint32_t *keylist, uint32_t *counters,
                     cudaStream_t st) {
    const unsigned blocks = (n + 255) / 256;
    k_kg_insert<<<blocks, 256, 0, st>>>(n, KgXY<C>{qx, qy}, seed, hmask, htab, rep, kcnt);
    k_kg_assign<<<blocks, 256, 0, st>>>(n, rep, kcnt, threshold, max_keys, keyid, keylist, counters);
    return cudaGetLastError();
}

inline cudaError_t op_route(uint32_t n, const uint32_t *rep, const int32_t *keyid, int32_t *item_kid, uint32_t *klist, uint32_t *glist,
                            uint32_t *counters, cudaStream_t st) {
    k_kg_route<<<(n + 255) / 256, 256, 0, st>>>(n, rep, keyid, item_kid, klist, glist, counters);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_gpart(uint32_t n, const uint32_t *uw, const uint32_t *gtab, uint32_t *gacc, cudaStream_t st) {
    constexpr int BLOCK = 64;
    k_gpart<C, BLOCK, Cfg<C>::GPART_MINB><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, st>>>(n, uw, reinterpret_cast<const uint4 *>(gtab), gacc);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_coz(uint32_t n, const uint8_t *qx, const uint8_t *qy, const uint8_t *r, const uint32_t *uw, const uint8_t *flags,
                   const uint32_t *gtab, uint32_t *tscr, uint8_t *ok, const uint32_t *list, const uint32_t *count, cudaStream_t st) {
    constexpr int BLOCK = 64;
    const size_t smem = (size_t)7 * 2 * C::N * 4 * BLOCK;  // < 48 KB for both curves: no opt-in attribute needed
    k_verify_coz<C, BLOCK, Cfg<C>::COZ_MINB><<<(n + BLOCK - 1) / BLOCK, BLOCK, smem, st>>>(
        n, qx, qy, r, uw, flags, reinterpret_cast<const uint4 *>(gtab), tscr, ok, list, count);
    return cudaGetLastError();
}

// window tables (registered keys; P-384 keys grouped inside a launch)
template <class C, int W>
cudaError_t op_kt_build(const uint32_t *nkeys_ptr, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy,
                        uint32_t *bases, uint32_t *hs, uint32_t *ztop, uint32_t *pref, uint32_t *ktab, uint8_t *keyflags, cudaStream_t st) {
    using KT = KeyTab<32 * C::N, W>;
    const unsigned kb = (cap + 63) / 64;
    const unsigned wb = (unsigned)(((size_t)cap * KT::NWIN + 63) / 64);
    k_kt_bases4<C, KT><<<(unsigned)(((size_t)cap * 4 + 127) / 128), 128, 0, st>>>(nkeys_ptr, cap, keylist, qx, qy, bases, keyflags);
    k_kt_fill<C, W><<<wb, 64, 0, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop, ktab);
    k_kt_inv<C, KT><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keyflags, ztop, pref);
    k_kt_final<C, KT><<<wb, 64, 0, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop, ktab);
    return cudaGetLastError();
}

template <class C, int W>
cudaError_t op_kt_verify_grouped(uint32_t n, const int32_t *kidmap, const uint8_t *keyflags, const uint8_t *r, const uint32_t *uw, const uint8_t *flags,
                                 const uint32_t *gtab, const uint32_t *ktab, uint8_t *ok, const uint32_t *list, const uint32_t *count,
                                 const uint32_t *gacc, cudaStream_t st) {
    constexpr int BLOCK = 64;
    k_verify_kt<C, W, BLOCK, Cfg<C>::KT_MINB, false, Cfg<C>::KT_INL><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, st>>>(
        n, nullptr, kidmap, 0, keyflags, r, uw, flags, reinterpret_cast<const uint4 *>(gtab), reinterpret_cast<const uint4 *>(ktab), ok, list, count,
        gacc);
    return cudaGetLastError();
}

template <class C, int W>
cudaError_t op_kt_verify_registered(uint32_t n, const uint32_t *slot, const int32_t *slot2local, uint32_t n_slots, const uint8_t *keyflags,
                                    const uint8_t *r, const uint32_t *uw, const uint8_t *flags, const uint32_t *gtab, const uint32_t *ktab,
                                    uint8_t *ok, int warp, cudaStream_t st) {
    constexpr int BLOCK = 64;
    const uint4 *g4 = reinterpret_cast<const uint4 *>(gtab), *k4 = reinterpret_cast<const uint4 *>(ktab);
    if (warp)
        k_verify_kt_warp<C, W><<<(unsigned)(((size_t)n * 32 + 127) / 128), 128, 0, st>>>(n, slot, slot2local, n_slots, keyflags, r, uw, flags, g4, k4, ok);
    else
        k_verify_kt<C, W, BLOCK, Cfg<C>::KT_MINB, true, Cfg<C>::KT_INL><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, st>>>(
            n, slot, slot2local, n_slots, keyflags, r, uw, flags, g4, k4, ok, nullptr, nullptr, nullptr);
    return cudaGetLastError();
}

// comb tables (P-256 keys grouped inside a launch)
template <class C>
cudaError_t op_comb_build(const uint32_t *nkeys_ptr, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy,
                          uint32_t *bases, uint32_t *hs, uint32_t *ztop, uint32_t *pref, uint32_t *ktab, uint8_t *keyflags, cudaStream_t st) {
    using CT = CombTab<C>;
    const unsigned kb = (cap + 63) / 64;
    const unsigned wb = (unsigned)(((size_t)cap * 32 + 63) / 64);  // a warp per key
    constexpr bool INL = Cfg<C>::COMB_INL;
    constexpr size_t fill_smem = (size_t)2 * CT::NBASE * 2 * C::N * 4;                 // two warps x 16 affine bases
    constexpr size_t final_smem = (size_t)2 * 32 * (CT::ENT / 2 * 2 * C::N / 4 + 1) * 16;  // two warps x 32 half chains
    k_kt_bases2<C, CT, INL><<<(unsigned)(((size_t)cap * 2 + 127) / 128), 128, 0, st>>>(nkeys_ptr, cap, keylist, qx, qy, bases, keyflags);
    k_comb_affine<C><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keyflags, bases, pref);
    k_comb_fill_warp<C, INL><<<wb, 64, fill_smem, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop);
    k_kt_inv<C, CT, CombScr<C>><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keyflags, ztop, pref);
    k_comb_final<C, INL><<<wb, 64, final_smem, st>>>(nkeys_ptr, cap, keyflags, hs, ztop, ktab);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_comb_verify(uint32_t n, const int32_t *kidmap, const uint8_t *keyflags, const uint8_t *r, const uint32_t *uw, const uint8_t *flags,
                           const uint32_t * /* gtab: u1*G comes in gacc */, const uint32_t *ktab, uint8_t *ok, const uint32_t *list,
                           const uint32_t *count, const uint32_t *gacc, cudaStream_t st) {
    constexpr int BLOCK = 64;
    k_verify_comb<C, BLOCK, Cfg<C>::COMB_MINB, Cfg<C>::COMB_INL><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, st>>>(
        n, kidmap, keyflags, r, uw, flags, reinterpret_cast<const uint4 *>(ktab), ok, list, count, gacc);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_kc_lookup(const uint32_t *nkeys_ptr, uint32_t kcap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy, KcMap c, uint32_t tw4,
                         int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab, cudaStream_t st) {
    k_kc_lookup<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(nkeys_ptr, kcap, keylist, KcXY<C>{qx, qy}, c, tw4, keyid, lk, keyflags,
                                                                            reinterpret_cast<uint4 *>(ktab));
    return cudaGetLastError();
}

template <class C>
cudaError_t op_kc_insert(uint32_t kcap, const uint32_t *lk, const uint8_t *qx, const uint8_t *qy, KcMap c, uint32_t tw4, const uint8_t *keyflags,
                         const uint32_t *ktab, cudaStream_t st) {
    k_kc_insert<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(kcap, lk, KcXY<C>{qx, qy}, c, tw4, keyflags,
                                                                            reinterpret_cast<const uint4 *>(ktab));
    return cudaGetLastError();
}

template <class C>
cudaError_t op_kca_lookup(const uint32_t *nkeys_ptr, uint32_t kcap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy, KcaMap c,
                          unsigned long long now, uint32_t tw4, int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab, cudaStream_t st) {
    k_kca_lookup<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(nkeys_ptr, kcap, keylist, KcXY<C>{qx, qy}, c, now, tw4, keyid, lk,
                                                                             keyflags, reinterpret_cast<uint4 *>(ktab));
    return cudaGetLastError();
}

template <class C>
cudaError_t op_kca_insert(uint32_t kcap, const uint32_t *lk, const uint8_t *qx, const uint8_t *qy, KcaMap c, unsigned long long now, uint32_t tw4,
                          const uint8_t *keyflags, const uint32_t *ktab, cudaStream_t st) {
    k_kca_insert<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(kcap, lk, KcXY<C>{qx, qy}, c, now, tw4, keyflags,
                                                                             reinterpret_cast<const uint4 *>(ktab));
    return cudaGetLastError();
}

template <class C, class KT>
constexpr KtGeom kt_geom() {
    using KS = KtSizes<C, KT>;
    return KtGeom{KS::bases_words(1), KS::hs_words(1), KS::ztop_words(1), KS::ktab_words(1)};
}

}  // namespace sbv
