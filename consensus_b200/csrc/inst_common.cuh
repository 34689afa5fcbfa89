// inst_common.cuh — launcher templates behind ops.h.  Each inst_*.cu instantiates one group for one curve.
#pragma once
#include "keygroup.cuh"
#include "ops.h"
#include <cstdlib>

namespace sbv {

template <class C> struct Cfg;
// P-256: the fixed-base kernels run with their multiplications inlined at 6 blocks of 64 threads per SM (window kernel 168
// registers, comb kernel 153, no spills; the window kernel is equal or slightly ahead of the out-of-line build at 7
// blocks, which spills);
// the generic kernel likewise at 6 blocks (no spills) now that it only sees the keys that do not repeat.
template <> struct Cfg<P256> { static constexpr int COZ_MINB = 6, KT_MINB = 7, KT_VARIANT = 2, COMB_MINB = 6; static constexpr bool COMB_INL = true; };
template <> struct Cfg<P384> { static constexpr int COZ_MINB = 4, KT_MINB = 4, KT_VARIANT = 0; };

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
                     uint32_t *kcnt, uint32_t threshold, uint32_t max_keys, int32_t *keyid, uint32_t *keylist, int32_t *item_kid,
                     uint32_t *klist, uint32_t *glist, uint32_t *counters, int route, cudaStream_t st) {
    const unsigned blocks = (n + 255) / 256;
    k_kg_insert<C><<<blocks, 256, 0, st>>>(n, qx, qy, seed, hmask, htab, rep, kcnt);
    k_kg_assign<<<blocks, 256, 0, st>>>(n, rep, kcnt, threshold, max_keys, keyid, keylist, counters);
    if (route) k_kg_route<<<blocks, 256, 0, st>>>(n, rep, keyid, item_kid, klist, glist, counters);
    return cudaGetLastError();
}

[[maybe_unused]] static cudaError_t op_route(uint32_t n, const uint32_t *rep, const int32_t *keyid, int32_t *item_kid, uint32_t *klist, uint32_t *glist,
                            uint32_t *counters, cudaStream_t st) {
    k_kg_route<<<(n + 255) / 256, 256, 0, st>>>(n, rep, keyid, item_kid, klist, glist, counters);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_gpart(uint32_t n, const uint32_t *uw, const uint32_t *gtab, uint32_t *gacc, cudaStream_t st) {
    constexpr int BLOCK = 64;
    k_gpart<C, BLOCK, Cfg<C>::KT_MINB - 1><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, st>>>(n, uw, reinterpret_cast<const uint4 *>(gtab), gacc);
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
    static const int bases_variant = getenv("SBV_KT_BASES") ? atoi(getenv("SBV_KT_BASES")) : 0;  // A/B: 1 = one thread per key (inlined), 2 = (out of line)
    if (bases_variant == 2) k_kt_bases<C, KT, false><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keylist, qx, qy, bases, keyflags);
    else if (bases_variant == 1) k_kt_bases<C, KT, true><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keylist, qx, qy, bases, keyflags);
    else k_kt_bases4<C, KT><<<(unsigned)(((size_t)cap * 4 + 127) / 128), 128, 0, st>>>(nkeys_ptr, cap, keylist, qx, qy, bases, keyflags);
    k_kt_fill<C, W><<<wb, 64, 0, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop, ktab);
    k_kt_inv<C, KT><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keyflags, ztop, pref);
    k_kt_final<C, KT><<<wb, 64, 0, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop, ktab);
    return cudaGetLastError();
}

template <class C, int W>
cudaError_t op_kt_verify(int reg, int warp, uint32_t n, const uint32_t *slot, const int32_t *kidmap, uint32_t n_slots,
                         const uint8_t *keyflags, const uint8_t *r, const uint32_t *uw, const uint8_t *flags, const uint32_t *gtab,
                         const uint32_t *ktab, uint8_t *ok, const uint32_t *list, const uint32_t *count, const uint32_t *gacc, cudaStream_t st) {
    constexpr int BLOCK = 64, MINB = Cfg<C>::KT_MINB;
    static const int variant = getenv("SBV_KT_VARIANT") ? atoi(getenv("SBV_KT_VARIANT")) : Cfg<C>::KT_VARIANT;
    const uint4 *g4 = reinterpret_cast<const uint4 *>(gtab), *k4 = reinterpret_cast<const uint4 *>(ktab);
    const unsigned blocks = (n + BLOCK - 1) / BLOCK;
#define SBV_KT_ARGS n, slot, kidmap, n_slots, keyflags, r, uw, flags, g4, k4, ok, list, count, gacc
    if (warp) {
        k_verify_kt_warp<C, W><<<(unsigned)(((size_t)n * 32 + 127) / 128), 128, 0, st>>>(n, slot, kidmap, n_slots, keyflags, r, uw, flags, g4, k4, ok);
    } else if (reg) {
        if (variant == 1) k_verify_kt<C, W, BLOCK, MINB, true, true><<<blocks, BLOCK, 0, st>>>(SBV_KT_ARGS);
        else if (variant == 2) k_verify_kt<C, W, BLOCK, MINB - 1, true, true><<<blocks, BLOCK, 0, st>>>(SBV_KT_ARGS);
        else k_verify_kt<C, W, BLOCK, MINB, true, false><<<blocks, BLOCK, 0, st>>>(SBV_KT_ARGS);
    } else {
        if (variant == 1) k_verify_kt<C, W, BLOCK, MINB, false, true><<<blocks, BLOCK, 0, st>>>(SBV_KT_ARGS);          // multiplications inlined
        else if (variant == 2) k_verify_kt<C, W, BLOCK, MINB - 1, false, true><<<blocks, BLOCK, 0, st>>>(SBV_KT_ARGS); // inlined, one block fewer per SM
        else k_verify_kt<C, W, BLOCK, MINB, false, false><<<blocks, BLOCK, 0, st>>>(SBV_KT_ARGS);                      // multiplications out of line
    }
#undef SBV_KT_ARGS
    return cudaGetLastError();
}

// comb tables (P-256 keys grouped inside a launch)
template <class C>
cudaError_t op_comb_build(const uint32_t *nkeys_ptr, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy,
                          uint32_t *bases, uint32_t *hs, uint32_t *ztop, uint32_t *pref, uint32_t *ktab, uint8_t *keyflags, cudaStream_t st) {
    using CT = CombTab<C>;
    const unsigned kb = (cap + 63) / 64;
    const unsigned cb = (unsigned)(((size_t)cap * CT::NCHAIN + 63) / 64);
    k_kt_bases4<C, CT><<<(unsigned)(((size_t)cap * 4 + 127) / 128), 128, 0, st>>>(nkeys_ptr, cap, keylist, qx, qy, bases, keyflags);
    k_comb_affine<C><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keyflags, bases, pref);
    k_comb_fill<C><<<cb, 64, 0, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop, ktab);
    k_kt_inv<C, CT><<<kb, 64, 0, st>>>(nkeys_ptr, cap, keyflags, ztop, pref);
    k_kt_final<C, CT><<<cb, 64, 0, st>>>(nkeys_ptr, cap, bases, keyflags, hs, ztop, ktab);
    return cudaGetLastError();
}

template <class C>
cudaError_t op_comb_verify(int reg, int warp, uint32_t n, const uint32_t *slot, const int32_t *kidmap, uint32_t n_slots,
                           const uint8_t *keyflags, const uint8_t *r, const uint32_t *uw, const uint8_t *flags, const uint32_t *gtab,
                           const uint32_t *ktab, uint8_t *ok, const uint32_t *list, const uint32_t *count, const uint32_t *gacc, cudaStream_t st) {
    constexpr int BLOCK = 64;
    (void)slot; (void)n_slots;
    if (reg || warp || !list || !count) return cudaErrorInvalidValue;  // comb tables serve the grouped items of a launch only
    k_verify_comb<C, BLOCK, Cfg<C>::COMB_MINB, Cfg<C>::COMB_INL><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, st>>>(
        n, kidmap, keyflags, r, uw, flags, reinterpret_cast<const uint4 *>(gtab), reinterpret_cast<const uint4 *>(ktab), ok, list, count, gacc);
    return cudaGetLastError();
}

template <class C, class KT>
constexpr KtGeom kt_geom() {
    using KS = KtSizes<C, KT>;
    return KtGeom{KS::bases_words(1), KS::hs_words(1), KS::ztop_words(1), KS::ktab_words(1)};
}

}  // namespace sbv
