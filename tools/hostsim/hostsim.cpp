// hostsim.cpp — TEST INFRASTRUCTURE: the device headers of libsbv compiled for the CPU (see csrc/hostsim.h) and
// driven one simulated thread at a time.  tests/test_hostsim.py (-m "not gpu") compares the results with Python
// big integers and with the oracle, so limb-level mistakes are caught without a GPU.  Not linked into libsbv.so.
#define SBV_HOSTSIM 1
#include <stdint.h>
#include <algorithm>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../consensus_b200/csrc/hostsim.h"
thread_local hostsim_dim3 threadIdx, blockIdx, blockDim, gridDim;
thread_local hostsim_warp *hostsim_ctx = nullptr;
namespace sbv { uint32_t tab[1 << 18]; }
#include "../../consensus_b200/csrc/debug_ops.cuh"
#include "../../consensus_b200/csrc/keygroup.cuh"
#include "../../consensus_b200/csrc/key_cache.cuh"
#include "../../consensus_b200/csrc/key_cache_assoc.cuh"
#include "../../consensus_b200/csrc/sha256.cuh"
#include "../../consensus_b200/csrc/sha384.cuh"
#include "../../consensus_b200/csrc/quorum.cuh"
#include "../../consensus_b200/csrc/ed25519_debug.cuh"
#include "../../consensus_b200/csrc/sha512.cuh"
#include "../../consensus_b200/csrc/ed25519_verify.cuh"
#include "../../consensus_b200/csrc/ed25519_keyed.cuh"
#include "../../consensus_b200/csrc/ed25519_comb.cuh"
#include "../../consensus_b200/csrc/shards.h"
#include "../../consensus_b200/csrc/mixed.cuh"
#include "../../consensus_b200/csrc/mixed_hash.cuh"
#include "../../consensus_b200/csrc/rsa.cuh"
#include "../../consensus_b200/csrc/rsa_debug.cuh"
#include "../../consensus_b200/csrc/sha512_batch.cuh"

using namespace sbv;

// G comb for the simulation: T[i][b] = b * 2^(GW*i) * G, built incrementally (running sum + one batched inversion per
// window) — the device kernel k_gtable_init builds every entry independently, which a CPU cannot afford.
template <class C>
static void build_comb_host(uint32_t *tab) {
    constexpr int N = C::N;
    const size_t per = (size_t)1 << C::GW;
    Jac<C> base;
    C::get_gx(base.X); C::get_gy(base.Y); C::get_one(base.Z);
    std::vector<uint32_t> jac(per * 3 * N), pref(per * N);
    for (int win = 0; win < C::GWINS; win++) {
        if (win) for (int d = 0; d < C::GW; d++) pt_double<C>(base);
        Jac<C> acc = base;
        uint32_t run[N];
        C::get_one(run);
        for (size_t b = 1; b < per; b++) {
            if (b > 1) pt_add<C, false>(acc, base.X, base.Y, base.Z, false, false);
            memcpy(&jac[b * 3 * N], acc.X, 4 * N); memcpy(&jac[b * 3 * N + N], acc.Y, 4 * N); memcpy(&jac[b * 3 * N + 2 * N], acc.Z, 4 * N);
            memcpy(&pref[b * N], run, 4 * N);
            C::fmul(run, run, acc.Z);
        }
        uint32_t inv[N];
        f_inv<C>(inv, run);
        uint32_t *out = tab + ((size_t)win << C::GW) * 2 * N;
        memset(out, 0, 2 * N * 4);
        for (size_t b = per - 1; b >= 1; b--) {
            uint32_t pv[N], z[N], zi[N], z2[N], z3[N], x[N], y[N];
            memcpy(pv, &pref[b * N], 4 * N); memcpy(z, &jac[b * 3 * N + 2 * N], 4 * N);
            memcpy(x, &jac[b * 3 * N], 4 * N); memcpy(y, &jac[b * 3 * N + N], 4 * N);
            C::fmul(zi, inv, pv);
            C::fmul(inv, inv, z);
            C::fsqr(z2, zi); C::fmul(z3, z2, zi);
            C::fmul(x, x, z2); C::fmul(y, y, z3);
            memcpy(out + b * 2 * N, x, 4 * N); memcpy(out + b * 2 * N + N, y, 4 * N);
        }
    }
}

template <class F>
static void run_grid(unsigned blocks, unsigned threads, F &&body) {
    gridDim.x = blocks; blockDim.x = threads;
    for (unsigned b = 0; b < blocks; b++)
        for (unsigned t = 0; t < threads; t++) { blockIdx.x = b; threadIdx.x = t; body(); }
}

extern "C" int hs_debug_op(int curve, int op, size_t n, const uint32_t *a, const uint32_t *b, uint32_t *out) {
    for (size_t i = 0; i < n; i++) {
        if (curve == 0) debug_op_dispatch<P256>(op, (uint32_t)i, a, b, out);
        else debug_op_dispatch<P384>(op, (uint32_t)i, a, b, out);
    }
    return 0;
}

// LOCKSTEP form for warp-cooperative kernels: the 32 lanes of a warp are 32 OS threads that meet at every shuffle / ballot
// (hostsim.h); warps run one after the other.
template <class F>
static void run_grid_lockstep(unsigned blocks, unsigned threads, F &&body) {
    for (unsigned b = 0; b < blocks; b++)
        for (unsigned w0 = 0; w0 < threads; w0 += 32) {
            hostsim_warp ctx;
            std::vector<std::thread> lanes;
            for (unsigned t = w0; t < w0 + 32 && t < threads; t++)
                lanes.emplace_back([&, t] {
                    gridDim.x = blocks; blockDim.x = threads; blockIdx.x = b; threadIdx.x = t;
                    hostsim_ctx = &ctx;
                    body();
                    hostsim_ctx = nullptr;
                });
            for (auto &l : lanes) l.join();
        }
}

// the product's construction kernels for a window table (KT = KeyTab) or a comb table (KT = CombTab) of up to `cap` keys,
// *cnt of them, key k = item keylist[k] of qx / qy (keylist NULL: item k).  four == 1: the doubling chain by k_kt_bases4
// (four lanes per key, in lockstep), four == 2: by k_kt_bases2 (two lanes per key, in lockstep; what libsbv.so runs for a
// comb), else by the one-thread-per-key k_kt_bases.  ktab: KtSizes::ktab_words(cap) words of
// final affine tables, kflags: cap validity flags.
template <class C, class KT>
static void bases_t(const uint32_t *cnt, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy, int four, uint32_t *bases,
                    uint8_t *kflags) {
    constexpr bool COMB = std::is_same<KT, CombTab<C>>::value;  // the comb build runs inlined multiplications, as in libsbv.so
    if (four == 2) run_grid_lockstep((unsigned)(((size_t)cap * 2 + 127) / 128), 128, [&] { k_kt_bases2<C, KT, COMB>(cnt, cap, keylist, qx, qy, bases, kflags); });
    else if (four) run_grid_lockstep((unsigned)(((size_t)cap * 4 + 127) / 128), 128, [&] { k_kt_bases4<C, KT>(cnt, cap, keylist, qx, qy, bases, kflags); });
    else run_grid((cap + 63) / 64, 64, [&] { k_kt_bases<C, KT>(cnt, cap, keylist, qx, qy, bases, kflags); });
}

// What the comb build leaves between its kernels, in one order whatever the scratch layout (key k = 0..cap-1, chain ch):
// jac [k][ch][slot][2N] the fill's Jacobian X, Y; hs [k][ch][slot-1][N] its Z ratios; ztop [k][ch][N] 1 / Z of slot 15
// after k_kt_inv.  NULL: not wanted.
struct CombInner {
    uint32_t *jac = nullptr, *hs = nullptr, *ztop = nullptr;
};

// The comb part of the build after the doubling chain: warp = 1 as libsbv.so runs it (k_comb_fill_warp and k_comb_final,
// a warp per key, in lockstep; CombScr scratch), warp = 0 by the one-thread-per-chain reference (k_comb_fill and
// k_kt_final over the window tables' scratch layout).
template <class C>
static void comb_t(const uint32_t *cnt, uint32_t cap, bool warp, uint32_t *bases, uint32_t *ktab, uint8_t *kflags, const CombInner &in) {
    using CT = CombTab<C>;
    using KS = KtSizes<C, CT>;
    using S = CombScr<C>;
    constexpr int N = C::N;
    std::vector<uint32_t> hs(KS::hs_words(cap)), ztop(KS::ztop_words(cap)), pref(KS::ztop_words(cap));
    const unsigned kb = (cap + 63) / 64, cb = (unsigned)(((size_t)cap * CT::NCHAIN + 63) / 64), wb = (unsigned)(((size_t)cap * 32 + 63) / 64);
    run_grid(kb, 64, [&] { k_comb_affine<C>(cnt, cap, kflags, bases, pref.data()); });
    // word i of slot `slot` of chain ch of key k in each layout; jac: w = 0 .. 2N-1 over X then Y
    auto jac_at = [&](uint32_t k, int ch, int slot, int i) -> uint32_t {
        return warp ? hs[(S::jac(k, slot, i / 4) + ch) * 4 + (i & 3)] : ktab[((size_t)(k * CT::NCHAIN + ch) * CT::ENT + slot) * 2 * N + i];
    };
    auto hs_at = [&](uint32_t k, int ch, int slot, int i) -> uint32_t {
        return warp ? hs[(S::hs(k, slot, i / 4) + ch) * 4 + (i & 3)] : hs[(((size_t)ch * (CT::ENT - 1) + slot - 1) * N + i) * cap + k];
    };
    if (warp) run_grid_lockstep(wb, 64, [&] { k_comb_fill_warp<C, true>(cnt, cap, bases, kflags, hs.data(), ztop.data()); });
    else run_grid(cb, 64, [&] { k_comb_fill<C, true>(cnt, cap, bases, kflags, hs.data(), ztop.data(), ktab); });
    for (uint32_t k = 0; k < cap; k++)
        for (int ch = 0; ch < CT::NCHAIN; ch++)
            for (int slot = 0; slot < CT::ENT; slot++) {
                for (int i = 0; in.jac && i < 2 * N; i++) in.jac[((size_t)(k * CT::NCHAIN + ch) * CT::ENT + slot) * 2 * N + i] = jac_at(k, ch, slot, i);
                for (int i = 0; in.hs && slot && i < N; i++) in.hs[((size_t)(k * CT::NCHAIN + ch) * (CT::ENT - 1) + slot - 1) * N + i] = hs_at(k, ch, slot, i);
            }
    if (warp) run_grid(kb, 64, [&] { k_kt_inv<C, CT, S>(cnt, cap, kflags, ztop.data(), pref.data()); });
    else run_grid(kb, 64, [&] { k_kt_inv<C, CT>(cnt, cap, kflags, ztop.data(), pref.data()); });
    for (uint32_t k = 0; in.ztop && k < cap; k++)
        for (int ch = 0; ch < CT::NCHAIN; ch++)
            for (int i = 0; i < N; i++)
                in.ztop[((size_t)k * CT::NCHAIN + ch) * N + i] = ztop[warp ? S::at(k, ch, i, cap) : ZByChain<N>::at(k, ch, i, cap)];
    if (warp) run_grid_lockstep(wb, 64, [&] { k_comb_final<C, true>(cnt, cap, kflags, hs.data(), ztop.data(), ktab); });
    else run_grid(cb, 64, [&] { k_kt_final<C, CT, true>(cnt, cap, bases, kflags, hs.data(), ztop.data(), ktab); });
}

template <class C, class KT>
static void build_t(const uint32_t *cnt, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy, int four, uint32_t *ktab,
                    uint8_t *kflags) {
    using KS = KtSizes<C, KT>;
    std::vector<uint32_t> bases(KS::bases_words(cap));
    bases_t<C, KT>(cnt, cap, keylist, qx, qy, four, bases.data(), kflags);
    if constexpr (std::is_same<KT, CombTab<C>>::value) {
        comb_t<C>(cnt, cap, true, bases.data(), ktab, kflags, CombInner{});
    } else {
        std::vector<uint32_t> hs(KS::hs_words(cap)), ztop(KS::ztop_words(cap)), pref(KS::ztop_words(cap));
        const unsigned kb = (cap + 63) / 64, cb = (unsigned)(((size_t)cap * KT::NCHAIN + 63) / 64);
        run_grid(cb, 64, [&] { k_kt_fill<C, KT::STEP>(cnt, cap, bases.data(), kflags, hs.data(), ztop.data(), ktab); });
        run_grid(kb, 64, [&] { k_kt_inv<C, KT>(cnt, cap, kflags, ztop.data(), pref.data()); });
        run_grid(cb, 64, [&] { k_kt_final<C, KT>(cnt, cap, bases.data(), kflags, hs.data(), ztop.data(), ktab); });
    }
}

// P-256 comb tables of nkeys keys in a build of capacity cap >= nkeys (the surplus slots stay untouched: zeros), by the
// path `warp` selects (comb_t), with what the build leaves between its kernels (CombInner; each output may be NULL)
extern "C" int hs_comb_build(int warp, size_t nkeys, size_t cap, const uint8_t *qx, const uint8_t *qy, uint32_t *ktab_out, uint32_t *jac_out,
                             uint32_t *hs_out, uint32_t *ztop_out, uint8_t *flags_out) {
    using KS = KtSizes<P256, CombTab<P256>>;
    if (nkeys > cap) return -1;
    const uint32_t cnt = (uint32_t)nkeys, c = (uint32_t)cap;
    std::vector<uint32_t> bases(KS::bases_words(cap)), ktab(KS::ktab_words(cap), 0);
    std::vector<uint8_t> kflags(cap, 0);
    bases_t<P256, CombTab<P256>>(&cnt, c, nullptr, qx, qy, 2, bases.data(), kflags.data());
    comb_t<P256>(&cnt, c, warp != 0, bases.data(), ktab.data(), kflags.data(), CombInner{jac_out, hs_out, ztop_out});
    memcpy(ktab_out, ktab.data(), ktab.size() * 4);
    memcpy(flags_out, kflags.data(), cap);
    return 0;
}

template <class C, class KT>
static void tables_t(uint32_t nkeys, const uint8_t *qx, const uint8_t *qy, int four, uint32_t *ktab_out, uint8_t *flags_out) {
    std::vector<uint32_t> ktab(KtSizes<C, KT>::ktab_words(nkeys), 0);
    std::vector<uint8_t> kflags(nkeys, 0);
    build_t<C, KT>(&nkeys, nkeys, nullptr, qx, qy, four, ktab.data(), kflags.data());
    memcpy(ktab_out, ktab.data(), ktab.size() * 4);
    memcpy(flags_out, kflags.data(), nkeys);
}

// kind: 0 = 5-bit windows, 1 = 8-bit windows, 2 = comb (P-256 only, as in the product)
extern "C" size_t hs_ktab_words(int curve, int kind, size_t nkeys) {
    if (curve == 0) return kind == 2 ? KtSizes<P256, CombTab<P256>>::ktab_words(nkeys)
                         : kind ? KtSizes<P256, KeyTab<256, 8>>::ktab_words(nkeys) : KtSizes<P256, KeyTab<256, 5>>::ktab_words(nkeys);
    return kind == 2 ? 0 : kind ? KtSizes<P384, KeyTab<384, 8>>::ktab_words(nkeys) : KtSizes<P384, KeyTab<384, 5>>::ktab_words(nkeys);
}
extern "C" int hs_tables(int curve, int kind, size_t nkeys, const uint8_t *qx, const uint8_t *qy, int four, uint32_t *ktab_out, uint8_t *flags_out) {
    const uint32_t k = (uint32_t)nkeys;
    if (curve == 0 && kind == 2) tables_t<P256, CombTab<P256>>(k, qx, qy, four, ktab_out, flags_out);
    else if (curve == 0 && kind == 1) tables_t<P256, KeyTab<256, 8>>(k, qx, qy, four, ktab_out, flags_out);
    else if (curve == 0) tables_t<P256, KeyTab<256, 5>>(k, qx, qy, four, ktab_out, flags_out);
    else if (kind == 2) return -1;
    else if (kind == 1) tables_t<P384, KeyTab<384, 8>>(k, qx, qy, four, ktab_out, flags_out);
    else tables_t<P384, KeyTab<384, 5>>(k, qx, qy, four, ktab_out, flags_out);
    return 0;
}

// the Jacobian bases of P-256 comb tables for keys 0..nkeys-1, by the chain `four` selects (as in build_t), before
// k_comb_affine: KtSizes::bases_words(nkeys) words, layout [c][3N words][nkeys]
extern "C" int hs_comb_bases(size_t nkeys, const uint8_t *qx, const uint8_t *qy, int four, uint32_t *bases_out, uint8_t *flags_out) {
    const uint32_t k = (uint32_t)nkeys;
    memset(bases_out, 0, KtSizes<P256, CombTab<P256>>::bases_words(nkeys) * 4);
    bases_t<P256, CombTab<P256>>(&k, k, nullptr, qx, qy, four, bases_out, flags_out);
    return 0;
}

// kg_hash (the probe start of k_kg_insert) of items 0..n-1 of (qx, qy) under `seed`
extern "C" int hs_kg_hash(int curve, size_t n, const uint8_t *qx, const uint8_t *qy, uint32_t seed, uint32_t *out) {
    for (size_t i = 0; i < n; i++) out[i] = curve == 0 ? kg_hash<P256>(qx, qy, (uint32_t)i, seed) : kg_hash<P384>(qx, qy, (uint32_t)i, seed);
    return 0;
}

// k_sha256 over a ragged batch, one message per simulated thread (perm: optional processing order, as the counting sort gives it)
extern "C" int hs_sha256(size_t n, const uint8_t *msgs, const uint64_t *off, uint64_t base, const uint32_t *perm, uint8_t *digest_out) {
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_sha256((uint32_t)n, msgs, off, base, digest_out, perm); });
    return 0;
}
// k_sha384 over a ragged batch, as hs_sha256 (digest_out: 48 bytes per message)
extern "C" int hs_sha384(size_t n, const uint8_t *msgs, const uint64_t *off, uint64_t base, const uint32_t *perm, uint8_t *digest_out) {
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_sha384((uint32_t)n, msgs, off, base, digest_out, perm); });
    return 0;
}

// quorum counting (k_quorum_count + k_quorum_reached) for the instances [inst_base, inst_base + n_instances), as one device of a
// sharded engine runs it; ok may be NULL (prepares)
extern "C" int hs_quorum(size_t n_votes, const uint32_t *instance, const uint16_t *sender, const uint16_t *signer, const uint8_t *digest_match,
                         const uint8_t *ok, const uint16_t *self_id, uint32_t inst_base, size_t n_instances, uint32_t threshold, uint32_t *valid_count,
                         uint8_t *reached) {
    memset(valid_count, 0, n_instances * 4);
    run_grid((unsigned)((n_votes + 255) / 256), 256, [&] {
        k_quorum_count((uint32_t)n_votes, instance, sender, signer, digest_match, ok, self_id, inst_base, (uint32_t)n_instances, valid_count);
    });
    run_grid((unsigned)((n_instances + 255) / 256), 256, [&] { k_quorum_reached((uint32_t)n_instances, valid_count, threshold, reached); });
    return 0;
}
// k_pack_bits in lockstep (a warp ballot per 32 verdicts)
extern "C" int hs_pack_bits(size_t n, const uint8_t *ok, uint32_t *mask) {
    run_grid_lockstep((unsigned)((n + 255) / 256), 256, [&] { k_pack_bits((uint32_t)n, ok, mask); });
    return 0;
}

// the shards of a multi-device engine (shards.h, host code of libsbv itself): a plain batch of n items (votes == 0) or n
// commit votes grouped by instance.  ranges: [G][4] = item lo, item count, instance lo, instance count; words = wv, wi.
static Shards make_shards(int votes, size_t n, const uint32_t *instance, size_t n_instances, int G) {
    return votes ? quorum_shards(n, instance, n_instances, G) : batch_shards(n, G);
}
extern "C" int hs_shards(int votes, size_t n, const uint32_t *instance, size_t n_instances, int G, size_t *ranges, size_t *words) {
    const Shards s = make_shards(votes, n, instance, n_instances, G);
    for (int g = 0; g < G; g++) {
        const Range ir = s.ir.empty() ? Range{0, 0} : s.ir[g];
        const size_t r[4] = {s.vr[g].lo, s.vr[g].n, ir.lo, ir.n};
        memcpy(ranges + 4 * g, r, sizeof r);
    }
    words[0] = s.wv;
    words[1] = s.wi;
    return 0;
}
// the host unpack of the gathered words (G * (wv + wi) words) into verdict and reached bytes
extern "C" int hs_unpack_shards(int votes, size_t n, const uint32_t *instance, size_t n_instances, int G, const uint32_t *gathered, uint8_t *ok,
                                uint8_t *reached) {
    unpack_shards(make_shards(votes, n, instance, n_instances, G), gathered, ok, reached);
    return 0;
}

// registered-key path (sbv_set_keys / sbv_verify_registered): 8-bit window tables for `nkeys` keys, then k_prep and the
// fixed-base kernel with the key taken by slot — thread per signature, or (warp != 0) ONE SIGNATURE PER WARP in lockstep
// (k_verify_kt_warp: lanes add their table points, shuffle-tree reduction)
template <class C>
static void registered_t(uint32_t n, uint32_t nkeys, const uint8_t *kx, const uint8_t *ky, const uint32_t *slot, const uint8_t *r, const uint8_t *s,
                         const uint8_t *dig, uint32_t dlen, const uint4 *gtab, int warp, uint8_t *ok) {
    constexpr int N = C::N, S = 8, W = 8;
    using KT = KeyTab<32 * N, W>;
    std::vector<uint32_t> ktab(KtSizes<C, KT>::ktab_words(nkeys));
    std::vector<uint8_t> kflags(nkeys);
    tables_t<C, KT>(nkeys, kx, ky, 0, ktab.data(), kflags.data());
    // one entry past the slots, mapped to key 0: a slot check that admits slot == n_slots reads a valid key there and
    // accepts, where the device would read past the end of the map
    std::vector<int32_t> s2l(nkeys + 1, 0);
    for (uint32_t i = 0; i < nkeys; i++) s2l[i] = (int32_t)i;
    std::vector<uint32_t> uw((size_t)2 * N * n);
    std::vector<uint8_t> flags(n);
    run_grid(((n + S - 1) / S + 127) / 128, 128, [&] { k_prep<C, S>(n, r, s, dig, dlen, uw.data(), flags.data()); });
    const uint4 *k4 = reinterpret_cast<const uint4 *>(ktab.data());
    if (warp)
        run_grid_lockstep((unsigned)(((size_t)n * 32 + 127) / 128), 128,
                          [&] { k_verify_kt_warp<C, W>(n, slot, s2l.data(), nkeys, kflags.data(), r, uw.data(), flags.data(), gtab, k4, ok); });
    else
        run_grid((n + 63) / 64, 64, [&] {
            k_verify_kt<C, W, 64, 1, true, false>(n, slot, s2l.data(), nkeys, kflags.data(), r, uw.data(), flags.data(), gtab, k4, ok, nullptr, nullptr, nullptr);
        });
}

template <class C> static const uint4 *gtab_for(int idx);
extern "C" int hs_verify_registered(int curve, size_t n, size_t nkeys, const uint8_t *kx, const uint8_t *ky, const uint32_t *slot, const uint8_t *r,
                                    const uint8_t *s, const uint8_t *dig, uint32_t dlen, int warp, uint8_t *ok) {
    if (curve == 0) registered_t<P256>((uint32_t)n, (uint32_t)nkeys, kx, ky, slot, r, s, dig, dlen, gtab_for<P256>(0), warp, ok);
    else registered_t<P384>((uint32_t)n, (uint32_t)nkeys, kx, ky, slot, r, s, dig, dlen, gtab_for<P384>(1), warp, ok);
    return 0;
}

// keys-per-item path: k_prep + k_verify_coz, exactly the kernels of the product, thread by thread
template <class C, int BLOCK>
static void verify_coz_t(uint32_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy, const uint8_t *dig,
                         uint32_t dlen, const uint4 *gtab, uint8_t *ok) {
    constexpr int N = C::N, S = 8;
    std::vector<uint32_t> uw((size_t)2 * N * n);
    std::vector<uint8_t> flags(n);
    std::vector<uint32_t> tscr((size_t)12 * N * n);
    const unsigned pthreads = (n + S - 1) / S;
    run_grid((pthreads + 127) / 128, 128, [&] { k_prep<C, S>(n, r, s, dig, dlen, uw.data(), flags.data()); });
    run_grid((n + BLOCK - 1) / BLOCK, BLOCK, [&] {
        k_verify_coz<C, BLOCK, 1>(n, qx, qy, r, uw.data(), flags.data(), gtab, tscr.data(), ok, nullptr, nullptr);
    });
}

// grouped path: k_prep, key grouping, table construction and the fixed-base kernel for repeated keys (P-256: comb tables and
// k_verify_comb; P-384: 5-bit window tables and k_verify_kt, as in the product), k_verify_coz for the rest.  The second half
// runs chunk by chunk (chunk = items per chunk; 0: the whole batch as one chunk), as sbv_launch_verify_chunk
// (csrc/pipeline.cu) enqueues it: the items [lo, lo + cn) are a batch of their own for every per-item array (word-major,
// stride = the chunk's size, base = words per item * lo); the grouping (rep, keyid) and the key tables are shared; routing
// is per chunk, chunk-local indices, the chunk's own counters.
template <class C>
static void verify_grouped_t(uint32_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy, const uint8_t *dig,
                             uint32_t dlen, const uint4 *gtab, uint32_t threshold, uint32_t max_keys, uint8_t *ok, uint32_t *stats,
                             uint32_t chunk = 0) {
    constexpr int N = C::N, S = 8;
    std::vector<uint32_t> uw((size_t)2 * N * n);
    std::vector<uint8_t> flags(n);
    std::vector<uint32_t> tscr((size_t)12 * N * n);
    uint32_t hsize = 1;
    while (hsize < 2 * n) hsize <<= 1;
    std::vector<uint32_t> htab(hsize, KG_EMPTY), rep(n), kcnt(n, 0), keylist(max_keys ? max_keys : 1), klist(n), glist(n), counters(4, 0);
    std::vector<int32_t> keyid(n), item_kid(n);
    run_grid((n + 255) / 256, 256, [&] { k_kg_insert(n, KgXY<C>{qx, qy}, 0x1234567u, hsize - 1, htab.data(), rep.data(), kcnt.data()); });
    run_grid((n + 255) / 256, 256, [&] { k_kg_assign(n, rep.data(), kcnt.data(), threshold, max_keys, keyid.data(), keylist.data(), counters.data()); });
    const size_t cap = max_keys ? max_keys : 1;
    constexpr bool comb = std::is_same<C, P256>::value;
    using KT = typename std::conditional<comb, CombTab<C>, KeyTab<32 * N, 5>>::type;
    std::vector<uint32_t> ktab(KtSizes<C, KT>::ktab_words(cap));
    std::vector<uint8_t> kflags(cap, 0);
    build_t<C, KT>(counters.data(), (uint32_t)cap, keylist.data(), qx, qy, 0, ktab.data(), kflags.data());
    const uint4 *k4 = reinterpret_cast<const uint4 *>(ktab.data());
    std::vector<uint32_t> gacc((size_t)3 * N * n);
    const size_t L = C::BYTES;
    const uint32_t per = chunk ? chunk : n;
    uint32_t kt_total = 0, gen_total = 0;
    for (uint32_t lo = 0; lo < n; lo += per) {
        const uint32_t cn = n - lo < per ? n - lo : per;
        std::vector<uint32_t> cc(4, 0);
        uint32_t *uwc = uw.data() + (size_t)2 * N * lo, *tsc = tscr.data() + (size_t)12 * N * lo, *gac = gacc.data() + (size_t)3 * N * lo;
        uint8_t *flc = flags.data() + lo;
        const uint8_t *rc = r + lo * L;
        const int32_t *kid = item_kid.data() + lo;
        const uint32_t *kl = klist.data() + lo;
        run_grid(((cn + S - 1) / S + 127) / 128, 128, [&] { k_prep<C, S>(cn, rc, s + lo * L, dig + (size_t)lo * dlen, dlen, uwc, flc); });
        run_grid((cn + 255) / 256, 256, [&] { k_kg_route(cn, rep.data() + lo, keyid.data(), item_kid.data() + lo, klist.data() + lo, glist.data() + lo, cc.data()); });
        run_grid((cn + 63) / 64, 64, [&] { k_verify_coz<C, 64, 1>(cn, qx + lo * L, qy + lo * L, rc, uwc, flc, gtab, tsc, ok + lo, glist.data() + lo, cc.data() + 2); });
        run_grid((cn + 63) / 64, 64, [&] { k_gpart<C, 64, 1>(cn, uwc, gtab, gac); });
        run_grid((cn + 63) / 64, 64, [&] {
            if constexpr (comb) k_verify_comb<C, 64, 1, false>(cn, kid, kflags.data(), rc, uwc, flc, k4, ok + lo, kl, cc.data() + 1, gac);
            else k_verify_kt<C, 5, 64, 1, false, false>(cn, nullptr, kid, 0, kflags.data(), rc, uwc, flc, gtab, k4, ok + lo, kl, cc.data() + 1, gac);
        });
        kt_total += cc[1]; gen_total += cc[2];
    }
    if (stats) { stats[0] = counters[0]; stats[1] = kt_total; stats[2] = gen_total; }
}

static std::vector<uint32_t> g_gtab[2];
template <class C>
static const uint4 *gtab_for(int idx) {
    auto &g = g_gtab[idx];
    if (g.empty()) {
        const size_t entries = (size_t)C::GWINS << C::GW;
        g.resize(entries * 2 * C::N);
        // incremental construction (the device kernel builds every entry independently, far too slow for a CPU)
        build_comb_host<C>(g.data());
    }
    return reinterpret_cast<const uint4 *>(g.data());
}

// the same with the second half run chunk by chunk (chunk = items per chunk), as a chunked host-buffer call does
extern "C" int hs_verify_chunked(int curve, size_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy, const uint8_t *dig,
                      uint32_t dlen, uint32_t threshold, uint32_t max_keys, uint32_t chunk, uint8_t *ok, uint32_t *stats) {
    if (curve == 0) verify_grouped_t<P256>((uint32_t)n, r, s, qx, qy, dig, dlen, gtab_for<P256>(0), threshold, max_keys, ok, stats, chunk);
    else verify_grouped_t<P384>((uint32_t)n, r, s, qx, qy, dig, dlen, gtab_for<P384>(1), threshold, max_keys, ok, stats, chunk);
    return 0;
}

extern "C" int hs_verify(int curve, size_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy, const uint8_t *dig, uint32_t dlen,
              uint8_t *ok) {
    if (curve == 0) verify_coz_t<P256, 64>((uint32_t)n, r, s, qx, qy, dig, dlen, gtab_for<P256>(0), ok);
    else verify_coz_t<P384, 64>((uint32_t)n, r, s, qx, qy, dig, dlen, gtab_for<P384>(1), ok);
    return 0;
}

// grouped (fixed-base for repeated keys) path; stats = {keys found, items on the fixed-base path, items on the generic path}
extern "C" int hs_verify_grouped(int curve, size_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy, const uint8_t *dig,
                      uint32_t dlen, uint32_t threshold, uint32_t max_keys, uint8_t *ok, uint32_t *stats) {
    if (curve == 0) verify_grouped_t<P256>((uint32_t)n, r, s, qx, qy, dig, dlen, gtab_for<P256>(0), threshold, max_keys, ok, stats);
    else verify_grouped_t<P384>((uint32_t)n, r, s, qx, qy, dig, dlen, gtab_for<P384>(1), threshold, max_keys, ok, stats);
    return 0;
}


// ---- Ed25519 (ed25519.cuh, sha512.cuh, ed25519_verify.cuh) ----
// field / decode / mod-L operations of ed25519_debug.cuh, 24-word slots
extern "C" int hs_ed25519_op(int op, size_t n, const uint32_t *in, uint32_t *out) {
    for (size_t i = 0; i < n; i++) ed_debug_dispatch(op, (uint32_t)i, in, out);
    return 0;
}
// point operations of ed25519_debug.cuh, ED_POINT_WORDS-word slots; -1 for an op the dispatch does not run, as
// sbv_debug_ed25519_point refuses it
extern "C" int hs_ed25519_point(int op, size_t n, const uint32_t *in, uint32_t *out) {
    if (!ed_point_op_ok(op)) return -1;
    for (size_t i = 0; i < n; i++) ed_point_dispatch(op, (uint32_t)i, in, out);
    return 0;
}
// k_ed_sha512 over a ragged batch (perm: optional processing order): k word-major [8][n], and the 16 digest limbs per item
extern "C" int hs_ed25519_sha512(size_t n, const uint8_t *msgs, const uint64_t *off, uint64_t base, const uint8_t *sig, const uint8_t *pub,
                                 const uint32_t *perm, uint32_t *k_out, uint32_t *dig_out) {
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_ed_sha512((uint32_t)n, sig, pub, msgs, off, base, k_out, perm, dig_out); });
    return 0;
}
static std::vector<uint32_t> &ed_btab_host() {
    static std::vector<uint32_t> t;
    if (t.empty()) {
        t.resize(ED_BTAB_WORDS);
        run_grid((ED_BWINS * ED_BENT + 63) / 64, 64, [&] { k_ed_btab_init(t.data()); });
    }
    return t;
}
// the fixed-base table of B as k_ed_btab_init builds it
extern "C" int hs_ed25519_btab(uint32_t *out) {
    memcpy(out, ed_btab_host().data(), ED_BTAB_WORDS * 4);
    return 0;
}
// the whole pipeline of sbv_ed25519_verify_batch on one device: k_ed_sha512, then k_ed_verify with blocks of 32 threads
extern "C" int hs_ed25519_verify(size_t n, const uint8_t *msgs, const uint64_t *off, const uint8_t *sig, const uint8_t *pub, uint8_t *ok) {
    std::vector<uint32_t> k(8 * n + 8);
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_ed_sha512((uint32_t)n, sig, pub, msgs, off, 0, k.data(), nullptr, nullptr); });
    const uint4 *bt = reinterpret_cast<const uint4 *>(ed_btab_host().data());
    run_grid((unsigned)((n + 31) / 32), 32, [&] { k_ed_verify<32>((uint32_t)n, sig, pub, k.data(), bt, ok, nullptr, nullptr); });
    return 0;
}
// k_ed_verify alone with the caller's k (8 little-endian limbs per item, each < L; -1 otherwise), as
// sbv_debug_ed25519_verify_k runs it on the device
extern "C" int hs_ed25519_verify_k(size_t n, const uint8_t *sig, const uint8_t *pub, const uint32_t *k_in, uint8_t *ok) {
    uint32_t Lm[8];
    ed_order(Lm);
    std::vector<uint32_t> k(8 * n + 8);
    for (size_t i = 0; i < n; i++) {
        uint32_t ki[8];
        for (int w = 0; w < 8; w++) k[(size_t)w * n + i] = ki[w] = k_in[i * 8 + w];
        if (!mp_lt<8>(ki, Lm)) return -1;
    }
    const uint4 *bt = reinterpret_cast<const uint4 *>(ed_btab_host().data());
    run_grid((unsigned)((n + 31) / 32), 32, [&] { k_ed_verify<32>((uint32_t)n, sig, pub, k.data(), bt, ok, nullptr, nullptr); });
    return 0;
}

// ---- registered Ed25519 keys (ed25519_keyed.cuh) ----
// The registry of sbv_ed25519_set_keys, built by the same kernels: the registered bytes of every slot, slot -> table
// (-1: the key does not decode) and one table per decodable key.
static struct {
    std::vector<uint4> pub;  // 2 per slot (16-byte aligned, as cudaMalloc gives it)
    std::vector<int32_t> slot2local;
    std::vector<uint32_t> ktab;
    uint32_t n = 0;
} g_edk;

// chunk: keys per k_ed_ktab_build launch, as ed_keys_fill (inst_ed25519.cu) splits them; 0 = ED_KBUILD_MAX
extern "C" int hs_ed25519_set_keys(size_t n, const uint8_t *pub, uint32_t chunk) {
    g_edk.pub.assign(2 * n + 2, uint4{0, 0, 0, 0});
    if (n) memcpy(g_edk.pub.data(), pub, n * 32);
    const uint8_t *kp = reinterpret_cast<const uint8_t *>(g_edk.pub.data());
    std::vector<uint32_t> xy(16 * n + 16);
    std::vector<uint8_t> flag(n + 1);
    run_grid((unsigned)((n + 63) / 64), 64, [&] { k_ed_kdecode((uint32_t)n, kp, xy.data(), flag.data()); });
    g_edk.slot2local.assign(n + 1, -1);
    std::vector<uint32_t> slot_of;
    for (size_t i = 0; i < n; i++)
        if (flag[i]) { g_edk.slot2local[i] = (int32_t)slot_of.size(); slot_of.push_back((uint32_t)i); }
    // the entry past the last slot maps to slot 0's table: a slot check that admits slot == n then reads a valid table and
    // accepts slot 0's rows, where the device would read past the end of the map
    if (n) g_edk.slot2local[n] = g_edk.slot2local[0];
    const uint32_t cnt = (uint32_t)slot_of.size();
    g_edk.ktab.assign((size_t)cnt * ED_KTAB_WORDS + 4, 0);
    const uint32_t per = std::min(cnt, chunk ? chunk : ED_KBUILD_MAX);
    std::vector<uint32_t> pref((size_t)per * ED_BWINS * ED_BENT * 8 + 1);
    for (uint32_t c0 = 0; c0 < cnt; c0 += per) {
        const uint32_t cc = std::min(per, cnt - c0);
        run_grid((cc * ED_BWINS + 63) / 64, 64,
                 [&] { k_ed_ktab_build(cc, slot_of.data() + c0, xy.data(), g_edk.ktab.data() + (size_t)c0 * ED_KTAB_WORDS, pref.data()); });
    }
    g_edk.n = (uint32_t)n;
    return 0;
}
// the whole table (32 x 128 entries of 24 words) of a registered slot; -1 for an unknown slot or a key that does not decode
extern "C" int hs_ed25519_ktab(uint32_t slot, uint32_t *out) {
    if (slot >= g_edk.n || g_edk.slot2local[slot] < 0) return -1;
    memcpy(out, g_edk.ktab.data() + (size_t)g_edk.slot2local[slot] * ED_KTAB_WORDS, ED_KTAB_WORDS * 4);
    return 0;
}
static void ed_verify_keyed_host(size_t n, const uint32_t *key_slot, const uint8_t *sig, const uint32_t *k, uint8_t *ok) {
    const uint4 *bt = reinterpret_cast<const uint4 *>(ed_btab_host().data());
    const uint4 *kt = reinterpret_cast<const uint4 *>(g_edk.ktab.data());
    run_grid((unsigned)((n + 127) / 128), 128,
             [&] { k_ed_verify_keyed<128>((uint32_t)n, sig, key_slot, g_edk.n, g_edk.slot2local.data(), kt, k, bt, ok); });
}
// the pipeline of sbv_ed25519_verify_registered on one device: k_ed_key_gather, k_ed_sha512, k_ed_verify_keyed
extern "C" int hs_ed25519_verify_registered(size_t n, const uint8_t *msgs, const uint64_t *off, const uint32_t *key_slot, const uint8_t *sig,
                                            uint8_t *ok) {
    std::vector<uint4> pub(2 * n + 2);
    run_grid((unsigned)((2 * n + 255) / 256), 256,
             [&] { k_ed_key_gather((uint32_t)n, key_slot, g_edk.n, g_edk.pub.data(), pub.data()); });
    std::vector<uint32_t> k(8 * n + 8);
    const uint8_t *pb = reinterpret_cast<const uint8_t *>(pub.data());
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_ed_sha512((uint32_t)n, sig, pb, msgs, off, 0, k.data(), nullptr, nullptr); });
    ed_verify_keyed_host(n, key_slot, sig, k.data(), ok);
    return 0;
}
// k_ed_verify_keyed alone with the caller's k (8 little-endian limbs per item, each < L; -1 otherwise), as
// sbv_debug_ed25519_verify_registered_k runs it on the device
extern "C" int hs_ed25519_verify_registered_k(size_t n, const uint32_t *key_slot, const uint8_t *sig, const uint32_t *k_in, uint8_t *ok) {
    uint32_t Lm[8];
    ed_order(Lm);
    std::vector<uint32_t> k(8 * n + 8);
    for (size_t i = 0; i < n; i++) {
        uint32_t ki[8];
        for (int w = 0; w < 8; w++) k[(size_t)w * n + i] = ki[w] = k_in[i * 8 + w];
        if (!mp_lt<8>(ki, Lm)) return -1;
    }
    ed_verify_keyed_host(n, key_slot, sig, k.data(), ok);
    return 0;
}

// ---- Ed25519 keys grouped inside a keys-per-item launch (ed25519_comb.cuh) ----
// The first half of a grouped launch as sbv_launch_verify_begin (pipeline.cu) enqueues it for Ed25519: k_kg_insert over
// the 32 key bytes, k_kg_assign (threshold T, kcap table slots), the four comb construction kernels; then k_kg_route.
struct EdGroup {
    std::vector<uint32_t> rep, keylist, klist, glist, counters, ctab;
    std::vector<int32_t> keyid, item_kid;
    std::vector<uint8_t> kflags;
};
static void ed_group_host(uint32_t n, const uint8_t *pub, uint32_t T, uint32_t kcap, EdGroup &g) {
    uint32_t hsize = 1;
    while (hsize < 2 * n) hsize <<= 1;
    const uint32_t cap = kcap ? kcap : 1;
    std::vector<uint32_t> htab(hsize, KG_EMPTY), kcnt(n, 0);
    std::vector<uint32_t> bases(EDC_BASES_WORDS * cap), hs(EDC_HS_WORDS * cap), ztop(EDC_ZTOP_WORDS * cap), pref(EDC_ZTOP_WORDS * cap);
    g.rep.assign(n, 0); g.klist.assign(n, 0); g.glist.assign(n, 0); g.counters.assign(4, 0);
    g.keyid.assign(n, -1); g.item_kid.assign(n, -1);
    g.keylist.assign(cap, 0); g.kflags.assign(cap, 0); g.ctab.assign((size_t)cap * EDC_TAB_WORDS, 0);
    uint32_t *cnt = g.counters.data();
    run_grid((n + 255) / 256, 256, [&] { k_kg_insert(n, KgKey32{pub}, 0x1234567u, hsize - 1, htab.data(), g.rep.data(), kcnt.data()); });
    run_grid((n + 255) / 256, 256, [&] { k_kg_assign(n, g.rep.data(), kcnt.data(), T, kcap, g.keyid.data(), g.keylist.data(), cnt); });
    const unsigned kb = (cap + 63) / 64, cb = (cap * EDC_NCHAIN + 63) / 64;
    run_grid(kb, 64, [&] { k_edc_bases(cnt, cap, g.keylist.data(), pub, bases.data(), g.kflags.data()); });
    run_grid(cb, 64, [&] { k_edc_fill(cnt, cap, bases.data(), g.kflags.data(), hs.data(), ztop.data(), g.ctab.data()); });
    run_grid(kb, 64, [&] { k_edc_inv(cnt, cap, g.kflags.data(), ztop.data(), pref.data()); });
    run_grid(cb, 64, [&] { k_edc_final(cnt, cap, g.kflags.data(), hs.data(), ztop.data(), g.ctab.data()); });
    run_grid((n + 255) / 256, 256, [&] { k_kg_route(n, g.rep.data(), g.keyid.data(), g.item_kid.data(), g.klist.data(), g.glist.data(), cnt); });
}
// table slots of a launch of n items, as group_slots (pipeline.cu) counts them with no minimum batch; 0: no grouping
static uint32_t ed_group_cap_host(uint32_t n, uint32_t T, uint32_t max_keys) {
    if (T == 0 || n < T || max_keys == 0) return 0;
    const uint32_t k = std::min(n / T, max_keys);
    return k ? k : 1;
}
// The comb tables of a launch of the n keys of pub at threshold T with at most max_keys tables, as
// sbv_debug_ed25519_comb_tab reports them: per query item, status 0 and the table (510 x 24 words) at out + q * 12240;
// 1: no table; 2: a table slot, but the key does not decode.
extern "C" int hs_ed25519_comb_tab(size_t n, const uint8_t *pub, uint32_t T, uint32_t max_keys, size_t m, const uint32_t *items, int32_t *status,
                                   uint32_t *out) {
    const uint32_t kcap = ed_group_cap_host((uint32_t)n, T, max_keys);
    EdGroup g;
    if (kcap) ed_group_host((uint32_t)n, pub, T, kcap, g);
    for (size_t q = 0; q < m; q++) {
        if (items[q] >= n) return -1;
        const int32_t kid = kcap ? g.keyid[g.rep[items[q]]] : -1;
        status[q] = kid < 0 ? 1 : g.kflags[kid] ? 0 : 2;
        if (status[q] == 0) memcpy(out + q * EDC_TAB_WORDS, g.ctab.data() + (size_t)kid * EDC_TAB_WORDS, EDC_TAB_WORDS * 4);
    }
    return 0;
}
// k_ed_verify_comb with the caller's k (8 little-endian limbs per item, each < L; -1 otherwise), every distinct key with a
// table, as sbv_debug_ed25519_verify_comb_k runs it on the device
extern "C" int hs_ed25519_verify_comb_k(size_t n, const uint8_t *sig, const uint8_t *pub, const uint32_t *k_in, uint8_t *ok) {
    uint32_t Lm[8];
    ed_order(Lm);
    std::vector<uint32_t> k(8 * n + 8);
    for (size_t i = 0; i < n; i++) {
        uint32_t ki[8];
        for (int w = 0; w < 8; w++) k[(size_t)w * n + i] = ki[w] = k_in[i * 8 + w];
        if (!mp_lt<8>(ki, Lm)) return -1;
    }
    if (n == 0) return 0;
    EdGroup g;
    ed_group_host((uint32_t)n, pub, 1, (uint32_t)n, g);
    const uint4 *bt = reinterpret_cast<const uint4 *>(ed_btab_host().data()), *ct = reinterpret_cast<const uint4 *>(g.ctab.data());
    run_grid((unsigned)((n + 127) / 128), 128,
             [&] { k_ed_verify_comb<128>((uint32_t)n, sig, g.item_kid.data(), g.kflags.data(), ct, k.data(), bt, ok, nullptr, nullptr); });
    return 0;
}
// the pipeline of sbv_ed25519_verify_batch on one device with grouping: the first half (ed_group_host), k_ed_sha512,
// k_ed_verify over the generic list and k_ed_verify_comb over the grouped one; T = 0 or fewer than T items: no grouping.
// stats = {keys found, items on the comb path, items on the generic path}
extern "C" int hs_ed25519_verify_grouped(size_t n, const uint8_t *msgs, const uint64_t *off, const uint8_t *sig, const uint8_t *pub, uint32_t T,
                                         uint32_t max_keys, uint8_t *ok, uint32_t *stats) {
    const uint32_t nn = (uint32_t)n, kcap = ed_group_cap_host(nn, T, max_keys);
    if (!kcap) {
        if (stats) { stats[0] = 0; stats[1] = 0; stats[2] = nn; }
        return hs_ed25519_verify(n, msgs, off, sig, pub, ok);
    }
    EdGroup g;
    ed_group_host(nn, pub, T, kcap, g);
    std::vector<uint32_t> k(8 * n + 8);
    run_grid((nn + 127) / 128, 128, [&] { k_ed_sha512(nn, sig, pub, msgs, off, 0, k.data(), nullptr, nullptr); });
    const uint4 *bt = reinterpret_cast<const uint4 *>(ed_btab_host().data()), *ct = reinterpret_cast<const uint4 *>(g.ctab.data());
    const uint32_t *cnt = g.counters.data();
    run_grid((nn + 31) / 32, 32, [&] { k_ed_verify<32>(nn, sig, pub, k.data(), bt, ok, g.glist.data(), cnt + 2); });
    run_grid((nn + 127) / 128, 128,
             [&] { k_ed_verify_comb<128>(nn, sig, g.item_kid.data(), g.kflags.data(), ct, k.data(), bt, ok, g.klist.data(), cnt + 1); });
    if (stats) { stats[0] = cnt[0]; stats[1] = cnt[1]; stats[2] = cnt[2]; }
    return 0;
}

// ---- mixed ECDSA / Ed25519 shards (mixed.cuh) ----
// The caller's arrays as the plan of a shard with m = {m0, m1, n - m0 - m1} items per family: idx, slot and ok hold the
// three families one after the other (n entries each), off their m_f + 1 offsets one after the other (n + 3 entries);
// r0 / s0 (32 B per item), r1 / s1 (48 B) and sig2 (64-byte rows) are per family; blob is the shared message buffer.
static MixPlan hs_plan(size_t n, uint32_t m0, uint32_t m1, uint32_t *idx, uint32_t *slot, uint8_t *r0, uint8_t *s0, uint8_t *r1, uint8_t *s1,
                       uint8_t *sig2, uint64_t *off, uint8_t *blob, uint8_t *ok) {
    const uint32_t at[3] = {0, m0, m0 + m1};
    MixPlan p;
    for (int f = 0; f < MIX_FAMILIES; f++)
        p.f[f] = MixFamily{idx ? idx + at[f] : nullptr, slot ? slot + at[f] : nullptr, f == 0 ? r0 : f == 1 ? r1 : sig2, f == 0 ? s0 : f == 1 ? s1 : nullptr,
                           off ? off + at[f] + f : nullptr, ok ? ok + at[f] : nullptr};
    p.blob = blob;
    (void)n;
    return p;
}
// k_mix_count, k_mix_scan (as one thread: the simulation has no block barrier) and k_mix_split over a shard whose offsets
// are off_in[0..n]
extern "C" int hs_mixed_split(size_t n, const uint8_t *tag, const uint32_t *slot_in, const uint8_t *sig96, const uint64_t *off_in, uint32_t m0, uint32_t m1,
                              uint32_t *idx, uint32_t *slot, uint8_t *r0, uint8_t *s0, uint8_t *r1, uint8_t *s1, uint8_t *sig2, uint64_t *off_out) {
    const MixPlan p = hs_plan(n, m0, m1, idx, slot, r0, s0, r1, s1, sig2, off_out, nullptr, nullptr);
    const uint32_t nn = (uint32_t)n, ntiles = (uint32_t)((n + MIX_TILE - 1) / MIX_TILE);
    std::vector<uint32_t> tc((size_t)MIX_FAMILIES * ntiles + 1);
    std::vector<uint64_t> tb((size_t)MIX_FAMILIES * ntiles + 1);
    run_grid((ntiles + 255) / 256, 256, [&] { k_mix_count(nn, tag, off_in, ntiles, tc.data(), tb.data()); });
    run_grid(1, 1, [&] { k_mix_scan(ntiles, tc.data(), tb.data(), p); });
    run_grid((ntiles + 255) / 256, 256, [&] { k_mix_split(nn, tag, slot_in, sig96, off_in, ntiles, tc.data(), tb.data(), p); });
    return 0;
}
// k_mix_compact: the messages of src (offsets off_in from base; src readable 8 bytes past the last one) into blob at the
// split's offsets
extern "C" int hs_mixed_compact(size_t n, uint32_t m0, uint32_t m1, const uint8_t *src, const uint64_t *off_in, uint64_t base, const uint32_t *idx,
                                const uint64_t *off_out, uint8_t *blob) {
    const MixPlan p = hs_plan(n, m0, m1, const_cast<uint32_t *>(idx), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                              const_cast<uint64_t *>(off_out), blob, nullptr);
    run_grid((unsigned)((n * MIX_LANES + 255) / 256), 256, [&] { k_mix_compact((uint32_t)n, m0, m1, src, off_in, base, p); });
    return 0;
}
// k_mix_ok: the family verdicts ok_fam (compacted order) back to item order
extern "C" int hs_mixed_scatter(size_t n, uint32_t m0, uint32_t m1, const uint32_t *idx, const uint8_t *ok_fam, uint8_t *ok) {
    const MixPlan p = hs_plan(n, m0, m1, const_cast<uint32_t *>(idx), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                              const_cast<uint8_t *>(ok_fam));
    run_grid((unsigned)((n + 255) / 256), 256, [&] { k_mix_ok((uint32_t)n, m0, m1, p, ok); });
    return 0;
}
// The pipeline of sbv_mixed_verify_registered on one device: split, compaction, then per ECDSA family hs_sha256 and
// hs_verify_registered against the keys of that curve in the ECDSA registry (nkeys keys: curve tags, X || Y in 48-byte
// slots as sbv_set_keys takes them; a slot >= nkeys or of the other curve rejects), hs_ed25519_verify_registered against
// the registry of hs_ed25519_set_keys for the Ed25519 family, and the scatter.  Tags must be <= 2.
extern "C" int hs_mixed_verify_registered(size_t n, const uint8_t *tag, const uint8_t *msgs, const uint64_t *off, const uint32_t *slot_in,
                                          const uint8_t *sig96, size_t nkeys, const uint8_t *key_curve, const uint8_t *key_xy, uint8_t *ok) {
    uint32_t m[3] = {0, 0, 0};
    for (size_t i = 0; i < n; i++) {
        if (tag[i] > 2) return -1;
        m[tag[i]]++;
    }
    const uint64_t base = off[0], bytes = off[n] - base;
    std::vector<uint8_t> src(bytes + 16, 0);
    if (bytes) memcpy(src.data(), msgs + base, bytes);
    std::vector<uint32_t> idx(n + 1), slot(n + 1);
    std::vector<uint8_t> r0(32 * m[0] + 1), s0(32 * m[0] + 1), r1(48 * m[1] + 1), s1(48 * m[1] + 1), sig2(64 * m[2] + 1), blob(bytes + 128, 0), okf(n + 1, 0);
    std::vector<uint64_t> fo(n + 3);
    hs_mixed_split(n, tag, slot_in, sig96, off, m[0], m[1], idx.data(), slot.data(), r0.data(), s0.data(), r1.data(), s1.data(), sig2.data(), fo.data());
    hs_mixed_compact(n, m[0], m[1], src.data(), off, base, idx.data(), fo.data(), blob.data());
    const uint32_t at[3] = {0, m[0], m[0] + m[1]};
    for (int f = 0; f < 2; f++) {
        if (!m[f]) continue;
        const size_t L = f ? 48 : 32;
        std::vector<uint8_t> dig(32 * m[f]), kx, ky;
        hs_sha256(m[f], blob.data(), fo.data() + at[f] + f, 0, nullptr, dig.data());
        std::vector<int64_t> local(nkeys, -1);
        uint32_t nloc = 0;
        for (size_t k = 0; k < nkeys; k++)
            if (key_curve[k] == f) {
                local[k] = nloc++;
                kx.insert(kx.end(), key_xy + 96 * k + 48 - L, key_xy + 96 * k + 48);
                ky.insert(ky.end(), key_xy + 96 * k + 96 - L, key_xy + 96 * k + 96);
            }
        if (!nloc) continue;  // no key of this curve: every item rejects (okf is zero)
        std::vector<uint32_t> ls(m[f]);
        for (uint32_t j = 0; j < m[f]; j++) {
            const uint32_t s = slot[at[f] + j];
            ls[j] = s < nkeys && local[s] >= 0 ? (uint32_t)local[s] : nloc;
        }
        hs_verify_registered(f, m[f], nloc, kx.data(), ky.data(), ls.data(), f ? r1.data() : r0.data(), f ? s1.data() : s0.data(), dig.data(), 32, 0,
                             okf.data() + at[f]);
    }
    if (m[2]) hs_ed25519_verify_registered(m[2], blob.data(), fo.data() + at[2] + 2, slot.data() + at[2], sig2.data(), okf.data() + at[2]);
    hs_mixed_scatter(n, m[0], m[1], idx.data(), okf.data(), ok);
    return 0;
}

// ---- SHA-384 items in mixed shards (mixed_hash.cuh, sbv_mixed384_*) ----
// k_mix_alg over n tags in place: tags 3 and 4 become 0 and 1, sha384[i] = whether item i is over SHA-384
extern "C" int hs_mix_alg(size_t n, uint8_t *tag, uint8_t *sha384) {
    run_grid((unsigned)((n + 255) / 256), 256, [&] { k_mix_alg((uint32_t)n, tag, sha384); });
    return 0;
}
// k_sha2_sel over the n items of one family: messages at off[j] - base in msgs (readable 8 bytes past the last one), idx[j]
// their shard index, sha384 the shard's flags, dlen (32 or 48) bytes of e per item into digest_out; perm: optional
// processing order, as the counting sort gives it
extern "C" int hs_sha2_sel(size_t n, const uint8_t *msgs, const uint64_t *off, uint64_t base, const uint32_t *idx, const uint8_t *sha384, uint32_t dlen,
                           const uint32_t *perm, uint8_t *digest_out) {
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_sha2_sel((uint32_t)n, msgs, off, base, idx, sha384, dlen, digest_out, perm); });
    return 0;
}

// ---- mixed shards with keys per item (k_mix_split<true>, sbv_mixed_verify_batch) ----
// hs_mixed_split for a keys-per-item shard: key96 (one 96-byte row per item) instead of slots; besides the arrays of
// hs_mixed_split, qx0 / qy0 (32 B per item), qx1 / qy1 (48 B) and pub2 (32 B) receive the compacted keys
extern "C" int hs_mixed_split_keys(size_t n, const uint8_t *tag, const uint8_t *key96, const uint8_t *sig96, const uint64_t *off_in, uint32_t m0,
                                   uint32_t m1, uint32_t *idx, uint8_t *r0, uint8_t *s0, uint8_t *r1, uint8_t *s1, uint8_t *sig2, uint8_t *qx0,
                                   uint8_t *qy0, uint8_t *qx1, uint8_t *qy1, uint8_t *pub2, uint64_t *off_out) {
    const MixPlan p = hs_plan(n, m0, m1, idx, nullptr, r0, s0, r1, s1, sig2, off_out, nullptr, nullptr);
    const MixKeys k{{qx0, qx1}, {qy0, qy1}, pub2};
    const uint32_t nn = (uint32_t)n, ntiles = (uint32_t)((n + MIX_TILE - 1) / MIX_TILE);
    std::vector<uint32_t> tc((size_t)MIX_FAMILIES * ntiles + 1);
    std::vector<uint64_t> tb((size_t)MIX_FAMILIES * ntiles + 1);
    run_grid((ntiles + 255) / 256, 256, [&] { k_mix_count(nn, tag, off_in, ntiles, tc.data(), tb.data()); });
    run_grid(1, 1, [&] { k_mix_scan(ntiles, tc.data(), tb.data(), p); });
    run_grid((ntiles + 255) / 256, 256, [&] { k_mix_split<true>(nn, tag, nullptr, sig96, off_in, ntiles, tc.data(), tb.data(), p, key96, k); });
    return 0;
}
// The pipeline of sbv_mixed_verify_batch on one device: the split with keys, compaction, then per ECDSA family hs_sha256
// and hs_verify_grouped over the family's compacted keys, hs_ed25519_verify_grouped for the Ed25519 family (T, max_keys:
// the grouping settings of both), and the scatter.  Tags must be <= 2.
extern "C" int hs_mixed_verify_batch(size_t n, const uint8_t *tag, const uint8_t *msgs, const uint64_t *off, const uint8_t *sig96, const uint8_t *key96,
                                     uint32_t T, uint32_t max_keys, uint8_t *ok) {
    uint32_t m[3] = {0, 0, 0};
    for (size_t i = 0; i < n; i++) {
        if (tag[i] > 2) return -1;
        m[tag[i]]++;
    }
    const uint64_t base = off[0], bytes = off[n] - base;
    std::vector<uint8_t> src(bytes + 16, 0);
    if (bytes) memcpy(src.data(), msgs + base, bytes);
    std::vector<uint32_t> idx(n + 1);
    std::vector<uint8_t> r0(32 * m[0] + 1), s0(32 * m[0] + 1), r1(48 * m[1] + 1), s1(48 * m[1] + 1), sig2(64 * m[2] + 1), qx0(32 * m[0] + 1),
        qy0(32 * m[0] + 1), qx1(48 * m[1] + 1), qy1(48 * m[1] + 1), pub2(32 * m[2] + 1), blob(bytes + 128, 0), okf(n + 1, 0);
    std::vector<uint64_t> fo(n + 3);
    hs_mixed_split_keys(n, tag, key96, sig96, off, m[0], m[1], idx.data(), r0.data(), s0.data(), r1.data(), s1.data(), sig2.data(), qx0.data(), qy0.data(),
                        qx1.data(), qy1.data(), pub2.data(), fo.data());
    hs_mixed_compact(n, m[0], m[1], src.data(), off, base, idx.data(), fo.data(), blob.data());
    const uint32_t at[3] = {0, m[0], m[0] + m[1]};
    for (int f = 0; f < 2; f++) {
        if (!m[f]) continue;
        std::vector<uint8_t> dig(32 * m[f]);
        hs_sha256(m[f], blob.data(), fo.data() + at[f] + f, 0, nullptr, dig.data());
        hs_verify_grouped(f, m[f], f ? r1.data() : r0.data(), f ? s1.data() : s0.data(), f ? qx1.data() : qx0.data(), f ? qy1.data() : qy0.data(),
                          dig.data(), 32, T, max_keys, okf.data() + at[f], nullptr);
    }
    if (m[2]) hs_ed25519_verify_grouped(m[2], blob.data(), fo.data() + at[2] + 2, sig2.data(), pub2.data(), T, max_keys, okf.data() + at[2], nullptr);
    hs_mixed_scatter(n, m[0], m[1], idx.data(), okf.data(), ok);
    return 0;
}

// ---- the key cache (key_cache.cuh) ----
// The cache of one family on one device as caller-owned arrays (state / keys / pidx: smask + 1 slots; pool: cap tables of
// tw4 16-byte words; stats: 4 counters), so that a test can run launches against it and inspect or set any slot.
// fam: 0 = P-256 and 1 = P-384 (keys qx || qy of items of a, b), 2 = Ed25519 (32-byte keys of items of a; b unused).
static KcMap hs_kc_map(uint32_t *state, uint32_t *keys, uint32_t *pidx, uint32_t *pool, unsigned long long *stats, uint32_t smask, uint32_t cap,
                       uint32_t seed) {
    return KcMap{state, keys, pidx, pool, stats, smask, cap, seed};
}
template <class F>
static int hs_kc_fam(int fam, const uint8_t *a, const uint8_t *b, F &&f) {
    if (fam == 0) f(KcXY<P256>{a, b});
    else if (fam == 1) f(KcXY<P384>{a, b});
    else if (fam == 2) f(KcKey32{a});
    else return -1;
    return 0;
}
// k_kc_lookup over the launch's grouped keys (count *nkeys, key k = item keylist[k]); lk: 2 + kcap words, zeroed here
extern "C" int hs_kc_lookup(int fam, const uint8_t *a, const uint8_t *b, const uint32_t *nkeys, uint32_t kcap, const uint32_t *keylist,
                            uint32_t *state, uint32_t *keys, uint32_t *pidx, uint32_t *pool, unsigned long long *stats, uint32_t smask, uint32_t cap,
                            uint32_t seed, uint32_t tw4, int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab) {
    const KcMap c = hs_kc_map(state, keys, pidx, pool, stats, smask, cap, seed);
    lk[0] = lk[1] = 0;
    return hs_kc_fam(fam, a, b, [&](auto key) {
        run_grid_lockstep((unsigned)(((size_t)kcap * 32 + 127) / 128), 128, [&] {
            k_kc_lookup(nkeys, kcap, keylist, key, c, tw4, keyid, lk, keyflags, reinterpret_cast<uint4 *>(ktab));
        });
    });
}
// k_kc_insert after the build of the launch's misses (ktab[0, lk[0]), keyflags)
extern "C" int hs_kc_insert(int fam, const uint8_t *a, const uint8_t *b, uint32_t kcap, const uint32_t *lk, uint32_t *state, uint32_t *keys,
                            uint32_t *pidx, uint32_t *pool, unsigned long long *stats, uint32_t smask, uint32_t cap, uint32_t seed, uint32_t tw4,
                            const uint8_t *keyflags, const uint32_t *ktab) {
    const KcMap c = hs_kc_map(state, keys, pidx, pool, stats, smask, cap, seed);
    return hs_kc_fam(fam, a, b, [&](auto key) {
        run_grid_lockstep((unsigned)(((size_t)kcap * 32 + 127) / 128), 128, [&] {
            k_kc_insert(kcap, lk, key, c, tw4, keyflags, reinterpret_cast<const uint4 *>(ktab));
        });
    });
}
// the first probe slot of item i's key (kc_hash(key) & smask), or with fp != 0 its fingerprint (kc_fp)
extern "C" uint32_t hs_kc_slot(int fam, const uint8_t *a, const uint8_t *b, uint32_t i, uint32_t seed, uint32_t smask, int fp) {
    uint32_t h = 0;
    hs_kc_fam(fam, a, b, [&](auto key) {
        uint32_t w[decltype(key)::W];
        key.load(i, w);
        h = fp ? kc_fp(w, seed) : kc_hash(w, seed) & smask;
    });
    return h;
}

// ---- the evicting key cache (key_cache_assoc.cuh) ----
// The cache of one family as caller-owned arrays: state and stamp (u64) and keys of sets * KCA_WAYS ways, pool: one table
// of tw4 16-byte words per way, stats: 6 counters.  fam as for hs_kc_lookup; now: the launch's stamp.
static KcaMap hs_kca_map(unsigned long long *state, unsigned long long *stamp, uint32_t *keys, uint32_t *pool, unsigned long long *stats, uint32_t sets,
                         uint32_t seed) {
    return KcaMap{state, stamp, keys, pool, stats, sets, seed};
}
// k_kca_lookup over the launch's grouped keys (count *nkeys, key k = item keylist[k]); lk: 2 + kcap words, zeroed here
extern "C" int hs_kca_lookup(int fam, const uint8_t *a, const uint8_t *b, const uint32_t *nkeys, uint32_t kcap, const uint32_t *keylist,
                             unsigned long long *state, unsigned long long *stamp, uint32_t *keys, uint32_t *pool, unsigned long long *stats, uint32_t sets,
                             uint32_t seed, unsigned long long now, uint32_t tw4, int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab) {
    const KcaMap c = hs_kca_map(state, stamp, keys, pool, stats, sets, seed);
    lk[0] = lk[1] = 0;
    return hs_kc_fam(fam, a, b, [&](auto key) {
        run_grid_lockstep((unsigned)(((size_t)kcap * 32 + 127) / 128), 128, [&] {
            k_kca_lookup(nkeys, kcap, keylist, key, c, now, tw4, keyid, lk, keyflags, reinterpret_cast<uint4 *>(ktab));
        });
    });
}
// k_kca_insert after the build of the launch's misses (ktab[0, lk[0]), keyflags)
extern "C" int hs_kca_insert(int fam, const uint8_t *a, const uint8_t *b, uint32_t kcap, const uint32_t *lk, unsigned long long *state,
                             unsigned long long *stamp, uint32_t *keys, uint32_t *pool, unsigned long long *stats, uint32_t sets, uint32_t seed,
                             unsigned long long now, uint32_t tw4, const uint8_t *keyflags, const uint32_t *ktab) {
    const KcaMap c = hs_kca_map(state, stamp, keys, pool, stats, sets, seed);
    return hs_kc_fam(fam, a, b, [&](auto key) {
        run_grid_lockstep((unsigned)(((size_t)kcap * 32 + 127) / 128), 128, [&] {
            k_kca_insert(kcap, lk, key, c, now, tw4, keyflags, reinterpret_cast<const uint4 *>(ktab));
        });
    });
}
// the set of item i's key (its first way is set * KCA_WAYS), and in *fp its fingerprint as the state word holds it
extern "C" uint32_t hs_kca_set(int fam, const uint8_t *a, const uint8_t *b, uint32_t i, uint32_t seed, uint32_t sets, unsigned long long *fp) {
    uint32_t set = 0;
    hs_kc_fam(fam, a, b, [&](auto key) {
        uint32_t w[decltype(key)::W];
        key.load(i, w);
        const KcaMap c{nullptr, nullptr, nullptr, nullptr, nullptr, sets, seed};
        set = kca_base(c, w) / KCA_WAYS;
        *fp = kca_fp(w, seed);
    });
    return set;
}

// ---- RSA (rsa.cuh) and SHA-512 (sha512_batch.cuh) ----
extern "C" int hs_sha512(size_t n, const uint8_t *msgs, const uint64_t *off, uint64_t base, const uint32_t *perm, uint8_t *digest_out) {
    run_grid((unsigned)((n + 127) / 128), 128, [&] { k_sha512((uint32_t)n, msgs, off, base, digest_out, perm); });
    return 0;
}

// k_rsa_verify over n items of k = 64 * nl bytes, two groups of 16 lanes per simulated warp, in lockstep
extern "C" int hs_rsa_verify(int nl, size_t n, uint32_t hash, const uint8_t *sig, const uint8_t *mod, const uint32_t *pub_exp, const uint8_t *digest,
                             uint8_t *ok) {
    const unsigned blocks = (unsigned)((n * RSA_GROUP + 31) / 32);
    if (nl == 4) run_grid_lockstep(blocks, 32, [&] { k_rsa_verify<4>((uint32_t)n, hash, sig, mod, pub_exp, digest, ok); });
    else if (nl == 6) run_grid_lockstep(blocks, 32, [&] { k_rsa_verify<6>((uint32_t)n, hash, sig, mod, pub_exp, digest, ok); });
    else if (nl == 8) run_grid_lockstep(blocks, 32, [&] { k_rsa_verify<8>((uint32_t)n, hash, sig, mod, pub_exp, digest, ok); });
    else return -1;
    return 0;
}

// The arithmetic of rsa.cuh item by item: k_rsa_debug (rsa_debug.cuh) as libsbv.so's sbv_debug_rsa runs it, in blocks of
// 128 threads, with the same arguments.  -1 (and nothing written) for the calls rsa_debug_args_ok refuses.
extern "C" int hs_rsa_debug(uint32_t mod_bytes, int op, size_t n, const uint8_t *a, const uint8_t *b, const uint8_t *mod, const uint32_t *exp,
                            uint8_t *out, uint32_t *aux) {
    if (!rsa_debug_args_ok(mod_bytes, op, n, a, b, mod, exp, out, aux)) return -1;
    const unsigned blocks = (unsigned)((n * RSA_GROUP + 127) / 128);
    if (mod_bytes == 256) run_grid_lockstep(blocks, 128, [&] { k_rsa_debug<4>(op, (uint32_t)n, a, b, mod, exp, out, aux); });
    else if (mod_bytes == 384) run_grid_lockstep(blocks, 128, [&] { k_rsa_debug<6>(op, (uint32_t)n, a, b, mod, exp, out, aux); });
    else run_grid_lockstep(blocks, 128, [&] { k_rsa_debug<8>(op, (uint32_t)n, a, b, mod, exp, out, aux); });
    return 0;
}

// Ops 0-3 of hs_rsa_debug in the older layout: k = 64 * nl bytes, ninv[i] = aux, and for op 3 the 16 lazy words of item i
// packed at b + 64 i (not spread over a k-byte row).
extern "C" int hs_rsa_op(int nl, int op, size_t n, const uint8_t *a, const uint8_t *b, const uint8_t *mod, uint8_t *out, uint32_t *ninv) {
    if (op < RSA_DBG_MONT || op > RSA_DBG_RESOLVE || nl <= 0) return -1;
    const size_t k = 64 * (size_t)nl;
    std::vector<uint8_t> rows;
    if (op == RSA_DBG_RESOLVE && b) {
        rows.assign(n * k, 0);
        for (size_t i = 0; i < n; i++) memcpy(&rows[i * k], b + i * 64, 64);
        b = rows.data();
    }
    std::vector<uint32_t> exp(n, 0), aux(n);
    const int rc = hs_rsa_debug((uint32_t)k, op, n, a, b, mod, exp.data(), out, aux.data());
    if (rc == 0 && op != RSA_DBG_RESOLVE)
        for (size_t i = 0; i < n; i++) ninv[i] = aux[i];
    return rc;
}
