// inst_ed25519.cu — launchers of the Ed25519 kernels (sha512.cuh, ed25519_verify.cuh, ed25519_keyed.cuh,
// ed25519_comb.cuh) behind engine.h, the Ed25519 entry of the grouping table (ops.h: GroupOps), and the registry of
// registered Ed25519 keys.
#include <vector>

#include "engine.h"
#include "ed25519_comb.cuh"
#include "ed25519_keyed.cuh"
#include "ed25519_verify.cuh"
#include "key_cache.cuh"
#include "key_cache_assoc.cuh"
#include "keygroup.cuh"
#include "sha512.cuh"

using namespace sbv;

namespace {
constexpr int ED_BLOCK = 32;  // 32 KiB of shared memory per block (the 1A..8A tables): no opt-in attribute needed
constexpr size_t ED_SMEM = (size_t)8 * 4 * 8 * 4 * ED_BLOCK;
constexpr int EDK_BLOCK = 128;  // k_ed_verify_keyed: no shared memory; see DESIGN.md §3 for registers and occupancy
constexpr int EDC_BLOCK = 128;  // k_ed_verify_comb: likewise
}  // namespace
static_assert(SBV_ED_BTAB_ENTRIES == (size_t)ED_BWINS * ED_BENT && SBV_ED_BTAB_ENTRY_WORDS == ED_BWORDS, "engine.h: table of B");

// The fixed-base table of B, built on the first Ed25519 call of each device.  Caller holds e->mu and has set the device.
// The build is synchronised before the pointer is published, so a verification on any stream sees a finished table.
int sbv_ed_btab_ensure(sbv_engine *e, Dev &d) {
    if (d.ed_btab) return 0;
    uint32_t *t = nullptr;
    CU(e, cudaMalloc(&t, ED_BTAB_WORDS * sizeof(uint32_t)));
    k_ed_btab_init<<<(ED_BWINS * ED_BENT + 63) / 64, 64, 0, d.stream>>>(t);
    e->launches += 1;
    cudaError_t st = cudaGetLastError();
    if (st == cudaSuccess) st = cudaStreamSynchronize(d.stream);
    if (st != cudaSuccess) {
        cudaFree(t);
        return sbv_fail(e, SBV_ERR_CUDA, "k_ed_btab_init: %s", cudaGetErrorString(st));
    }
    d.ed_btab = t;
    return 0;
}

// ---- keys per item ----
// A keys-per-item launch: the first half is sbv_launch_verify_begin (pipeline.cu) over the grouping table below, then
//
//   st     memsets  k_kg_insert  k_kg_assign ─┬─ k_kg_route  length sort  k_ed_sha512 ─┬──────────── (wait tables) k_ed_verify_comb ─ (wait generic) ─ done
//   s_tab                                     └─ k_edc_bases  k_edc_fill  k_edc_inv  k_edc_final ──┘
//   s_gen                                                                              └─ k_ed_verify (keys without a table) ─────────────────┘
//
// Keys whose 32 bytes occur at least group_threshold times get a comb table (ed25519_comb.cuh) and their items take
// k_ed_verify_comb; the table construction (latency-bound: one doubling chain per key) runs beside SHA-512.  With a key
// cache reserved, k_kc_lookup runs after k_kg_assign and k_kc_insert after k_edc_final, as for ECDSA (k_kca_lookup and
// k_kca_insert for an evicting cache).
namespace {
constexpr KtGeom ED_COMB_GEOM{EDC_BASES_WORDS, EDC_HS_WORDS, EDC_ZTOP_WORDS, EDC_TAB_WORDS};
static_assert(EDC_TAB_WORDS == 2 * 255 * SBV_ED_BTAB_ENTRY_WORDS, "debug.cu: sbv_debug_ed25519_comb_tab's table of 510 entries");

// The GroupOps of Ed25519: the key is (pub, nullptr).
cudaError_t edg_group(uint32_t n, const uint8_t *pub, const uint8_t *, uint32_t seed, uint32_t hmask, uint32_t *htab, uint32_t *rep, uint32_t *kcnt,
                      uint32_t threshold, uint32_t max_keys, int32_t *keyid, uint32_t *keylist, uint32_t *counters, cudaStream_t st) {
    const unsigned blocks = (n + 255) / 256;
    k_kg_insert<<<blocks, 256, 0, st>>>(n, KgKey32{pub}, seed, hmask, htab, rep, kcnt);
    k_kg_assign<<<blocks, 256, 0, st>>>(n, rep, kcnt, threshold, max_keys, keyid, keylist, counters);
    return cudaGetLastError();
}

cudaError_t edg_build(const uint32_t *nk, uint32_t cap, const uint32_t *kl, const uint8_t *pub, const uint8_t *, uint32_t *bases, uint32_t *hs,
                      uint32_t *ztop, uint32_t *pref, uint32_t *ktab, uint8_t *keyflags, cudaStream_t st) {
    const unsigned kb = (cap + 63) / 64, cb = (unsigned)(((size_t)cap * EDC_NCHAIN + 63) / 64);
    k_edc_bases<<<kb, 64, 0, st>>>(nk, cap, kl, pub, bases, keyflags);
    k_edc_fill<<<cb, 64, 0, st>>>(nk, cap, bases, keyflags, hs, ztop, ktab);
    k_edc_inv<<<kb, 64, 0, st>>>(nk, cap, keyflags, ztop, pref);
    k_edc_final<<<cb, 64, 0, st>>>(nk, cap, keyflags, hs, ztop, ktab);
    return cudaGetLastError();
}

cudaError_t edg_cache_lookup(const uint32_t *nkeys_ptr, uint32_t kcap, const uint32_t *keylist, const uint8_t *pub, const uint8_t *, KcMap c, uint32_t tw4,
                             int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab, cudaStream_t st) {
    k_kc_lookup<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(nkeys_ptr, kcap, keylist, KcKey32{pub}, c, tw4, keyid, lk, keyflags,
                                                                            reinterpret_cast<uint4 *>(ktab));
    return cudaGetLastError();
}

cudaError_t edg_cache_insert(uint32_t kcap, const uint32_t *lk, const uint8_t *pub, const uint8_t *, KcMap c, uint32_t tw4, const uint8_t *keyflags,
                             const uint32_t *ktab, cudaStream_t st) {
    k_kc_insert<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(kcap, lk, KcKey32{pub}, c, tw4, keyflags,
                                                                            reinterpret_cast<const uint4 *>(ktab));
    return cudaGetLastError();
}

cudaError_t edg_evict_lookup(const uint32_t *nkeys_ptr, uint32_t kcap, const uint32_t *keylist, const uint8_t *pub, const uint8_t *, KcaMap c,
                             unsigned long long now, uint32_t tw4, int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab, cudaStream_t st) {
    k_kca_lookup<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(nkeys_ptr, kcap, keylist, KcKey32{pub}, c, now, tw4, keyid, lk, keyflags,
                                                                             reinterpret_cast<uint4 *>(ktab));
    return cudaGetLastError();
}

cudaError_t edg_evict_insert(uint32_t kcap, const uint32_t *lk, const uint8_t *pub, const uint8_t *, KcaMap c, unsigned long long now, uint32_t tw4,
                             const uint8_t *keyflags, const uint32_t *ktab, cudaStream_t st) {
    k_kca_insert<<<(unsigned)(((size_t)kcap * 32 + 127) / 128), 128, 0, st>>>(kcap, lk, KcKey32{pub}, c, now, tw4, keyflags,
                                                                             reinterpret_cast<const uint4 *>(ktab));
    return cudaGetLastError();
}

const KtOps ED_COMB = {ED_COMB_GEOM, edg_build};

// k_kg_route after the first half: the items of keys with a table onto w->klist, the rest onto w->glist (counts at
// zeroed[1] / zeroed[2])
int ed_route(sbv_engine *e, const VerifyLaunch &vl, cudaStream_t st) {
    Dev::Scratch *w = vl.w;
    k_kg_route<<<(uint32_t)((vl.n + 255) / 256), 256, 0, st>>>((uint32_t)vl.n, w->rep, w->keyid, w->item_kid, w->klist, w->glist, w->zeroed);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

int ed_grouped(sbv_engine *e, Dev &d, const VerifyLaunch &vl, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint8_t *d_sig,
               const uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st) {
    if (int rc = ed_route(e, vl, st)) return rc;
    Dev::Scratch *w = vl.w;
    const uint32_t nn = (uint32_t)vl.n, *counters = w->zeroed;
    const uint32_t *perm = nullptr;
    if (int rc = sbv_launch_length_sort(e, vl.n, d_off, d_perm, st, &perm)) return rc;
    k_ed_sha512<<<(nn + 127) / 128, 128, 0, st>>>(nn, d_sig, d_pub, d_msgs, d_off, base, d_k, perm, nullptr);
    e->launches += 1;
    CU(e, cudaGetLastError());
    CU(e, cudaEventRecord(w->ev_prep, st));
    CU(e, cudaStreamWaitEvent(w->s_gen, w->ev_prep, 0));
    const uint4 *btab = reinterpret_cast<const uint4 *>(d.ed_btab);
    k_ed_verify<ED_BLOCK><<<(nn + ED_BLOCK - 1) / ED_BLOCK, ED_BLOCK, ED_SMEM, w->s_gen>>>(nn, d_sig, d_pub, d_k, btab, d_ok, w->glist, counters + 2);
    e->launches += 1;
    CU(e, cudaGetLastError());
    CU(e, cudaEventRecord(w->ev_gen, w->s_gen));
    CU(e, cudaStreamWaitEvent(st, w->ev_tab, 0));
    k_ed_verify_comb<EDC_BLOCK><<<(nn + EDC_BLOCK - 1) / EDC_BLOCK, EDC_BLOCK, 0, st>>>(
        nn, d_sig, w->item_kid, w->keyflags, reinterpret_cast<const uint4 *>((uint32_t *)w->ktab), d_k, btab, d_ok, w->klist, counters + 1);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

// the comb kernel over every item (no list) with the caller's k
int ed_comb_k(sbv_engine *e, Dev &d, const VerifyLaunch &vl, const uint8_t *d_sig, const uint32_t *d_k, uint8_t *d_ok, cudaStream_t st) {
    if (int rc = ed_route(e, vl, st)) return rc;
    Dev::Scratch *w = vl.w;
    const uint32_t nn = (uint32_t)vl.n;
    CU(e, cudaStreamWaitEvent(st, w->ev_tab, 0));
    k_ed_verify_comb<EDC_BLOCK><<<(nn + EDC_BLOCK - 1) / EDC_BLOCK, EDC_BLOCK, 0, st>>>(
        nn, d_sig, w->item_kid, w->keyflags, reinterpret_cast<const uint4 *>((uint32_t *)w->ktab), d_k, reinterpret_cast<const uint4 *>(d.ed_btab), d_ok,
        nullptr, nullptr);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
}  // namespace

const GroupOps sbv_group_ed25519 = {&ED_COMB, KcKey32::W, 4, edg_group, edg_cache_lookup, edg_cache_insert, edg_evict_lookup, edg_evict_insert};

int sbv_launch_ed25519(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint8_t *d_sig,
                       const uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st) {
    VerifyLaunch vl;
    if (int rc = sbv_launch_verify_begin(e, d, SBV_ED25519, n, d_pub, nullptr, st, &vl)) return rc;
    if (vl.grouping)
        return sbv_launch_verify_close(e, vl, st, ed_grouped(e, d, vl, d_msgs, d_off, base, d_sig, d_pub, d_k, d_perm, d_ok, st));
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_ed_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_sig, d_pub, d_msgs, d_off, base, d_k, perm, nullptr);
    k_ed_verify<ED_BLOCK><<<(uint32_t)((n + ED_BLOCK - 1) / ED_BLOCK), ED_BLOCK, ED_SMEM, st>>>(
        (uint32_t)n, d_sig, d_pub, d_k, reinterpret_cast<const uint4 *>(d.ed_btab), d_ok, nullptr, nullptr);
    e->launches += 2;
    CU(e, cudaGetLastError());
    return 0;
}

// test hook (debug.cu): k_ed_verify_comb with the caller's k over every item, every distinct key with a table
int sbv_launch_ed_verify_comb_k(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_sig, const uint8_t *d_pub, const uint32_t *d_k, uint8_t *d_ok,
                                cudaStream_t st) {
    VerifyLaunch vl;
    if (int rc = sbv_launch_verify_begin(e, d, SBV_ED25519, n, d_pub, nullptr, st, &vl, 1, true)) return rc;
    return sbv_launch_verify_close(e, vl, st, ed_comb_k(e, d, vl, d_sig, d_k, d_ok, st));
}

// test hook (debug.cu): the production SHA-512 kernel with its digests written out as well
int sbv_launch_ed_sha512_digest(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, const uint8_t *d_sig, const uint8_t *d_pub,
                                uint32_t *d_k, uint32_t *d_dig, cudaStream_t st) {
    k_ed_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_sig, d_pub, d_msgs, d_off, 0, d_k, nullptr, d_dig);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

// test hook (debug.cu): the production verification kernel with the caller's k (word-major, every k < L) in place of
// SHA-512's.  The table of B must exist (sbv_ed_btab_ensure).
int sbv_launch_ed_verify_k(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_sig, const uint8_t *d_pub, const uint32_t *d_k, uint8_t *d_ok,
                           cudaStream_t st) {
    k_ed_verify<ED_BLOCK><<<(uint32_t)((n + ED_BLOCK - 1) / ED_BLOCK), ED_BLOCK, ED_SMEM, st>>>(
        (uint32_t)n, d_sig, d_pub, d_k, reinterpret_cast<const uint4 *>(d.ed_btab), d_ok, nullptr, nullptr);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

// ---- registered Ed25519 keys ----
void sbv_ed_keys_free(Dev &d) {
    void *p[] = {d.ed_kpub, d.ed_slot2local, d.ed_ktab};
    for (void *x : p) if (x) cudaFree(x);
    d.ed_kpub = nullptr;
    d.ed_slot2local = nullptr;
    d.ed_ktab = nullptr;
    d.ed_n_slots = 0;
    d.ed_n_local = 0;
}

namespace {
struct DevTemp {  // device temporaries of one registry build, freed on every exit path
    std::vector<void *> p;
    ~DevTemp() { for (void *x : p) cudaFree(x); }
    template <class T>
    cudaError_t alloc(T **out, size_t bytes) {
        void *q = nullptr;
        const cudaError_t st = cudaMalloc(&q, bytes);
        if (st == cudaSuccess) { p.push_back(q); *out = static_cast<T *>(q); }
        return st;
    }
};

// The registry of device d from the n keys of pub: the registered bytes, k_ed_kdecode for the flags, the map of the
// decodable slots to tables, and k_ed_ktab_build for their tables, at most ED_KBUILD_MAX keys per launch.
int ed_keys_fill(sbv_engine *e, Dev &d, size_t n, const uint8_t *pub) {
    const uint32_t ns = (uint32_t)n;
    CU(e, cudaMalloc(&d.ed_kpub, n * 32));
    CU(e, cudaMalloc(&d.ed_slot2local, n * sizeof(int32_t)));
    DevTemp tmp;
    uint32_t *xy = nullptr;
    uint8_t *flag = nullptr;
    CU(e, tmp.alloc(&xy, n * 16 * sizeof(uint32_t)));
    CU(e, tmp.alloc(&flag, n));
    CU(e, cudaMemcpyAsync(d.ed_kpub, pub, n * 32, cudaMemcpyHostToDevice, d.stream));
    k_ed_kdecode<<<(ns + 63) / 64, 64, 0, d.stream>>>(ns, d.ed_kpub, xy, flag);
    e->launches += 1;
    CU(e, cudaGetLastError());
    std::vector<uint8_t> hflag(n);
    CU(e, cudaMemcpyAsync(hflag.data(), flag, n, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    std::vector<int32_t> map(n, -1);
    std::vector<uint32_t> slot_of;
    for (size_t i = 0; i < n; i++)
        if (hflag[i]) { map[i] = (int32_t)slot_of.size(); slot_of.push_back((uint32_t)i); }
    const size_t cnt = slot_of.size();
    CU(e, cudaMemcpyAsync(d.ed_slot2local, map.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, d.stream));
    if (cnt) {
        CU(e, cudaMalloc(&d.ed_ktab, cnt * ED_KTAB_WORDS * sizeof(uint32_t)));
        const size_t chunk = std::min(cnt, (size_t)ED_KBUILD_MAX);
        uint32_t *d_slot_of = nullptr, *pref = nullptr;
        CU(e, tmp.alloc(&d_slot_of, cnt * sizeof(uint32_t)));
        CU(e, tmp.alloc(&pref, chunk * ED_BWINS * ED_BENT * 8 * sizeof(uint32_t)));
        CU(e, cudaMemcpyAsync(d_slot_of, slot_of.data(), cnt * sizeof(uint32_t), cudaMemcpyHostToDevice, d.stream));
        for (size_t c0 = 0; c0 < cnt; c0 += chunk) {
            const uint32_t cc = (uint32_t)std::min(chunk, cnt - c0), threads = cc * ED_BWINS;
            k_ed_ktab_build<<<(threads + 63) / 64, 64, 0, d.stream>>>(cc, d_slot_of + c0, xy, d.ed_ktab + c0 * ED_KTAB_WORDS, pref);
            e->launches += 1;
            CU(e, cudaGetLastError());
        }
    }
    CU(e, cudaStreamSynchronize(d.stream));
    d.ed_n_slots = ns;
    d.ed_n_local = (uint32_t)cnt;
    return 0;
}
}  // namespace

int sbv_ed_keys_build(sbv_engine *e, Dev &d, size_t n, const uint8_t *pub) {
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, cudaDeviceSynchronize());  // no launch on any lane may still read the old registry
    sbv_ed_keys_free(d);
    if (n == 0) return 0;
    const int rc = ed_keys_fill(e, d, n, pub);
    if (rc) {
        cudaStreamSynchronize(d.stream);
        sbv_ed_keys_free(d);
    }
    return rc;
}

int sbv_launch_ed25519_registered(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint32_t *d_slot,
                                  const uint8_t *d_sig, uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st) {
    k_ed_key_gather<<<(uint32_t)((2 * n + 255) / 256), 256, 0, st>>>((uint32_t)n, d_slot, d.ed_n_slots, reinterpret_cast<const uint4 *>(d.ed_kpub),
                                                                      reinterpret_cast<uint4 *>(d_pub));
    e->launches += 1;
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_ed_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_sig, d_pub, d_msgs, d_off, base, d_k, perm, nullptr);
    k_ed_verify_keyed<EDK_BLOCK><<<(uint32_t)((n + EDK_BLOCK - 1) / EDK_BLOCK), EDK_BLOCK, 0, st>>>(
        (uint32_t)n, d_sig, d_slot, d.ed_n_slots, d.ed_slot2local, reinterpret_cast<const uint4 *>(d.ed_ktab), d_k,
        reinterpret_cast<const uint4 *>(d.ed_btab), d_ok);
    e->launches += 2;
    CU(e, cudaGetLastError());
    return 0;
}

// test hook (debug.cu): the production registered-key kernel with the caller's k (word-major, every k < L)
int sbv_launch_ed_verify_registered_k(sbv_engine *e, Dev &d, size_t n, const uint32_t *d_slot, const uint8_t *d_sig, const uint32_t *d_k, uint8_t *d_ok,
                                      cudaStream_t st) {
    k_ed_verify_keyed<EDK_BLOCK><<<(uint32_t)((n + EDK_BLOCK - 1) / EDK_BLOCK), EDK_BLOCK, 0, st>>>(
        (uint32_t)n, d_sig, d_slot, d.ed_n_slots, d.ed_slot2local, reinterpret_cast<const uint4 *>(d.ed_ktab), d_k,
        reinterpret_cast<const uint4 *>(d.ed_btab), d_ok);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
