// inst_ed25519.cu — launchers of the Ed25519 kernels (sha512.cuh, ed25519_verify.cuh, ed25519_keyed.cuh,
// ed25519_comb.cuh) behind engine.h, and the registry of registered Ed25519 keys.
#include <vector>

#include "engine.h"
#include "ed25519_comb.cuh"
#include "ed25519_keyed.cuh"
#include "ed25519_verify.cuh"
#include "key_cache.cuh"
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
// A keys-per-item launch (pipeline.cu draws the same for ECDSA):
//
//   st     memsets  k_kg_insert  k_kg_assign ─┬─ k_kg_route  length sort  k_ed_sha512 ─┬──────────── (wait tables) k_ed_verify_comb ─ (wait generic) ─ done
//   s_tab                                     └─ k_edc_bases  k_edc_fill  k_edc_inv  k_edc_final ──┘
//   s_gen                                                                              └─ k_ed_verify (keys without a table) ─────────────────┘
//
// Keys whose 32 bytes occur at least group_threshold times get a comb table (ed25519_comb.cuh) and their items take
// k_ed_verify_comb; the table construction (latency-bound: one doubling chain per key) runs beside SHA-512.  With a key
// cache reserved, k_kc_lookup runs after k_kg_assign and k_kc_insert after k_edc_final, as in pipeline.cu.
namespace {
constexpr KtGeom ED_COMB_GEOM{EDC_BASES_WORDS, EDC_HS_WORDS, EDC_ZTOP_WORDS, EDC_TAB_WORDS};
static_assert(SBV_ED_COMB_ENTRIES * SBV_ED_BTAB_ENTRY_WORDS == EDC_TAB_WORDS, "engine.h: comb table");

// table slots of a launch of n items at threshold T, as the ECDSA launches count them; 0: the launch does not group
size_t ed_group_cap(const sbv_engine *e, size_t n, uint32_t T) {
    if (T == 0 || n < T || n < (size_t)e->group_min_batch || e->group_max_keys <= 0) return 0;
    size_t kcap = n / T;
    if (kcap > (size_t)e->group_max_keys) kcap = (size_t)e->group_max_keys;
    return kcap ? kcap : 1;
}

// On st: the grouping of the n keys of d_pub (at most kcap of them with >= T items get a table slot) and the routing onto
// w->klist / w->glist (counts at zeroed[1] / zeroed[2]); on w->s_tab: the comb tables, then w->ev_tab.
int ed_group(sbv_engine *e, Dev &d, Dev::Scratch *w, size_t n, const uint8_t *d_pub, uint32_t T, size_t kcap, cudaStream_t st) {
    const uint32_t nn = (uint32_t)n, cap = (uint32_t)kcap, blocks = (nn + 255) / 256;
    uint32_t *counters = w->zeroed, *kcnt = w->zeroed + 4;
    CU(e, cudaMemsetAsync(w->htab, 0xff, (size_t)w->hsize * 4, st));
    CU(e, cudaMemsetAsync(w->zeroed, 0, (n + 4) * 4, st));
    k_kg_insert<<<blocks, 256, 0, st>>>(nn, KgKey32{d_pub}, e->hash_seed, w->hsize - 1, w->htab, w->rep, kcnt);
    k_kg_assign<<<blocks, 256, 0, st>>>(nn, w->rep, kcnt, T, cap, w->keyid, w->keylist, counters);
    CU(e, cudaGetLastError());
    // with a key cache: the lookup renumbers the keys (misses first), copies the hits' tables, and the build makes the misses
    const Dev::KeyCache &kc = d.kc[SBV_ED25519];
    uint32_t *lk = sbv_key_cache_area(d, SBV_ED25519, w, kcap);
    const unsigned wb = (unsigned)(((size_t)cap * 32 + 127) / 128);
    if (lk) {
        CU(e, cudaMemsetAsync(lk, 0, 8, st));
        k_kc_lookup<<<wb, 128, 0, st>>>(counters, cap, w->keylist, KcKey32{d_pub}, kc.map, (uint32_t)kc.tw4, w->keyid, lk, w->keyflags,
                                        reinterpret_cast<uint4 *>((uint32_t *)w->ktab));
        CU(e, cudaGetLastError());
    }
    CU(e, cudaEventRecord(w->ev_group, st));
    CU(e, cudaStreamWaitEvent(w->s_tab, w->ev_group, 0));
    const unsigned kb = (cap + 63) / 64, cb = (unsigned)(((size_t)cap * EDC_NCHAIN + 63) / 64);
    const uint32_t *nk = lk ? lk : counters, *kl = lk ? lk + 2 : (const uint32_t *)w->keylist;
    k_edc_bases<<<kb, 64, 0, w->s_tab>>>(nk, cap, kl, d_pub, w->bases, w->keyflags);
    k_edc_fill<<<cb, 64, 0, w->s_tab>>>(nk, cap, w->bases, w->keyflags, w->hs, w->ztop, w->ktab);
    k_edc_inv<<<kb, 64, 0, w->s_tab>>>(nk, cap, w->keyflags, w->ztop, w->pref);
    k_edc_final<<<cb, 64, 0, w->s_tab>>>(nk, cap, w->keyflags, w->hs, w->ztop, w->ktab);
    if (lk)
        k_kc_insert<<<wb, 128, 0, w->s_tab>>>(cap, lk, KcKey32{d_pub}, kc.map, (uint32_t)kc.tw4, w->keyflags,
                                              reinterpret_cast<const uint4 *>((uint32_t *)w->ktab));
    CU(e, cudaGetLastError());
    CU(e, cudaEventRecord(w->ev_tab, w->s_tab));
    k_kg_route<<<blocks, 256, 0, st>>>(nn, w->rep, w->keyid, w->item_kid, w->klist, w->glist, counters);
    e->launches += 7 + (lk ? 2 : 0);
    CU(e, cudaGetLastError());
    return 0;
}

// Hands the set back behind everything the launch enqueued on its side streams: on success and after a fault alike.
int ed_close(sbv_engine *e, Dev::Scratch *w, cudaStream_t st, int rc) {
    if (rc) cudaStreamWaitEvent(st, w->ev_tab, 0);  // a fault before the join: the tables may still be in flight
    const cudaError_t a = cudaStreamWaitEvent(st, w->ev_gen, 0), b = cudaEventRecord(w->done, st);
    if (rc) return rc;
    CU(e, a);
    CU(e, b);
    return 0;
}

int ed_grouped(sbv_engine *e, Dev &d, Dev::Scratch *w, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint8_t *d_sig,
               const uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, uint32_t T, size_t kcap, cudaStream_t st) {
    if (int rc = ed_group(e, d, w, n, d_pub, T, kcap, st)) return rc;
    const uint32_t nn = (uint32_t)n, *counters = w->zeroed;
    const uint32_t *perm = nullptr;
    if (int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm)) return rc;
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
}  // namespace

int sbv_launch_ed25519(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint8_t *d_sig,
                       const uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st) {
    const uint32_t T = e->group_threshold > 0 ? (uint32_t)e->group_threshold : 0;
    const size_t kcap = ed_group_cap(e, n, T);
    if (kcap) {
        Dev::Scratch *w = nullptr;
        if (int rc = sbv_take_scratch(e, d, 0, &ED_COMB_GEOM, n, kcap, st, &w)) return rc;
        return ed_close(e, w, st, ed_grouped(e, d, w, n, d_msgs, d_off, base, d_sig, d_pub, d_k, d_perm, d_ok, T, kcap, st));
    }
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

// test hook (debug.cu): the first half of a grouped launch, synchronised
int sbv_launch_ed_comb_tables(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_pub, cudaStream_t st, Dev::Scratch **out) {
    *out = nullptr;
    const uint32_t T = e->group_threshold > 0 ? (uint32_t)e->group_threshold : 0;
    const size_t kcap = ed_group_cap(e, n, T);
    if (!kcap) return 0;
    Dev::Scratch *w = nullptr;
    if (int rc = sbv_take_scratch(e, d, 0, &ED_COMB_GEOM, n, kcap, st, &w)) return rc;
    int rc = ed_group(e, d, w, n, d_pub, T, kcap, st);
    if (!rc) {
        const cudaError_t a = cudaStreamWaitEvent(st, w->ev_tab, 0);
        rc = a != cudaSuccess ? sbv_fail(e, SBV_ERR_CUDA, "cudaStreamWaitEvent: %s", cudaGetErrorString(a)) : 0;
    }
    if (!rc) {
        const cudaError_t a = cudaStreamSynchronize(st);
        rc = a != cudaSuccess ? sbv_fail(e, SBV_ERR_CUDA, "k_edc_*: %s", cudaGetErrorString(a)) : 0;
    }
    if (rc) return ed_close(e, w, st, rc);
    *out = w;
    return 0;
}

// test hook (debug.cu): k_ed_verify_comb with the caller's k over every item, every distinct key with a table
int sbv_launch_ed_verify_comb_k(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_sig, const uint8_t *d_pub, const uint32_t *d_k, uint8_t *d_ok,
                                cudaStream_t st) {
    Dev::Scratch *w = nullptr;
    if (int rc = sbv_take_scratch(e, d, 0, &ED_COMB_GEOM, n, n, st, &w)) return rc;
    int rc = ed_group(e, d, w, n, d_pub, 1, n, st);
    if (!rc) {
        const uint32_t nn = (uint32_t)n;
        const cudaError_t a = cudaStreamWaitEvent(st, w->ev_tab, 0);
        if (a == cudaSuccess)
            k_ed_verify_comb<EDC_BLOCK><<<(nn + EDC_BLOCK - 1) / EDC_BLOCK, EDC_BLOCK, 0, st>>>(
                nn, d_sig, w->item_kid, w->keyflags, reinterpret_cast<const uint4 *>((uint32_t *)w->ktab), d_k, reinterpret_cast<const uint4 *>(d.ed_btab),
                d_ok, nullptr, nullptr);
        e->launches += 1;
        const cudaError_t b = a != cudaSuccess ? a : cudaGetLastError();
        rc = b != cudaSuccess ? sbv_fail(e, SBV_ERR_CUDA, "k_ed_verify_comb: %s", cudaGetErrorString(b)) : 0;
    }
    return ed_close(e, w, st, rc);
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
