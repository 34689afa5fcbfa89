// key_cache.cu — the grouped-key cache of each device: reserve, free and statistics (sbv_key_cache_reserve /
// sbv_key_cache_reserve_evicting / sbv_key_cache_stats / sbv_key_cache_stats_ex).  The kernels are in key_cache.cuh
// (fill once) and key_cache_assoc.cuh (evicting); pipeline.cu enqueues them through the grouping table (ops.h).
#include <cstring>

#include "engine.h"

namespace {
// One allocation: pool [cap][table words], stats [4] (u64), state [slots], pidx [slots], keys [slots][key words], then the
// SBV_SCRATCH launch areas.  The part after the pool is zeroed: an empty map and zero counters.
int kc_alloc(sbv_engine *e, Dev &d, int s, size_t cap) {
    if (cap == 0) return 0;
    if (cap > ((size_t)1 << 30)) return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve: %zu tables for scheme %d", cap, s);
    uint32_t slots = 1;
    while (slots < 2 * cap) slots <<= 1;
    const GroupOps &g = sbv_group_ops(s);
    const size_t tw = g.kt->geom.ktab_words, kw = g.key_words;
    const size_t lkw = 2 + (size_t)(e->group_max_keys > 0 ? e->group_max_keys : 0);
    if (cap > SIZE_MAX / (tw * 4)) return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve: %zu tables for scheme %d", cap, s);
    const size_t pool = cap * tw * 4, rest = 32 + (size_t)slots * (2 + kw) * 4 + SBV_SCRATCH * lkw * 4;
    if (pool > SIZE_MAX - rest) return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve: %zu tables for scheme %d", cap, s);
    Dev::KeyCache &k = d.kc[s];
    if (cudaMalloc(&k.mem, pool + rest) != cudaSuccess) {
        cudaGetLastError();
        k.mem = nullptr;
        return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve: %zu bytes for scheme %d on device %d", pool + rest, s, d.ordinal);
    }
    uint8_t *b = static_cast<uint8_t *>(k.mem);
    k.map.pool = reinterpret_cast<uint32_t *>(b);
    k.map.stats = reinterpret_cast<unsigned long long *>(b + pool);
    k.map.state = reinterpret_cast<uint32_t *>(b + pool + 32);
    k.map.pidx = k.map.state + slots;
    k.map.keys = k.map.pidx + slots;
    k.map.smask = slots - 1;
    k.map.cap = (uint32_t)cap;
    k.capacity = cap;
    k.map.seed = (e->hash_seed ^ 0x6a09e667u) * (uint32_t)(2 * s + 3);  // per family, independent of the grouping's probes
    k.lk = k.map.keys + (size_t)slots * kw;
    k.lk_words = lkw;
    k.tw4 = tw / 4;
    CU(e, cudaMemsetAsync(b + pool, 0, rest, d.stream));
    return 0;
}

// The evicting cache: cap rounded up to a multiple of KCA_WAYS ways.  One allocation: pool [ways][table words], stats [8]
// (u64: six used), state [ways] (u64), stamp [ways] (u64), keys [ways][key words], then the SBV_SCRATCH launch areas.
// The part after the pool is zeroed: every way EMPTY, every stamp and counter 0.
int kca_alloc(sbv_engine *e, Dev &d, int s, size_t cap) {
    if (cap == 0) return 0;
    if (cap > ((size_t)1 << 30)) return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve_evicting: %zu tables for scheme %d", cap, s);
    const size_t ways = (cap + KCA_WAYS - 1) / KCA_WAYS * KCA_WAYS;
    const GroupOps &g = sbv_group_ops(s);
    const size_t tw = g.kt->geom.ktab_words, kw = g.key_words;
    const size_t lkw = 2 + (size_t)(e->group_max_keys > 0 ? e->group_max_keys : 0);
    if (ways > SIZE_MAX / (tw * 4)) return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve_evicting: %zu tables for scheme %d", cap, s);
    const size_t pool = ways * tw * 4, rest = 64 + ways * (16 + kw * 4) + SBV_SCRATCH * lkw * 4;
    if (pool > SIZE_MAX - rest) return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve_evicting: %zu tables for scheme %d", cap, s);
    Dev::KeyCache &k = d.kc[s];
    if (cudaMalloc(&k.mem, pool + rest) != cudaSuccess) {
        cudaGetLastError();
        k.mem = nullptr;
        return sbv_fail(e, SBV_ERR_NOMEM, "sbv_key_cache_reserve_evicting: %zu bytes for scheme %d on device %d", pool + rest, s, d.ordinal);
    }
    uint8_t *b = static_cast<uint8_t *>(k.mem);
    k.evicting = true;
    k.amap.pool = reinterpret_cast<uint32_t *>(b);
    k.amap.stats = reinterpret_cast<unsigned long long *>(b + pool);
    k.amap.state = k.amap.stats + 8;
    k.amap.stamp = k.amap.state + ways;
    k.amap.keys = reinterpret_cast<uint32_t *>(k.amap.stamp + ways);
    k.amap.sets = (uint32_t)(ways / KCA_WAYS);
    k.amap.seed = (e->hash_seed ^ 0x6a09e667u) * (uint32_t)(2 * s + 3);
    k.capacity = ways;
    k.lk = k.amap.keys + ways * kw;
    k.lk_words = lkw;
    k.tw4 = tw / 4;
    CU(e, cudaMemsetAsync(b + pool, 0, rest, d.stream));
    return 0;
}

// Replaces every device's caches with caches of the given mode.  Excludes concurrent launches as sbv_ed25519_set_keys
// does: the registry lock, the engine lock, then a drain of every device, so no launch still reads or fills the old maps.
// A fault frees them all.
int reserve(sbv_engine *e, const size_t cap[3], bool evicting) {
    std::unique_lock<std::shared_mutex> reg(e->ed_reg_mu);
    std::lock_guard<std::mutex> lk(e->mu);
    for (Dev &d : e->devs) {
        CU(e, cudaSetDevice(d.ordinal));
        CU(e, cudaDeviceSynchronize());
        sbv_key_cache_free(d);
    }
    for (Dev &d : e->devs) {
        int rc = 0;
        const cudaError_t a = cudaSetDevice(d.ordinal);
        if (a != cudaSuccess) rc = sbv_fail(e, SBV_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(a));
        for (int s = 0; s < 3 && !rc; s++) rc = evicting ? kca_alloc(e, d, s, cap[s]) : kc_alloc(e, d, s, cap[s]);
        if (!rc) {
            const cudaError_t b = cudaStreamSynchronize(d.stream);
            if (b != cudaSuccess) rc = sbv_fail(e, SBV_ERR_CUDA, "sbv_key_cache_reserve: %s", cudaGetErrorString(b));
        }
        if (rc) {
            for (Dev &o : e->devs) {
                cudaSetDevice(o.ordinal);
                cudaDeviceSynchronize();
                sbv_key_cache_free(o);
            }
            return rc;
        }
    }
    return SBV_OK;
}

// capacity, resident, hits, misses, evictions, given up of one scheme, summed over devices; caller holds e->mu
int stats(sbv_engine *e, uint8_t scheme, uint64_t (&sum)[6]) {
    for (uint64_t &v : sum) v = 0;
    for (Dev &d : e->devs) {
        const Dev::KeyCache &k = d.kc[scheme];
        if (!k.mem) continue;
        unsigned long long st[6] = {0, 0, 0, 0, 0, 0};
        CU(e, cudaSetDevice(d.ordinal));
        if (k.evicting) CU(e, cudaMemcpy(st, k.amap.stats, sizeof st, cudaMemcpyDeviceToHost));
        else CU(e, cudaMemcpy(st, k.map.stats, 4 * sizeof st[0], cudaMemcpyDeviceToHost));
        sum[0] += k.capacity;
        for (int i = 1; i < 6; i++) sum[i] += st[i];
    }
    return 0;
}
}  // namespace

void sbv_key_cache_free(Dev &d) {
    for (Dev::KeyCache &k : d.kc) {
        if (k.mem) cudaFree(k.mem);
        k = Dev::KeyCache{};
    }
}

uint32_t *sbv_key_cache_area(Dev &d, int s, const Dev::Scratch *w, size_t kcap) {
    const Dev::KeyCache &k = d.kc[s];
    return k.mem && kcap + 2 <= k.lk_words ? k.lk + (size_t)(w - d.ws) * k.lk_words : nullptr;
}

extern "C" {

int sbv_key_cache_reserve(sbv_engine *e, size_t p256, size_t p384, size_t ed25519) {
    if (!e) return SBV_ERR_ARG;
    const size_t cap[3] = {p256, p384, ed25519};
    return reserve(e, cap, false);
}

int sbv_key_cache_reserve_evicting(sbv_engine *e, size_t p256, size_t p384, size_t ed25519) {
    if (!e) return SBV_ERR_ARG;
    const size_t cap[3] = {p256, p384, ed25519};
    return reserve(e, cap, true);
}

int sbv_key_cache_stats(sbv_engine *e, uint8_t scheme, uint64_t out[4]) {
    if (!e) return SBV_ERR_ARG;
    if (scheme > SBV_ED25519 || !out) return sbv_fail(e, SBV_ERR_ARG, "sbv_key_cache_stats: bad argument");
    std::lock_guard<std::mutex> lk(e->mu);
    uint64_t sum[6];
    if (int rc = stats(e, scheme, sum)) return rc;
    memcpy(out, sum, 4 * sizeof sum[0]);
    return SBV_OK;
}

int sbv_key_cache_stats_ex(sbv_engine *e, uint8_t scheme, uint64_t out[6]) {
    if (!e) return SBV_ERR_ARG;
    if (scheme > SBV_ED25519 || !out) return sbv_fail(e, SBV_ERR_ARG, "sbv_key_cache_stats_ex: bad argument");
    std::lock_guard<std::mutex> lk(e->mu);
    uint64_t sum[6];
    if (int rc = stats(e, scheme, sum)) return rc;
    memcpy(out, sum, sizeof sum);
    return SBV_OK;
}

}  // extern "C"
