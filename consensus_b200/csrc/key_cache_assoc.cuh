// key_cache_assoc.cuh — the evicting mode of the grouped-key cache (sbv_key_cache_reserve_evicting).
//
// The same two places in a keys-per-item launch as the fill-once cache (key_cache.cuh), the same launch area and the same
// contract with the build:
//
//   k_kca_lookup  on st, after k_kg_assign: one warp per grouped key.  Misses get ids [0, m) (lk[0] = m), hits ids
//                 [m, k) (lk[1]), lk[2 + id] and keyid[] follow; a hit's table is copied into its ktab slot and its key flag
//                 set.  The build kernels then make exactly the missed tables, ktab[0, m).
//   k_kca_insert  on s_tab, after the build: one warp per missed key whose build flagged it valid.  It takes a way of the
//                 key's set (an EMPTY one, else the least recently used one it may replace), writes the key and the table
//                 and publishes READY.
//
// The map: capacity rounded up to a multiple of KCA_WAYS (16) ways, sets = ways / 16.  A hash of the exact key bytes picks
// the set, a second hash the 32-bit fingerprint.  Way i of the map is pool entry i: no index, no pool counter.  Per way:
//   state  64 bits: fingerprint << 32 | pins << 2 | EMPTY / BUSY / READY  (0 is EMPTY: a memset empties the map)
//   keys   the key words of a READY way, compared word for word before any hit
//   stamp  the launch sequence number (per device and scheme, one per grouped launch, from 1) of the last hit or insert
// Replacement: least recently stamped within the set, among READY ways with no pin and a stamp older than the launch's.
// Nothing waits on another thread: no spin on BUSY, no spin on a pin; every loop is bounded.
//
// Why the races are harmless:
//  * No READY on an incomplete table.  A way becomes BUSY by one CAS, from EMPTY or from READY with no pin; the warp that
//    won it writes the stamp, the key words and the whole table, fences, and only then release-stores READY with its own
//    fingerprint and no pin.  Readers load the state with acquire semantics and the key and table through L2 (ld.cg).
//  * No table copied out of a way that can change under the copy.  A hit first pins the way: a CAS from the exact READY
//    word it read to that word plus one pin.  A claim needs a word with no pin, so from the pin until the unpin no insert
//    can take the way; the copy completes (every lane's loads, a warp barrier and a fence) before the unpin.  A pin lost to
//    another pin is retried from the new word, a bounded number of times; a pin lost to a claim is a miss.
//  * ABA.  Between the read of a READY word and the pin, the way may have been evicted and refilled by another key with the
//    same fingerprint, leaving the very same word: the CAS succeeds.  So the key words are compared after the pin (and a
//    fence), never before: a mismatch unpins and counts as a miss.  A refill with the same key holds the same table (a
//    table is a pure function of the key bytes), so it is a correct hit.
//  * A launch never evicts a table it has just used.  A hit stamps the way (atomicMax) before the launch's insert kernel
//    runs (stream order: the insert waits for ev_group), and an insert only replaces ways stamped before its own launch.
//    Ways the launch inserts carry its stamp too, so within one launch the inserts of a set take min(c, 16) ways of c keys,
//    exactly, and give up on the rest.
//  * Duplicates are harmless.  An insert gives up when its key is READY in the set or a BUSY way has its fingerprint, but
//    two launches inserting one key at once can both pass that scan and take two ways.  Both hold the same table; a
//    lookup takes whichever it pins first, and the spare one ages out.  No verdict depends on a key being in one way.
//  * Counters are statistics only: hits + misses is every grouped valid key, resident counts EMPTY ways filled, an eviction
//    is a READY way replaced, a give-up is a valid miss that found no way it could take (every way BUSY with another key,
//    pinned, or used by this launch or a later one) or lost KCA_CLAIM_TRIES claims in a row.  An insert that stops because
//    its key is already there or being inserted counts as neither.
#pragma once
#include "key_cache.cuh"

namespace sbv {

constexpr unsigned long long KCA_PIN = 4;                // one pin, in the state word
constexpr unsigned long long KCA_PINS = 0xfffffffcull;   // the pin count's bits
constexpr int KCA_PIN_TRIES = 8, KCA_CLAIM_TRIES = KCA_WAYS + 1;
constexpr unsigned KCA_FULL = 0xffffffffu;

SBV_DEV unsigned long long kca_load_acquire(const unsigned long long *p) {
#if defined(__CUDA_ARCH__)
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
#else
    return *(const volatile unsigned long long *)p;
#endif
}
SBV_DEV void kca_store_release(unsigned long long *p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
    *(volatile unsigned long long *)p = v;
#endif
}

// the first way of key w's set, and its fingerprint in the state word's upper half
template <int W>
SBV_DEV uint32_t kca_base(const KcaMap &c, const uint32_t (&w)[W]) {
    return __umulhi(kc_hash<W>(w, c.seed), c.sets) * KCA_WAYS;
}
template <int W>
SBV_DEV unsigned long long kca_fp(const uint32_t (&w)[W], uint32_t seed) {
    return (unsigned long long)kc_hash<W>(w, seed ^ 0xa54ff53au) << 32;
}
template <int W>
SBV_DEV bool kca_same(const KcaMap &c, uint32_t way, const uint32_t (&w)[W]) {
    const uint32_t *s = c.keys + (size_t)way * W;
    uint32_t diff = 0;
#pragma unroll
    for (int k = 0; k < W; k++) diff |= kc_ld(s + k) ^ w[k];
    return diff == 0;
}
SBV_DEV unsigned long long kca_shfl_xor(unsigned long long v, int d) {
    const uint32_t src = (threadIdx.x & 31) ^ (uint32_t)d;
    const uint32_t lo = __shfl_sync(KCA_FULL, (uint32_t)v, (int)src), hi = __shfl_sync(KCA_FULL, (uint32_t)(v >> 32), (int)src);
    return (unsigned long long)hi << 32 | lo;
}

// Pins `way` if it is READY with fingerprint fp and holds key w: returns the way, else -1 (with no pin left behind).
template <int W>
SBV_DEV int32_t kca_pin(const KcaMap &c, uint32_t way, unsigned long long fp, const uint32_t (&w)[W]) {
    const unsigned long long ready = fp | KC_READY;
    unsigned long long s = kca_load_acquire(c.state + way);
    for (int t = 0; t < KCA_PIN_TRIES && (s & ~KCA_PINS) == ready; t++) {
        const unsigned long long o = atomicCAS(c.state + way, s, s + KCA_PIN);
        if (o != s) { s = o; continue; }  // another pin (retry from the new word) or a claim (the loop ends)
        __threadfence();                  // the key words and the table its READY store published
        if (kca_same<W>(c, way, w)) return (int32_t)way;
        atomicAdd(c.state + way, 0ull - KCA_PIN);  // refilled with another key of this fingerprint: a miss
        return -1;
    }
    return -1;
}

// One warp per grouped key k < min(*nkeys_ptr, kcap), key k = item keylist[k].  lk: the launch area, lk[0] = lk[1] = 0 on
// entry; on exit lk[0] = misses m, lk[1] = hits, lk[2 + id] = the item of key id.  now: the launch's stamp.
template <class KV>
__global__ void __launch_bounds__(128) k_kca_lookup(const uint32_t *__restrict__ nkeys_ptr, uint32_t kcap, const uint32_t *__restrict__ keylist, KV key,
                                                    KcaMap c, unsigned long long now, uint32_t tw4, int32_t *__restrict__ keyid,
                                                    uint32_t *__restrict__ lk, uint8_t *__restrict__ keyflags, uint4 *__restrict__ ktab) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nk = __ldg(nkeys_ptr);
    if (nk > kcap) nk = kcap;
    if (k >= nk) return;  // a warp leaves together
    const uint32_t item = keylist[k];
    uint32_t w[KV::W];
    key.load(item, w);
    const uint32_t base = kca_base<KV::W>(c, w);
    const unsigned long long fp = kca_fp<KV::W>(w, c.seed);
    const unsigned long long s = lane < KCA_WAYS ? kca_load_acquire(c.state + base + lane) : 0;
    unsigned cand = __ballot_sync(KCA_FULL, lane < KCA_WAYS && (s & ~KCA_PINS) == (fp | KC_READY));
    int32_t id = 0, way = -1;
    if (lane == 0) {
        for (; cand && way < 0; cand &= cand - 1) way = kca_pin<KV::W>(c, base + (uint32_t)(__ffs((int)cand) - 1), fp, w);
        if (way < 0) {
            id = (int32_t)atomicAdd(lk + 0, 1u);
        } else {
            id = (int32_t)(nk - 1 - atomicAdd(lk + 1, 1u));
            keyflags[id] = 1;
            atomicMax(c.stamp + way, now);
            atomicAdd(c.stats + 2, 1ull);
        }
        lk[2 + id] = item;
        keyid[item] = id;
    }
    way = __shfl_sync(KCA_FULL, way, 0);
    if (way < 0) return;
    id = __shfl_sync(KCA_FULL, id, 0);
    const uint4 *src = reinterpret_cast<const uint4 *>(c.pool) + (size_t)way * tw4;
    uint4 *dst = ktab + (size_t)id * tw4;
    for (uint32_t i = lane; i < tw4; i += 32) dst[i] = kc_ld(src + i);
    __syncwarp();  // every lane's loads, then lane 0's fence and unpin
    if (lane == 0) {
        __threadfence();
        atomicAdd(c.state + way, 0ull - KCA_PIN);
    }
}

// One warp per missed key k < lk[0] (after the build: ktab[k], keyflags[k]); invalid keys are never inserted.
template <class KV>
__global__ void __launch_bounds__(128) k_kca_insert(uint32_t kcap, const uint32_t *__restrict__ lk, KV key, KcaMap c, unsigned long long now,
                                                    uint32_t tw4, const uint8_t *__restrict__ keyflags, const uint4 *__restrict__ ktab) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t m = lk[0];
    if (m > kcap) m = kcap;
    if (k >= m || !keyflags[k]) return;  // a warp leaves together
    uint32_t w[KV::W];
    key.load(lk[2 + k], w);
    const uint32_t base = kca_base<KV::W>(c, w);
    const unsigned long long fp = kca_fp<KV::W>(w, c.seed);
    if (lane == 0) atomicAdd(c.stats + 3, 1ull);
    int32_t way = -1;
    bool evict = false, there = false;
    for (int t = 0; t < KCA_CLAIM_TRIES && way < 0 && !there; t++) {
        const unsigned long long s = lane < KCA_WAYS ? kca_load_acquire(c.state + base + lane) : 0;
        const uint32_t st = (uint32_t)s & 3u;
        const bool mine = lane < KCA_WAYS && (s >> 32) == (fp >> 32) && (st == KC_BUSY || (st == KC_READY && kca_same<KV::W>(c, base + lane, w)));
        if (__ballot_sync(KCA_FULL, mine)) { there = true; break; }  // resident, or being inserted by another launch
        const unsigned empty = __ballot_sync(KCA_FULL, lane < KCA_WAYS && s == 0);
        unsigned long long age = ~0ull;
        if (lane < KCA_WAYS && st == KC_READY && (s & KCA_PINS) == 0) {
            const unsigned long long a = kc_ld(c.stamp + base + lane);
            if (a < now) age = a;
        }
        unsigned long long lo = age;  // the least recent stamp of the set's replaceable ways
        for (int d = 16; d; d >>= 1) {
            const unsigned long long o = kca_shfl_xor(lo, d);
            lo = o < lo ? o : lo;
        }
        const unsigned pick = empty ? empty : __ballot_sync(KCA_FULL, age != ~0ull && age == lo);
        if (!pick) break;  // no way this key may take
        const int v = __ffs((int)pick) - 1;
        int won = 0;
        if ((int)lane == v && atomicCAS(c.state + base + lane, s, fp | KC_BUSY) == s) {
            won = 1;
            __threadfence();  // the unpin of the last reader before this warp's writes
        }
        if (__shfl_sync(KCA_FULL, won, v)) {
            way = (int32_t)(base + (uint32_t)v);
            evict = !empty;
        }
    }
    if (way < 0) {
        if (lane == 0 && !there) atomicAdd(c.stats + 5, 1ull);
        return;
    }
    __syncwarp();
    if (lane == 0) {
        c.stamp[way] = now;
        uint32_t *kw = c.keys + (size_t)way * KV::W;
#pragma unroll
        for (int i = 0; i < KV::W; i++) kw[i] = w[i];
    }
    const uint4 *src = ktab + (size_t)k * tw4;
    uint4 *dst = reinterpret_cast<uint4 *>(c.pool) + (size_t)way * tw4;
    for (uint32_t i = lane; i < tw4; i += 32) dst[i] = src[i];
    __threadfence();  // every lane's writes, then the warp barrier, then lane 0's release
    __syncwarp();
    if (lane == 0) {
        kca_store_release(c.state + way, fp | KC_READY);
        atomicAdd(c.stats + (evict ? 4 : 1), 1ull);
    }
}

}  // namespace sbv
