// key_cache.cuh — the opt-in cache of grouped-key tables across launches (sbv_key_cache_reserve).
//
// A keys-per-item launch builds a table for every key it groups (keygroup.cuh; ed25519_comb.cuh for Ed25519).  With a
// cache reserved, two kernels bracket that build and nothing else of the launch changes:
//
//   k_kc_lookup   on st, after k_kg_assign: one warp per grouped key.  Lane 0 looks the key up; the launch's key ids are
//                 renumbered so that the misses come first (ids [0, m), in the launch area's keylist, count lk[0]) and
//                 the hits last (ids [m, k)), keyid[] follows.  A hit's table is copied from the pool into its ktab slot
//                 (16-byte coherent loads, the warp's lanes side by side) and its key flag set.  The build kernels then
//                 run unchanged with count lk[0] and keylist lk + 2: they build exactly the missed tables, ktab[0, m).
//   k_kc_insert   on s_tab, after the build: one warp per missed key whose build flagged it valid.  It claims a map slot
//                 (EMPTY -> BUSY by CAS) and a pool entry, copies the table in and publishes READY with release
//                 semantics.
//
// Every table is a pure function of the key bytes, so where a table comes from changes nothing downstream: routing and the
// verify kernels read the same ktab / keyflags / item_kid as without a cache, and the verdicts are bit for bit the same.
//
// The map: open addressing over a power of two >= 2 x capacity slots, linear probing, keyed by the exact key bytes (a hash
// picks the first slot and a second one the fingerprint in the state word; a READY slot matches only when all its key
// words are equal).  A slot's state only moves EMPTY -> BUSY -> READY; nothing is ever removed, and sbv_key_cache_reserve
// empties the map with no launch in flight.  Nothing waits on another thread: a BUSY slot is passed or given up on.
//
// Why the races are harmless:
//  * No READY on an incomplete table.  READY is stored once per slot, by lane 0 of the one warp whose CAS took the slot,
//    after that warp wrote the key words, the pool index and the whole table (pool entry `at` comes from a counter, so no
//    other warp ever writes it) and fenced; the store is a release at GPU scope.  A reader loads the state with acquire
//    semantics before it reads the key, the index or the table, and reads them through L2 (ld.global.cg), never through the
//    non-coherent path.  A BUSY slot is never a hit.
//  * No claimed slot without a table forever while its key keeps missing.  A claim is followed, in the same warp and with
//    no wait on any other thread, by the pool claim and then the publication.  The one exception is a pool claim that
//    finds the pool exhausted: that slot stays BUSY, but with the pool full no key can get a table again until a reserve
//    empties the map, so no key stays missing because of that slot.
//  * At most one READY slot per key.  An insert claims only the first EMPTY slot of its key's probe sequence and gives up
//    at a BUSY slot of its fingerprint or a READY slot of its key.  States never go back to EMPTY, so two inserts of one
//    key (two launches at once) meet at the same first EMPTY slot: one wins the CAS, the other finds it BUSY or READY with
//    the same fingerprint and does not insert; that launch still verified with its own build, and the next launch hits.
//  * A lookup that stops at EMPTY misses nothing: an insert takes the first EMPTY slot of the probe sequence, and a slot
//    never becomes EMPTY again.
#pragma once
#include "keygroup.cuh"
#include "key_cache.h"

namespace sbv {

constexpr uint32_t KC_EMPTY = 0, KC_BUSY = 1, KC_READY = 2;  // EMPTY = 0: a memset empties the map

// Key views: the exact bytes of key `item` as W words.
template <class C>
struct KcXY {  // ECDSA: qx || qy
    static constexpr int W = 2 * C::N;
    const uint8_t *qx_be, *qy_be;
    SBV_DEV void load(uint32_t item, uint32_t (&w)[W]) const {
        const uint32_t *x = reinterpret_cast<const uint32_t *>(qx_be + (size_t)item * C::BYTES);
        const uint32_t *y = reinterpret_cast<const uint32_t *>(qy_be + (size_t)item * C::BYTES);
#pragma unroll
        for (int k = 0; k < C::N; k++) { w[k] = __ldg(x + k); w[C::N + k] = __ldg(y + k); }
    }
};
struct KcKey32 {  // Ed25519: the 32-byte encoding
    static constexpr int W = 8;
    const uint8_t *pub;
    SBV_DEV void load(uint32_t item, uint32_t (&w)[W]) const {
        const uint32_t *x = reinterpret_cast<const uint32_t *>(pub + (size_t)item * 32);
#pragma unroll
        for (int k = 0; k < W; k++) w[k] = __ldg(x + k);
    }
};

SBV_DEV uint32_t kc_load_acquire(const uint32_t *p) {
#if defined(__CUDA_ARCH__)
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#else
    return *(const volatile uint32_t *)p;
#endif
}
SBV_DEV void kc_store_release(uint32_t *p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#else
    *(volatile uint32_t *)p = v;
#endif
}
// coherent loads (L2): data another kernel published while this one may be running
template <class T>
SBV_DEV T kc_ld(const T *p) {
#if defined(__CUDA_ARCH__)
    return __ldcg(p);
#else
    return *p;
#endif
}

template <int W>
SBV_DEV uint32_t kc_hash(const uint32_t (&w)[W], uint32_t seed) {
    uint32_t h = seed;
#pragma unroll
    for (int k = 0; k < W; k++) h = kg_mix(h, w[k]);
    return h ^ (h >> 16);
}
template <int W>
SBV_DEV bool kc_same(const KcMap &c, uint32_t slot, const uint32_t (&w)[W]) {
    const uint32_t *s = c.keys + (size_t)slot * W;
    uint32_t diff = 0;
#pragma unroll
    for (int k = 0; k < W; k++) diff |= kc_ld(s + k) ^ w[k];
    return diff == 0;
}

// The state word of a slot: KC_EMPTY, or KC_BUSY / KC_READY in the low two bits with a 30-bit fingerprint of the key
// above them (a second hash), set by the claim.  An insert that meets a BUSY slot of another fingerprint knows the slot
// holds another key and probes on; one of the same fingerprint gives up (the same key, being inserted by another launch, or
// rarely another key: that one is inserted by a later launch, once the slot is READY and its key can be compared).
template <int W>
SBV_DEV uint32_t kc_fp(const uint32_t (&w)[W], uint32_t seed) {
    return kc_hash<W>(w, seed ^ 0x3c6ef372u) << 2;
}

// the READY slot of key w, or -1
template <int W>
SBV_DEV int32_t kc_find(const KcMap &c, const uint32_t (&w)[W]) {
    const uint32_t ready = kc_fp<W>(w, c.seed) | KC_READY;
    uint32_t h = kc_hash<W>(w, c.seed) & c.smask;
    for (uint32_t p = 0; p <= c.smask; p++, h = (h + 1) & c.smask) {
        const uint32_t s = kc_load_acquire(c.state + h);
        if (s == KC_EMPTY) return -1;
        if (s == ready && kc_same<W>(c, h, w)) return (int32_t)h;
    }
    return -1;
}

// a slot claimed for key w (EMPTY -> BUSY), or -1: the pool is full, the key is being or has been inserted, an insert of
// a key of the same fingerprint is in progress on the probe sequence, or the map is full
template <int W>
SBV_DEV int32_t kc_claim(const KcMap &c, const uint32_t (&w)[W]) {
    if (*(const volatile unsigned long long *)c.stats >= c.cap) return -1;
    const uint32_t fp = kc_fp<W>(w, c.seed);
    uint32_t h = kc_hash<W>(w, c.seed) & c.smask;
    for (uint32_t p = 0; p <= c.smask; p++, h = (h + 1) & c.smask) {
        uint32_t s = kc_load_acquire(c.state + h);
        if (s == KC_EMPTY) {
            if (atomicCAS(c.state + h, KC_EMPTY, fp | KC_BUSY) == KC_EMPTY) return (int32_t)h;
            s = kc_load_acquire(c.state + h);  // BUSY or READY now
        }
        if ((s & ~3u) != fp) continue;
        if ((s & 3u) == KC_BUSY) return -1;
        if (kc_same<W>(c, h, w)) return -1;
    }
    return -1;
}

// One warp per grouped key k < min(*nkeys_ptr, kcap), key k = item keylist[k].  lk: the launch area, lk[0] = lk[1] = 0 on
// entry; on exit lk[0] = misses m, lk[1] = hits, lk[2 + id] = the item of key id.  tw4: 16-byte words per table.
template <class KV>
__global__ void __launch_bounds__(128) k_kc_lookup(const uint32_t *__restrict__ nkeys_ptr, uint32_t kcap, const uint32_t *__restrict__ keylist, KV key,
                                                   KcMap c, uint32_t tw4, int32_t *__restrict__ keyid, uint32_t *__restrict__ lk,
                                                   uint8_t *__restrict__ keyflags, uint4 *__restrict__ ktab) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nk = __ldg(nkeys_ptr);
    if (nk > kcap) nk = kcap;
    if (k >= nk) return;  // a warp leaves together
    int32_t id = 0, at = -1;
    if (lane == 0) {
        const uint32_t item = keylist[k];
        uint32_t w[KV::W];
        key.load(item, w);
        const int32_t slot = kc_find<KV::W>(c, w);
        if (slot < 0) {
            id = (int32_t)atomicAdd(lk + 0, 1u);
        } else {
            id = (int32_t)(nk - 1 - atomicAdd(lk + 1, 1u));
            at = (int32_t)kc_ld(c.pidx + slot);
            keyflags[id] = 1;
            atomicAdd(c.stats + 2, 1ull);
        }
        lk[2 + id] = item;
        keyid[item] = id;
    }
    at = __shfl_sync(0xffffffffu, at, 0);
    if (at < 0) return;
    id = __shfl_sync(0xffffffffu, id, 0);
    const uint4 *src = reinterpret_cast<const uint4 *>(c.pool) + (size_t)at * tw4;
    uint4 *dst = ktab + (size_t)id * tw4;
    for (uint32_t i = lane; i < tw4; i += 32) dst[i] = kc_ld(src + i);
}

// One warp per missed key k < lk[0] (after the build: ktab[k], keyflags[k]); invalid keys are never inserted.
template <class KV>
__global__ void __launch_bounds__(128) k_kc_insert(uint32_t kcap, const uint32_t *__restrict__ lk, KV key, KcMap c, uint32_t tw4,
                                                   const uint8_t *__restrict__ keyflags, const uint4 *__restrict__ ktab) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t m = lk[0];
    if (m > kcap) m = kcap;
    if (k >= m || !keyflags[k]) return;  // a warp leaves together
    int32_t slot = -1, at = 0;
    uint32_t w[KV::W];
    if (lane == 0) {
        atomicAdd(c.stats + 3, 1ull);
        key.load(lk[2 + k], w);
        slot = kc_claim<KV::W>(c, w);
        if (slot >= 0) {
            const unsigned long long t = atomicAdd(c.stats + 0, 1ull);
            if (t < c.cap) {
                at = (int32_t)t;
                uint32_t *kw = c.keys + (size_t)slot * KV::W;
#pragma unroll
                for (int i = 0; i < KV::W; i++) kw[i] = w[i];
                c.pidx[slot] = (uint32_t)at;
            } else {
                slot = -1;  // the pool is full: the slot stays BUSY (see the header)
            }
        }
    }
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (slot < 0) return;
    at = __shfl_sync(0xffffffffu, at, 0);
    const uint4 *src = ktab + (size_t)k * tw4;
    uint4 *dst = reinterpret_cast<uint4 *>(c.pool) + (size_t)at * tw4;
    for (uint32_t i = lane; i < tw4; i += 32) dst[i] = src[i];
    __threadfence();  // every lane's writes, then the warp barrier, then lane 0's release
    __syncwarp();
    if (lane == 0) {
        kc_store_release(c.state + slot, kc_fp<KV::W>(w, c.seed) | KC_READY);
        atomicAdd(c.stats + 1, 1ull);
    }
}

}  // namespace sbv
