// key_cache.h — the device view of one family's key cache on one device (sbv_key_cache_reserve; kernels in key_cache.cuh;
// the evicting mode of sbv_key_cache_reserve_evicting: key_cache_assoc.cuh).
// Plain pointers only, so that the host code, ops.h and the CPU simulation share it.
#pragma once
#include <stdint.h>

struct KcMap {
    uint32_t *state;            // [smask + 1] KC_EMPTY / KC_BUSY / KC_READY
    uint32_t *keys;             // [smask + 1][key words] the key of a READY slot
    uint32_t *pidx;             // [smask + 1] pool index of a READY slot
    uint32_t *pool;             // [cap][table words]
    unsigned long long *stats;  // [0] pool entries claimed, [1] resident tables, [2] hits, [3] misses
    uint32_t smask, cap, seed;  // slots - 1 (slots: a power of two >= 2 * cap), pool entries, hash seed
};

// Ways per set of the evicting cache: a set's state words are one ballot of half a warp (and one 128-byte line), and a
// key competes with 15 others for its set, close enough to a fully associative LRU for a cache of a few hundred keys up.
constexpr uint32_t KCA_WAYS = 16;

// The evicting cache: sets * KCA_WAYS ways; way i is pool entry i.
struct KcaMap {
    unsigned long long *state;  // [ways] fingerprint << 32 | pins << 2 | KC_EMPTY / KC_BUSY / KC_READY (0: EMPTY)
    unsigned long long *stamp;  // [ways] launch sequence number of the way's last hit or insert
    uint32_t *keys;             // [ways][key words] the key of a READY way
    uint32_t *pool;             // [ways][table words]
    unsigned long long *stats;  // [0] unused, [1] resident tables, [2] hits, [3] misses, [4] evictions, [5] inserts given up
    uint32_t sets, seed;
};
