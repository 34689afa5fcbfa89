// key_cache.h — the device view of one family's key cache on one device (sbv_key_cache_reserve; kernels in key_cache.cuh).
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
