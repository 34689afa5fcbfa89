// ops.h — per-curve kernel launchers behind plain function pointers, so that the host pipeline (pipeline.cu) is
// written once and the heavy kernel templates are compiled in parallel, one translation unit per group
// (inst_<curve>_{prep,coz,comb|kt5,kt8}.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "key_cache.h"

struct KtGeom {  // words per key of a per-key table and of its construction scratch
    size_t bases_words, hs_words, ztop_words, ktab_words;
};

struct KtOps {  // one kind of per-key table: its geometry and its construction kernels, enqueued back to back on st
    KtGeom geom;
    cudaError_t (*build)(const uint32_t *nkeys_ptr, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy,
                         uint32_t *bases, uint32_t *hs, uint32_t *ztop, uint32_t *pref, uint32_t *ktab, uint8_t *keyflags, cudaStream_t st);
};
// Tables of the keys grouped inside a launch.  Fixed-base verification of items list[0 .. *count): the key of item i is
// kidmap[i], and gacc holds u1*G of every item (gpart).
struct GroupedKtOps : KtOps {
    cudaError_t (*verify)(uint32_t n, const int32_t *kidmap, const uint8_t *keyflags, const uint8_t *r, const uint32_t *uw, const uint8_t *flags,
                          const uint32_t *gtab, const uint32_t *ktab, uint8_t *ok, const uint32_t *list, const uint32_t *count, const uint32_t *gacc,
                          cudaStream_t st);
};
// Tables of the registered keys (sbv_set_keys).  Fixed-base verification of every item: the key of item i is
// slot2local[slot[i]]; warp: one signature per warp.
struct RegisteredKtOps : KtOps {
    cudaError_t (*verify)(uint32_t n, const uint32_t *slot, const int32_t *slot2local, uint32_t n_slots, const uint8_t *keyflags, const uint8_t *r,
                          const uint32_t *uw, const uint8_t *flags, const uint32_t *gtab, const uint32_t *ktab, uint8_t *ok, int warp, cudaStream_t st);
};

struct CurveOps {
    int N, bytes;
    size_t gtab_entries;
    cudaError_t (*gtable_init)(uint32_t *gtab, cudaStream_t st);
    cudaError_t (*prep)(uint32_t n, const uint8_t *r, const uint8_t *s, const uint8_t *dig, uint32_t dlen, uint32_t *uw, uint8_t *flags,
                        cudaStream_t st);
    // routing of a range of items onto the fixed-base and the generic list (launches route chunk by chunk: rep / item_kid /
    // klist / glist point at the chunk, the indices written to the lists are chunk-local, counters are the chunk's own)
    cudaError_t (*route)(uint32_t n, const uint32_t *rep, const int32_t *keyid, int32_t *item_kid, uint32_t *klist, uint32_t *glist,
                         uint32_t *counters, cudaStream_t st);
    // u1*G of every item into gacc[3N][n] (the half of the fixed-base verification that does not need the key tables)
    cudaError_t (*gpart)(uint32_t n, const uint32_t *uw, const uint32_t *gtab, uint32_t *gacc, cudaStream_t st);
    cudaError_t (*coz)(uint32_t n, const uint8_t *qx, const uint8_t *qy, const uint8_t *r, const uint32_t *uw, const uint8_t *flags,
                       const uint32_t *gtab, uint32_t *tscr, uint8_t *ok, const uint32_t *list, const uint32_t *count, cudaStream_t st);
    // keys grouped inside a launch (P-256: comb tables; P-384: 5-bit window tables) / registered keys (8-bit windows)
    const GroupedKtOps *grouped;
    const RegisteredKtOps *kt8;
};

// The first half of a keys-per-item launch of one scheme (pipeline.cu: sbv_launch_verify_begin): the grouping of the
// repeated keys, the key cache and the tables of the grouped keys.  A key comes in as (qx, qy) for ECDSA and as (the
// 32-byte encoding, nullptr) for Ed25519.
struct GroupOps {
    const KtOps *kt;      // the geometry and the construction of the tables (P-256: comb; P-384: 5-bit windows; Ed25519: comb)
    size_t key_words;     // 32-bit words of a key as the cache stores and compares it
    int build_launches;   // kernels kt->build enqueues
    // insert + assign (two launches); buffers zeroed / 0xff-filled by the caller
    cudaError_t (*group)(uint32_t n, const uint8_t *qx, const uint8_t *qy, uint32_t seed, uint32_t hmask, uint32_t *htab, uint32_t *rep,
                         uint32_t *kcnt, uint32_t threshold, uint32_t max_keys, int32_t *keyid, uint32_t *keylist, uint32_t *counters, cudaStream_t st);
    // the key cache (key_cache.cuh): k_kc_lookup after the grouping, k_kc_insert after the table construction; tw4 = 16-byte
    // words per table
    cudaError_t (*cache_lookup)(const uint32_t *nkeys_ptr, uint32_t kcap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy, KcMap c,
                                uint32_t tw4, int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab, cudaStream_t st);
    cudaError_t (*cache_insert)(uint32_t kcap, const uint32_t *lk, const uint8_t *qx, const uint8_t *qy, KcMap c, uint32_t tw4, const uint8_t *keyflags,
                                const uint32_t *ktab, cudaStream_t st);
    // the evicting cache (key_cache_assoc.cuh): k_kca_lookup / k_kca_insert in the same places; now = the launch's stamp
    cudaError_t (*evict_lookup)(const uint32_t *nkeys_ptr, uint32_t kcap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy, KcaMap c,
                                unsigned long long now, uint32_t tw4, int32_t *keyid, uint32_t *lk, uint8_t *keyflags, uint32_t *ktab, cudaStream_t st);
    cudaError_t (*evict_insert)(uint32_t kcap, const uint32_t *lk, const uint8_t *qx, const uint8_t *qy, KcaMap c, unsigned long long now, uint32_t tw4,
                                const uint8_t *keyflags, const uint32_t *ktab, cudaStream_t st);
};

#define SBV_COZ_DECL(NAME)                                                                                                          \
    cudaError_t NAME(uint32_t n, const uint8_t *qx, const uint8_t *qy, const uint8_t *r, const uint32_t *uw, const uint8_t *flags, \
                     const uint32_t *gtab, uint32_t *tscr, uint8_t *ok, const uint32_t *list, const uint32_t *count, cudaStream_t st)
SBV_COZ_DECL(sbv_coz_p256);
SBV_COZ_DECL(sbv_coz_p384);
extern const CurveOps sbv_ops_p256, sbv_ops_p384;
extern const GroupedKtOps sbv_comb_p256, sbv_kt5_p384;
extern const RegisteredKtOps sbv_kt8_p256, sbv_kt8_p384;
inline const CurveOps &sbv_ops(int curve) { return curve == 0 ? sbv_ops_p256 : sbv_ops_p384; }
extern const GroupOps sbv_group_p256, sbv_group_p384, sbv_group_ed25519;
// by scheme tag: SBV_P256, SBV_P384, SBV_ED25519
inline const GroupOps &sbv_group_ops(int scheme) { return scheme == 0 ? sbv_group_p256 : scheme == 1 ? sbv_group_p384 : sbv_group_ed25519; }
