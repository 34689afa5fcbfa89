// ops.h — per-curve kernel launchers behind plain function pointers, so that the host pipeline (pipeline.cu) is
// written once and the heavy kernel templates are compiled in parallel, one translation unit per group
// (inst_<curve>_{prep,coz,comb|kt5,kt8}.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

struct KtGeom {  // words per key of a per-key table and of its construction scratch
    size_t bases_words, hs_words, ztop_words, ktab_words;
};

struct KtOps {
    KtGeom geom;
    // the table-construction kernels, enqueued back to back on st
    cudaError_t (*build)(const uint32_t *nkeys_ptr, uint32_t cap, const uint32_t *keylist, const uint8_t *qx, const uint8_t *qy,
                         uint32_t *bases, uint32_t *hs, uint32_t *ztop, uint32_t *pref, uint32_t *ktab, uint8_t *keyflags, cudaStream_t st);
    // fixed-base verification; reg: keys by slot (registered) or by item (grouped); warp: one signature per warp
    // (registered only)
    cudaError_t (*verify)(int reg, int warp, uint32_t n, const uint32_t *slot, const int32_t *kidmap, uint32_t n_slots,
                          const uint8_t *keyflags, const uint8_t *r, const uint32_t *uw, const uint8_t *flags, const uint32_t *gtab,
                          const uint32_t *ktab, uint8_t *ok, const uint32_t *list, const uint32_t *count, const uint32_t *gacc, cudaStream_t st);
};

struct CurveOps {
    int N, bytes;
    size_t gtab_entries;
    cudaError_t (*gtable_init)(uint32_t *gtab, cudaStream_t st);
    cudaError_t (*prep)(uint32_t n, const uint8_t *r, const uint8_t *s, const uint8_t *dig, uint32_t dlen, uint32_t *uw, uint8_t *flags,
                        cudaStream_t st);
    // key grouping: insert + assign (+ route when `route`: three launches); buffers zeroed / 0xff-filled by the caller
    cudaError_t (*group)(uint32_t n, const uint8_t *qx, const uint8_t *qy, uint32_t seed, uint32_t hmask, uint32_t *htab, uint32_t *rep,
                         uint32_t *kcnt, uint32_t threshold, uint32_t max_keys, int32_t *keyid, uint32_t *keylist, int32_t *item_kid,
                         uint32_t *klist, uint32_t *glist, uint32_t *counters, int route, cudaStream_t st);
    // the routing step alone, for a range of items (chunked launches route chunk by chunk: rep / item_kid / klist / glist
    // point at the chunk, the indices written to the lists are chunk-local, counters are the chunk's own)
    cudaError_t (*route)(uint32_t n, const uint32_t *rep, const int32_t *keyid, int32_t *item_kid, uint32_t *klist, uint32_t *glist,
                         uint32_t *counters, cudaStream_t st);
    // u1*G of every item into gacc[3N][n] (the half of the fixed-base verification that does not need the key tables)
    cudaError_t (*gpart)(uint32_t n, const uint32_t *uw, const uint32_t *gtab, uint32_t *gacc, cudaStream_t st);
    cudaError_t (*coz)(uint32_t n, const uint8_t *qx, const uint8_t *qy, const uint8_t *r, const uint32_t *uw, const uint8_t *flags,
                       const uint32_t *gtab, uint32_t *tscr, uint8_t *ok, const uint32_t *list, const uint32_t *count, cudaStream_t st);
    // keys grouped inside a launch (P-256: comb tables; P-384: 5-bit window tables) / registered keys (8-bit windows)
    const KtOps *grouped, *kt8;
};

#define SBV_COZ_DECL(NAME)                                                                                                          \
    cudaError_t NAME(uint32_t n, const uint8_t *qx, const uint8_t *qy, const uint8_t *r, const uint32_t *uw, const uint8_t *flags, \
                     const uint32_t *gtab, uint32_t *tscr, uint8_t *ok, const uint32_t *list, const uint32_t *count, cudaStream_t st)
SBV_COZ_DECL(sbv_coz_p256);
SBV_COZ_DECL(sbv_coz_p384);
extern const CurveOps sbv_ops_p256, sbv_ops_p384;
extern const KtOps sbv_comb_p256, sbv_kt8_p256, sbv_kt5_p384, sbv_kt8_p384;
inline const CurveOps &sbv_ops(int curve) { return curve == 0 ? sbv_ops_p256 : sbv_ops_p384; }
