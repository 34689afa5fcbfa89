// mixed.cuh — the split of a mixed ECDSA / Ed25519 shard into its three families (P-256, P-384, Ed25519) and the
// scatter of the family verdicts back into item order (sbv_mixed_verify_registered, sbv_mixed_verify_quorum,
// sbv_mixed_verify_batch).
//
// A shard is uploaded as the caller holds it: a scheme tag, a slot or a 96-byte key row, a 96-byte signature row and a
// message per item.  The split is a stable partition done in tiles of MIX_TILE consecutive items, one thread per tile:
//   k_mix_count    per tile and family: the item count and the message bytes;
//   k_mix_scan     one block: the exclusive prefixes of both over the tiles, per family, and where each family's messages
//                  start in the shared message buffer;
//   k_mix_split    per tile, in item order: each item's index, slot, signature (r and s arrays of width L for ECDSA,
//                  64-byte R || S rows for Ed25519) and message offset, at the item's rank inside its family; with
//                  KEYS, the key row instead of the slot (qx and qy arrays of width L for ECDSA, 32-byte rows for
//                  Ed25519);
//   k_mix_compact  MIX_LANES threads per item copy its message bytes to the family's region of the shared buffer, 16
//                  aligned bytes per store (byte stores only where a 16-byte word is shared with a neighbour);
//   k_mix_ok       after the family pipelines: ok[idx_f[j]] = ok_f[j].
// The family regions of the message buffer start 16-byte aligned and each is followed by at least 16 bytes of slack, so
// k_sha256 and k_ed_sha512 read them as they read a staged blob (aligned 32-bit loads, 8 bytes past the last message).
// Offsets are positions in the shared buffer, so the hash kernels take base 0.
#pragma once
#include <stdint.h>

namespace sbv {

constexpr int MIX_FAMILIES = 3;   // 0 = P-256, 1 = P-384, 2 = Ed25519 (the scheme tags of sbv.h)
constexpr uint32_t MIX_TILE = 16;  // items per thread of k_mix_count / k_mix_split
constexpr int MIX_SCAN_THREADS = 1024;
constexpr uint32_t MIX_LANES = 8;  // threads per item of k_mix_compact: 128 bytes per pass

// The compacted arrays of one family: items [0, m) in the order they have in the shard.
struct MixFamily {
    uint32_t *idx;   // item index inside the shard
    uint32_t *slot;  // registry slot
    uint8_t *r, *s;  // ECDSA: r and s, L bytes each; Ed25519: r = 64-byte R || S rows, s unused
    uint64_t *off;   // m + 1 message offsets into the shared buffer
    uint8_t *ok;     // verdicts of the family pipeline
};
struct MixPlan {
    MixFamily f[MIX_FAMILIES];
    uint8_t *blob;   // the shared message buffer
};
// The compacted keys of a keys-per-item shard, in the order of MixFamily: a separate parameter, so that the plan, and
// with it every kernel of a registered shard, stays as it is.
struct MixKeys {
    uint8_t *qx[2], *qy[2];  // P-256 (32 bytes each), P-384 (48 bytes each)
    uint8_t *pub;            // Ed25519: 32-byte encodings
};

__device__ __forceinline__ uint64_t mix_align16(uint64_t x) { return (x + 15) & ~(uint64_t)15; }
// selects instead of a dynamic index into the parameter block, which would copy it to local memory
__device__ __forceinline__ MixFamily mix_family(const MixPlan &p, uint32_t f) { return f == 0 ? p.f[0] : f == 1 ? p.f[1] : p.f[2]; }

__global__ void __launch_bounds__(256) k_mix_count(uint32_t n, const uint8_t *__restrict__ tag, const uint64_t *__restrict__ off,
                                                   uint32_t ntiles, uint32_t *__restrict__ tile_cnt, uint64_t *__restrict__ tile_bytes) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    uint32_t c[MIX_FAMILIES] = {0, 0, 0};
    uint64_t b[MIX_FAMILIES] = {0, 0, 0};
    const uint32_t lo = t * MIX_TILE, hi = n - lo < MIX_TILE ? n : lo + MIX_TILE;
    for (uint32_t i = lo; i < hi; i++) {
        const uint32_t f = tag[i];
        const uint64_t len = off[i + 1] - off[i];
#pragma unroll
        for (int k = 0; k < MIX_FAMILIES; k++) {
            c[k] += f == (uint32_t)k ? 1u : 0u;
            b[k] += f == (uint32_t)k ? len : 0u;
        }
    }
#pragma unroll
    for (int k = 0; k < MIX_FAMILIES; k++) {
        tile_cnt[(size_t)k * ntiles + t] = c[k];
        tile_bytes[(size_t)k * ntiles + t] = b[k];
    }
}

// One block.  Thread t owns a contiguous run of tiles: it sums them, the block scans the sums (Hillis-Steele in shared
// memory), and the thread rewrites its tiles with exclusive prefixes; the byte prefixes include the family's start in the
// shared buffer.  Thread 0 closes every family's offsets with off_f[m_f] = its end.  Correct for any blockDim.x <=
// MIX_SCAN_THREADS.
__global__ void __launch_bounds__(MIX_SCAN_THREADS) k_mix_scan(uint32_t ntiles, uint32_t *__restrict__ tile_cnt, uint64_t *__restrict__ tile_bytes,
                                                               MixPlan p) {
    __shared__ uint32_t sc[MIX_FAMILIES][MIX_SCAN_THREADS];
    __shared__ uint64_t sb[MIX_FAMILIES][MIX_SCAN_THREADS];
    const uint32_t T = blockDim.x, tid = threadIdx.x;
    const uint32_t per = (ntiles + T - 1) / T, lo = tid * per < ntiles ? tid * per : ntiles, hi = ntiles - lo < per ? ntiles : lo + per;
    uint32_t c[MIX_FAMILIES] = {0, 0, 0};
    uint64_t b[MIX_FAMILIES] = {0, 0, 0};
    for (uint32_t t = lo; t < hi; t++)
#pragma unroll
        for (int k = 0; k < MIX_FAMILIES; k++) {
            c[k] += tile_cnt[(size_t)k * ntiles + t];
            b[k] += tile_bytes[(size_t)k * ntiles + t];
        }
#pragma unroll
    for (int k = 0; k < MIX_FAMILIES; k++) { sc[k][tid] = c[k]; sb[k][tid] = b[k]; }
    __syncthreads();
    for (uint32_t d = 1; d < T; d <<= 1) {
        uint32_t vc[MIX_FAMILIES] = {0, 0, 0};
        uint64_t vb[MIX_FAMILIES] = {0, 0, 0};
        if (tid >= d)
#pragma unroll
            for (int k = 0; k < MIX_FAMILIES; k++) { vc[k] = sc[k][tid - d]; vb[k] = sb[k][tid - d]; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < MIX_FAMILIES; k++) { sc[k][tid] += vc[k]; sb[k][tid] += vb[k]; }
        __syncthreads();
    }
    uint64_t start[MIX_FAMILIES];
    start[0] = 0;
    start[1] = mix_align16(sb[0][T - 1] + 16);
    start[2] = start[1] + mix_align16(sb[1][T - 1] + 16);
#pragma unroll
    for (int k = 0; k < MIX_FAMILIES; k++) {
        uint32_t rc = sc[k][tid] - c[k];
        uint64_t rb = start[k] + sb[k][tid] - b[k];
        for (uint32_t t = lo; t < hi; t++) {
            const uint32_t tc = tile_cnt[(size_t)k * ntiles + t];
            const uint64_t tb = tile_bytes[(size_t)k * ntiles + t];
            tile_cnt[(size_t)k * ntiles + t] = rc;
            tile_bytes[(size_t)k * ntiles + t] = rb;
            rc += tc;
            rb += tb;
        }
        if (tid == 0) p.f[k].off[sc[k][T - 1]] = start[k] + sb[k][T - 1];
    }
}

__device__ __forceinline__ void mix_copy16(uint8_t *dst, const uint8_t *src, int words16) {
    for (int w = 0; w < words16; w++) reinterpret_cast<uint4 *>(dst)[w] = __ldg(reinterpret_cast<const uint4 *>(src) + w);
}

// KEYS: the shard carries a 96-byte key row per item (key96, packed as sig96 is) instead of a slot; the registered
// instantiation never reads key96 or k.
template <bool KEYS = false>
__global__ void __launch_bounds__(256) k_mix_split(uint32_t n, const uint8_t *__restrict__ tag, const uint32_t *__restrict__ slot,
                                                   const uint8_t *__restrict__ sig96, const uint64_t *__restrict__ off, uint32_t ntiles,
                                                   const uint32_t *__restrict__ tile_cnt, const uint64_t *__restrict__ tile_bytes, MixPlan p,
                                                   const uint8_t *__restrict__ key96 = nullptr, MixKeys k = MixKeys{}) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    uint32_t rank[MIX_FAMILIES];
    uint64_t pos[MIX_FAMILIES];
#pragma unroll
    for (int k = 0; k < MIX_FAMILIES; k++) { rank[k] = tile_cnt[(size_t)k * ntiles + t]; pos[k] = tile_bytes[(size_t)k * ntiles + t]; }
    const uint32_t lo = t * MIX_TILE, hi = n - lo < MIX_TILE ? n : lo + MIX_TILE;
    for (uint32_t i = lo; i < hi; i++) {
        const uint32_t f = tag[i];
        const MixFamily F = mix_family(p, f);
        const uint32_t j = f == 0 ? rank[0] : f == 1 ? rank[1] : rank[2];
        const uint64_t at = f == 0 ? pos[0] : f == 1 ? pos[1] : pos[2];
        const uint64_t len = off[i + 1] - off[i];
#pragma unroll
        for (int k = 0; k < MIX_FAMILIES; k++)
            if (f == (uint32_t)k) { rank[k]++; pos[k] += len; }
        F.idx[j] = i;
        if constexpr (!KEYS) F.slot[j] = slot[i];
        F.off[j] = at;
        const uint8_t *row = sig96 + (size_t)i * 96;
        if (f == 0) {
            mix_copy16(F.r + (size_t)j * 32, row, 2);
            mix_copy16(F.s + (size_t)j * 32, row + 32, 2);
            if constexpr (KEYS) mix_copy16(k.qx[0] + (size_t)j * 32, key96 + (size_t)i * 96, 2);
            if constexpr (KEYS) mix_copy16(k.qy[0] + (size_t)j * 32, key96 + (size_t)i * 96 + 32, 2);
        } else if (f == 1) {
            mix_copy16(F.r + (size_t)j * 48, row, 3);
            mix_copy16(F.s + (size_t)j * 48, row + 48, 3);
            if constexpr (KEYS) mix_copy16(k.qx[1] + (size_t)j * 48, key96 + (size_t)i * 96, 3);
            if constexpr (KEYS) mix_copy16(k.qy[1] + (size_t)j * 48, key96 + (size_t)i * 96 + 48, 3);
        } else {
            mix_copy16(F.r + (size_t)j * 64, row, 4);
            if constexpr (KEYS) mix_copy16(k.pub + (size_t)j * 32, key96 + (size_t)i * 96, 2);
        }
    }
}

// Item g of the compacted order (family 0's m0 items, then family 1's m1, then family 2's) is copied by MIX_LANES threads;
// thread l writes the 16-byte words l, l + MIX_LANES, ... of the item's destination range.  A word wholly inside the item
// is assembled from aligned 32-bit loads of the source (PRMT) and stored as one uint4; the first and last words, which
// the neighbouring items may share, are written byte by byte.  src: the staged shard, whose offsets start at base.
__global__ void __launch_bounds__(256) k_mix_compact(uint32_t n, uint32_t m0, uint32_t m1, const uint8_t *__restrict__ src,
                                                     const uint64_t *__restrict__ off, uint64_t base, MixPlan p) {
    const uint64_t tix = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t g = (uint32_t)(tix / MIX_LANES), lane = (uint32_t)(tix % MIX_LANES);
    if (g >= n) return;
    const uint32_t f = g < m0 ? 0 : g < m0 + m1 ? 1 : 2, j = g - (f == 0 ? 0 : f == 1 ? m0 : m0 + m1);
    const MixFamily F = mix_family(p, f);
    const uint32_t i = F.idx[j];
    const uint64_t s = off[i] - base, len = off[i + 1] - off[i], d = F.off[j];
    if (len == 0) return;
    const uint64_t w0 = d >> 4, w1 = (d + len - 1) >> 4;
    for (uint64_t w = w0 + lane; w <= w1; w += MIX_LANES) {
        const uint64_t lo = w << 4;
        uint8_t *out = p.blob + lo;
        if (lo >= d && lo + 16 <= d + len) {
            const uint64_t sp = lo - d + s;
            const uint32_t *words = reinterpret_cast<const uint32_t *>(src + (sp & ~(uint64_t)3));
            const uint32_t sh = (uint32_t)(sp & 3), sel = sh | ((sh + 1) << 4) | ((sh + 2) << 8) | ((sh + 3) << 12);
            uint32_t v[5];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = __ldg(words + k);
            v[4] = sh ? __ldg(words + 4) : 0u;
            *reinterpret_cast<uint4 *>(out) = make_uint4(__byte_perm(v[0], v[1], sel), __byte_perm(v[1], v[2], sel), __byte_perm(v[2], v[3], sel),
                                                         __byte_perm(v[3], v[4], sel));
        } else {
            const uint64_t a = lo > d ? lo : d, b = lo + 16 < d + len ? lo + 16 : d + len;
            for (uint64_t q = a; q < b; q++) p.blob[q] = src[q - d + s];
        }
    }
}

// verdicts of the compacted order back to item order
__global__ void __launch_bounds__(256) k_mix_ok(uint32_t n, uint32_t m0, uint32_t m1, MixPlan p, uint8_t *__restrict__ ok) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const uint32_t f = g < m0 ? 0 : g < m0 + m1 ? 1 : 2, j = g - (f == 0 ? 0 : f == 1 ? m0 : m0 + m1);
    const MixFamily F = mix_family(p, f);
    ok[F.idx[j]] = F.ok[j];
}

}  // namespace sbv
