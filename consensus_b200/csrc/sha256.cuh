// sha256.cuh — SHA-256 over a ragged batch, one message per thread (FIPS 180-4).
//
// Replaces the reference's crypto/sha256 call sites on the verification path:
// /root/reference/pkg/types/types.go:64-69 (computeDigest), internal/bft/util.go:583-585.
// Messages are concatenated in one device buffer with byte offsets off[n+1]; a thread walks its
// message with ALIGNED 32-bit loads and re-aligns with PRMT (byte_perm), so arbitrary byte
// offsets cost no byte loads.  The buffer must be readable 8 bytes past the last message.
#pragma once
#include <stdint.h>

#include "sha256_core.cuh"

namespace sbv {

// The SHA-256 state h after message idx of the batch (offsets off relative to base): the per-message body of k_sha256,
// shared with k_sha2_sel (mixed_hash.cuh).
__device__ __forceinline__ void sha256_msg(uint32_t (&h)[8], const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                           uint32_t idx) {
    const uint64_t o = off[idx] - base;
    const uint64_t len = off[idx + 1] - off[idx];
    const uint32_t *words = reinterpret_cast<const uint32_t *>(msgs + (o & ~(uint64_t)3));
    const uint32_t sh = (uint32_t)(o & 3);
    const uint32_t sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
    h[0] = 0x6a09e667; h[1] = 0xbb67ae85; h[2] = 0x3c6ef372; h[3] = 0xa54ff53a;
    h[4] = 0x510e527f; h[5] = 0x9b05688c; h[6] = 0x1f83d9ab; h[7] = 0x5be0cd19;
    const uint64_t nblocks = (len + 9 + 63) / 64;
    for (uint64_t blk = 0; blk < nblocks; blk++) {
        uint32_t w[16];
        const uint64_t bpos = blk * 64;
        if (bpos + 64 <= len) {
            uint32_t prev = __ldg(words + blk * 16);
#pragma unroll
            for (int j = 0; j < 16; j++) {
                uint32_t next = (sh || j < 15) ? __ldg(words + blk * 16 + j + 1) : 0u;
                w[j] = __byte_perm(prev, next, sel);
                prev = next;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const uint64_t p = bpos + 4 * (uint64_t)j;
                uint32_t v = 0;
                if (p < len) {
                    uint32_t a = __ldg(words + blk * 16 + j), b = __ldg(words + blk * 16 + j + 1);
                    v = __byte_perm(a, b, sel);
                    uint32_t rem = (uint32_t)(len - p);  // valid bytes in this word (>= 1)
                    if (rem < 4) v = (v & (0xffffffffu << (8 * (4 - rem)))) | (0x80u << (8 * (3 - rem)));
                } else if (p == len) {
                    v = 0x80000000u;
                }
                w[j] = v;
            }
            if (blk == nblocks - 1) {
                const uint64_t bits = len * 8;
                w[14] = (uint32_t)(bits >> 32);
                w[15] = (uint32_t)bits;
            }
        }
        sha256_compress(h, w);
    }
}

// digest_out: 32 bytes per message, big-endian words (the byte string SHA-256 defines)
// perm (optional): message processed by thread t is perm[t] — the launcher sorts messages by block
// count (longest first) so the 32 lanes of a warp hash messages of equal length instead of all
// waiting for the longest one.
__global__ void __launch_bounds__(128) k_sha256(uint32_t n, const uint8_t *__restrict__ msgs,
                                                const uint64_t *__restrict__ off, uint64_t base, uint8_t *__restrict__ digest_out,
                                                const uint32_t *__restrict__ perm) {
    const uint32_t tix = blockIdx.x * blockDim.x + threadIdx.x;
    if (tix >= n) return;
    const uint32_t idx = perm ? perm[tix] : tix;
    uint32_t h[8];
    sha256_msg(h, msgs, off, base, idx);
    uint4 *out = reinterpret_cast<uint4 *>(digest_out + (size_t)idx * 32);
    out[0] = make_uint4(__byte_perm(h[0], 0, 0x0123), __byte_perm(h[1], 0, 0x0123), __byte_perm(h[2], 0, 0x0123), __byte_perm(h[3], 0, 0x0123));
    out[1] = make_uint4(__byte_perm(h[4], 0, 0x0123), __byte_perm(h[5], 0, 0x0123), __byte_perm(h[6], 0, 0x0123), __byte_perm(h[7], 0, 0x0123));
}

// ---- counting sort of the messages by SHA-256 block count (descending) ----
constexpr int SHA_BINS = 1024;  // bin = min(nblocks, 1023): exact up to 65 KB messages
__device__ __forceinline__ uint32_t sha_bin(const uint64_t *off, uint32_t i) {
    const uint64_t nb = (off[i + 1] - off[i] + 9 + 63) / 64;
    return nb < SHA_BINS ? (uint32_t)nb : SHA_BINS - 1;
}
__global__ void k_sha_hist(uint32_t n, const uint64_t *__restrict__ off, uint32_t *__restrict__ hist) {
    __shared__ uint32_t h[SHA_BINS];
    for (int i = threadIdx.x; i < SHA_BINS; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&h[sha_bin(off, i)], 1u);
    __syncthreads();
    for (int b = threadIdx.x; b < SHA_BINS; b += blockDim.x) if (h[b]) atomicAdd(&hist[b], h[b]);
}
// one block of SHA_BINS threads: start[b] = number of messages in bins > b (longest first); cursor = 0
__global__ void k_sha_scan(const uint32_t *__restrict__ hist, uint32_t *__restrict__ start, uint32_t *__restrict__ cursor) {
    __shared__ uint32_t s[SHA_BINS];
    const int b = threadIdx.x;
    s[b] = hist[SHA_BINS - 1 - b];  // reversed: position b holds bin SHA_BINS-1-b
    __syncthreads();
    for (int d = 1; d < SHA_BINS; d <<= 1) {
        uint32_t v = b >= d ? s[b - d] : 0u;
        __syncthreads();
        s[b] += v;
        __syncthreads();
    }
    start[SHA_BINS - 1 - b] = s[b] - hist[SHA_BINS - 1 - b];  // exclusive
    cursor[b] = 0;
}
__global__ void k_sha_scatter(uint32_t n, const uint64_t *__restrict__ off, const uint32_t *__restrict__ start,
                              uint32_t *__restrict__ cursor, uint32_t *__restrict__ perm) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < n;
    const uint32_t b = valid ? sha_bin(off, i) : 0xffffffffu;
    // warp-aggregated: one atomic per distinct bin per warp (a batch of equal-length messages would
    // otherwise serialise a million atomics on one counter); ranks keep the input order inside a warp
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t peers = __match_any_sync(0xffffffffu, b);
    const int leader = __ffs((int)peers) - 1;
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    uint32_t base = 0;
    if (valid && (int)lane == leader) base = atomicAdd(&cursor[b], (uint32_t)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    if (valid) perm[start[b] + base + rank] = i;
}

}  // namespace sbv
