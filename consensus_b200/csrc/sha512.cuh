// sha512.cuh — SHA-512 (FIPS 180-4) of R || A || M over a ragged batch, one item per thread, reduced mod L: the
// challenge k = SHA-512(R || A || M) mod L of Ed25519 verification (RFC 8032 §5.1.7).
//
// R (the first half of the signature) and A (the public key) come from their own arrays and M from the message blob at
// off[i], so nothing is concatenated on the host.  M is read with ALIGNED 32-bit loads and re-aligned with PRMT, as
// k_sha256 does; the blob must be readable 8 bytes past the last message.  The compression function and the message
// loader are those of sha512_core.cuh, which SHA-384 shares.
#pragma once
#include <stdint.h>

#include "ed25519.cuh"
#include "sha512_core.cuh"

namespace sbv {

// The 64-byte digest of R || A || M for item idx (16 little-endian limbs of the digest read as a little-endian
// integer, as RFC 8032 reads it).  sig: 64 bytes per item (R || S); pub: 32 bytes per item.
SBV_DEV void ed_sha512_item(uint32_t (&dig)[16], uint32_t idx, const uint8_t *__restrict__ sig, const uint8_t *__restrict__ pub,
                            const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base) {
    const uint64_t o = off[idx] - base;
    const uint64_t len = off[idx + 1] - off[idx];
    const uint32_t *words = reinterpret_cast<const uint32_t *>(msgs + (o & ~(uint64_t)3));
    const uint32_t sh = (uint32_t)(o & 3);
    const uint32_t sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
    uint64_t h[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                     0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    const uint64_t total = 64 + len;  // bytes hashed
    const uint64_t nblocks = (total + 17 + 127) / 128;
    for (uint64_t blk = 0; blk < nblocks; blk++) {
        uint32_t w32[32];
        if (blk == 0) {  // R || A
            const uint4 *r4 = reinterpret_cast<const uint4 *>(sig + (size_t)idx * 64);
            const uint4 *a4 = reinterpret_cast<const uint4 *>(pub + (size_t)idx * 32);
            const uint4 v[4] = {__ldg(r4), __ldg(r4 + 1), __ldg(a4), __ldg(a4 + 1)};
#pragma unroll
            for (int q = 0; q < 4; q++) {
                w32[4 * q] = bswap32(v[q].x); w32[4 * q + 1] = bswap32(v[q].y);
                w32[4 * q + 2] = bswap32(v[q].z); w32[4 * q + 3] = bswap32(v[q].w);
            }
        } else {
            sha512_msg16(w32, blk * 128 - 64, len, words, sel, sh);
        }
        sha512_msg16(w32 + 16, blk * 128, len, words, sel, sh);
        uint64_t w[16];
#pragma unroll
        for (int j = 0; j < 16; j++) w[j] = ((uint64_t)w32[2 * j] << 32) | w32[2 * j + 1];
        if (blk == nblocks - 1) w[15] = total * 8;  // the 128-bit length; its high half (w[14]) is zero
        sha512_compress(h, w);
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
        dig[2 * u] = bswap32((uint32_t)(h[u] >> 32));
        dig[2 * u + 1] = bswap32((uint32_t)h[u]);
    }
}

// k = SHA-512(R || A || M) mod L, written word-major: k_out[w * n + idx], w = 0..7 (little-endian limbs), which the
// verify kernel reads coalesced.  perm (optional): thread t hashes item perm[t] — the items sorted by length (the
// block-count sort of sha256.cuh), so that the lanes of a warp hash messages of about the same length.
// dig_out (optional, tests only): the 16 digest limbs of item idx at dig_out[16 * idx].
__global__ void __launch_bounds__(128) k_ed_sha512(uint32_t n, const uint8_t *__restrict__ sig, const uint8_t *__restrict__ pub,
                                                   const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                                   uint32_t *__restrict__ k_out, const uint32_t *__restrict__ perm,
                                                   uint32_t *__restrict__ dig_out) {
    const uint32_t tix = blockIdx.x * blockDim.x + threadIdx.x;
    if (tix >= n) return;
    const uint32_t idx = perm ? perm[tix] : tix;
    uint32_t dig[16], k[8];
    ed_sha512_item(dig, idx, sig, pub, msgs, off, base);
    if (dig_out) {
#pragma unroll
        for (int w = 0; w < 16; w++) dig_out[(size_t)idx * 16 + w] = dig[w];
    }
    sc_reduce512(k, dig);
#pragma unroll
    for (int w = 0; w < 8; w++) k_out[(size_t)w * n + idx] = k[w];
}

}  // namespace sbv
