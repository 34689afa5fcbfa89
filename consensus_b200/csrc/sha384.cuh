// sha384.cuh — SHA-384 over a ragged batch, one message per thread (FIPS 180-4 §6.5): the SHA-512 compression of
// sha512_core.cuh from the SHA-384 initial value (§5.3.4), the digest truncated to its first 48 bytes.  The e of an
// ECDSA signature made with SHA-384 (Go's x509 ECDSAWithSHA384, JOSE ES384, TLS ecdsa_secp384r1_sha384).
//
// Same contract as k_sha256: messages concatenated in one device buffer with byte offsets off[n+1] relative to `base`,
// read with ALIGNED 32-bit loads and re-aligned with PRMT; the buffer must be readable 8 bytes past the last message.
// The block-count sort of sha256.cuh orders the messages for it too (it is monotone in the length).
#pragma once
#include <stdint.h>

#include "sha512_core.cuh"

namespace sbv {

// The SHA-512 state h after message idx of the batch from the SHA-384 initial value (offsets off relative to base); the
// digest is the first six words.  The per-message body of k_sha384, shared with k_sha2_sel (mixed_hash.cuh).
__device__ __forceinline__ void sha384_msg(uint64_t (&h)[8], const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                           uint32_t idx) {
    const uint64_t o = off[idx] - base;
    const uint64_t len = off[idx + 1] - off[idx];
    const uint32_t *words = reinterpret_cast<const uint32_t *>(msgs + (o & ~(uint64_t)3));
    const uint32_t sh = (uint32_t)(o & 3);
    const uint32_t sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
    h[0] = 0xcbbb9d5dc1059ed8ull; h[1] = 0x629a292a367cd507ull; h[2] = 0x9159015a3070dd17ull; h[3] = 0x152fecd8f70e5939ull;
    h[4] = 0x67332667ffc00b31ull; h[5] = 0x8eb44a8768581511ull; h[6] = 0xdb0c2e0d64f98fa7ull; h[7] = 0x47b5481dbefa4fa4ull;
    const uint64_t nblocks = (len + 17 + 127) / 128;  // the 0x80 byte and the 128-bit length fit after the message
    for (uint64_t blk = 0; blk < nblocks; blk++) {
        uint32_t w32[32];
        sha512_msg16(w32, blk * 128, len, words, sel, sh);
        sha512_msg16(w32 + 16, blk * 128 + 64, len, words, sel, sh);
        uint64_t w[16];
#pragma unroll
        for (int j = 0; j < 16; j++) w[j] = ((uint64_t)w32[2 * j] << 32) | w32[2 * j + 1];
        if (blk == nblocks - 1) {  // the bit length as a 128-bit big-endian integer
            w[14] = len >> 61;
            w[15] = len << 3;
        }
        sha512_compress(h, w);
    }
}

// digest_out: 48 bytes per message at idx * 48, big-endian words (the byte string SHA-384 defines), which is the layout
// k_prep reads with dlen = 48.  perm (optional): message processed by thread t is perm[t] (see k_sha256).
__global__ void __launch_bounds__(128) k_sha384(uint32_t n, const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                                uint8_t *__restrict__ digest_out, const uint32_t *__restrict__ perm) {
    const uint32_t tix = blockIdx.x * blockDim.x + threadIdx.x;
    if (tix >= n) return;
    const uint32_t idx = perm ? perm[tix] : tix;
    uint64_t h[8];
    sha384_msg(h, msgs, off, base, idx);
    uint4 *out = reinterpret_cast<uint4 *>(digest_out + (size_t)idx * 48);
    out[0] = make_uint4(bswap32((uint32_t)(h[0] >> 32)), bswap32((uint32_t)h[0]), bswap32((uint32_t)(h[1] >> 32)), bswap32((uint32_t)h[1]));
    out[1] = make_uint4(bswap32((uint32_t)(h[2] >> 32)), bswap32((uint32_t)h[2]), bswap32((uint32_t)(h[3] >> 32)), bswap32((uint32_t)h[3]));
    out[2] = make_uint4(bswap32((uint32_t)(h[4] >> 32)), bswap32((uint32_t)h[4]), bswap32((uint32_t)(h[5] >> 32)), bswap32((uint32_t)h[5]));
}

}  // namespace sbv
