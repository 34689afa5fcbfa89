// sha512_batch.cuh — SHA-512 over a ragged batch, one message per thread (FIPS 180-4 §6.4): the compression function
// and message loader of sha512_core.cuh from the SHA-512 initial value (§5.3.5), the whole 64-byte digest out.  The
// digest of an RSA signature made with SHA-512 (Go's x509 SHA512WithRSA), and sbv_sha512_batch.
//
// Same contract as k_sha256 and k_sha384: messages concatenated in one device buffer with byte offsets off[n+1] relative
// to `base`, read with ALIGNED 32-bit loads; the buffer must be readable 8 bytes past the last message.  The block-count
// sort of sha256.cuh orders the messages for it too.
#pragma once
#include <stdint.h>

#include "sha512_core.cuh"

namespace sbv {

// digest_out: 64 bytes per message at idx * 64 (the byte string SHA-512 defines).  perm (optional): message processed by
// thread t is perm[t] (see k_sha256).
__global__ void __launch_bounds__(128) k_sha512(uint32_t n, const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                                uint8_t *__restrict__ digest_out, const uint32_t *__restrict__ perm) {
    const uint32_t tix = blockIdx.x * blockDim.x + threadIdx.x;
    if (tix >= n) return;
    const uint32_t idx = perm ? perm[tix] : tix;
    const uint64_t o = off[idx] - base;
    const uint64_t len = off[idx + 1] - off[idx];
    const uint32_t *words = reinterpret_cast<const uint32_t *>(msgs + (o & ~(uint64_t)3));
    const uint32_t sh = (uint32_t)(o & 3);
    const uint32_t sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
    uint64_t h[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                     0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
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
    uint4 *out = reinterpret_cast<uint4 *>(digest_out + (size_t)idx * 64);
#pragma unroll
    for (int q = 0; q < 4; q++)
        out[q] = make_uint4(bswap32((uint32_t)(h[2 * q] >> 32)), bswap32((uint32_t)h[2 * q]), bswap32((uint32_t)(h[2 * q + 1] >> 32)),
                            bswap32((uint32_t)h[2 * q + 1]));
}

}  // namespace sbv
