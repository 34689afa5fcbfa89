// mixed_hash.cuh — SHA-384 items in mixed shards (sbv_mixed384_verify_registered, sbv_mixed384_verify_batch,
// sbv_mixed384_verify_quorum): ECDSA over SHA-384 beside ECDSA over SHA-256 and Ed25519 in one call.
//
// The split of mixed.cuh knows three families (P-256, P-384, Ed25519) and stays as it is.  A shard that holds a tag of
// SBV_P256_SHA384 (3) or SBV_P384_SHA384 (4) runs one kernel before it:
//   k_mix_alg   per item: the tag becomes its curve family in place (3 -> 0, 4 -> 1) and sha384[i] records whether
//               item i is hashed with SHA-384;
// and each ECDSA family that holds a SHA-384 item is hashed by k_sha2_sel instead of k_sha256, behind the same
// block-count sort:
//   k_sha2_sel  one message per thread; family item j is hashed with SHA-384 iff sha384[idx[j]], and e is written in the
//               layout k_prep reads with the family's dlen:
//                 dlen 32 (P-256)  the SHA-256 digest, or the first 32 bytes of SHA-384 (crypto/ecdsa's truncation);
//                 dlen 48 (P-384)  the SHA-384 digest, or 16 zero bytes and the SHA-256 digest: the integer e of dlen 32.
// The per-message bodies are those of k_sha256 and k_sha384 (sha256_msg, sha384_msg), so both hashes are computed
// exactly as the single-hash calls compute them.
#pragma once
#include <stdint.h>

#include "sha256.cuh"
#include "sha384.cuh"

namespace sbv {

constexpr uint32_t MIX_TAG_SHA384 = 3;  // tags MIX_TAG_SHA384 + f: family f (P-256, P-384) over SHA-384

__global__ void __launch_bounds__(256) k_mix_alg(uint32_t n, uint8_t *__restrict__ tag, uint8_t *__restrict__ sha384) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t t = tag[i];
    const bool wide = t >= MIX_TAG_SHA384;
    tag[i] = (uint8_t)(wide ? t - MIX_TAG_SHA384 : t);
    sha384[i] = wide ? 1 : 0;
}

// n items of one family: messages at off[j] - base in msgs (readable 8 bytes past the last one), idx[j] = the item's index
// in the shard, sha384 = the flags of k_mix_alg in shard order.  digest_out: dlen (32 or 48) bytes per item at j * dlen.
// perm (optional): item processed by thread t is perm[t] (see k_sha256).
__global__ void __launch_bounds__(128) k_sha2_sel(uint32_t n, const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                                  const uint32_t *__restrict__ idx, const uint8_t *__restrict__ sha384, uint32_t dlen,
                                                  uint8_t *__restrict__ digest_out, const uint32_t *__restrict__ perm) {
    const uint32_t tix = blockIdx.x * blockDim.x + threadIdx.x;
    if (tix >= n) return;
    const uint32_t j = perm ? perm[tix] : tix;
    uint4 *out = reinterpret_cast<uint4 *>(digest_out + (size_t)j * dlen);
    if (sha384[idx[j]]) {
        uint64_t h[8];
        sha384_msg(h, msgs, off, base, j);
        out[0] = make_uint4(bswap32((uint32_t)(h[0] >> 32)), bswap32((uint32_t)h[0]), bswap32((uint32_t)(h[1] >> 32)), bswap32((uint32_t)h[1]));
        out[1] = make_uint4(bswap32((uint32_t)(h[2] >> 32)), bswap32((uint32_t)h[2]), bswap32((uint32_t)(h[3] >> 32)), bswap32((uint32_t)h[3]));
        if (dlen == 48)
            out[2] = make_uint4(bswap32((uint32_t)(h[4] >> 32)), bswap32((uint32_t)h[4]), bswap32((uint32_t)(h[5] >> 32)), bswap32((uint32_t)h[5]));
    } else {
        uint32_t h[8];
        sha256_msg(h, msgs, off, base, j);
        if (dlen == 48) *out++ = make_uint4(0u, 0u, 0u, 0u);
        out[0] = make_uint4(bswap32(h[0]), bswap32(h[1]), bswap32(h[2]), bswap32(h[3]));
        out[1] = make_uint4(bswap32(h[4]), bswap32(h[5]), bswap32(h[6]), bswap32(h[7]));
    }
}

}  // namespace sbv
