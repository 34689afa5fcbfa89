// rsa_quorum.cuh — the split of a shard of RSA commit votes (sbv_rsa_verify_quorum) into its three key sizes.
//
// A shard is uploaded as the caller holds it: a family tag (rsa_shard.h: rsa_family of the signature's length), a slot,
// a ragged signature and a message per vote; the messages are hashed in vote order first.  The split reuses the kernels of
// mixed.cuh with the signature offsets in place of the message offsets: k_mix_count and k_mix_scan (tag RSA_NO_FAMILY
// counts in no family), then k_rsa_split below, then k_mix_compact, which copies each signature into its family's region
// of the plan's blob, k bytes per row.  A region starts 16-byte aligned (rsa_family_start) and its rows are k bytes, so
// every row is aligned for the group kernels' loads.  After the per-family rsa_launch_shard, k_mix_ok scatters the
// family verdicts back into vote order over a zeroed array, so that votes of no family reject.
//
// The plan's families: idx, slot, off and ok as for a mixed shard; r holds the hLen-byte digest rows; s is unused.
#pragma once
#include <stdint.h>

#include "mixed.cuh"
#include "rsa_shard.h"

namespace sbv {

static_assert(RSA_FAMILIES == MIX_FAMILIES, "one plan family per RSA key size");

// One thread per tile of MIX_TILE votes, in vote order, after k_mix_scan: each family vote's index, slot and destination
// offset in the compacted blob at its rank inside its family, and its digest row (hlen bytes, a multiple of 16, from the
// vote-order digests dig) copied to the family's digest rows.
__global__ void __launch_bounds__(256) k_rsa_split(uint32_t n, const uint8_t *__restrict__ tag, const uint32_t *__restrict__ slot,
                                                   const uint8_t *__restrict__ dig, uint32_t hlen, const uint64_t *__restrict__ off, uint32_t ntiles,
                                                   const uint32_t *__restrict__ tile_cnt, const uint64_t *__restrict__ tile_bytes, MixPlan p) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    uint32_t rank[MIX_FAMILIES];
    uint64_t pos[MIX_FAMILIES];
#pragma unroll
    for (int k = 0; k < MIX_FAMILIES; k++) { rank[k] = tile_cnt[(size_t)k * ntiles + t]; pos[k] = tile_bytes[(size_t)k * ntiles + t]; }
    const uint32_t lo = t * MIX_TILE, hi = n - lo < MIX_TILE ? n : lo + MIX_TILE;
    for (uint32_t i = lo; i < hi; i++) {
        const uint32_t f = tag[i];
        if (f >= (uint32_t)MIX_FAMILIES) continue;
        const MixFamily F = mix_family(p, f);
        const uint32_t j = f == 0 ? rank[0] : f == 1 ? rank[1] : rank[2];
        const uint64_t at = f == 0 ? pos[0] : f == 1 ? pos[1] : pos[2];
        const uint64_t len = off[i + 1] - off[i];
#pragma unroll
        for (int k = 0; k < MIX_FAMILIES; k++)
            if (f == (uint32_t)k) { rank[k]++; pos[k] += len; }
        F.idx[j] = i;
        F.slot[j] = slot[i];
        F.off[j] = at;
        mix_copy16(F.r + (size_t)j * hlen, dig + (size_t)i * hlen, (int)(hlen / 16));
    }
}

}  // namespace sbv
