// inst_mixed.cu — launchers of the split / scatter kernels of mixed ECDSA / Ed25519 shards (mixed.cuh) behind engine.h,
// and the layout of their device scratch.
#include "engine.h"
#include "mixed.cuh"

using namespace sbv;

namespace {
size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

MixPlan plan_of(const MixBufs &b) {
    MixPlan p;
    for (int f = 0; f < MIX_FAMILIES; f++) p.f[f] = MixFamily{b.idx[f], b.slot[f], b.r[f], b.s[f], b.off[f], b.ok[f]};
    p.blob = b.blob;
    return p;
}
}  // namespace
static_assert(MIX_FAMILIES == SBV_ED25519 + 1, "one family per scheme tag");

size_t sbv_mix_carve(uint8_t *base, size_t n, const uint32_t m[3], uint64_t bytes, bool keys, MixBufs *out, const uint32_t *m384) {
    MixBufs b{};
    size_t at = 0;
    auto take = [&](size_t sz) {
        uint8_t *p = base ? base + at : nullptr;
        at += al256(sz);
        return p;
    };
    const size_t ntiles = (n + MIX_TILE - 1) / MIX_TILE;
    b.tag = take(n);
    if (keys) b.key96 = take(n * 96);
    else b.slot_in = (uint32_t *)take(n * 4);
    b.sig96 = take(n * 96);
    b.tile_cnt = (uint32_t *)take(ntiles * MIX_FAMILIES * 4);
    b.tile_bytes = (uint64_t *)take(ntiles * MIX_FAMILIES * 8);
    b.blob = take(bytes + MIX_FAMILIES * 32);  // three regions, each 16-byte aligned and followed by >= 16 bytes of slack
    for (int f = 0; f < MIX_FAMILIES; f++) {
        const size_t k = m[f], L = f == SBV_P256 ? 32 : f == SBV_P384 ? 48 : 64;
        b.idx[f] = (uint32_t *)take(k * 4);
        if (!keys) b.slot[f] = (uint32_t *)take(k * 4);
        else if (f != SBV_ED25519) {
            b.qx[f] = take(k * L);
            b.qy[f] = take(k * L);
        }
        b.r[f] = take(k * L);
        b.s[f] = f == SBV_ED25519 ? nullptr : take(k * L);
        b.off[f] = (uint64_t *)take((k + 1) * 8);
        b.ok[f] = take(k);
        b.perm[f] = (uint32_t *)take((k + 3 * 1024) * 4);
        // ECDSA: e, 32 bytes per item, or 48 for a P-384 family with SHA-384 items; Ed25519: k, word-major
        b.dig[f] = take(k * (f == SBV_P384 && m384 && m384[SBV_P384] ? 48 : 32));
        b.pub[f] = f == SBV_ED25519 ? take(k * 32) : nullptr;
    }
    if (m384 && (m384[SBV_P256] || m384[SBV_P384])) b.alg = take(n);
    if (out) *out = b;
    return at;
}

int sbv_launch_mix_split(sbv_engine *e, const MixBufs &b, size_t n, const uint32_t m[3], const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base,
                         cudaStream_t st) {
    const uint32_t nn = (uint32_t)n, ntiles = (uint32_t)((n + MIX_TILE - 1) / MIX_TILE);
    const MixPlan p = plan_of(b);
    k_mix_count<<<(ntiles + 255) / 256, 256, 0, st>>>(nn, b.tag, d_off, ntiles, b.tile_cnt, b.tile_bytes);
    k_mix_scan<<<1, MIX_SCAN_THREADS, 0, st>>>(ntiles, b.tile_cnt, b.tile_bytes, p);
    if (b.key96)
        k_mix_split<true><<<(ntiles + 255) / 256, 256, 0, st>>>(nn, b.tag, nullptr, b.sig96, d_off, ntiles, b.tile_cnt, b.tile_bytes, p, b.key96,
                                                                 MixKeys{{b.qx[0], b.qx[1]}, {b.qy[0], b.qy[1]}, b.pub[SBV_ED25519]});
    else
        k_mix_split<<<(ntiles + 255) / 256, 256, 0, st>>>(nn, b.tag, b.slot_in, b.sig96, d_off, ntiles, b.tile_cnt, b.tile_bytes, p);
    k_mix_compact<<<(uint32_t)(((uint64_t)n * MIX_LANES + 255) / 256), 256, 0, st>>>(nn, m[0], m[1], d_msgs, d_off, base, p);
    e->launches += 4;
    CU(e, cudaGetLastError());
    return 0;
}

int sbv_launch_mix_ok(sbv_engine *e, const MixBufs &b, size_t n, const uint32_t m[3], uint8_t *d_ok, cudaStream_t st) {
    k_mix_ok<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, m[0], m[1], plan_of(b), d_ok);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
