// shards.h — how a multi-device engine splits one call between its devices, and the layout of the packed words they
// all-gather.  Pure host code (no CUDA), shared by engine.cu and the CPU simulation, which checks it against
// consensus_b200/sharding.py.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace sbv {

struct Range { size_t lo, n; };

// device g of G owns items [n*g/G, n*(g+1)/G)
inline Range shard_range(size_t n, int g, int G) {
    const size_t lo = n * g / G, hi = n * (g + 1) / G;
    return {lo, hi - lo};
}

// The items (votes) and instances of every device, and the gather buffer's layout: device g's slot starts at word
// g * wp() and holds wv words of verdict bits, then wi words of reached bits (k_pack_bits: bit i of word i / 32).
struct Shards {
    std::vector<Range> vr, ir;  // ir is empty for a plain batch
    size_t wv = 0, wi = 0;
    size_t wp() const { return wv + wi; }
};

// a plain batch: contiguous items, no instances
inline Shards batch_shards(size_t n, int G) {
    Shards s;
    for (int g = 0; g < G; g++) {
        s.vr.push_back(shard_range(n, g, G));
        s.wv = std::max(s.wv, (s.vr[g].n + 31) / 32);
    }
    return s;
}

// Commit votes, grouped by non-decreasing instance (checked by the caller): device g owns the contiguous instances
// shard_range(n_instances, g, G) and the votes that carry them, so every count is local.  The last device also takes
// trailing votes whose instance is out of range.
inline Shards quorum_shards(size_t n_votes, const uint32_t *instance, size_t n_instances, int G) {
    Shards s;
    for (int g = 0; g < G; g++) {
        const Range ir = shard_range(n_instances, g, G);
        const uint32_t *a = std::lower_bound(instance, instance + n_votes, (uint32_t)ir.lo);
        const uint32_t *b = g == G - 1 ? instance + n_votes : std::lower_bound(instance, instance + n_votes, (uint32_t)(ir.lo + ir.n));
        s.vr.push_back({(size_t)(a - instance), (size_t)(b - a)});
        s.ir.push_back(ir);
        s.wv = std::max(s.wv, (s.vr[g].n + 31) / 32);
        s.wi = std::max(s.wi, (ir.n + 31) / 32);
    }
    return s;
}

// the gathered words of all devices -> verdict bytes (and reached bytes, when there are instances)
inline void unpack_shards(const Shards &s, const uint32_t *words, uint8_t *ok, uint8_t *reached) {
    auto bit = [](const uint32_t *w, size_t i) { return (uint8_t)((w[i >> 5] >> (i & 31)) & 1u); };
    for (size_t g = 0; g < s.vr.size(); g++) {
        const uint32_t *w = words + s.wp() * g;
        for (size_t i = 0; i < s.vr[g].n; i++) ok[s.vr[g].lo + i] = bit(w, i);
        if (!s.ir.empty())
            for (size_t i = 0; i < s.ir[g].n; i++) reached[s.ir[g].lo + i] = bit(w + s.wv, i);
    }
}

}  // namespace sbv
