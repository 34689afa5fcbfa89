// rsa_shard.h — what one RSA launch is given, shared by libsbv.so and the CPU simulation (tools/hostsim): the description
// of a shard of RSA items and the two maps from a call's shape to the kernels' template arguments.  Pure host code;
// rsa_launch_shard (rsa_keyed.cuh) turns a shard into launches.
#pragma once
#include <cstddef>
#include <cstdint>
#include <type_traits>

struct uint4;  // CUDA's vector type (hostsim.h in the simulation)

namespace sbv {

enum class RsaPad { pkcs1, pss };

// n items of k bytes (256, 384 or 512) each, device pointers (the simulation: host pointers).  sig: n * k bytes, big-endian,
// EM written over it with PSS; digest: n * hLen bytes (hash: SBV_HASH_SHA256 / 384 / 512); ok: n verdicts.  The key of
// each item is (mod: n * k bytes, exp: n words), or, with slot set, the registry slot slot[i] of nslots (rec and pool as
// k_rsa_kprep writes them; null for an empty registry).
struct RsaShard {
    uint32_t k, hash;
    RsaPad pad;
    int32_t salt_len;  // PSS: >= -1, as in sbv_rsa_pss_verify_batch
    size_t n;
    uint8_t *sig;
    const uint8_t *digest;
    uint8_t *ok;
    const uint8_t *mod = nullptr;
    const uint32_t *exp = nullptr;
    const uint32_t *slot = nullptr;
    uint32_t nslots = 0;
    const uint4 *rec = nullptr;
    const uint32_t *pool = nullptr;
};

// The limbs per lane NL = k / 64 of a k-byte modulus: f(std::integral_constant<int, NL>{}) for k = 256, 384 or 512,
// false (f not called) for any other k.
template <class F>
bool rsa_nl(uint32_t k, F &&f) {
    switch (k) {
        case 256: f(std::integral_constant<int, 4>{}); return true;
        case 384: f(std::integral_constant<int, 6>{}); return true;
        case 512: f(std::integral_constant<int, 8>{}); return true;
    }
    return false;
}

// The hash instance H of k_rsa_pss for hash tag h: f(std::integral_constant<int, H>{}) for SBV_HASH_SHA256 / 384 / 512
// (H = 0 / 1 / 2), false (f not called) for any other tag.
template <class F>
bool rsa_h(uint32_t h, F &&f) {
    switch (h) {
        case 0: f(std::integral_constant<int, 0>{}); return true;
        case 1: f(std::integral_constant<int, 1>{}); return true;
        case 2: f(std::integral_constant<int, 2>{}); return true;
    }
    return false;
}

inline bool rsa_size_ok(uint32_t k) { return rsa_nl(k, [](auto) {}); }
inline bool rsa_hash_ok(uint32_t h) { return rsa_h(h, [](auto) {}); }

// The RSA commit votes (sbv_rsa_verify_quorum) carry signatures of the signer's key size, and the length alone decides a
// vote's family, as Go's VerifyPKCS1v15 / VerifyPSS reject len(sig) != pub.Size(): 0 / 1 / 2 for 256 / 384 / 512 bytes,
// RSA_NO_FAMILY for any other length (the vote rejects without reaching a kernel).
constexpr int RSA_FAMILIES = 3;
constexpr uint8_t RSA_NO_FAMILY = 3;
inline uint8_t rsa_family(uint64_t len) { return len == 256 ? 0 : len == 384 ? 1 : len == 512 ? 2 : RSA_NO_FAMILY; }
inline uint32_t rsa_family_k(int f) { return 256u + 128u * (uint32_t)f; }
// Where family f's k-byte rows start in the compacted signature buffer of a split shard with m[c] votes of family c: the
// region starts k_mix_scan lays out (each 16-byte aligned, after the previous region and 16 bytes of slack).
inline uint64_t rsa_family_start(const uint32_t (&m)[RSA_FAMILIES], int f) {
    uint64_t at = 0;
    for (int c = 0; c < f; c++) at += ((uint64_t)m[c] * rsa_family_k(c) + 16 + 15) & ~(uint64_t)15;
    return at;
}

// Every RSA kernel runs in blocks of 128 threads, `lanes` threads per item (a group of 16, or 1): the grid of `items`.
constexpr uint32_t RSA_BLOCK = 128;
inline uint32_t rsa_grid(size_t items, uint32_t lanes) { return (uint32_t)((items * lanes + RSA_BLOCK - 1) / RSA_BLOCK); }

}  // namespace sbv
