// rsa_keyed.cuh — registered RSA keys (sbv_rsa_set_keys / sbv_rsa_verify_registered and the PSS and fused-hash forms): the
// key-only work of rsa.cuh done once per key set instead of once per signature.
//
// The registry of n slots is two arrays on every device:
//   rec   two uint4 per slot: {k, valid, ntop, n0'} and {e, off_lo, off_hi, 0}.  k = the slot's modulus size in bytes (256,
//         384 or 512); valid = 1 iff the key rule of rsa.cuh passed (N odd, N's leading byte nonzero, 2 <= e <= 2^31 - 1);
//         ntop = N's leading byte (the emLen of PSS); n0' = -N^-1 mod 2^32; off = the word offset of the slot's limbs in
//         pool.
//   pool  per slot, K = k / 4 little-endian 32-bit limbs of N, then K of R^2 mod N.
//         n0' and R^2 are built for every key rsa_r2 can take (N odd, top limb nonzero), the invalid ones among them too,
//         so that a registered key is refused by its validity flag alone; they are zero for the others.  Lane l of a
//         group holds limbs [l*NL, l*NL + NL), which are contiguous, so each operand is NL / 4 (NL = 4, 8) or NL / 2
//         (NL = 6) vector loads per lane.  The slots lie in slot order, slot i at word off_i = (the byte offset of modulus
//         i in the registered moduli) / 2: 16-byte aligned, as every modulus is a multiple of 256 bytes.
// 32 + 2k bytes per key: 544, 800 and 1,056 for 2048-, 3072- and 4096-bit keys.
//
//   k_rsa_kprep<NL>       a group of 16 lanes per key of one size: the record and limbs of its slot, with rsa_ninv and
//                         rsa_r2 (skipped for an even N or a zero top limb, which rsa_r2 cannot take).
//   k_rsa_verify_reg<NL>  PKCS #1 v1.5 as k_rsa_verify with the key read from the item's slot: the slot bound, the size,
//                         the validity flag, S < N, then rsa_pow_tail and rsa_pkcs1_match.
//   k_rsa_em_reg<NL>      as k_rsa_em with the key read from the slot: EM over the signature, the key and range verdict.
//   k_rsa_pss_reg<H>      pss_decode after k_rsa_em_reg, ntop taken from the record.
#pragma once
#include <stdint.h>

#include "rsa.cuh"
#include "rsa_pss.cuh"
#include "rsa_shard.h"

namespace sbv {

// This lane's NL limbs at p (16-byte aligned for NL = 4 and 8, 8-byte aligned for NL = 6), and back.
template <int NL>
SBV_DEV void rsa_limbs_load(uint32_t (&x)[NL], const uint32_t *p) {
    if constexpr (NL % 4 == 0) {
#pragma unroll
        for (int j = 0; j < NL / 4; j++) {
            const uint4 v = reinterpret_cast<const uint4 *>(p)[j];
            x[4 * j] = v.x, x[4 * j + 1] = v.y, x[4 * j + 2] = v.z, x[4 * j + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < NL / 2; j++) {
            const uint2 v = reinterpret_cast<const uint2 *>(p)[j];
            x[2 * j] = v.x, x[2 * j + 1] = v.y;
        }
    }
}
template <int NL>
SBV_DEV void rsa_limbs_store(uint32_t *p, const uint32_t (&x)[NL]) {
    if constexpr (NL % 4 == 0) {
#pragma unroll
        for (int j = 0; j < NL / 4; j++) reinterpret_cast<uint4 *>(p)[j] = uint4{x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]};
    } else {
#pragma unroll
        for (int j = 0; j < NL / 2; j++) reinterpret_cast<uint2 *>(p)[j] = uint2{x[2 * j], x[2 * j + 1]};
    }
}

// One key per group of 16 lanes: key j of the launch is slot slots[j], of k = 64 * NL bytes; its modulus is at mods +
// mod_off[slot] (big-endian), its exponent exps[slot].  Writes the slot's record and limbs (layout above).  The minimum of
// one block per SM lets ptxas keep the 4096-bit form in registers (with (128) alone it picks 80 and spills).
template <int NL>
__global__ void __launch_bounds__(128, 1) k_rsa_kprep(uint32_t cnt, const uint32_t *__restrict__ slots, const uint8_t *__restrict__ mods,
                                                      const uint64_t *__restrict__ mod_off, const uint32_t *__restrict__ exps, uint4 *__restrict__ rec,
                                                      uint32_t *__restrict__ pool) {
    const uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / RSA_GROUP;
    if (j >= cnt) return;  // the whole group
    constexpr int K = RSA_GROUP * NL;
    constexpr uint32_t k = 4 * K;
    const RsaLanes g = rsa_lanes();
    const uint32_t slot = slots[j], e = exps[slot];
    const uint64_t off = mod_off[slot];
    uint32_t n[NL], x[NL];
    rsa_load(g, n, mods + off, k);
    const uint32_t lo = rsa_from(g, n[0], 0), hi = rsa_from(g, n[NL - 1], RSA_GROUP - 1);
    // the key rule of rsa_recover, once per key; n0' and R^2 for every key rsa_r2 can take (N odd, top limb nonzero), so
    // that the validity flag alone refuses the rest of the invalid keys
    const bool valid = (lo & 1) != 0 && hi >= (1u << 24) && e >= 2 && e <= 0x7fffffffu;
    uint32_t ninv = 0;
    if ((lo & 1) != 0 && hi != 0) {
        ninv = rsa_ninv(g, n);
        rsa_r2(g, x, n, ninv);
    } else {
#pragma unroll
        for (int i = 0; i < NL; i++) x[i] = 0;
    }
    uint32_t *p = pool + off / 2 + g.l * NL;
    rsa_limbs_store(p, n);
    rsa_limbs_store(p + K, x);
    if (g.l == 0) {
        rec[2 * (size_t)slot] = uint4{k, valid ? 1u : 0u, hi >> 24, ninv};
        rec[2 * (size_t)slot + 1] = uint4{e, (uint32_t)(off / 2), (uint32_t)(off / 2 >> 32), 0u};
    }
}

// Steps 1-3 with the key of registry slot `slot` (the same in every lane of the group): false for a slot outside the
// registry, a key of another size than k = 64 * NL, a key the rule refused or S >= N; else tail(em) as rsa_recover.
template <int NL, class Tail>
SBV_DEV bool rsa_recover_reg(const RsaLanes &g, const uint8_t *sig, uint32_t slot, uint32_t nslots, const uint4 *rec, const uint32_t *pool,
                             Tail &&tail) {
    constexpr int K = RSA_GROUP * NL;
    constexpr uint32_t k = 4 * K;
    if (slot >= nslots) return false;
    const uint4 r0 = rec[2 * (size_t)slot], r1 = rec[2 * (size_t)slot + 1];
    if (r0.x != k) return false;
    if (r0.y == 0) return false;
    const uint32_t *p = pool + (((uint64_t)r1.z << 32) | r1.y) + g.l * NL;
    uint32_t n[NL], s[NL], x[NL];
    rsa_limbs_load(n, p);
    rsa_load(g, s, sig, k);
    const uint32_t below = rsa_sub(g, x, s, n);  // 1 iff S < N
    if (!below) return false;
    rsa_limbs_load(x, p + K);  // R^2 mod N
    uint32_t sm[NL], acc[NL];
    return rsa_pow_tail<NL>(g, s, x, n, r0.w, r1.x, sm, acc, tail);
}

// One item per group of 16 lanes: ok[i] = 1 iff sig i (k = 64 * NL bytes) is a valid PKCS #1 v1.5 signature of digest i
// (hLen bytes) under the key of registry slot key_slot[i].
template <int NL>
__global__ void __launch_bounds__(128) k_rsa_verify_reg(uint32_t n, uint32_t hash, const uint8_t *__restrict__ sig, const uint32_t *__restrict__ key_slot,
                                                        uint32_t nslots, const uint4 *__restrict__ rec, const uint32_t *__restrict__ pool,
                                                        const uint8_t *__restrict__ digest, uint8_t *__restrict__ ok) {
    const uint64_t item = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / RSA_GROUP;
    if (item >= n) return;  // the whole group
    constexpr uint32_t k = 64 * NL;
    const RsaLanes g = rsa_lanes();
    const uint8_t *h = digest + item * (32 + 16 * hash);
    const bool v = rsa_recover_reg<NL>(g, sig + item * k, key_slot[item], nslots, rec, pool,
                                       [&](const uint32_t (&em)[NL]) { return rsa_pkcs1_match<NL>(g, em, h, hash); });
    if (g.l == 0) ok[item] = v ? 1 : 0;
}

// k_rsa_em with the key of registry slot key_slot[i]: EM = S^e mod N over sig where the slot, the key and S < N accept
// the item, and ok[i] = 1 there, else 0 (sig left as it was).  (128, 1) as for k_rsa_kprep: no spill at 4096 bits.
template <int NL>
__global__ void __launch_bounds__(128, 1) k_rsa_em_reg(uint32_t n, uint8_t *__restrict__ sig, const uint32_t *__restrict__ key_slot, uint32_t nslots,
                                                       const uint4 *__restrict__ rec, const uint32_t *__restrict__ pool, uint8_t *__restrict__ ok) {
    const uint64_t item = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / RSA_GROUP;
    if (item >= n) return;  // the whole group
    constexpr uint32_t k = 64 * NL;
    const RsaLanes g = rsa_lanes();
    uint8_t *s = sig + item * k;
    const bool v = rsa_recover_reg<NL>(g, s, key_slot[item], nslots, rec, pool, [&](const uint32_t (&em)[NL]) {
        rsa_store(g, s, em, k);
        return true;
    });
    if (g.l == 0) ok[item] = v ? 1 : 0;
}

// One item per thread after k_rsa_em_reg: em k bytes per item, digest HL bytes per item; ok[i] &= the PSS verdict, N's
// leading byte read from the record of the item's slot (ok[i] = 1 only where that slot exists).
template <int H>
__global__ void __launch_bounds__(128) k_rsa_pss_reg(uint32_t n, uint32_t k, int32_t salt_len, uint8_t *__restrict__ em,
                                                     const uint32_t *__restrict__ key_slot, const uint4 *__restrict__ rec,
                                                     const uint8_t *__restrict__ digest, uint8_t *__restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !ok[i]) return;
    const uint32_t ntop = rec[2 * (size_t)key_slot[i]].z;
    const bool v = pss_decode<H>(em + (size_t)i * k, k, ntop, digest + (size_t)i * PssSha<H>::HL, salt_len);
    ok[i] = v ? 1 : 0;
}

// Host side of the build (the engine and the CPU simulation): mod_off[i] = the byte offset of modulus i in the registered
// moduli (mod_bytes in slot order, each 256, 384 or 512); slots = the slot indices grouped by size, those of size 256 +
// 128 c at [first[c], first[c + 1]), one k_rsa_kprep launch each.  Returns the total bytes of the moduli: the pool holds
// total / 2 words.
inline uint64_t rsa_reg_layout(size_t n, const uint32_t *mod_bytes, uint64_t *mod_off, uint32_t *slots, size_t (&first)[4]) {
    uint64_t t = 0;
    for (size_t i = 0; i < n; i++) {
        mod_off[i] = t;
        t += mod_bytes[i];
    }
    size_t m = 0;
    for (int c = 0; c < 3; c++) {
        first[c] = m;
        for (size_t i = 0; i < n; i++)
            if (mod_bytes[i] == 256u + 128u * c) slots[m++] = (uint32_t)i;
    }
    first[3] = m;
    return t;
}

// ---- the launch plan of the RSA kernels, for the engine and the CPU simulation alike ----
// launch(kernel, lanes, items, args...) runs kernel(args...) over rsa_grid(items, lanes) blocks of RSA_BLOCK threads and
// returns 0 or an error code; lanes = RSA_GROUP for the kernels of a group per item, 1 for one thread per item.

// The shards the plan launches: a size and a hash tag of the set, and for PSS a salt length >= -1.
inline bool rsa_shard_ok(const RsaShard &s) {
    return rsa_size_ok(s.k) && rsa_hash_ok(s.hash) && (s.pad == RsaPad::pkcs1 || s.salt_len >= PSS_SALT_EQUALS_HASH);
}

// The PSS decoding of a shard alone: k_rsa_pss (with a slot per item k_rsa_pss_reg) over the EMs in s.sig, for the items
// s.ok accepts.  -1 with nothing launched for a shard rsa_shard_ok refuses.
template <class Launch>
int rsa_launch_pss_decode(const RsaShard &s, Launch &&launch) {
    if (!rsa_shard_ok(s)) return -1;
    if (s.n == 0) return 0;
    const uint32_t n = (uint32_t)s.n;
    int rc = 0;
    rsa_h(s.hash, [&](auto h) {
        constexpr int H = decltype(h)::value;
        if (s.slot) rc = launch(k_rsa_pss_reg<H>, 1, s.n, n, s.k, s.salt_len, s.sig, s.slot, s.rec, s.digest, s.ok);
        else rc = launch(k_rsa_pss<H>, 1, s.n, n, s.k, s.salt_len, s.sig, s.mod, s.digest, s.ok);
    });
    return rc;
}

// The kernels of one shard: PKCS #1 v1.5 k_rsa_verify; PSS k_rsa_em, which writes EM over s.sig, then the decoding.  With a
// slot per item, their _reg forms.  -1 with nothing launched for a shard rsa_shard_ok refuses; n = 0 launches nothing.
template <class Launch>
int rsa_launch_shard(const RsaShard &s, Launch &&launch) {
    if (!rsa_shard_ok(s)) return -1;
    if (s.n == 0) return 0;
    const bool pss = s.pad == RsaPad::pss, reg = s.slot != nullptr;
    const uint32_t n = (uint32_t)s.n;
    int rc = 0;
    rsa_nl(s.k, [&](auto nl) {
        constexpr int NL = decltype(nl)::value;
        if (!pss && reg) rc = launch(k_rsa_verify_reg<NL>, RSA_GROUP, s.n, n, s.hash, s.sig, s.slot, s.nslots, s.rec, s.pool, s.digest, s.ok);
        else if (!pss) rc = launch(k_rsa_verify<NL>, RSA_GROUP, s.n, n, s.hash, s.sig, s.mod, s.exp, s.digest, s.ok);
        else if (reg) rc = launch(k_rsa_em_reg<NL>, RSA_GROUP, s.n, n, s.sig, s.slot, s.nslots, s.rec, s.pool, s.ok);
        else rc = launch(k_rsa_em<NL>, RSA_GROUP, s.n, n, s.sig, s.mod, s.exp, s.ok);
    });
    if (rc || !pss) return rc;
    return rsa_launch_pss_decode(s, launch);
}

// The registry build: one k_rsa_kprep launch per modulus size present, over the slots of that size (slots, first and
// mod_off as rsa_reg_layout wrote them; mods and exps the registered moduli and exponents).
template <class Launch>
int rsa_launch_kprep(const uint32_t *slots, const size_t (&first)[4], const uint8_t *mods, const uint64_t *mod_off, const uint32_t *exps, uint4 *rec,
                     uint32_t *pool, Launch &&launch) {
    int rc = 0;
    for (int c = 0; c < 3 && !rc; c++) {
        const uint32_t cnt = (uint32_t)(first[c + 1] - first[c]);
        if (cnt == 0) continue;
        rsa_nl(256 + 128 * c, [&](auto nl) {
            rc = launch(k_rsa_kprep<decltype(nl)::value>, RSA_GROUP, cnt, cnt, slots + first[c], mods, mod_off, exps, rec, pool);
        });
    }
    return rc;
}

}  // namespace sbv
