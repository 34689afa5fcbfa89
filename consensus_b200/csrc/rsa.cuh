// rsa.cuh — RSA PKCS #1 v1.5 signature verification (RFC 8017 §8.2.2, Go's crypto/rsa.VerifyPKCS1v15) for moduli of
// 2048, 3072 and 4096 bits (k = 256, 384 or 512 bytes), a group of 16 lanes per signature, two signatures per warp.  The
// key rule, the range check and the exponentiation (rsa_recover) serve RSA-PSS too (rsa_pss.cuh); the exponentiation from
// S * R onward (rsa_pow_tail) and the encoding compare (rsa_pkcs1_match) serve the registered keys (rsa_keyed.cuh).
//
// Layout.  A k-byte number is K = k/4 little-endian 32-bit limbs; lane l of the group holds limbs [l*NL, l*NL + NL),
// NL = K/16 = 4, 6 or 8, of every operand.  Values cross the group only by shuffle and ballot under the group's mask.
//
// Montgomery multiplication (R = 2^(32K)), row form: for each limb a_i of a (broadcast from its owner lane), every lane
// adds a_i*b over its limbs; the quotient digit q = t_0 * n0' is taken from the lowest limb of the group (lane 0's t[0],
// which is exact: every pending carry sits above it), every lane adds q*N, and the accumulator moves down one limb, the
// lowest limb of lane l+1 into the top limb of lane l.  The carries out of each lane's top limb stay lazy in one word per
// lane (`cz`, weight 2^(32(l*NL+NL))) that rides along with the shift; they are resolved once after the K rows: every lane
// adds the word of the lane below, and the remaining 0/1 carries between lanes are settled with a ballot of
// generate / propagate bits.  The final conditional subtraction resolves its borrows the same way.
//
// Setup, with no division: n0' = -N^-1 mod 2^32 by Newton iteration; R^2 mod N by modular doublings and five Montgomery
// squarings (rsa_r2).  Then S -> S*R, left-to-right square-and-multiply over the bits of e, and one product by 1 leaves
// EM = S^e mod N, which is compared limb by limb with the expected encoding built in registers from (k, hash, H).  EM is
// never written to memory.
#pragma once
#include <stdint.h>

#include "hostsim.h"

#ifndef SBV_DEV
#define SBV_DEV __device__ __forceinline__
#endif

namespace sbv {

constexpr int RSA_GROUP = 16;  // lanes per signature

// the DigestInfo prefixes of RFC 8017 §9.2 note 1 (with the NULL parameters): SHA-256, SHA-384, SHA-512
__constant__ uint8_t RSA_DIGEST_INFO[3][19] = {
    {0x30, 0x31, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x01, 0x05, 0x00, 0x04, 0x20},
    {0x30, 0x41, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x02, 0x05, 0x00, 0x04, 0x30},
    {0x30, 0x51, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x03, 0x05, 0x00, 0x04, 0x40}};

// This lane's place in its group: the group's shuffle mask, the warp lane of its lane 0, and its index in the group.
struct RsaLanes {
    unsigned mask;
    int base, l;
};
SBV_DEV RsaLanes rsa_lanes() {
    const int lane = (int)(threadIdx.x & 31);
    return RsaLanes{0xffffu << (lane & 16), lane & 16, lane & 15};
}
SBV_DEV uint32_t rsa_from(const RsaLanes &g, uint32_t v, int src) { return __shfl_sync(g.mask, v, g.base + src); }
// bit l = p of group lane l
SBV_DEV uint32_t rsa_bits(const RsaLanes &g, bool p) { return (__ballot_sync(g.mask, p) >> g.base) & 0xffffu; }

// The limbs of this lane from a k-byte big-endian number at p (4-byte aligned), and back.
template <int NL>
SBV_DEV void rsa_load(const RsaLanes &g, uint32_t (&x)[NL], const uint8_t *p, uint32_t k) {
#pragma unroll
    for (int j = 0; j < NL; j++) x[j] = __byte_perm(*reinterpret_cast<const uint32_t *>(p + k - 4 * (g.l * NL + j) - 4), 0, 0x0123);
}
template <int NL>
SBV_DEV void rsa_store(const RsaLanes &g, uint8_t *p, const uint32_t (&x)[NL], uint32_t k) {
#pragma unroll
    for (int j = 0; j < NL; j++) *reinterpret_cast<uint32_t *>(p + k - 4 * (g.l * NL + j) - 4) = __byte_perm(x[j], 0, 0x0123);
}

// d = x - y over the whole group; returns the borrow out of the top limb (1: x < y).  Each lane subtracts its limbs with
// a local borrow chain; the borrows between lanes are resolved at once: lane l generates a borrow if its chain does, and
// propagates one if its difference is zero, so the borrow into each lane is ((G << 1) + P) ^ P, bit 16 the borrow out.
template <int NL>
SBV_DEV uint32_t rsa_sub(const RsaLanes &g, uint32_t (&d)[NL], const uint32_t (&x)[NL], const uint32_t (&y)[NL]) {
    uint32_t b = 0, z = 0;
#pragma unroll
    for (int j = 0; j < NL; j++) {
        const uint64_t s = (uint64_t)x[j] - y[j] - b;
        d[j] = (uint32_t)s;
        b = (uint32_t)(s >> 63);
        z |= d[j];
    }
    const uint32_t gen = rsa_bits(g, b != 0), prop = rsa_bits(g, z == 0);
    const uint32_t bin = ((gen << 1) + prop) ^ prop;
    uint32_t c = (bin >> g.l) & 1;
#pragma unroll
    for (int j = 0; j < NL; j++) {
        const uint64_t s = (uint64_t)d[j] - c;
        d[j] = (uint32_t)s;
        c = (uint32_t)(s >> 63);
    }
    return (bin >> 16) & 1;
}

// x + top*R < 2N (top: 0 or 1, the same in every lane) -> x mod N
template <int NL>
SBV_DEV void rsa_csub(const RsaLanes &g, uint32_t (&x)[NL], uint32_t top, const uint32_t (&n)[NL]) {
    uint32_t d[NL];
    const uint32_t borrow = rsa_sub(g, d, x, n);
    if (top || !borrow) {
#pragma unroll
        for (int j = 0; j < NL; j++) x[j] = d[j];
    }
}

// (t, cz) += x * y over this lane's limbs: the carry out of the top limb goes to the lazy word cz
template <int NL>
SBV_DEV void rsa_row(uint32_t (&t)[NL], uint64_t &cz, uint32_t x, const uint32_t (&y)[NL]) {
    uint32_t c = 0;
#pragma unroll
    for (int j = 0; j < NL; j++) {
        const uint64_t p = (uint64_t)x * y[j] + t[j] + c;
        t[j] = (uint32_t)p;
        c = (uint32_t)(p >> 32);
    }
    cz += c;
}

// The end of a Montgomery product: the value t + czl * 2^(32(l*NL+NL)) summed over the lanes (czl <= 3, t any limbs) is
// below 2N; it leaves t = that value mod N.  Carry resolution: every lane adds the lazy word of the lane below; the 0/1
// carries that leaves between lanes are settled by ballot (generate: the lane's add carried out; propagate: the lane is
// all ones), bit 16 being the carry out of the top lane.  Then the conditional subtraction.
template <int NL>
SBV_DEV void rsa_resolve(const RsaLanes &g, uint32_t (&t)[NL], uint32_t czl, const uint32_t (&n)[NL]) {
    uint32_t c = rsa_from(g, czl, g.l ? g.l - 1 : 0), ones = 0xffffffffu;
    if (g.l == 0) c = 0;
#pragma unroll
    for (int j = 0; j < NL; j++) {
        const uint64_t s = (uint64_t)t[j] + c;
        t[j] = (uint32_t)s;
        c = (uint32_t)(s >> 32);
        ones &= t[j];
    }
    const uint32_t gen = rsa_bits(g, c != 0), prop = rsa_bits(g, ones == 0xffffffffu);
    const uint32_t cin = ((gen << 1) + prop) ^ prop;
    c = (cin >> g.l) & 1;
#pragma unroll
    for (int j = 0; j < NL; j++) {
        const uint64_t s = (uint64_t)t[j] + c;
        t[j] = (uint32_t)s;
        c = (uint32_t)(s >> 32);
    }
    const uint32_t top = ((cin >> 16) & 1) + rsa_from(g, czl, RSA_GROUP - 1);
    rsa_csub(g, t, top, n);
}

// r = a * b * R^-1 mod N for a, b < N (r may be a or b).  ninv = -N^-1 mod 2^32.
//
// Bound of the lazy word: it is at most 3 when a row starts (0 at the first); the two products add at most 2^32 - 1
// each, and the shift takes it back to (t + cz) >> 32 <= (2^32 - 1 + 3 + 2^33 - 2) >> 32 = 3.  So after the K rows it
// fits a limb, and the accumulator is below 2N < 2R (a, b < N), so the top after resolution is 0 or 1.
template <int NL>
SBV_DEV void rsa_mont(const RsaLanes &g, uint32_t (&r)[NL], const uint32_t (&a)[NL], const uint32_t (&b)[NL], const uint32_t (&n)[NL], uint32_t ninv) {
    uint32_t t[NL];
#pragma unroll
    for (int j = 0; j < NL; j++) t[j] = 0;
    uint64_t cz = 0;
    const int up = g.l < RSA_GROUP - 1 ? g.l + 1 : g.l;
#pragma unroll 1
    for (int o = 0; o < RSA_GROUP; o++) {
#pragma unroll
        for (int jj = 0; jj < NL; jj++) {
            rsa_row(t, cz, rsa_from(g, a[jj], o), b);  // a_i, i = o*NL + jj
            const uint32_t q = rsa_from(g, t[0], 0) * ninv;
            rsa_row(t, cz, q, n);  // the lowest limb of the group is now 0
            uint32_t nx = rsa_from(g, t[0], up);
            if (g.l == RSA_GROUP - 1) nx = 0;
#pragma unroll
            for (int j = 0; j < NL - 1; j++) t[j] = t[j + 1];
            const uint64_t s = (uint64_t)nx + cz;
            t[NL - 1] = (uint32_t)s;
            cz = s >> 32;
        }
    }
    rsa_resolve(g, t, (uint32_t)cz, n);
#pragma unroll
    for (int j = 0; j < NL; j++) r[j] = t[j];
}

// -N^-1 mod 2^32 for odd N: x = n0 is an inverse mod 2^3 (n0^2 = 1 mod 8), and each Newton step x *= 2 - n0*x doubles the
// correct bits: 6, 12, 24, 48.
template <int NL>
SBV_DEV uint32_t rsa_ninv(const RsaLanes &g, const uint32_t (&n)[NL]) {
    const uint32_t n0 = rsa_from(g, n[0], 0);
    uint32_t x = n0;
#pragma unroll
    for (int i = 0; i < 4; i++) x *= 2u - n0 * x;
    return 0u - x;
}

// R^2 mod N for an odd N whose top limb is nonzero.  With b = bit length of N, x = 2^(b-1) < N (N is odd, so it is not
// 2^(b-1) itself).  33K - b + 1 modular doublings take x to 2^(33K) = R * 2^K mod N; a Montgomery squaring maps
// R * 2^s to R * 2^(2s), so five of them give R * 2^(32K) = R^2 mod N.  (For k = 256 that is R * 2^64 and 65 to 72
// doublings; K + 1 to K + 32 doublings in general.)
template <int NL>
SBV_DEV void rsa_r2(const RsaLanes &g, uint32_t (&x)[NL], const uint32_t (&n)[NL], uint32_t ninv) {
    constexpr int K = RSA_GROUP * NL;
    const uint32_t ntop = rsa_from(g, n[NL - 1], RSA_GROUP - 1);
    const int b = 32 * K - __clz((int)ntop);
    const int pos = b - 1;
#pragma unroll
    for (int j = 0; j < NL; j++) x[j] = (g.l * NL + j == (pos >> 5)) ? 1u << (pos & 31) : 0u;
    const int down = g.l ? g.l - 1 : 0;
#pragma unroll 1
    for (int i = 0; i < 33 * K - b + 1; i++) {
        const uint32_t hi = x[NL - 1] >> 31;
        uint32_t in = rsa_from(g, hi, down);
        if (g.l == 0) in = 0;
        const uint32_t top = rsa_from(g, hi, RSA_GROUP - 1);
#pragma unroll
        for (int j = NL - 1; j > 0; j--) x[j] = (x[j] << 1) | (x[j - 1] >> 31);
        x[0] = (x[0] << 1) | in;
        rsa_csub(g, x, top, n);
    }
#pragma unroll 1
    for (int i = 0; i < 5; i++) rsa_mont(g, x, x, x, n, ninv);
}

// Step 3 from S * R onward, shared by the keys carried per item (rsa_recover) and the registered keys (rsa_keyed.cuh):
// s = S < N, x = R^2 mod N on entry (scratch after), ninv = -N^-1 mod 2^32, e the public exponent; returns tail(em), em =
// S^e mod N, this lane's limbs.  sm (S * R) and acc are the caller's arrays: declared there, ahead of rsa_r2, the keys-per-
// item kernels compile to the same instructions as before this function was split out.
template <int NL, class Tail>
SBV_DEV bool rsa_pow_tail(const RsaLanes &g, const uint32_t (&s)[NL], uint32_t (&x)[NL], const uint32_t (&n)[NL], uint32_t ninv, uint32_t e,
                          uint32_t (&sm)[NL], uint32_t (&acc)[NL], Tail &&tail) {
    rsa_mont(g, sm, s, x, n, ninv);  // S * R mod N
    // left to right over the bits of e below its top bit: square, and multiply by S*R where the bit is set
#pragma unroll
    for (int j = 0; j < NL; j++) acc[j] = sm[j];
    int i = 30 - __clz((int)e);
    bool mul = false;
#pragma unroll 1
    while (i >= 0) {
        uint32_t m[NL];
#pragma unroll
        for (int j = 0; j < NL; j++) m[j] = mul ? sm[j] : acc[j];
        rsa_mont(g, acc, acc, m, n, ninv);
        if (mul) { mul = false; i--; }
        else if ((e >> i) & 1) mul = true;
        else i--;
    }
#pragma unroll
    for (int j = 0; j < NL; j++) x[j] = (g.l == 0 && j == 0) ? 1u : 0u;
    rsa_mont(g, acc, acc, x, n, ninv);  // EM = S^e mod N
    return tail(acc);
}

// Steps 1-3 of both paddings (the same in every lane of the group): false if the key rule or S < N refuses the item, else
// tail(em), em = S^e mod N, this lane's limbs.  sig, mod: k bytes big-endian; e: the public exponent.  The padding's part
// is a callable rather than a caller testing a flag, so that every refusal returns straight out of the kernel's item.
template <int NL, class Tail>
SBV_DEV bool rsa_recover(const RsaLanes &g, const uint8_t *sig, const uint8_t *mod, uint32_t e, Tail &&tail) {
    constexpr int K = RSA_GROUP * NL;
    constexpr uint32_t k = 4 * K;
    uint32_t n[NL], s[NL], x[NL];
    rsa_load(g, n, mod, k);
    rsa_load(g, s, sig, k);
    // the key: N odd, N's leading byte nonzero, 2 <= e <= 2^31 - 1
    const uint32_t n0 = rsa_from(g, n[0], 0), ntop = rsa_from(g, n[NL - 1], RSA_GROUP - 1);
    if (!(n0 & 1) || (ntop >> 24) == 0 || e < 2 || e > 0x7fffffffu) return false;
    // the range: S < N
    if (!rsa_sub(g, x, s, n)) return false;
    const uint32_t ninv = rsa_ninv(g, n);
    uint32_t sm[NL], acc[NL];
    rsa_r2(g, x, n, ninv);
    return rsa_pow_tail<NL>(g, s, x, n, ninv, e, sm, acc, tail);
}

// Step 4 of PKCS #1 v1.5 (the same in every lane of the group): em = this lane's limbs of S^e mod N; h: the hLen-byte
// digest, hash 0 / 1 / 2 = SHA-256 / SHA-384 / SHA-512.
template <int NL>
SBV_DEV bool rsa_pkcs1_match(const RsaLanes &g, const uint32_t (&acc)[NL], const uint8_t *h, uint32_t hash) {
    constexpr uint32_t k = 64 * NL;
    // EM = 00 || 01 || FF..FF || 00 || DigestInfo || H, by bytes counted from the end (r = 0 is the last byte)
    const uint32_t hl = 32 + 16 * hash, tl = hl + 19;
    uint32_t bad = 0;
#pragma unroll
    for (int j = 0; j < NL; j++) {
        uint32_t w = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t r = 4 * (g.l * NL + j) + q;
            uint32_t v;
            if (r < hl) v = h[hl - 1 - r];
            else if (r < tl) v = RSA_DIGEST_INFO[hash][tl - 1 - r];
            else if (r == tl) v = 0x00;
            else if (r < k - 2) v = 0xff;
            else if (r == k - 2) v = 0x01;
            else v = 0x00;
            w |= v << (8 * q);
        }
        bad |= w ^ acc[j];
    }
    return rsa_bits(g, bad != 0) == 0;
}

// The PKCS #1 v1.5 verdict of one item (the same in every lane of the group).  sig, mod: k bytes big-endian; e: the public
// exponent; h: the hLen-byte digest, hash 0 / 1 / 2 = SHA-256 / SHA-384 / SHA-512.
template <int NL>
SBV_DEV bool rsa_verify_item(const RsaLanes &g, const uint8_t *sig, const uint8_t *mod, uint32_t e, const uint8_t *h, uint32_t hash) {
    return rsa_recover<NL>(g, sig, mod, e, [&](const uint32_t (&acc)[NL]) { return rsa_pkcs1_match<NL>(g, acc, h, hash); });
}

// One item per group of 16 lanes: ok[i] = 1 iff sig i (k bytes) is a valid PKCS #1 v1.5 signature of digest i (hLen
// bytes) under the key (mod i, pub_exp[i]); k = 64 * NL.
template <int NL>
__global__ void __launch_bounds__(128) k_rsa_verify(uint32_t n, uint32_t hash, const uint8_t *__restrict__ sig, const uint8_t *__restrict__ mod,
                                                    const uint32_t *__restrict__ pub_exp, const uint8_t *__restrict__ digest, uint8_t *__restrict__ ok) {
    // 64-bit: a grid of n < 2^31 items has up to 2^35 threads
    const uint64_t item = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / RSA_GROUP;
    if (item >= n) return;  // the whole group
    constexpr uint32_t k = 64 * NL;
    const RsaLanes g = rsa_lanes();
    const bool v = rsa_verify_item<NL>(g, sig + item * k, mod + item * k, pub_exp[item], digest + item * (32 + 16 * hash), hash);
    if (g.l == 0) ok[item] = v ? 1 : 0;
}

}  // namespace sbv
