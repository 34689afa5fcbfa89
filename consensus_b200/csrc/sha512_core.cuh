// sha512_core.cuh — the SHA-512 compression function and message loader (FIPS 180-4 §6.4), shared by SHA-512 (the
// Ed25519 challenge, sha512.cuh) and SHA-384 (the ECDSA digests of sbv_hash384_*, sha384.cuh).  No curve code here, so
// the ECDSA translation units include it without the Ed25519 headers.
//
// 64-bit words are register pairs: rotations are funnel shifts of the halves, additions carry-chained.  Messages are read
// with ALIGNED 32-bit loads and re-aligned with PRMT, as k_sha256 does.
#pragma once
#include <stdint.h>

#include "hostsim.h"

#ifndef SBV_DEV
#define SBV_DEV __device__ __forceinline__
#endif

namespace sbv {

__constant__ uint64_t SHA512_K[80] = {
    0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull,
    0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull,
    0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull,
    0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,
    0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull,
    0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,
    0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull,
    0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,
    0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull,
    0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull,
    0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull,
    0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
    0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull,
    0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull,
    0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull,
    0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull};

// rotate right by a constant: two funnel shifts of the 32-bit halves
SBV_DEV uint64_t rotr64(uint64_t x, int n) {
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    uint32_t rl, rh;
    if (n < 32) { rl = __funnelshift_r(lo, hi, n); rh = __funnelshift_r(hi, lo, n); }
    else { rl = __funnelshift_r(hi, lo, n - 32); rh = __funnelshift_r(lo, hi, n - 32); }
    return ((uint64_t)rh << 32) | rl;
}

SBV_DEV void sha512_compress(uint64_t (&h)[8], uint64_t (&w)[16]) {
    uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
    for (int i = 0; i < 80; i++) {
        if (i >= 16) {
            const uint64_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            const uint64_t s0 = rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7);
            const uint64_t s1 = rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6);
            w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
        }
        const uint64_t S1 = rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41);
        const uint64_t ch = (e & f) ^ (~e & g);
        const uint64_t t1 = hh + S1 + ch + SHA512_K[i] + w[i & 15];
        const uint64_t S0 = rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39);
        const uint64_t mj = (a & b) ^ (a & c) ^ (b & c);
        const uint64_t t2 = S0 + mj;
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// 16 big-endian words of the message stream from message byte mp on (mp a multiple of 4), with the 0x80 pad byte at
// message byte len and zeros after it.  words/sel/sh: the aligned view of the message (see k_sha256).
SBV_DEV void sha512_msg16(uint32_t *w, uint64_t mp, uint64_t len, const uint32_t *__restrict__ words, uint32_t sel, uint32_t sh) {
    const uint32_t *p = words + (mp >> 2);
    if (mp + 64 <= len) {
        uint32_t prev = __ldg(p);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const uint32_t next = (sh || j < 15) ? __ldg(p + j + 1) : 0u;
            w[j] = __byte_perm(prev, next, sel);
            prev = next;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const uint64_t q = mp + 4 * (uint64_t)j;
            uint32_t v = 0;
            if (q < len) {
                v = __byte_perm(__ldg(p + j), __ldg(p + j + 1), sel);
                const uint32_t rem = (uint32_t)(len - q);  // valid bytes in this word (>= 1)
                if (rem < 4) v = (v & (0xffffffffu << (8 * (4 - rem)))) | (0x80u << (8 * (3 - rem)));
            } else if (q == len) {
                v = 0x80000000u;
            }
            w[j] = v;
        }
    }
}

SBV_DEV uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

}  // namespace sbv
