// rsa_pss.cuh — RSA-PSS signature verification (RFC 8017 §8.1.2 with the EMSA-PSS decoding of §9.1.2, Go's
// crypto/rsa.VerifyPSS) for the moduli of rsa.cuh, MGF1 over the message hash (SHA-256, SHA-384 or SHA-512).  Two kernels:
//
//   k_rsa_em<NL>  a group of 16 lanes per item, as k_rsa_verify: the key rule, S < N and EM = S^e mod N (rsa_recover),
//                 EM written big-endian over the item's signature, and the key and range verdict into ok;
//   k_rsa_pss<H>  one thread per item over that EM (the items ok refuses are skipped): steps 2-8 of the accept set in
//                 include/sbv.h, the verdict ANDed into ok.  DB is unmasked in place over maskedDB.
//
// The byte logic runs in plain per-thread code, away from the shuffles of the exponentiation.  Every MGF1 block is one
// compression (hLen + 4 bytes fit one block of each hash); M' = 0^8 || mHash || salt takes one to nine.
#pragma once
#include <stdint.h>

#include "rsa.cuh"
#include "sha256_core.cuh"
#include "sha512_core.cuh"

namespace sbv {

constexpr int32_t PSS_SALT_EQUALS_HASH = -1, PSS_SALT_AUTO = 0;  // salt_len as Go's PSSOptions.SaltLength

// One item per group of 16 lanes: EM = S^e mod N over sig (k = 64 * NL bytes per item) where the key rule and S < N
// accept the item, and ok[i] = 1 there, else 0 (sig left as it was).
template <int NL>
__global__ void __launch_bounds__(128) k_rsa_em(uint32_t n, uint8_t *__restrict__ sig, const uint8_t *__restrict__ mod, const uint32_t *__restrict__ pub_exp,
                                                uint8_t *__restrict__ ok) {
    // 64-bit: a grid of n < 2^31 items has up to 2^35 threads
    const uint64_t item = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / RSA_GROUP;
    if (item >= n) return;  // the whole group
    constexpr uint32_t k = 64 * NL;
    const RsaLanes g = rsa_lanes();
    uint8_t *s = sig + item * k;
    const bool v = rsa_recover<NL>(g, s, mod + item * k, pub_exp[item], [&](const uint32_t (&em)[NL]) {
        rsa_store(g, s, em, k);  // each lane writes the limbs it loaded
        return true;
    });
    if (g.l == 0) ok[item] = v ? 1 : 0;
}

// The big-endian word at p (any alignment)
SBV_DEV uint32_t pss_be32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

// The hash of tag H (0 / 1 / 2: SHA-256 / SHA-384 / SHA-512) over messages given as 32-bit big-endian words, BW of them
// per block; word(i) is the i-th big-endian word of the digest (i < HL / 4).
template <int H> struct PssSha;
template <> struct PssSha<0> {
    static constexpr uint32_t HL = 32, BW = 16;
    uint32_t h[8];
    SBV_DEV PssSha() {
        h[0] = 0x6a09e667; h[1] = 0xbb67ae85; h[2] = 0x3c6ef372; h[3] = 0xa54ff53a;
        h[4] = 0x510e527f; h[5] = 0x9b05688c; h[6] = 0x1f83d9ab; h[7] = 0x5be0cd19;
    }
    SBV_DEV void compress(uint32_t (&w)[BW]) { sha256_compress(h, w); }
    SBV_DEV uint32_t word(int i) const { return h[i]; }
};
template <int H> struct PssSha {
    static_assert(H == 1 || H == 2, "hash tag");
    static constexpr uint32_t HL = H == 1 ? 48 : 64, BW = 32;
    uint64_t h[8];
    SBV_DEV PssSha() {
        if (H == 1) {
            h[0] = 0xcbbb9d5dc1059ed8ull; h[1] = 0x629a292a367cd507ull; h[2] = 0x9159015a3070dd17ull; h[3] = 0x152fecd8f70e5939ull;
            h[4] = 0x67332667ffc00b31ull; h[5] = 0x8eb44a8768581511ull; h[6] = 0xdb0c2e0d64f98fa7ull; h[7] = 0x47b5481dbefa4fa4ull;
        } else {
            h[0] = 0x6a09e667f3bcc908ull; h[1] = 0xbb67ae8584caa73bull; h[2] = 0x3c6ef372fe94f82bull; h[3] = 0xa54ff53a5f1d36f1ull;
            h[4] = 0x510e527fade682d1ull; h[5] = 0x9b05688c2b3e6c1full; h[6] = 0x1f83d9abfb41bd6bull; h[7] = 0x5be0cd19137e2179ull;
        }
    }
    SBV_DEV void compress(uint32_t (&w)[BW]) {
        uint64_t x[16];
#pragma unroll
        for (int j = 0; j < 16; j++) x[j] = ((uint64_t)w[2 * j] << 32) | w[2 * j + 1];
        sha512_compress(h, x);
    }
    SBV_DEV uint32_t word(int i) const { return (uint32_t)(h[i >> 1] >> ((i & 1) ? 0 : 32)); }
};

// Hash(M') for M' = 0^8 || mHash || salt (slen bytes of salt), read byte by byte; the padding of FIPS 180-4 §5.1 with a
// bit length below 2^32.
template <int H>
SBV_DEV void pss_mprime(PssSha<H> &s, const uint8_t *mhash, const uint8_t *salt, uint32_t slen) {
    constexpr uint32_t HL = PssSha<H>::HL, BW = PssSha<H>::BW, B = 4 * BW, Z = 8;  // Z: the zero bytes that open M'
    const uint32_t len = Z + HL + slen;
    const uint32_t nb = (len + 1 + B / 8 + B - 1) / B;  // the 0x80 byte and the 8- or 16-byte length fit after M'
    for (uint32_t b = 0; b < nb; b++) {
        uint32_t w[BW];
#pragma unroll
        for (uint32_t j = 0; j < BW; j++) {
            uint32_t v = 0;
#pragma unroll
            for (uint32_t q = 0; q < 4; q++) {
                const uint32_t p = b * B + 4 * j + q;
                uint32_t c = 0;
                if (p >= Z && p < Z + HL) c = mhash[p - Z];
                else if (p >= Z + HL && p < len) c = salt[p - Z - HL];
                else if (p == len) c = 0x80;
                v = (v << 8) | c;
            }
            w[j] = v;
        }
        if (b == nb - 1) w[BW - 1] = len * 8;
        s.compress(w);
    }
}

// Steps 2-8 of the accept set for one item: em = EM (k bytes, unmasked in place), ntop = N's leading byte (nonzero: the key
// rule has passed), mhash = the HL-byte digest.
template <int H>
SBV_DEV bool pss_decode(uint8_t *em, uint32_t k, uint32_t ntop, const uint8_t *mhash, int32_t salt_len) {
    using Sha = PssSha<H>;
    constexpr uint32_t HL = Sha::HL, HW = HL / 4;
    // 2. emBits = bitlen(N) - 1 and emLen = ceil(emBits / 8): k - 1 when N's leading byte is 01, and then EM's leading byte
    //    must be 0 and is dropped.  zb = 8 emLen - emBits, the top bits of maskedDB[0] that must be clear.
    const uint32_t lead = ntop == 1 ? 1 : 0;
    if (lead && em[0] != 0) return false;
    em += lead;
    const uint32_t emLen = k - lead, zb = lead ? 0 : (uint32_t)__clz((int)ntop) - 23, keep = 0xffu >> zb;
    // 3. the salt length (hLen for EqualsHash, 0 for the bound in auto mode), compared in 64 bits
    const int64_t sl = salt_len == PSS_SALT_EQUALS_HASH ? (int64_t)HL : (int64_t)salt_len;
    if ((int64_t)emLen < (int64_t)HL + sl + 2) return false;
    // 4. the trailer
    if (em[emLen - 1] != 0xbc) return false;
    // 5. maskedDB = the first dbLen bytes, H_em the next HL bytes
    const uint32_t dbLen = emLen - HL - 1;
    if (em[0] & ~keep) return false;
    const uint8_t *hem = em + dbLen;
    uint32_t hw[HW];  // H_em, big-endian words
#pragma unroll
    for (uint32_t j = 0; j < HW; j++) hw[j] = pss_be32(hem + 4 * j);
    // 6. DB = maskedDB ^ MGF1(H_em, dbLen), block c = Hash(H_em || BE32(c)); then the top zb bits of DB[0] cleared
    uint8_t *db = em;
    for (uint32_t c = 0; c * HL < dbLen; c++) {
        uint32_t w[Sha::BW];
#pragma unroll
        for (uint32_t j = 0; j < Sha::BW; j++) w[j] = j < HW ? hw[j] : j == HW ? c : j == HW + 1 ? 0x80000000u : 0u;
        w[Sha::BW - 1] = (HL + 4) * 8;
        Sha s;
        s.compress(w);
#pragma unroll
        for (uint32_t t = 0; t < HL; t++) {
            const uint32_t p = c * HL + t;
            if (p < dbLen) db[p] ^= (uint8_t)(s.word(t >> 2) >> (24 - 8 * (t & 3)));
        }
    }
    db[0] &= keep;
    // 7. PS = zero bytes up to the 01 separator; the salt is everything after it, of the length salt_len asks for
    uint32_t ps = 0;
    while (ps < dbLen && db[ps] == 0) ps++;
    if (ps == dbLen || db[ps] != 0x01) return false;
    const uint32_t slen = dbLen - ps - 1;
    if (salt_len != PSS_SALT_AUTO && (int64_t)slen != sl) return false;
    // 8. accept iff Hash(0^8 || mHash || salt) = H_em (read again: hw is not kept live across the hash)
    Sha s;
    pss_mprime<H>(s, mhash, db + ps + 1, slen);
    uint32_t diff = 0;
#pragma unroll
    for (uint32_t j = 0; j < HW; j++) diff |= s.word(j) ^ pss_be32(hem + 4 * j);
    return diff == 0;
}

// One item per thread after k_rsa_em: em and mod k bytes per item, digest HL bytes per item; ok[i] &= the PSS verdict.
template <int H>
__global__ void __launch_bounds__(128) k_rsa_pss(uint32_t n, uint32_t k, int32_t salt_len, uint8_t *__restrict__ em, const uint8_t *__restrict__ mod,
                                                 const uint8_t *__restrict__ digest, uint8_t *__restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !ok[i]) return;
    const bool v = pss_decode<H>(em + (size_t)i * k, k, mod[(size_t)i * k], digest + (size_t)i * PssSha<H>::HL, salt_len);
    ok[i] = v ? 1 : 0;
}

}  // namespace sbv
