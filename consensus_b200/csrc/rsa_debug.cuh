// rsa_debug.cuh — test hook of the RSA arithmetic of rsa.cuh (debug.cu on the device, tools/hostsim on the CPU): the
// production primitives item by item, in the production layout (blocks of 128 threads, two groups of 16 lanes per warp).
//
// Item i of every buffer: a, b, mod and out hold k = 64 * NL bytes big-endian, exp and aux one word.
//   op 0  out = a * b * R^-1 mod N (a, b < N), aux = n0' = -N^-1 mod 2^32
//   op 1  out = R^2 mod N, aux = n0'
//   op 2  out = a - N mod R, aux = the borrow out of the top limb (1: a < N)
//   op 3  out = the end of a product (rsa_resolve) on the limbs a and the lazy words b: lane l's word is the l-th
//         little-endian 32-bit word of b's item, weight 2^(32(l*NL+NL)); aux = 0
//   op 4  out = a^e mod N for a < N and e = exp[i], aux = n0'
// N = mod is odd with a nonzero top limb (rsa_r2 needs both, and every op takes n0').
#pragma once
#include <stddef.h>

#include "rsa.cuh"
#include "rsa_shard.h"

namespace sbv {

enum RsaDebugOp { RSA_DBG_MONT = 0, RSA_DBG_R2 = 1, RSA_DBG_SUB = 2, RSA_DBG_RESOLVE = 3, RSA_DBG_POW = 4 };

// The calls the hook runs: a modulus size of rsa.cuh, a known op, every buffer present and n < 2^31.
inline bool rsa_debug_args_ok(uint32_t mod_bytes, int op, size_t n, const void *a, const void *b, const void *mod, const void *exp, const void *out,
                              const void *aux) {
    return rsa_size_ok(mod_bytes) && op >= RSA_DBG_MONT && op <= RSA_DBG_POW && a && b && mod && exp && out && aux &&
           n < ((size_t)1 << 31);
}

// S^e mod N by the production primitives: S into Montgomery form (rsa_r2, rsa_mont), left-to-right square-and-multiply
// from acc = R mod N over every bit of e from its top bit down, and the product by 1.  A loop of its own, not the one of
// rsa_verify_item: it checks long chains of products, and the verdict sets check that loop.
template <int NL>
SBV_DEV void rsa_debug_pow(const RsaLanes &g, uint32_t (&r)[NL], const uint32_t (&s)[NL], uint32_t e, const uint32_t (&n)[NL], uint32_t ninv) {
    uint32_t r2[NL], sm[NL], one[NL];
    rsa_r2(g, r2, n, ninv);
    rsa_mont(g, sm, s, r2, n, ninv);
#pragma unroll
    for (int j = 0; j < NL; j++) one[j] = (g.l == 0 && j == 0) ? 1u : 0u;
    rsa_mont(g, r, r2, one, n, ninv);  // R mod N: 1 in Montgomery form
#pragma unroll 1
    for (int i = 31 - __clz((int)e); i >= 0; i--) {
        rsa_mont(g, r, r, r, n, ninv);
        if ((e >> i) & 1) rsa_mont(g, r, r, sm, n, ninv);
    }
    rsa_mont(g, r, r, one, n, ninv);
}

template <int NL>
__global__ void __launch_bounds__(128) k_rsa_debug(int op, uint32_t n, const uint8_t *__restrict__ a, const uint8_t *__restrict__ b,
                                                   const uint8_t *__restrict__ mod, const uint32_t *__restrict__ exp, uint8_t *__restrict__ out,
                                                   uint32_t *__restrict__ aux) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / RSA_GROUP;
    if (i >= n) return;  // the whole group
    constexpr uint32_t k = 64 * NL;
    const RsaLanes g = rsa_lanes();
    uint32_t x[NL], y[NL], nn[NL], r[NL];
    rsa_load(g, nn, mod + i * k, k);
    rsa_load(g, x, a + i * k, k);
    uint32_t w = 0;
    if (op == RSA_DBG_RESOLVE) {
        rsa_resolve(g, x, reinterpret_cast<const uint32_t *>(b + i * k)[g.l], nn);
#pragma unroll
        for (int j = 0; j < NL; j++) r[j] = x[j];
    } else if (op == RSA_DBG_SUB) {
        w = rsa_sub(g, r, x, nn);
    } else {
        w = rsa_ninv(g, nn);
        if (op == RSA_DBG_MONT) {
            rsa_load(g, y, b + i * k, k);
            rsa_mont(g, r, x, y, nn, w);
        } else if (op == RSA_DBG_R2) {
            rsa_r2(g, r, nn, w);
        } else {
            rsa_debug_pow(g, r, x, exp[i], nn, w);
        }
    }
    rsa_store(g, out + i * k, r, k);
    if (g.l == 0) aux[i] = w;
}

}  // namespace sbv
