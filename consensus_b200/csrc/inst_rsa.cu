// inst_rsa.cu — launchers of the RSA verification kernel (rsa.cuh, one instance per modulus size) and of k_sha512
// (sha512_batch.cuh) behind engine.h.
#include "engine.h"
#include "rsa.cuh"
#include "sha512_batch.cuh"

using namespace sbv;

int sbv_launch_sha512(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                      cudaStream_t st) {
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_msgs, d_off, base, d_digest, perm);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

int sbv_launch_rsa(sbv_engine *e, uint32_t mod_bytes, uint8_t hash, size_t n, const uint8_t *d_sig, const uint8_t *d_mod, const uint32_t *d_exp,
                   const uint8_t *d_digest, uint8_t *d_ok, cudaStream_t st) {
    if (n == 0) return 0;
    const uint32_t blocks = (uint32_t)((n * RSA_GROUP + 127) / 128);
    switch (mod_bytes) {
        case 256: k_rsa_verify<4><<<blocks, 128, 0, st>>>((uint32_t)n, hash, d_sig, d_mod, d_exp, d_digest, d_ok); break;
        case 384: k_rsa_verify<6><<<blocks, 128, 0, st>>>((uint32_t)n, hash, d_sig, d_mod, d_exp, d_digest, d_ok); break;
        case 512: k_rsa_verify<8><<<blocks, 128, 0, st>>>((uint32_t)n, hash, d_sig, d_mod, d_exp, d_digest, d_ok); break;
        default: return fail(e, SBV_ERR_ARG, "mod_bytes must be 256, 384 or 512");
    }
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
