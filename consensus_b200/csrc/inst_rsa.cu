// inst_rsa.cu — launchers of the RSA verification kernels (rsa.cuh, rsa_pss.cuh and, for registered keys, rsa_keyed.cuh: one
// instance per modulus size, and per hash for the PSS decoding), the build of the RSA key registry and k_sha512
// (sha512_batch.cuh) behind engine.h.
#include "engine.h"
#include "rsa.cuh"
#include "sha512_batch.cuh"
// after sha512_batch.cuh: SHA256_K (sha256_core.cuh) then lands after SHA512_K in the constant bank, where k_sha512 does
// not see it move
#include "rsa_pss.cuh"
#include "rsa_keyed.cuh"

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

int sbv_launch_rsa_pss(sbv_engine *e, uint32_t mod_bytes, uint8_t hash, int32_t salt_len, size_t n, uint8_t *d_sig, const uint8_t *d_mod,
                       const uint32_t *d_exp, const uint8_t *d_digest, uint8_t *d_ok, cudaStream_t st) {
    if (n == 0) return 0;
    const uint32_t blocks = (uint32_t)((n * RSA_GROUP + 127) / 128);
    switch (mod_bytes) {
        case 256: k_rsa_em<4><<<blocks, 128, 0, st>>>((uint32_t)n, d_sig, d_mod, d_exp, d_ok); break;
        case 384: k_rsa_em<6><<<blocks, 128, 0, st>>>((uint32_t)n, d_sig, d_mod, d_exp, d_ok); break;
        case 512: k_rsa_em<8><<<blocks, 128, 0, st>>>((uint32_t)n, d_sig, d_mod, d_exp, d_ok); break;
        default: return fail(e, SBV_ERR_ARG, "mod_bytes must be 256, 384 or 512");
    }
    e->launches += 1;
    CU(e, cudaGetLastError());
    const uint32_t tblocks = (uint32_t)((n + 127) / 128);
    switch (hash) {
        case SBV_HASH_SHA256: k_rsa_pss<0><<<tblocks, 128, 0, st>>>((uint32_t)n, mod_bytes, salt_len, d_sig, d_mod, d_digest, d_ok); break;
        case SBV_HASH_SHA384: k_rsa_pss<1><<<tblocks, 128, 0, st>>>((uint32_t)n, mod_bytes, salt_len, d_sig, d_mod, d_digest, d_ok); break;
        case SBV_HASH_SHA512: k_rsa_pss<2><<<tblocks, 128, 0, st>>>((uint32_t)n, mod_bytes, salt_len, d_sig, d_mod, d_digest, d_ok); break;
        default: return fail(e, SBV_ERR_ARG, "hash must be SBV_HASH_SHA256, SBV_HASH_SHA384 or SBV_HASH_SHA512");
    }
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

// ---- registered RSA keys ----
void sbv_rsa_keys_free(Dev &d) {
    if (d.rsa_rec) cudaFree(d.rsa_rec);
    if (d.rsa_pool) cudaFree(d.rsa_pool);
    d.rsa_rec = nullptr;
    d.rsa_pool = nullptr;
    d.rsa_n_slots = 0;
}

namespace {
// The registry of device d from the n keys: the moduli, their offsets and the exponents uploaded, then one k_rsa_kprep
// launch per modulus size present over the slots of that size.
int rsa_keys_fill(sbv_engine *e, Dev &d, size_t n, const uint32_t *mod_bytes, const uint8_t *modulus, const uint32_t *pub_exp) {
    std::vector<uint64_t> off(n);
    std::vector<uint32_t> slots(n);
    size_t first[4];
    const uint64_t total = rsa_reg_layout(n, mod_bytes, off.data(), slots.data(), first);
    CU(e, cudaMalloc(&d.rsa_rec, n * 2 * sizeof(uint4)));
    CU(e, cudaMalloc(&d.rsa_pool, total * 2));  // total / 2 words
    DevTemp tmp;
    uint8_t *d_mods = nullptr;
    uint64_t *d_off = nullptr;
    uint32_t *d_exp = nullptr, *d_slots = nullptr;
    CU(e, tmp.alloc(&d_mods, total));
    CU(e, tmp.alloc(&d_off, n * 8));
    CU(e, tmp.alloc(&d_exp, n * 4));
    CU(e, tmp.alloc(&d_slots, n * 4));
    CU(e, cudaMemcpyAsync(d_mods, modulus, total, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(d_off, off.data(), n * 8, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(d_exp, pub_exp, n * 4, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(d_slots, slots.data(), n * 4, cudaMemcpyHostToDevice, d.stream));
    for (int c = 0; c < 3; c++) {
        const uint32_t cnt = (uint32_t)(first[c + 1] - first[c]);
        if (cnt == 0) continue;
        const uint32_t blocks = (uint32_t)(((uint64_t)cnt * RSA_GROUP + 127) / 128);
        const uint32_t *sl = d_slots + first[c];
        if (c == 0) k_rsa_kprep<4><<<blocks, 128, 0, d.stream>>>(cnt, sl, d_mods, d_off, d_exp, d.rsa_rec, d.rsa_pool);
        else if (c == 1) k_rsa_kprep<6><<<blocks, 128, 0, d.stream>>>(cnt, sl, d_mods, d_off, d_exp, d.rsa_rec, d.rsa_pool);
        else k_rsa_kprep<8><<<blocks, 128, 0, d.stream>>>(cnt, sl, d_mods, d_off, d_exp, d.rsa_rec, d.rsa_pool);
        e->launches += 1;
        CU(e, cudaGetLastError());
    }
    CU(e, cudaStreamSynchronize(d.stream));  // before the temporaries are freed
    d.rsa_n_slots = (uint32_t)n;
    return 0;
}
}  // namespace

int sbv_rsa_keys_build(sbv_engine *e, Dev &d, size_t n, const uint32_t *mod_bytes, const uint8_t *modulus, const uint32_t *pub_exp) {
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, cudaDeviceSynchronize());  // no launch on any lane may still read the old registry
    sbv_rsa_keys_free(d);
    if (n == 0) return 0;
    const int rc = rsa_keys_fill(e, d, n, mod_bytes, modulus, pub_exp);
    if (rc) {
        cudaStreamSynchronize(d.stream);
        sbv_rsa_keys_free(d);
    }
    return rc;
}

int sbv_launch_rsa_reg(sbv_engine *e, Dev &d, uint32_t mod_bytes, uint8_t hash, size_t n, const uint8_t *d_sig, const uint32_t *d_slot,
                       const uint8_t *d_digest, uint8_t *d_ok, cudaStream_t st) {
    if (n == 0) return 0;
    const uint32_t blocks = (uint32_t)((n * RSA_GROUP + 127) / 128), ns = d.rsa_n_slots;
    switch (mod_bytes) {
        case 256: k_rsa_verify_reg<4><<<blocks, 128, 0, st>>>((uint32_t)n, hash, d_sig, d_slot, ns, d.rsa_rec, d.rsa_pool, d_digest, d_ok); break;
        case 384: k_rsa_verify_reg<6><<<blocks, 128, 0, st>>>((uint32_t)n, hash, d_sig, d_slot, ns, d.rsa_rec, d.rsa_pool, d_digest, d_ok); break;
        case 512: k_rsa_verify_reg<8><<<blocks, 128, 0, st>>>((uint32_t)n, hash, d_sig, d_slot, ns, d.rsa_rec, d.rsa_pool, d_digest, d_ok); break;
        default: return fail(e, SBV_ERR_ARG, "mod_bytes must be 256, 384 or 512");
    }
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

int sbv_launch_rsa_pss_reg(sbv_engine *e, Dev &d, uint32_t mod_bytes, uint8_t hash, int32_t salt_len, size_t n, uint8_t *d_sig, const uint32_t *d_slot,
                           const uint8_t *d_digest, uint8_t *d_ok, cudaStream_t st) {
    if (n == 0) return 0;
    const uint32_t blocks = (uint32_t)((n * RSA_GROUP + 127) / 128), ns = d.rsa_n_slots;
    switch (mod_bytes) {
        case 256: k_rsa_em_reg<4><<<blocks, 128, 0, st>>>((uint32_t)n, d_sig, d_slot, ns, d.rsa_rec, d.rsa_pool, d_ok); break;
        case 384: k_rsa_em_reg<6><<<blocks, 128, 0, st>>>((uint32_t)n, d_sig, d_slot, ns, d.rsa_rec, d.rsa_pool, d_ok); break;
        case 512: k_rsa_em_reg<8><<<blocks, 128, 0, st>>>((uint32_t)n, d_sig, d_slot, ns, d.rsa_rec, d.rsa_pool, d_ok); break;
        default: return fail(e, SBV_ERR_ARG, "mod_bytes must be 256, 384 or 512");
    }
    e->launches += 1;
    CU(e, cudaGetLastError());
    const uint32_t tblocks = (uint32_t)((n + 127) / 128);
    switch (hash) {
        case SBV_HASH_SHA256: k_rsa_pss_reg<0><<<tblocks, 128, 0, st>>>((uint32_t)n, mod_bytes, salt_len, d_sig, d_slot, d.rsa_rec, d_digest, d_ok); break;
        case SBV_HASH_SHA384: k_rsa_pss_reg<1><<<tblocks, 128, 0, st>>>((uint32_t)n, mod_bytes, salt_len, d_sig, d_slot, d.rsa_rec, d_digest, d_ok); break;
        case SBV_HASH_SHA512: k_rsa_pss_reg<2><<<tblocks, 128, 0, st>>>((uint32_t)n, mod_bytes, salt_len, d_sig, d_slot, d.rsa_rec, d_digest, d_ok); break;
        default: return fail(e, SBV_ERR_ARG, "hash must be SBV_HASH_SHA256, SBV_HASH_SHA384 or SBV_HASH_SHA512");
    }
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
