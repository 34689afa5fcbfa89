// inst_ed25519.cu — launchers of the Ed25519 kernels (sha512.cuh, ed25519_verify.cuh) behind engine.h.
#include "engine.h"
#include "ed25519_verify.cuh"
#include "sha512.cuh"

using namespace sbv;

namespace {
constexpr int ED_BLOCK = 32;  // 32 KiB of shared memory per block (the 1A..8A tables): no opt-in attribute needed
constexpr size_t ED_SMEM = (size_t)8 * 4 * 8 * 4 * ED_BLOCK;
}  // namespace
static_assert(SBV_ED_BTAB_ENTRIES == (size_t)ED_BWINS * ED_BENT && SBV_ED_BTAB_ENTRY_WORDS == ED_BWORDS, "engine.h: table of B");

// The fixed-base table of B, built on the first Ed25519 call of each device.  Caller holds e->mu and has set the device.
// The build is synchronised before the pointer is published, so a verification on any stream sees a finished table.
int sbv_ed_btab_ensure(sbv_engine *e, Dev &d) {
    if (d.ed_btab) return 0;
    uint32_t *t = nullptr;
    CU(e, cudaMalloc(&t, ED_BTAB_WORDS * sizeof(uint32_t)));
    k_ed_btab_init<<<(ED_BWINS * ED_BENT + 63) / 64, 64, 0, d.stream>>>(t);
    e->launches += 1;
    cudaError_t st = cudaGetLastError();
    if (st == cudaSuccess) st = cudaStreamSynchronize(d.stream);
    if (st != cudaSuccess) {
        cudaFree(t);
        return sbv_fail(e, SBV_ERR_CUDA, "k_ed_btab_init: %s", cudaGetErrorString(st));
    }
    d.ed_btab = t;
    return 0;
}

int sbv_launch_ed25519(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint8_t *d_sig,
                       const uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st) {
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_ed_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_sig, d_pub, d_msgs, d_off, base, d_k, perm, nullptr);
    k_ed_verify<ED_BLOCK><<<(uint32_t)((n + ED_BLOCK - 1) / ED_BLOCK), ED_BLOCK, ED_SMEM, st>>>(
        (uint32_t)n, d_sig, d_pub, d_k, reinterpret_cast<const uint4 *>(d.ed_btab), d_ok);
    e->launches += 2;
    CU(e, cudaGetLastError());
    return 0;
}

// test hook (debug.cu): the production SHA-512 kernel with its digests written out as well
int sbv_launch_ed_sha512_digest(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, const uint8_t *d_sig, const uint8_t *d_pub,
                                uint32_t *d_k, uint32_t *d_dig, cudaStream_t st) {
    k_ed_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_sig, d_pub, d_msgs, d_off, 0, d_k, nullptr, d_dig);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}

// test hook (debug.cu): the production verification kernel with the caller's k (word-major, every k < L) in place of
// SHA-512's.  The table of B must exist (sbv_ed_btab_ensure).
int sbv_launch_ed_verify_k(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_sig, const uint8_t *d_pub, const uint32_t *d_k, uint8_t *d_ok,
                           cudaStream_t st) {
    k_ed_verify<ED_BLOCK><<<(uint32_t)((n + ED_BLOCK - 1) / ED_BLOCK), ED_BLOCK, ED_SMEM, st>>>(
        (uint32_t)n, d_sig, d_pub, d_k, reinterpret_cast<const uint4 *>(d.ed_btab), d_ok);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
