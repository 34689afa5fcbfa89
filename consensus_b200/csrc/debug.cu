#include "engine.h"
#include "debug_ops.cuh"
using namespace sbv;
// debug.cu — arithmetic-layer test hooks (used only by tests/; not part of include/sbv.h).
// Operands are little-endian 32-bit limb arrays, 2N limbs per slot (unused limbs zero).
namespace {
template <class C>
__global__ void k_debug_op(int op, uint32_t n, const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    debug_op_dispatch<C>(op, i, a, b, out);
}
}  // namespace

// op: see debug_ops.cuh (low byte: the operation; DEBUG_INL / DEBUG_NEG / DEBUG_SKIP flags above it)
extern "C" int sbv_debug_op(sbv_engine *e, uint8_t curve, int op, size_t n, const uint32_t *a, const uint32_t *b, uint32_t *out) {
    if (!e || curve > SBV_P384) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    const size_t N = curve == SBV_P256 ? 8 : 12, bytes = n * 2 * N * 4;
    int rc = sbv_ensure_scratch(e, d, 3 * bytes + 1024);
    if (rc) return rc;
    uint32_t *da = (uint32_t *)d.d_scratch, *db = da + n * 2 * N, *dout = db + n * 2 * N;
    CU(e, cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, d.stream));
    if (curve == SBV_P256) k_debug_op<P256><<<(uint32_t)((n + 63) / 64), 64, 0, d.stream>>>(op, (uint32_t)n, da, db, dout);
    else k_debug_op<P384><<<(uint32_t)((n + 63) / 64), 64, 0, d.stream>>>(op, (uint32_t)n, da, db, dout);
    CU(e, cudaGetLastError());
    CU(e, cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// Copies entries [first, first + count) of device 0's fixed-base table of G (k_gtable_init: entry (i << GW) + b is
// b * 2^(GW*i) * G, affine Montgomery x then y, 2N limbs) to the host.
extern "C" int sbv_debug_gtable(sbv_engine *e, uint8_t curve, size_t first, size_t count, uint32_t *out) {
    if (!e || curve > SBV_P384 || !out) return SBV_ERR_ARG;
    const CurveOps &ops = sbv_ops(curve);
    if (first > ops.gtab_entries || count > ops.gtab_entries - first) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    const size_t words = 2 * (size_t)ops.N;
    CU(e, cudaMemcpyAsync(out, d.gtab[curve] + first * words, count * words * 4, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}
