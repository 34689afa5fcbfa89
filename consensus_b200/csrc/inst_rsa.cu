// inst_rsa.cu — the RSA launches of libsbv.so: every RSA shard and the build of the RSA key registry go through the launch
// plan of rsa_keyed.cuh (one kernel instance per modulus size, and per hash for the PSS decoding), and k_sha512
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

namespace {
// The plan's launch on the engine: blocks of RSA_BLOCK threads on st, counted in e->launches.
auto engine_launch(sbv_engine *e, cudaStream_t st) {
    return [e, st](auto kernel, uint32_t lanes, size_t items, auto... args) -> int {
        kernel<<<rsa_grid(items, lanes), RSA_BLOCK, 0, st>>>(args...);
        e->launches += 1;
        CU(e, cudaGetLastError());
        return 0;
    };
}
}  // namespace

int sbv_launch_rsa(sbv_engine *e, const RsaShard &shard, cudaStream_t st) {
    if (!rsa_shard_ok(shard)) return fail(e, SBV_ERR_ARG, "RSA shard of a size, hash tag or salt length outside the set");
    return rsa_launch_shard(shard, engine_launch(e, st));
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
    if (int rc = rsa_launch_kprep(d_slots, first, d_mods, d_off, d_exp, d.rsa_rec, d.rsa_pool, engine_launch(e, d.stream))) return rc;
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
