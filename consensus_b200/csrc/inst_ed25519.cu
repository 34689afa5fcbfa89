// inst_ed25519.cu — launchers of the Ed25519 kernels (sha512.cuh, ed25519_verify.cuh, ed25519_keyed.cuh) behind engine.h,
// and the registry of registered Ed25519 keys.
#include <vector>

#include "engine.h"
#include "ed25519_keyed.cuh"
#include "ed25519_verify.cuh"
#include "sha512.cuh"

using namespace sbv;

namespace {
constexpr int ED_BLOCK = 32;  // 32 KiB of shared memory per block (the 1A..8A tables): no opt-in attribute needed
constexpr size_t ED_SMEM = (size_t)8 * 4 * 8 * 4 * ED_BLOCK;
constexpr int EDK_BLOCK = 128;  // k_ed_verify_keyed: no shared memory; see DESIGN.md §3 for registers and occupancy
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

// ---- registered Ed25519 keys ----
void sbv_ed_keys_free(Dev &d) {
    void *p[] = {d.ed_kpub, d.ed_slot2local, d.ed_ktab};
    for (void *x : p) if (x) cudaFree(x);
    d.ed_kpub = nullptr;
    d.ed_slot2local = nullptr;
    d.ed_ktab = nullptr;
    d.ed_n_slots = 0;
    d.ed_n_local = 0;
}

namespace {
struct DevTemp {  // device temporaries of one registry build, freed on every exit path
    std::vector<void *> p;
    ~DevTemp() { for (void *x : p) cudaFree(x); }
    template <class T>
    cudaError_t alloc(T **out, size_t bytes) {
        void *q = nullptr;
        const cudaError_t st = cudaMalloc(&q, bytes);
        if (st == cudaSuccess) { p.push_back(q); *out = static_cast<T *>(q); }
        return st;
    }
};

// The registry of device d from the n keys of pub: the registered bytes, k_ed_kdecode for the flags, the map of the
// decodable slots to tables, and k_ed_ktab_build for their tables, at most ED_KBUILD_MAX keys per launch.
int ed_keys_fill(sbv_engine *e, Dev &d, size_t n, const uint8_t *pub) {
    const uint32_t ns = (uint32_t)n;
    CU(e, cudaMalloc(&d.ed_kpub, n * 32));
    CU(e, cudaMalloc(&d.ed_slot2local, n * sizeof(int32_t)));
    DevTemp tmp;
    uint32_t *xy = nullptr;
    uint8_t *flag = nullptr;
    CU(e, tmp.alloc(&xy, n * 16 * sizeof(uint32_t)));
    CU(e, tmp.alloc(&flag, n));
    CU(e, cudaMemcpyAsync(d.ed_kpub, pub, n * 32, cudaMemcpyHostToDevice, d.stream));
    k_ed_kdecode<<<(ns + 63) / 64, 64, 0, d.stream>>>(ns, d.ed_kpub, xy, flag);
    e->launches += 1;
    CU(e, cudaGetLastError());
    std::vector<uint8_t> hflag(n);
    CU(e, cudaMemcpyAsync(hflag.data(), flag, n, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    std::vector<int32_t> map(n, -1);
    std::vector<uint32_t> slot_of;
    for (size_t i = 0; i < n; i++)
        if (hflag[i]) { map[i] = (int32_t)slot_of.size(); slot_of.push_back((uint32_t)i); }
    const size_t cnt = slot_of.size();
    CU(e, cudaMemcpyAsync(d.ed_slot2local, map.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, d.stream));
    if (cnt) {
        CU(e, cudaMalloc(&d.ed_ktab, cnt * ED_KTAB_WORDS * sizeof(uint32_t)));
        const size_t chunk = std::min(cnt, (size_t)ED_KBUILD_MAX);
        uint32_t *d_slot_of = nullptr, *pref = nullptr;
        CU(e, tmp.alloc(&d_slot_of, cnt * sizeof(uint32_t)));
        CU(e, tmp.alloc(&pref, chunk * ED_BWINS * ED_BENT * 8 * sizeof(uint32_t)));
        CU(e, cudaMemcpyAsync(d_slot_of, slot_of.data(), cnt * sizeof(uint32_t), cudaMemcpyHostToDevice, d.stream));
        for (size_t c0 = 0; c0 < cnt; c0 += chunk) {
            const uint32_t cc = (uint32_t)std::min(chunk, cnt - c0), threads = cc * ED_BWINS;
            k_ed_ktab_build<<<(threads + 63) / 64, 64, 0, d.stream>>>(cc, d_slot_of + c0, xy, d.ed_ktab + c0 * ED_KTAB_WORDS, pref);
            e->launches += 1;
            CU(e, cudaGetLastError());
        }
    }
    CU(e, cudaStreamSynchronize(d.stream));
    d.ed_n_slots = ns;
    d.ed_n_local = (uint32_t)cnt;
    return 0;
}
}  // namespace

int sbv_ed_keys_build(sbv_engine *e, Dev &d, size_t n, const uint8_t *pub) {
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, cudaDeviceSynchronize());  // no launch on any lane may still read the old registry
    sbv_ed_keys_free(d);
    if (n == 0) return 0;
    const int rc = ed_keys_fill(e, d, n, pub);
    if (rc) {
        cudaStreamSynchronize(d.stream);
        sbv_ed_keys_free(d);
    }
    return rc;
}

int sbv_launch_ed25519_registered(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint32_t *d_slot,
                                  const uint8_t *d_sig, uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st) {
    k_ed_key_gather<<<(uint32_t)((2 * n + 255) / 256), 256, 0, st>>>((uint32_t)n, d_slot, d.ed_n_slots, reinterpret_cast<const uint4 *>(d.ed_kpub),
                                                                      reinterpret_cast<uint4 *>(d_pub));
    e->launches += 1;
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_ed_sha512<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_sig, d_pub, d_msgs, d_off, base, d_k, perm, nullptr);
    k_ed_verify_keyed<EDK_BLOCK><<<(uint32_t)((n + EDK_BLOCK - 1) / EDK_BLOCK), EDK_BLOCK, 0, st>>>(
        (uint32_t)n, d_sig, d_slot, d.ed_n_slots, d.ed_slot2local, reinterpret_cast<const uint4 *>(d.ed_ktab), d_k,
        reinterpret_cast<const uint4 *>(d.ed_btab), d_ok);
    e->launches += 2;
    CU(e, cudaGetLastError());
    return 0;
}

// test hook (debug.cu): the production registered-key kernel with the caller's k (word-major, every k < L)
int sbv_launch_ed_verify_registered_k(sbv_engine *e, Dev &d, size_t n, const uint32_t *d_slot, const uint8_t *d_sig, const uint32_t *d_k, uint8_t *d_ok,
                                      cudaStream_t st) {
    k_ed_verify_keyed<EDK_BLOCK><<<(uint32_t)((n + EDK_BLOCK - 1) / EDK_BLOCK), EDK_BLOCK, 0, st>>>(
        (uint32_t)n, d_sig, d_slot, d.ed_n_slots, d.ed_slot2local, reinterpret_cast<const uint4 *>(d.ed_ktab), d_k,
        reinterpret_cast<const uint4 *>(d.ed_btab), d_ok);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
