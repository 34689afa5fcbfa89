// hostsim.h — TEST INFRASTRUCTURE ONLY.  Lets the device headers (mp.cuh, curve.cuh, kernels.cuh, keygroup.cuh)
// compile with plain g++ so that the limb arithmetic, the group law and the kernels can be run on the CPU — thread-per-item
// kernels one "thread" at a time, warp-cooperative ones in lockstep (one OS thread per lane) — and compared with Python big
// integers and the oracle (tests/test_hostsim.py, -m "not gpu").
// It is never part of libsbv.so: the product has no CPU path.  Only defined when SBV_HOSTSIM is set and the
// compiler is not nvcc.
#pragma once
#if defined(SBV_HOSTSIM) && !defined(__CUDACC__)
#include <stdint.h>
#include <string.h>

#include <condition_variable>
#include <map>
#include <mutex>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __shared__
#define __constant__ static const
#define __launch_bounds__(...)

struct hostsim_dim3 { unsigned x = 1, y = 1, z = 1; };
extern thread_local hostsim_dim3 threadIdx, blockIdx, blockDim, gridDim;
struct uint4 { uint32_t x, y, z, w; };
struct uint2 { uint32_t x, y; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

template <class T> static inline T __ldg(const T *p) { return *p; }
static inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {
    const uint64_t v = ((uint64_t)y << 32) | x;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t sel = (s >> (4 * i)) & 0xf;
        uint32_t byte = (uint32_t)(v >> (8 * (sel & 7))) & 0xff;
        if (sel & 8) byte = (byte & 0x80) ? 0xff : 0;
        r |= byte << (8 * i);
    }
    return r;
}
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) {
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31));
}
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t sh) {
    return (uint32_t)(((((uint64_t)hi << 32) | lo) << (sh & 31)) >> 32);
}
static inline int __ffs(int x) { return x ? __builtin_ctz((unsigned)x) + 1 : 0; }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static inline void __syncthreads() {}
static inline void __threadfence() {}
// Warp primitives.  Default: one simulated thread at a time — a "ballot" sees only the caller, a shuffle returns the caller's
// own value (thread-per-item kernels never depend on them).  LOCKSTEP mode (hostsim_ctx set by the driver, one OS thread
// per lane): the lanes named by `mask` meet at every primitive and exchange their values, which is what the
// warp-cooperative kernels (k_kt_bases4: four lanes per key) need.
struct hostsim_warp {
    std::mutex m;
    std::condition_variable cv;
    struct Slot { unsigned arrived = 0, gen = 0; uint32_t in[32] = {}, out[32] = {}; };
    std::map<unsigned, Slot> slots;  // one meeting point per participant mask
};
extern thread_local hostsim_warp *hostsim_ctx;
// every lane of `mask` contributes v; returns the 32 contributions (lanes outside the mask: stale / zero)
static inline void hostsim_exchange(unsigned mask, uint32_t v, uint32_t (&all)[32]) {
    hostsim_warp *w = hostsim_ctx;
    std::unique_lock<std::mutex> lk(w->m);
    hostsim_warp::Slot &s = w->slots[mask];
    s.in[threadIdx.x & 31] = v;
    if (++s.arrived == (unsigned)__builtin_popcount(mask)) {
        memcpy(s.out, s.in, sizeof s.in);
        s.arrived = 0;
        s.gen++;
        w->cv.notify_all();
    } else {
        const unsigned g = s.gen;
        w->cv.wait(lk, [&] { return s.gen != g; });
    }
    memcpy(all, s.out, sizeof s.out);  // still under the lock: the next meeting cannot complete before every lane has left this one
}
// LOCKSTEP mode: a barrier of the lanes of `mask` (the warp's shared memory is the extern `tab`, one array that the lanes
// of the running warp share)
static inline void __syncwarp(unsigned mask = 0xffffffffu) {
    if (!hostsim_ctx) return;
    uint32_t all[32];
    hostsim_exchange(mask, 0, all);
}
static inline unsigned __ballot_sync(unsigned mask, int p) {
    if (!hostsim_ctx) return p ? 1u : 0u;
    uint32_t all[32];
    hostsim_exchange(mask, p ? 1u : 0u, all);
    unsigned r = 0;
    for (int i = 0; i < 32; i++) if (((mask >> i) & 1) && all[i]) r |= 1u << i;
    return r;
}
static inline unsigned __activemask() { return 1u; }
static inline unsigned __match_any_sync(unsigned mask, uint32_t v) {
    if (!hostsim_ctx) return 1u << (threadIdx.x & 31);
    uint32_t all[32];
    hostsim_exchange(mask, v, all);
    unsigned r = 0;
    for (int i = 0; i < 32; i++) if (((mask >> i) & 1) && all[i] == v) r |= 1u << i;
    return r;
}
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src) {
    static_assert(sizeof(T) == 4, "32-bit shuffles only");
    if (!hostsim_ctx) return v;
    uint32_t u, all[32];
    memcpy(&u, &v, 4);
    hostsim_exchange(mask, u, all);
    T r;
    memcpy(&r, &all[src & 31], 4);
    return r;
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, int delta) {
    if (!hostsim_ctx) return v;
    const int src = (int)(threadIdx.x & 31) + delta;
    const T r = __shfl_sync(mask, v, src > 31 ? (int)(threadIdx.x & 31) : src);
    return src > 31 ? v : r;
}
template <class T> static inline T atomicAdd(T *p, T v) { T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicCAS(T *p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }
template <class T> static inline T atomicMax(T *p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicOr(T *p, T v) { T o = *p; *p = o | v; return o; }
typedef int cudaError_t;
typedef void *cudaStream_t;
#endif
