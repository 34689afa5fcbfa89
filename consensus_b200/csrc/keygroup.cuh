// keygroup.cuh — per-key fixed-base tables, built on the device, and the grouping of a keys-per-item batch by key.
//
// In the reference a Verifier sees the same few keys over and over: the n consenters sign every commit vote
// (/root/reference/internal/bft/view.go:519-551: up to n-1 votes per sequence from the same n-1 nodes) and clients
// sign many requests each (controller.go:233-246).  The C ABI still takes the key with every item (sbv_verify_batch:
// qx, qy per item), so the engine finds the repetition itself:
//
//   k_kg_insert   every item hashes its key (64/96 bytes of (qx, qy), or a 32-byte Ed25519 encoding: the key views
//                 KgXY / KgKey32) into an open-addressing table (CAS on the item index,
//                 full-key compare on collision): rep[i] = first item with the same key; warp-aggregated count
//   k_kg_assign   representatives whose key occurs >= T times (and while table slots last) get a dense key id
//   k_kg_route    items are appended to the fixed-base list (their key has a table) or to the generic list
//   k_kt_bases4   four lanes per key (window tables) / k_kt_bases2 two lanes per key (comb): validate the key, the
//                 bases B_i = 2^(STEP*i) * Q of its table — a chain of doublings whose independent multiplications run
//                 on different lanes (k_kt_bases, one thread per key, is their reference in the CPU simulation)
//   k_comb_affine one thread per key (comb): the 16 bases to affine with one inversion
//   k_comb_fill_warp  a warp per key, lane = chain (comb): the 16 entries of a chain, one mixed addition per Gray-code step
//   k_kt_fill     one thread per (key, window) (window table): e*B_w for e = 1..2^(W-1) with co-Z additions (5M+2S
//                 each — the chain of Z ratios that comes with them is exactly what the inversion needs)
//   k_kt_inv      one thread per key: ONE field inversion for all chains of the key (Montgomery's trick across
//                 the chains' top Z's)
//   k_kt_final    one thread per (key, chain): back-substitute the Z ratios, convert to affine, in place
//   k_comb_final  a warp per key, lane = chain (comb): the same conversion, the table written once in whole lines
//
// Keys grouped inside a launch get a comb table (CombTab, kernels.cuh), read by k_verify_comb: P-256: 240 doublings +
// 512 mixed additions (~11 multiplications) + 512 conversions (~6) + two inversions per key ~ 3.5 generic verifications;
// a comb verification (15 doublings + 32 additions + the u1*G half) is ~5x cheaper than a generic one, so T = 16 pays.
// In issued warp instructions (sm_90a SASS) a P-256 comb table costs ~16 K in the doubling chain (1,037 per doubling
// for 16 keys), ~39 K in k_comb_fill_warp (2,167 per mixed addition, inlined; 18 steps of a warp carry one) and ~15 K
// in k_comb_final (911 per entry, inlined), against ~266 K for the 64 verifications of a key in k_verify_comb and k_gpart.
// Registered keys (sbv_set_keys) get a window table (KeyTab, W = 8), read by k_verify_kt: built once per key set, so
// its verifications are the ones to make cheapest — no doublings at all.
#pragma once
#include "kernels.cuh"

namespace sbv {

constexpr uint32_t KG_EMPTY = 0xffffffffu;

// One word into the running hash: two multiplications with a shift between them, so that no difference in w comes out
// of the step independent of h (a single multiplication passes a difference in bit 31 through unchanged, and the next
// word could cancel it for every seed).
SBV_DEV uint32_t kg_mix(uint32_t h, uint32_t w) {
    h = (h ^ w) * 0x9E3779B1u;
    h ^= h >> 15;
    return h * 0x85EBCA77u;
}
// Every word of x and of y enters the hash: keys that differ anywhere hash apart for most seeds, so an adversary who
// picks the keys of a batch cannot make them share one probe sequence without knowing the engine's seed.
template <class C>
SBV_DEV uint32_t kg_hash(const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be, uint32_t i, uint32_t seed) {
    const uint32_t *x = reinterpret_cast<const uint32_t *>(qx_be + (size_t)i * C::BYTES);
    const uint32_t *y = reinterpret_cast<const uint32_t *>(qy_be + (size_t)i * C::BYTES);
    uint32_t h = seed;
#pragma unroll
    for (int k = 0; k < C::N; k++) {
        h = kg_mix(h, __ldg(x + k));
        h = kg_mix(h, __ldg(y + k));
    }
    return h ^ (h >> 16);  // the probe index takes the low bits
}
template <class C>
SBV_DEV bool kg_same_key(const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be, uint32_t i, uint32_t j) {
    const uint32_t *xi = reinterpret_cast<const uint32_t *>(qx_be + (size_t)i * C::BYTES);
    const uint32_t *xj = reinterpret_cast<const uint32_t *>(qx_be + (size_t)j * C::BYTES);
    const uint32_t *yi = reinterpret_cast<const uint32_t *>(qy_be + (size_t)i * C::BYTES);
    const uint32_t *yj = reinterpret_cast<const uint32_t *>(qy_be + (size_t)j * C::BYTES);
    uint32_t diff = 0;
#pragma unroll
    for (int k = 0; k < C::N; k++) diff |= (__ldg(xi + k) ^ __ldg(xj + k)) | (__ldg(yi + k) ^ __ldg(yj + k));
    return diff == 0;
}

// Key views of k_kg_insert: which bytes of item i make its key.
// KgXY<C>: the coordinates (qx, qy) of curve C, C::BYTES each (ECDSA).
template <class C>
struct KgXY {
    const uint8_t *qx_be, *qy_be;
    SBV_DEV uint32_t hash(uint32_t i, uint32_t seed) const { return kg_hash<C>(qx_be, qy_be, i, seed); }
    SBV_DEV bool same(uint32_t i, uint32_t j) const { return kg_same_key<C>(qx_be, qy_be, i, j); }
};
// KgKey32: a 32-byte encoding, 16-byte aligned per item (Ed25519, grouped by bytes rather than by the point they decode to)
struct KgKey32 {
    const uint8_t *pub;
    SBV_DEV uint32_t hash(uint32_t i, uint32_t seed) const {
        const uint32_t *x = reinterpret_cast<const uint32_t *>(pub + (size_t)i * 32);
        uint32_t h = seed;
#pragma unroll
        for (int k = 0; k < 8; k += 2) {
            h = (h ^ __ldg(x + k)) * 0x9E3779B1u;
            h = (h ^ __ldg(x + k + 1)) * 0x85EBCA77u;
            h ^= h >> 15;
        }
        return h;
    }
    SBV_DEV bool same(uint32_t i, uint32_t j) const {
        const uint32_t *xi = reinterpret_cast<const uint32_t *>(pub + (size_t)i * 32);
        const uint32_t *xj = reinterpret_cast<const uint32_t *>(pub + (size_t)j * 32);
        uint32_t diff = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) diff |= __ldg(xi + k) ^ __ldg(xj + k);
        return diff == 0;
    }
};

// htab: hmask + 1 slots, all KG_EMPTY on entry; kcnt: n zeros on entry.  KV: a key view (KgXY, KgKey32).
template <class KV>
__global__ void __launch_bounds__(256) k_kg_insert(uint32_t n, KV key, uint32_t seed, uint32_t hmask, uint32_t *__restrict__ htab,
                                                   uint32_t *__restrict__ rep, uint32_t *__restrict__ kcnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t h = key.hash(i, seed) & hmask;
    uint32_t r;
    for (;;) {
        uint32_t cur = htab[h];
        if (cur == KG_EMPTY) {
            cur = atomicCAS(htab + h, KG_EMPTY, i);
            if (cur == KG_EMPTY) { r = i; break; }
        }
        if (key.same(i, cur)) { r = cur; break; }
        h = (h + 1) & hmask;
    }
    rep[i] = r;
#if defined(__CUDA_ARCH__)
    // warp-aggregated count: a consensus batch has a handful of keys, i.e. thousands of items per counter
    const uint32_t peers = __match_any_sync(__activemask(), r);
    if ((threadIdx.x & 31) == (uint32_t)(__ffs((int)peers) - 1)) atomicAdd(kcnt + r, (uint32_t)__popc(peers));
#else
    atomicAdd(kcnt + r, 1u);
#endif
}

// keyid[i] (i a representative) = dense key id, or -1.  counters[0] = number of keys (may exceed max_keys: clamp
// when reading), counters[1] / counters[2] = fill of the fixed-base / generic lists; all zero on entry.
static __global__ void __launch_bounds__(256) k_kg_assign(uint32_t n, const uint32_t *__restrict__ rep, const uint32_t *__restrict__ kcnt,
                                                   uint32_t threshold, uint32_t max_keys, int32_t *__restrict__ keyid,
                                                   uint32_t *__restrict__ keylist, uint32_t *__restrict__ counters) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int32_t id = -1;
    if (rep[i] == i && kcnt[i] >= threshold) {
        const uint32_t k = atomicAdd(counters + 0, 1u);
        if (k < max_keys) { id = (int32_t)k; keylist[k] = i; }
    }
    keyid[i] = id;
}

// item_kid[i] = key id of item i's key (or -1); klist / glist = the two work lists
static __global__ void __launch_bounds__(256) k_kg_route(uint32_t n, const uint32_t *__restrict__ rep, const int32_t *__restrict__ keyid,
                                                  int32_t *__restrict__ item_kid, uint32_t *__restrict__ klist, uint32_t *__restrict__ glist,
                                                  uint32_t *__restrict__ counters) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    const int32_t kid = live ? keyid[rep[i]] : -1;
    if (live) item_kid[i] = kid;
#if defined(__CUDA_ARCH__)
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t mk = __ballot_sync(0xffffffffu, live && kid >= 0), mg = __ballot_sync(0xffffffffu, live && kid < 0);
    uint32_t bk = 0, bg = 0;
    if (lane == 0) {
        if (mk) bk = atomicAdd(counters + 1, (uint32_t)__popc(mk));
        if (mg) bg = atomicAdd(counters + 2, (uint32_t)__popc(mg));
    }
    bk = __shfl_sync(0xffffffffu, bk, 0);
    bg = __shfl_sync(0xffffffffu, bg, 0);
    const uint32_t below = (1u << lane) - 1u;
    if (live && kid >= 0) klist[bk + __popc(mk & below)] = i;
    if (live && kid < 0) glist[bg + __popc(mg & below)] = i;
#else
    if (live && kid >= 0) klist[atomicAdd(counters + 1, 1u)] = i;
    if (live && kid < 0) glist[atomicAdd(counters + 2, 1u)] = i;
#endif
}

// ---- table construction -------------------------------------------------------------------------------------
// Scratch layout of the window tables and of the comb's bases (cap = key capacity of the buffers; lanes of a warp are
// consecutive keys, so every access below is coalesced; the rest of the comb's scratch is CombScr):
//   bases [i][3N words][cap]                Jacobian B_i = 2^(STEP*i) * Q (the comb's are made affine in place)
//   hs    [win][e = 2..ENT][N words][cap]   Z ratios along chain win: Z_e = Z_{e-1} * H_e  (window: H_2 = 2*Y_B, Z_1 = Z_B)
//   ztop  [win][N words][cap]               Z_ENT of the chain; k_kt_inv overwrites it with its inverse
//   pref  [win][N words][cap]               prefix products of the inversions
//   ktab  [kid][win][e-1][2N words]         Jacobian X, Y from the fill kernel; affine x, y after k_kt_final

// nkeys_ptr: device counter (clamped to cap) — the grid is sized for the worst case and surplus threads leave.
// key k is item keylist[k] of (qx_be, qy_be); for registered keys keylist is the identity over the key array.
// One thread per key: the reference for k_kt_bases4 in the CPU simulation (tools/hostsim); libsbv.so launches k_kt_bases4.
template <class C, class KT>
__global__ void __launch_bounds__(64) k_kt_bases(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ keylist,
                                                 const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be,
                                                 uint32_t *__restrict__ bases, uint8_t *__restrict__ keyflags) {
    constexpr int N = C::N;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys) return;
    const uint32_t item = keylist ? keylist[k] : k;
    Jac<C> B;
    const bool good = load_key<C>(B.X, B.Y, qx_be, qy_be, item);
    keyflags[k] = good ? 1 : 0;
    if (!good) return;  // no table: every item of this key rejects (k_verify_kt checks the flag)
    C::get_one(B.Z);
#pragma unroll 1
    for (int win = 0; win < KT::NBASE; win++) {
        if (win) {
#pragma unroll 1
            for (int d = 0; d < KT::STEP; d++) pt_double<C>(B);
        }
        uint32_t *o = bases + (size_t)win * 3 * N * cap + k;
#pragma unroll
        for (int i = 0; i < N; i++) { o[(size_t)i * cap] = B.X[i]; o[(size_t)(N + i) * cap] = B.Y[i]; o[(size_t)(2 * N + i) * cap] = B.Z[i]; }
    }
}

// k_kt_bases4 — the same chain with FOUR LANES PER KEY (three of them working): the eight multiplications of a doubling
// form four dependent levels, and the independent ones of a level run on different lanes:
//   level 1   lane 0: delta = Z*Z          lane 1: bb = (2Y)*(2Y)        lane 2: Z3 = (2Y)*Z
//   level 2   lane 0: (X-delta)*(X+delta)  lane 1: beta4 = X*bb          lane 2: bb*bb
//   level 3   lane 0: alpha*alpha          (alpha = 3*(X-delta)(X+delta))
//   level 4   lane 0: alpha*(beta4 - X3)
// with six 8-word quad broadcasts per doubling (bb, beta4, 8Y^4, and the new X, Y, Z).  The kernel is one dependent
// chain on an otherwise idle sub-partition, so halving the number of dependent multiplications halves its duration.
template <class C, class KT>
__global__ void __launch_bounds__(128) k_kt_bases4(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ keylist,
                                                   const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be,
                                                   uint32_t *__restrict__ bases, uint8_t *__restrict__ keyflags) {
    constexpr int N = C::N;
    const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t k = gt >> 2, role = gt & 3;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys) return;  // a quad leaves together
    const unsigned qbase = (threadIdx.x & 31) & ~3u, qmask = 0xFu << qbase;
    const uint32_t item = keylist ? keylist[k] : k;
    uint32_t X[N], Y[N], Z[N];
    const bool good = load_key<C>(X, Y, qx_be, qy_be, item);  // the four lanes agree
    if (role == 0) keyflags[k] = good ? 1 : 0;
    if (!good) return;
    C::get_one(Z);
    auto bcast = [&](uint32_t (&v)[N], unsigned src) {
#pragma unroll
        for (int i = 0; i < N; i++) v[i] = __shfl_sync(qmask, v[i], qbase + src);
    };
#pragma unroll 1
    for (int win = 0; win < KT::NBASE; win++) {
        if (win) {
#pragma unroll 1
            for (int d = 0; d < KT::STEP; d++) {
                uint32_t s[N], a[N], b[N], r1[N], r2[N], r3[N], r4[N], t1[N], t2[N];
                C::fadd(s, Y, Y);
                // level 1: delta | bb | Z3 | (delta)
                mp_select<N>(a, role == 1 || role == 2, s, Z);
                mp_select<N>(b, role == 1, s, Z);
                C::fmul(r1, a, b);
                uint32_t bb[N];
                mp_copy<N>(bb, r1);
                bcast(bb, 1);
                // level 2: (X-delta)(X+delta) | X*bb | bb*bb
                C::fsub(t1, X, r1);
                C::fadd(t2, X, r1);
                mp_select<N>(a, role == 0, t1, X);
                mp_select<N>(a, role == 2, bb, a);
                mp_select<N>(b, role == 0, t2, bb);
                C::fmul(r2, a, b);
                // level 3 (lane 0): alpha = 3*r2, alpha^2 ; lane 2: 8Y^4 = r2 / 2 ; lane 1 holds beta4 = r2
                uint32_t alpha[N], half[N], beta4[N];
                C::fadd(t1, r2, r2);
                C::fadd(alpha, t1, r2);
                C::fhalf(half, r2);
                C::fmul(r3, alpha, alpha);
                mp_copy<N>(beta4, r2);
                bcast(beta4, 1);
                bcast(half, 2);
                // level 4 (lane 0): X3 = alpha^2 - 2*beta4 ; Y3 = alpha*(beta4 - X3) - 8Y^4
                uint32_t x3[N], y3[N];
                C::fadd(t1, beta4, beta4);
                C::fsub(x3, r3, t1);
                C::fsub(t2, beta4, x3);
                C::fmul(r4, alpha, t2);
                C::fsub(y3, r4, half);
                mp_copy<N>(X, x3); bcast(X, 0);
                mp_copy<N>(Y, y3); bcast(Y, 0);
                mp_copy<N>(Z, r1); bcast(Z, 2);
            }
        }
        if (role == 0) {
            uint32_t *o = bases + (size_t)win * 3 * N * cap + k;
#pragma unroll
            for (int i = 0; i < N; i++) { o[(size_t)i * cap] = X[i]; o[(size_t)(N + i) * cap] = Y[i]; o[(size_t)(2 * N + i) * cap] = Z[i]; }
        }
    }
}

// k_kt_bases2 — the same chain with TWO LANES PER KEY (the comb tables' builder): the eight multiplications of a doubling
// are two per level, so both lanes work at every level and the dependent length stays four:
//   level 1   lane 0: delta = Z^2                 lane 1: bb = (2Y)^2
//   level 2   lane 0: (X-delta)*(X+delta)         lane 1: beta4 = X*bb
//   level 3   lane 0: alpha^2                     lane 1: bb^2 (8Y^4 = half of it)
//   level 4   lane 0: alpha*(beta4 - X3)          lane 1: Z3 = (2Y)*Z
// with three 8-word pair exchanges per doubling (beta4 to lane 0; 8Y^4 and X3 crossing; Z3 and Y3 crossing).  Against
// k_kt_bases4 a warp carries 16 keys instead of 8 and both levels 1 and 3 are squarings, so a key costs about half the
// issued instructions for the same dependent chain.  Lane 0 holds (X, Y, Z) after every doubling and stores the bases.
template <class C, class KT, bool INL>
__global__ void __launch_bounds__(128) k_kt_bases2(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ keylist,
                                                   const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be,
                                                   uint32_t *__restrict__ bases, uint8_t *__restrict__ keyflags) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy of the doubling loop
    constexpr int N = C::N;
    const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t k = gt >> 1, role = gt & 1;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys) return;  // a pair leaves together
    const unsigned pbase = (threadIdx.x & 31) & ~1u, pmask = 3u << pbase, other = pbase + (role ^ 1);
    const uint32_t item = keylist ? keylist[k] : k;
    uint32_t X[N], Y[N], Z[N];
    const bool good = load_key<C>(X, Y, qx_be, qy_be, item);  // the two lanes agree
    if (role == 0) keyflags[k] = good ? 1 : 0;
    if (!good) return;
    C::get_one(Z);
    // v <- the other lane's v
    auto xchg = [&](uint32_t (&v)[N]) {
#pragma unroll
        for (int i = 0; i < N; i++) v[i] = __shfl_sync(pmask, v[i], other);
    };
#pragma unroll 1
    for (int win = 0; win < KT::NBASE; win++) {
        if (win) {
#pragma unroll 1
            for (int d = 0; d < KT::STEP; d++) {
                uint32_t s[N], a[N], b[N], r1[N], r2[N], r3[N], r4[N], t1[N], t2[N];
                C::fadd(s, Y, Y);
                // level 1: delta | bb
                mp_select<N>(a, role == 1, s, Z);
                A::fsqr(r1, a);
                // level 2: (X-delta)(X+delta) | beta4 = X*bb
                C::fsub(t1, X, r1);
                C::fadd(t2, X, r1);
                mp_select<N>(a, role == 1, X, t1);
                mp_select<N>(b, role == 1, r1, t2);
                A::fmul(r2, a, b);
                uint32_t beta4[N], alpha[N];
                mp_copy<N>(beta4, r2);
                xchg(beta4);  // lane 0 receives beta4 (lane 1 keeps its own in r2)
                // level 3: alpha^2 | bb^2
                C::fadd(t1, r2, r2);
                C::fadd(alpha, t1, r2);  // 3 (X - delta)(X + delta) on lane 0
                mp_select<N>(a, role == 1, r1, alpha);
                A::fsqr(r3, a);
                // lane 0: X3 = alpha^2 - 2*beta4 ; lane 1: 8Y^4 = bb^2 / 2 ; then each takes the other's
                uint32_t x3[N], c8[N];
                C::fadd(t1, beta4, beta4);
                C::fsub(t2, r3, t1);
                C::fhalf(t1, r3);
                mp_select<N>(x3, role == 1, t1, t2);
                xchg(x3);  // lane 0: 8Y^4 ; lane 1: X3
                mp_select<N>(c8, role == 1, t1, x3);
                mp_select<N>(x3, role == 1, x3, t2);
                // level 4: alpha*(beta4 - X3) | Z3 = 2Y*Z
                C::fsub(t1, beta4, x3);
                mp_select<N>(a, role == 1, s, alpha);
                mp_select<N>(b, role == 1, Z, t1);
                A::fmul(r4, a, b);
                // lane 0: Y3 = r4 - 8Y^4 ; lane 1: Z3 = r4 ; then each takes the other's
                C::fsub(t2, r4, c8);
                mp_select<N>(t1, role == 1, r4, t2);
                xchg(t1);  // lane 0: Z3 ; lane 1: Y3
                mp_copy<N>(X, x3);
                mp_select<N>(Y, role == 1, t1, t2);
                mp_select<N>(Z, role == 1, r4, t1);
            }
        }
        if (role == 0) {
            uint32_t *o = bases + (size_t)win * 3 * N * cap + k;
#pragma unroll
            for (int i = 0; i < N; i++) { o[(size_t)i * cap] = X[i]; o[(size_t)(N + i) * cap] = Y[i]; o[(size_t)(2 * N + i) * cap] = Z[i]; }
        }
    }
}

// One table entry (x, y: 2N words, 16-byte aligned) in 16-byte accesses.  The threads of a warp work on different chains,
// a chain's entries apart, so every access instruction touches 32 lines: 2N/4 vector accesses per entry instead of 2N
// scalar ones cut the memory requests of the table kernels fourfold.
template <int N>
SBV_DEV void st_entry(uint32_t *o, const uint32_t (&x)[N], const uint32_t (&y)[N]) {
    uint4 *v = reinterpret_cast<uint4 *>(o);
#pragma unroll
    for (int i = 0; i < N / 4; i++) {
        uint4 a, b;
        a.x = x[4 * i]; a.y = x[4 * i + 1]; a.z = x[4 * i + 2]; a.w = x[4 * i + 3];
        b.x = y[4 * i]; b.y = y[4 * i + 1]; b.z = y[4 * i + 2]; b.w = y[4 * i + 3];
        v[i] = a;
        v[N / 4 + i] = b;
    }
}
// plain loads (not __ldg: k_kt_final rewrites the entries it reads)
template <int N>
SBV_DEV void ld_entry(const uint32_t *o, uint32_t (&x)[N], uint32_t (&y)[N]) {
    const uint4 *v = reinterpret_cast<const uint4 *>(o);
#pragma unroll
    for (int i = 0; i < N / 4; i++) {
        const uint4 a = v[i], b = v[N / 4 + i];
        x[4 * i] = a.x; x[4 * i + 1] = a.y; x[4 * i + 2] = a.z; x[4 * i + 3] = a.w;
        y[4 * i] = b.x; y[4 * i + 1] = b.y; y[4 * i + 2] = b.z; y[4 * i + 3] = b.w;
    }
}

// co-Z addition (Meloni): P = (X1, Y1, Z) and Q = (X2, Y2, Z) share Z.  R = P + Q -> (X3, Y3, Z3) and P is
// re-expressed with the same Z3 = Z * (X1 - X2); h receives X1 - X2 (the ratio Z3 / Z).  5M + 2S.
// P != +-Q is the caller's business (multiples e*B, e >= 2, of a point of prime order never meet B).
template <class C>
SBV_DEV void zaddu(uint32_t (&X1)[C::N], uint32_t (&Y1)[C::N], const uint32_t (&X2)[C::N], const uint32_t (&Y2)[C::N],
                   uint32_t (&X3)[C::N], uint32_t (&Y3)[C::N], uint32_t (&h)[C::N]) {
    constexpr int N = C::N;
    uint32_t c[N], w1[N], w2[N], dy[N], d[N], a1[N], t[N];
    C::fsub(h, X1, X2);
    C::fsqr(c, h);
    C::fmul(w1, X1, c);
    C::fmul(w2, X2, c);
    C::fsub(dy, Y1, Y2);
    C::fsqr(d, dy);
    C::fsub(t, w1, w2);
    C::fmul(a1, Y1, t);
    C::fsub(X3, d, w1);
    C::fsub(X3, X3, w2);
    C::fsub(t, w1, X3);
    C::fmul(Y3, dy, t);
    C::fsub(Y3, Y3, a1);
    mp_copy<N>(X1, w1);
    mp_copy<N>(Y1, a1);
}

template <class C, int W>
__global__ void __launch_bounds__(64) k_kt_fill(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ bases,
                                                const uint8_t *__restrict__ keyflags, uint32_t *__restrict__ hs,
                                                uint32_t *__restrict__ ztop, uint32_t *__restrict__ ktab) {
    constexpr int N = C::N;
    using KT = KeyTab<32 * N, W>;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (t >= nkeys * KT::NWIN) return;
    const uint32_t k = t % nkeys, win = t / nkeys;
    if (!keyflags[k]) return;
    // B in Jacobian form with Z_B; entry 1 is B itself
    uint32_t bx[N], by[N], bz[N];
    {
        const uint32_t *o = bases + (size_t)win * 3 * N * cap + k;
#pragma unroll
        for (int i = 0; i < N; i++) { bx[i] = o[(size_t)i * cap]; by[i] = o[(size_t)(N + i) * cap]; bz[i] = o[(size_t)(2 * N + i) * cap]; }
    }
    uint32_t *out = ktab + ((size_t)k * KT::NWIN + win) * KT::ENT * 2 * N;
#pragma unroll
    for (int i = 0; i < N; i++) { out[i] = bx[i]; out[N + i] = by[i]; }
    // entry 2 = 2B (a = -3 Jacobian doubling); Z_2 = 2*Y_B*Z_B, so H_2 = 2*Y_B, and B is rescaled to Z_2:
    // (X_B * H^2, Y_B * H^3)
    Jac<C> P;
    mp_copy<N>(P.X, bx); mp_copy<N>(P.Y, by); mp_copy<N>(P.Z, bz);
    uint32_t h[N], h2[N], h3[N];
    C::fadd(h, by, by);
    pt_double<C>(P);
    C::fsqr(h2, h);
    C::fmul(h3, h2, h);
    C::fmul(bx, bx, h2);
    C::fmul(by, by, h3);
    uint32_t zacc[N];  // Z of the chain so far
    mp_copy<N>(zacc, P.Z);
    {
        uint32_t *hp = hs + ((size_t)win * (KT::ENT - 1) + 0) * N * cap + k;
#pragma unroll
        for (int i = 0; i < N; i++) { out[2 * N + i] = P.X[i]; out[3 * N + i] = P.Y[i]; hp[(size_t)i * cap] = h[i]; }
    }
    uint32_t px[N], py[N];
    mp_copy<N>(px, P.X); mp_copy<N>(py, P.Y);
#pragma unroll 1
    for (int e = 3; e <= KT::ENT; e++) {
        // (e)B = B + (e-1)B, both on the current Z; B is carried along to the new Z
        uint32_t x3[N], y3[N];
        zaddu<C>(bx, by, px, py, x3, y3, h);
        C::fmul(zacc, zacc, h);
        mp_copy<N>(px, x3); mp_copy<N>(py, y3);
        uint32_t *hp = hs + ((size_t)win * (KT::ENT - 1) + (e - 2)) * N * cap + k;
        uint32_t *oe = out + (size_t)(e - 1) * 2 * N;
#pragma unroll
        for (int i = 0; i < N; i++) { oe[i] = px[i]; oe[N + i] = py[i]; hp[(size_t)i * cap] = h[i]; }
    }
    uint32_t *zp = ztop + (size_t)win * N * cap + k;
#pragma unroll
    for (int i = 0; i < N; i++) zp[(size_t)i * cap] = zacc[i];
}

// Word i of chain ch's Z in ztop / pref: [chain][N words][cap] (window tables; the comb's layout is CombScr)
template <int N>
struct ZByChain {
    SBV_DEV static size_t at(uint32_t k, int ch, int i, uint32_t cap) { return ((size_t)ch * N + i) * cap + k; }
};

// ztop[win] <- 1 / ztop[win] for all chains of a key with one inversion (ZL: the layout of ztop and pref)
template <class C, class KT, class ZL = ZByChain<C::N>>
__global__ void __launch_bounds__(64) k_kt_inv(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint8_t *__restrict__ keyflags,
                                               uint32_t *__restrict__ ztop, uint32_t *__restrict__ pref) {
    constexpr int N = C::N;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys || !keyflags[k]) return;
    uint32_t run[N];
    C::get_one(run);
#pragma unroll 1
    for (int win = 0; win < KT::NCHAIN; win++) {
        uint32_t z[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            const size_t a = ZL::at(k, win, i, cap);
            z[i] = ztop[a];
            pref[a] = run[i];  // product of the windows before
        }
        C::fmul(run, run, z);
    }
    uint32_t inv[N];
    p_inv<C>(inv, run);  // binary extended GCD: this thread is alone on its chain, the dependent length is what counts
#pragma unroll 1
    for (int win = KT::NCHAIN - 1; win >= 0; win--) {
        uint32_t z[N], pv[N], zi[N];
#pragma unroll
        for (int i = 0; i < N; i++) { const size_t a = ZL::at(k, win, i, cap); z[i] = ztop[a]; pv[i] = pref[a]; }
        C::fmul(zi, inv, pv);
        C::fmul(inv, inv, z);
#pragma unroll
        for (int i = 0; i < N; i++) ztop[ZL::at(k, win, i, cap)] = zi[i];
    }
}

// INL: the multiplications inlined (Inl<C>); the comb tables' build takes it, its loop has a single conversion site.
template <class C, class KT, bool INL = false>
__global__ void __launch_bounds__(64) k_kt_final(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ bases,
                                                 const uint8_t *__restrict__ keyflags, const uint32_t *__restrict__ hs,
                                                 const uint32_t *__restrict__ ztop, uint32_t *__restrict__ ktab) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy
    constexpr int N = C::N;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (t >= nkeys * KT::NCHAIN) return;
    const uint32_t k = t % nkeys, win = t / nkeys;
    if (!keyflags[k]) return;
    uint32_t zi[N];  // 1 / Z_e, walking e = ENT .. 1
    {
        const uint32_t *zp = ztop + (size_t)win * N * cap + k;
#pragma unroll
        for (int i = 0; i < N; i++) zi[i] = zp[(size_t)i * cap];
    }
    uint32_t *out = ktab + ((size_t)k * KT::NCHAIN + win) * KT::ENT * 2 * N;
    // entry e-1 and its Z ratio are loaded before entry e is converted and stored (independent addresses: the loads
    // overlap the six multiplications)
    uint32_t x[N], y[N], h[N];
    {
        ld_entry<N>(out + (size_t)(KT::ENT - 1) * 2 * N, x, y);
    }
#pragma unroll 1
    for (int e = KT::ENT; e >= 1; e--) {
        uint32_t nx[N], ny[N], nh[N];
        if (e >= 2) {
            const uint32_t *hp = hs + ((size_t)win * (KT::ENT - 1) + (e - 2)) * N * cap + k;
            ld_entry<N>(out + (size_t)(e - 2) * 2 * N, nx, ny);
#pragma unroll
            for (int i = 0; i < N; i++) nh[i] = hp[(size_t)i * cap];
        }
        uint32_t z2[N], z3[N];
        A::fsqr(z2, zi);
        A::fmul(z3, z2, zi);
        A::fmul(x, x, z2);
        A::fmul(y, y, z3);
        st_entry<N>(out + (size_t)(e - 1) * 2 * N, x, y);
        if (e >= 2) {  // 1/Z_{e-1} = (1/Z_e) * H_e
            mp_copy<N>(h, nh);
            A::fmul(zi, zi, h);
            mp_copy<N>(x, nx); mp_copy<N>(y, ny);
        }
    }
    (void)bases;
}

// ---- comb tables (CombTab, kernels.cuh) -------------------------------------------------------------------------
// k_kt_bases4<C, CombTab<C>> leaves the 16 bases P_c = 2^(SPACING*c) * Q in Jacobian form; k_comb_affine makes them
// affine, k_comb_fill_warp walks the 32 chains a warp per key, k_kt_inv inverts the chains' top Z's as for a window
// table, and k_comb_final converts the entries and writes the table.

// bases -> affine (x, y in place of X, Y) with ONE inversion per key (Montgomery's trick over the 16 Z's; pref: prefix
// products, [c][N words][cap])
template <class C>
__global__ void __launch_bounds__(64) k_comb_affine(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint8_t *__restrict__ keyflags,
                                                    uint32_t *__restrict__ bases, uint32_t *__restrict__ pref) {
    constexpr int N = C::N;
    using CT = CombTab<C>;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys || !keyflags[k]) return;
    uint32_t run[N];
    C::get_one(run);
#pragma unroll 1
    for (int c = 0; c < CT::NBASE; c++) {
        uint32_t z[N];
        const uint32_t *zp = bases + ((size_t)c * 3 + 2) * N * cap + k;
        uint32_t *pp = pref + (size_t)c * N * cap + k;
#pragma unroll
        for (int i = 0; i < N; i++) { z[i] = zp[(size_t)i * cap]; pp[(size_t)i * cap] = run[i]; }
        C::fmul(run, run, z);
    }
    uint32_t inv[N];
    p_inv<C>(inv, run);
#pragma unroll 1
    for (int c = CT::NBASE - 1; c >= 0; c--) {
        uint32_t *o = bases + (size_t)c * 3 * N * cap + k;
        const uint32_t *pp = pref + (size_t)c * N * cap + k;
        uint32_t x[N], y[N], z[N], pv[N], zi[N], z2[N], z3[N];
#pragma unroll
        for (int i = 0; i < N; i++) { x[i] = o[(size_t)i * cap]; y[i] = o[(size_t)(N + i) * cap]; z[i] = o[(size_t)(2 * N + i) * cap]; pv[i] = pp[(size_t)i * cap]; }
        C::fmul(zi, inv, pv);
        C::fmul(inv, inv, z);
        C::fsqr(z2, zi);
        C::fmul(z3, z2, zi);
        C::fmul(x, x, z2);
        C::fmul(y, y, z3);
#pragma unroll
        for (int i = 0; i < N; i++) { o[(size_t)i * cap] = x[i]; o[(size_t)(N + i) * cap] = y[i]; }
    }
}

// One thread per (key, chain), chain = (block b, high nibble hi): slot 0 = the sum of the high teeth of hi, then the 15
// Gray codes of the low nibble, one mixed addition of +-P_(8b+t) per step (t = the bit the step flips).  Records what
// k_kt_final needs: Jacobian X, Y of every slot in ktab, the Z ratio H of every step in hs, the last Z in ztop.
// The reference for k_comb_fill_warp in the CPU simulation (tools/hostsim), with k_kt_inv and k_kt_final over the
// window tables' scratch layout; libsbv.so launches k_comb_fill_warp and k_comb_final.
// The chain of hi = 0 starts at infinity: its first step is a copy of P_(8b) (Z = 1, H = 1), and its slot 0 (m = 0,
// never read) is left as (0, 0).
// The high teeth are steps of the same loop ahead of the Gray walk, so the loop has ONE addition site and its
// multiplications can be inlined (INL: Inl<C>) within the instruction cache.
// No exceptional case arises: every point on a chain is s*Q with s a sum of distinct powers 2^(SPACING*c), so
// 0 < s < 2^(15*SPACING + 1) <= 2^361 < n, and Q has prime order n.  An addition of +P_t (t not in the sum) meets the
// accumulator only if s = 2^(SPACING*t) (impossible: distinct binary expansions) or s + 2^(SPACING*t) = n (too small);
// an addition of -P_t (t in the sum) only if s = -2^(SPACING*t) mod n (too small) or the sum becomes empty — and a Gray
// walk never returns to 0, while the chains with hi != 0 keep their high teeth.
template <class C, bool INL>
__global__ void __launch_bounds__(64) k_comb_fill(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ bases,
                                                  const uint8_t *__restrict__ keyflags, uint32_t *__restrict__ hs,
                                                  uint32_t *__restrict__ ztop, uint32_t *__restrict__ ktab) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy of the loop
    constexpr int N = C::N;
    using CT = CombTab<C>;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (t >= nkeys * CT::NCHAIN) return;
    const uint32_t k = t % nkeys, ch = t / nkeys;
    if (!keyflags[k]) return;
    const int b = (int)(ch >> 4), hi = (int)(ch & 15);
    auto base = [&](int c, uint32_t (&x)[N], uint32_t (&y)[N]) {
        const uint32_t *o = bases + (size_t)c * 3 * N * cap + k;
#pragma unroll
        for (int i = 0; i < N; i++) { x[i] = o[(size_t)i * cap]; y[i] = o[(size_t)(N + i) * cap]; }
    };
    uint32_t *out = ktab + ((size_t)k * CT::NCHAIN + ch) * CT::ENT * 2 * N;
    auto store = [&](int slot, const uint32_t (&x)[N], const uint32_t (&y)[N], const uint32_t (&h)[N]) {
        st_entry<N>(out + (size_t)slot * 2 * N, x, y);
        if (slot) {
            uint32_t *hp = hs + ((size_t)ch * (CT::ENT - 1) + (slot - 1)) * N * cap + k;
#pragma unroll
            for (int i = 0; i < N; i++) hp[(size_t)i * cap] = h[i];
        }
    };
    Jac<A> P;
    uint32_t x[N], y[N], h[N], zero[N];
#pragma unroll
    for (int i = 0; i < N; i++) zero[i] = 0;
    C::get_one(P.Z);
    C::get_one(h);
    if (hi == 0) store(0, zero, zero, h);
    const int nhigh = __popc(hi);  // steps before the Gray walk
    int rest = hi;                 // high teeth still to add
#pragma unroll 1
    for (int st = 0; st < nhigh + CT::ENT - 1; st++) {
        const int kk = st - nhigh + 1;  // the slot the step produces; <= 0 while the high teeth go in (0: the last of them)
        int tooth;
        bool sub = false;
        if (kk <= 0) {
            tooth = 4 + __ffs(rest) - 1;
            rest &= rest - 1;
        } else {
            tooth = __ffs(kk) - 1;                        // gray(kk - 1) -> gray(kk) flips this bit
            sub = !(((kk ^ (kk >> 1)) >> tooth) & 1);     // the bit goes off: subtract
        }
        base(CT::TEETH * b + tooth, x, y);
        if (sub) C::fsub(y, zero, y);
        if (st == 0) { mp_copy<N>(P.X, x); mp_copy<N>(P.Y, y); }  // from infinity: Z = 1, H = 1
        else pt_madd_table<A>(P, x, y, h);
        if (kk >= 0) store(kk, P.X, P.Y, h);
    }
    uint32_t *zp = ztop + (size_t)ch * N * cap + k;
#pragma unroll
    for (int i = 0; i < N; i++) zp[(size_t)i * cap] = P.Z[i];
}

// Scratch of the comb build as libsbv.so runs it (k_comb_fill_warp, k_kt_inv, k_comb_final): a warp per key, lane =
// chain, so every buffer is key-major with the chain innermost, in 16-byte words — one access of a warp covers 512
// contiguous bytes.  Indices in uint4:
//   hs   [key][ Z ratios [slot-1][N/4][chain] | Jacobian X, Y [slot][2N/4: X then Y][chain] ]
//   ztop [key][N/4][chain], pref alike   Z of slot 15 of the chain; k_kt_inv overwrites it with its inverse
// The affine table (ktab) keeps its layout (CombTab::slot) and is written once, by k_comb_final.
template <class C>
struct CombScr {
    using CT = CombTab<C>;
    static constexpr int Q = C::N / 4;  // 16-byte words per coordinate
    static constexpr size_t KEY = (size_t)((CT::ENT - 1) * Q + CT::ENT * 2 * Q) * CT::NCHAIN;  // uint4 of hs per key
    SBV_DEV static size_t hs(uint32_t k, int slot, int w) { return k * KEY + ((size_t)(slot - 1) * Q + w) * CT::NCHAIN; }
    SBV_DEV static size_t jac(uint32_t k, int slot, int w) { return k * KEY + ((size_t)(CT::ENT - 1) * Q + (size_t)slot * 2 * Q + w) * CT::NCHAIN; }
    SBV_DEV static size_t z(uint32_t k, int w) { return ((size_t)k * Q + w) * CT::NCHAIN; }
    // word i of chain ch's Z (k_kt_inv, one thread per key: ZL)
    SBV_DEV static size_t at(uint32_t k, int ch, int i, uint32_t) { return (z(k, i / 4) + ch) * 4 + (i & 3); }
};

template <int N>
SBV_DEV uint4 quad(const uint32_t (&v)[N], int w) { return make_uint4(v[4 * w], v[4 * w + 1], v[4 * w + 2], v[4 * w + 3]); }
template <int N>
SBV_DEV void unquad(uint32_t (&v)[N], int w, const uint4 q) { v[4 * w] = q.x; v[4 * w + 1] = q.y; v[4 * w + 2] = q.z; v[4 * w + 3] = q.w; }

// A warp per key, lane = chain (b, hi) = (lane >> 4, lane & 15): the chains of k_comb_fill, each lane doing exactly the
// steps, in the same order and with the same operands, that k_comb_fill's thread of that chain does — so the Jacobian
// entries, the Z ratios and the last Z are those of k_comb_fill, bit for bit.  What changes is when: a chain with popc(hi)
// high teeth takes popc(hi) + 15 steps, and it starts 4 - popc(hi) steps late, so that at step s every working lane makes
// slot s - 3 and the warp's stores of that slot are contiguous.  The 16 affine bases of the key (1 KiB) are read once per
// warp into shared memory (dynamic: 2N words per base and warp).
// No exceptional case arises, for the reason given above k_comb_fill: the additions of a chain are k_comb_fill's, and
// every point on it is s*Q with 0 < s < 2^(15*SPACING + 1) < n a sum of distinct powers 2^(SPACING*c); +P_t meets the
// accumulator only if s = 2^(SPACING*t) or s + 2^(SPACING*t) = n, -P_t only if s = -2^(SPACING*t) mod n or the sum empties,
// and neither the high teeth (always added, never removed) nor the Gray walk (never back to 0) empties it.
template <class C, bool INL>
__global__ void __launch_bounds__(64) k_comb_fill_warp(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint32_t *__restrict__ bases,
                                                       const uint8_t *__restrict__ keyflags, uint32_t *__restrict__ hs, uint32_t *__restrict__ ztop) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy of the loop
    constexpr int N = C::N, Q = N / 4, HT = CombTab<C>::TEETH / 2;  // HT: high teeth of a block
    using CT = CombTab<C>;
    using S = CombScr<C>;
    static_assert(CT::NCHAIN == 32 && CT::NBASE * 2 == 32, "a lane per chain; a lane per coordinate of a base");
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, ch = threadIdx.x & 31;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys || !keyflags[k]) return;  // a warp leaves together
    extern __shared__ uint32_t tab[];
    uint32_t *pb = tab + (threadIdx.x >> 5) * CT::NBASE * 2 * N;  // [c][x, y][N words]
    {
        const uint32_t *o = bases + ((size_t)(ch >> 1) * 3 + (ch & 1)) * N * cap + k;  // lane 2c + j: coordinate j of P_c
#pragma unroll
        for (int i = 0; i < N; i++) pb[ch * N + i] = o[(size_t)i * cap];
    }
    __syncwarp();
    uint4 *h4 = reinterpret_cast<uint4 *>(hs), *z4 = reinterpret_cast<uint4 *>(ztop);
    auto store = [&](int slot, const uint32_t (&x)[N], const uint32_t (&y)[N], const uint32_t (&h)[N]) {
#pragma unroll
        for (int w = 0; w < Q; w++) { h4[S::jac(k, slot, w) + ch] = quad<N>(x, w); h4[S::jac(k, slot, Q + w) + ch] = quad<N>(y, w); }
        if (slot) {
#pragma unroll
            for (int w = 0; w < Q; w++) h4[S::hs(k, slot, w) + ch] = quad<N>(h, w);
        }
    };
    const int b = (int)(ch >> 4), hi = (int)(ch & 15), nhigh = __popc(hi);
    Jac<A> P;
    uint32_t x[N], y[N], h[N], zero[N];
#pragma unroll
    for (int i = 0; i < N; i++) zero[i] = 0;
    C::get_one(P.Z);
    C::get_one(h);
    if (hi == 0) store(0, zero, zero, h);
    int rest = hi;  // high teeth still to add
#pragma unroll 1
    for (int s = 0; s < HT + CT::ENT - 1; s++) {
        const int st = s - (HT - nhigh);  // the chain's own step (k_comb_fill's st)
        if (st < 0) continue;
        const int kk = s - (HT - 1);      // the slot the step produces; <= 0 while the high teeth go in (0: the last of them)
        int tooth;
        bool neg = false;
        if (kk <= 0) {
            tooth = HT + __ffs(rest) - 1;
            rest &= rest - 1;
        } else {
            tooth = __ffs(kk) - 1;                       // gray(kk - 1) -> gray(kk) flips this bit
            neg = !(((kk ^ (kk >> 1)) >> tooth) & 1);    // the bit goes off: subtract
        }
        const uint32_t *pt = pb + (CT::TEETH * b + tooth) * 2 * N;
#pragma unroll
        for (int i = 0; i < N; i++) { x[i] = pt[i]; y[i] = pt[N + i]; }
        if (neg) C::fsub(y, zero, y);
        if (st == 0) { mp_copy<N>(P.X, x); mp_copy<N>(P.Y, y); }  // from infinity: Z = 1, H = 1
        else pt_madd_table<A>(P, x, y, h);
        if (kk >= 0) store(kk, P.X, P.Y, h);
    }
#pragma unroll
    for (int w = 0; w < Q; w++) z4[S::z(k, w) + ch] = quad<N>(P.Z, w);
}

// A warp per key, lane = chain: k_kt_final's conversion of the comb (1/Z_e walked from e = 16 down to 1, five
// multiplications per entry), reading k_comb_fill_warp's scratch, then the affine entries into ktab in its layout.  A
// chain's entries are contiguous there (CombTab::slot), so each lane stages half a chain (8 entries) in shared memory
// and the warp writes the 32 half chains one at a time: 512 contiguous bytes per store instruction.  Shared memory:
// 32 lanes x (8 entries x 2N/4 + 1 padding) 16-byte words per warp (P-256: 16.5 KiB); the padding word spreads the lanes'
// rows over the banks.
template <class C, bool INL>
__global__ void __launch_bounds__(64) k_comb_final(const uint32_t *__restrict__ nkeys_ptr, uint32_t cap, const uint8_t *__restrict__ keyflags,
                                                   const uint32_t *__restrict__ hs, const uint32_t *__restrict__ ztop, uint32_t *__restrict__ ktab) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy
    constexpr int N = C::N, Q = N / 4;
    using CT = CombTab<C>;
    using S = CombScr<C>;
    constexpr int HALF = CT::ENT / 2, ROW = HALF * 2 * Q + 1;  // entries per flush; stage row of a lane in uint4
    static_assert(CT::NCHAIN == 32 && HALF * 2 * Q == 32, "a lane per chain; a half chain is one 16-byte word per lane");
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, ch = threadIdx.x & 31;
    uint32_t nkeys = __ldg(nkeys_ptr);
    if (nkeys > cap) nkeys = cap;
    if (k >= nkeys || !keyflags[k]) return;  // a warp leaves together
    extern __shared__ uint32_t tab[];
    uint4 *stage = reinterpret_cast<uint4 *>(tab) + (threadIdx.x >> 5) * 32 * ROW;
    const uint4 *h4 = reinterpret_cast<const uint4 *>(hs), *z4 = reinterpret_cast<const uint4 *>(ztop);
    uint4 *out = reinterpret_cast<uint4 *>(ktab) + (size_t)k * CT::POINTS * 2 * Q;
    uint32_t zi[N];  // 1 / Z_e, walking e = ENT .. 1
#pragma unroll
    for (int w = 0; w < Q; w++) unquad<N>(zi, w, z4[S::z(k, w) + ch]);
    auto load = [&](int slot, uint32_t (&x)[N], uint32_t (&y)[N]) {
#pragma unroll
        for (int w = 0; w < Q; w++) { unquad<N>(x, w, h4[S::jac(k, slot, w) + ch]); unquad<N>(y, w, h4[S::jac(k, slot, Q + w) + ch]); }
    };
    // entry e-1 and its Z ratio are loaded before entry e is converted (independent addresses: the loads overlap the
    // multiplications)
    uint32_t x[N], y[N];
    load(CT::ENT - 1, x, y);
#pragma unroll 1
    for (int e = CT::ENT; e >= 1; e--) {
        uint32_t nx[N], ny[N], nh[N];
        if (e >= 2) {
            load(e - 2, nx, ny);
#pragma unroll
            for (int w = 0; w < Q; w++) unquad<N>(nh, w, h4[S::hs(k, e - 1, w) + ch]);
        }
        uint32_t z2[N], z3[N];
        A::fsqr(z2, zi);
        A::fmul(z3, z2, zi);
        A::fmul(x, x, z2);
        A::fmul(y, y, z3);
        uint4 *row = stage + ch * ROW + ((e - 1) % HALF) * 2 * Q;
#pragma unroll
        for (int w = 0; w < Q; w++) { row[w] = quad<N>(x, w); row[Q + w] = quad<N>(y, w); }
        if ((e - 1) % HALF == 0) {  // slots e-1 .. e-1+HALF-1 of every chain are staged: chain j's are word ch of its half
            __syncwarp();
            uint4 *o = out + (size_t)(e - 1) * 2 * Q + ch;
#pragma unroll 4
            for (int j = 0; j < CT::NCHAIN; j++) o[(size_t)j * CT::ENT * 2 * Q] = stage[j * ROW + ch];
            __syncwarp();
        }
        if (e >= 2) {  // 1/Z_{e-1} = (1/Z_e) * H_e
            A::fmul(zi, zi, nh);
            mp_copy<N>(x, nx); mp_copy<N>(y, ny);
        }
    }
}

template <class KT> struct IsComb { static constexpr bool value = false; };
template <class C> struct IsComb<CombTab<C>> { static constexpr bool value = true; };

// words of scratch the builder needs for `cap` keys (KT: KeyTab or CombTab)
template <class C, class KT_>
struct KtSizes {
    using KT = KT_;
    static constexpr size_t bases_words(size_t cap) { return (size_t)KT::NBASE * 3 * C::N * cap; }
    // the Z ratios; for a comb also the Jacobian entries (CombScr)
    static constexpr size_t hs_words(size_t cap) {
        return IsComb<KT>::value ? CombScr<C>::KEY * 4 * cap : (size_t)KT::NCHAIN * (KT::ENT - 1) * C::N * cap;
    }
    static constexpr size_t ztop_words(size_t cap) { return (size_t)KT::NCHAIN * C::N * cap; }
    static constexpr size_t ktab_words(size_t cap) { return KT::POINTS * 2 * C::N * cap; }
};

}  // namespace sbv
