// kernels.cuh — sm_90a kernels of the sbv hot path (ECDSA verify over NIST prime curves).
//
//   k_gtable_init        one-time: affine fixed-base comb table  T[i][b] = b * 2^(GW*i) * G  (Montgomery form;
//                        GW = 16 for both curves: 64 MiB for P-256, mostly in L2; 151 MB for P-384, in HBM)
//   k_prep               per batch: range checks, batched inversion of s mod n (Montgomery's trick over S items
//                        per thread, one binary-extended-GCD inversion per thread), u1 = e/s, u2 = r/s written
//                        word-major ([2N][n] words) so that every consumer reads them coalesced and cuts its own
//                        digits (comb digits of u1, Booth digits of u2 for whatever window it uses)
//   k_verify_coz         keys-per-item path for keys that occur ONCE (or too rarely) in a batch, one signature per
//                        thread: on-curve check, 4-bit signed window over a common-Z table of Q (shared memory,
//                        bank = lane, + coalesced global scratch), 256 doublings interleaved with 65 additions, 16
//                        comb additions for u1*G with the next gather in flight, final X == r*Z^2 comparison
//   k_gpart              u1*G alone, for the items of keys that repeat inside a batch (window 0 loaded, 15 additions)
//   k_verify_comb        FIXED-BASE path for P-256 keys that repeat inside a batch (comb table of the key, keygroup.cuh
//                        builds it on the fly): 31 comb additions (the first entry is loaded) and 15 doublings for
//                        u2*Q, then k_gpart's u1*G
//   k_verify_kt          FIXED-BASE path over a window table: registered keys (sbv_set_keys, 8-bit windows, built once
//                        per key set) and P-384 keys that repeat inside a batch (5-bit windows): no doublings,
//                        NWIN(W) signed-window additions for u2*Q + the comb additions for u1*G
//   k_verify_kt_warp     the same, ONE SIGNATURE PER WARP (small batches: lanes add their table points,
//                        shuffle-tree reduction)
//
// Reference boundary: api.Verifier.VerifyConsenterSig / VerifySignature / VerifyRequest
// (/root/reference/pkg/api/dependencies.go:54-71) — the arithmetic itself is Go crypto/ecdsa
// semantics (see include/sbv.h).
#pragma once
#include "curve.cuh"

namespace sbv {

template <int BITS, int W>
struct Windows {
    static constexpr int COUNT = (BITS + 1 + W - 1) / W;  // Booth windows covering BITS+1 bits
    static constexpr int ENTRIES = 1 << (W - 1);          // table holds 1..2^(W-1) times Q
};

template <class C>
SBV_DEV void load_affine(uint32_t (&x)[C::N], uint32_t (&y)[C::N], const uint4 *src) {
    constexpr int N = C::N;
#pragma unroll
    for (int i = 0; i < N / 4; i++) {
        uint4 v = __ldg(src + i);
        x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w;
        uint4 u = __ldg(src + N / 4 + i);
        y[4 * i] = u.x; y[4 * i + 1] = u.y; y[4 * i + 2] = u.z; y[4 * i + 3] = u.w;
    }
}

// ------------------------------------------------------------------------------------------------
template <class C>
__global__ void k_gtable_init(uint32_t *__restrict__ gtab) {
    constexpr int N = C::N;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= C::GWINS << C::GW) return;
    const int win = t >> C::GW, b = t & ((1 << C::GW) - 1);
    uint32_t *out = gtab + (size_t)t * 2 * N;
    if (b == 0) {
        for (int i = 0; i < 2 * N; i++) out[i] = 0;
        return;
    }
    Jac<C> base;
    C::get_gx(base.X); C::get_gy(base.Y); C::get_one(base.Z);
    for (int i = 0; i < C::GW * win; i++) pt_double<C>(base);
    Jac<C> acc;
    C::get_one(acc.X); C::get_one(acc.Y);
#pragma unroll
    for (int i = 0; i < N; i++) acc.Z[i] = 0;
    for (int bit = C::GW - 1; bit >= 0; bit--) {
        pt_double<C>(acc);
        pt_add<C, false>(acc, base.X, base.Y, base.Z, false, !((b >> bit) & 1));
    }
    uint32_t zi[N], zi2[N], zi3[N], x[N], y[N];
    f_inv<C>(zi, acc.Z);
    C::fsqr(zi2, zi);
    C::fmul(zi3, zi2, zi);
    C::fmul(x, acc.X, zi2);
    C::fmul(y, acc.Y, zi3);
    for (int i = 0; i < N; i++) { out[i] = x[i]; out[N + i] = y[i]; }
}

// ------------------------------------------------------------------------------------------------
// digest -> e: leftmost min(dlen, BYTES) bytes as a big-endian integer (crypto/ecdsa hashToNat).
template <class C>
SBV_DEV void load_digest(uint32_t (&e)[C::N], const uint8_t *d, uint32_t dlen) {
    constexpr int N = C::N;
    if (dlen == (uint32_t)C::BYTES) { load_be<N>(e, d); return; }
    const int L = dlen < (uint32_t)C::BYTES ? (int)dlen : C::BYTES;
#pragma unroll
    for (int j = 0; j < N; j++) {
        uint32_t v = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int pos = L - 1 - (4 * j + k);
            uint32_t byte = pos >= 0 ? (uint32_t)d[pos] : 0u;
            v |= byte << (8 * k);
        }
        e[j] = v;
    }
}

// ---- scalar digits, cut by the consumers from the word-major scalars uw[2N][n] (u1 words, then u2 words) ----
// comb digit `win` of u1 (GW bits, little-endian); GW divides 32
template <class C>
SBV_DEV uint32_t comb_digit_u1(const uint32_t *__restrict__ uw, uint32_t n, uint32_t idx, int win) {
    const int pos = win * C::GW;
    return (__ldg(uw + (size_t)(pos >> 5) * n + idx) >> (pos & 31)) & ((1u << C::GW) - 1u);
}
// Booth digit `win` of u2 for a W-bit signed window: looks at bits [W*win - 1, W*win + W - 1] (bit -1 and the bits
// above 32N are zero) and returns d in [-2^(W-1), 2^(W-1)]; sum d_i 2^(W i) = u2.
template <class C, int W>
SBV_DEV int booth_digit_u2(const uint32_t *__restrict__ uw, uint32_t n, uint32_t idx, int win) {
    constexpr int N = C::N;
    const uint32_t *u2 = uw + (size_t)N * n + idx;
    const int pos = W * win - 1;
    uint32_t b;
    if (pos < 0) {
        b = (__ldg(u2) << 1) & ((2u << W) - 1);
    } else {
        const int wd = pos >> 5, sh = pos & 31;
        const uint32_t lo = wd < N ? __ldg(u2 + (size_t)wd * n) : 0u;
        const uint32_t hi = wd + 1 < N ? __ldg(u2 + (size_t)(wd + 1) * n) : 0u;
        b = __funnelshift_r(lo, hi, sh) & ((2u << W) - 1);
    }
    const uint32_t sign = b >> W;
    uint32_t d = sign ? (((2u << W) - 1) - b) : b;
    d = (d + 1) >> 1;
    return sign ? -(int)d : (int)d;
}

template <class C, int S>
__global__ void __launch_bounds__(128) k_prep(uint32_t n, const uint8_t *__restrict__ r_be, const uint8_t *__restrict__ s_be,
                                              const uint8_t *__restrict__ dig_be, uint32_t dlen,
                                              uint32_t *__restrict__ uw, uint8_t *__restrict__ flags) {
    constexpr int N = C::N;
    const uint32_t T = gridDim.x * blockDim.x;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t sm[S][N];    // Montgomery form of s (or 1 when out of range)
    uint32_t pref[S][N];  // running products
    uint32_t nmod[N], rr[N];
    C::get_n(nmod);
    C::get_rr_n(rr);
    uint32_t run[N];
    C::get_one_n(run);
    int cnt = 0;
#pragma unroll 1
    for (int k = 0; k < S; k++) {
        uint32_t idx = t + (uint32_t)k * T;
        if (idx >= n) break;
        uint32_t s[N], r[N];
        load_be<N>(s, s_be + (size_t)idx * C::BYTES);
        load_be<N>(r, r_be + (size_t)idx * C::BYTES);
        bool ok = !mp_is_zero<N>(s) && mp_lt<N>(s, nmod) && !mp_is_zero<N>(r) && mp_lt<N>(r, nmod);
        flags[idx] = ok ? 1 : 0;
        uint32_t one[N];
#pragma unroll
        for (int i = 0; i < N; i++) one[i] = (i == 0);
        uint32_t sv[N];
        mp_select<N>(sv, ok, s, one);
        uint32_t m[N];
        C::nmul(m, sv, rr);
        C::nmul(run, run, m);
#pragma unroll
        for (int i = 0; i < N; i++) { sm[k][i] = m[i]; pref[k][i] = run[i]; }
        cnt++;
    }
    if (cnt == 0) return;
    uint32_t inv[N];
    n_inv<C>(inv, run);
#pragma unroll 1
    for (int k = cnt - 1; k >= 0; k--) {
        uint32_t idx = t + (uint32_t)k * T;
        uint32_t w[N], m[N];
#pragma unroll
        for (int i = 0; i < N; i++) m[i] = sm[k][i];
        if (k > 0) {
            uint32_t pv[N];
#pragma unroll
            for (int i = 0; i < N; i++) pv[i] = pref[k - 1][i];
            C::nmul(w, inv, pv);
            C::nmul(inv, inv, m);
        } else {
            mp_copy<N>(w, inv);
        }
        // w = s^-1 in Montgomery form; u = x * w (plain) for x < 2^(32N)
        uint32_t e[N], r[N], u1[N], u2[N];
        load_digest<C>(e, dig_be + (size_t)idx * dlen, dlen);
        load_be<N>(r, r_be + (size_t)idx * C::BYTES);
        C::nmul(u1, e, w);
        C::nmul(u2, r, w);
#pragma unroll
        for (int i = 0; i < N; i++) {
            uw[(size_t)i * n + idx] = u1[i];
            uw[(size_t)(N + i) * n + idx] = u2[i];
        }
    }
}

#ifdef __CUDACC__
// host-side launcher of k_prep
template <class C, int S>
inline cudaError_t launch_prep(uint32_t n, const uint8_t *d_r, const uint8_t *d_s, const uint8_t *d_dig, uint32_t dlen, uint32_t *uw,
                               uint8_t *flags, cudaStream_t st) {
    constexpr int PB = 128;
    const uint32_t pthreads = (n + S - 1) / S;
    k_prep<C, S><<<(pthreads + PB - 1) / PB, PB, 0, st>>>(n, d_r, d_s, d_dig, dlen, uw, flags);
    return cudaGetLastError();
}
#endif

// accept iff R != inf and R.x mod n == r  <=>  X == r*Z^2 or (r + n < p and X == (r+n)*Z^2)
template <class C>
SBV_DEV bool final_check(const Jac<C> &acc, const uint8_t *__restrict__ r_be, uint32_t idx) {
    constexpr int N = C::N;
    bool match = false;
    if (!mp_is_zero<N>(acc.Z)) {
        uint32_t zz[N], r[N], rr[N], rm[N], lhs[N], pmn[N];
        C::fsqr(zz, acc.Z);
        load_be<N>(r, r_be + (size_t)idx * C::BYTES);
        C::get_rr_p(rr);
        C::fmul(rm, r, rr);
        C::fmul(lhs, rm, zz);
        match = mp_eq<N>(lhs, acc.X);
        C::get_p_minus_n(pmn);
        if (!match && mp_lt<N>(r, pmn)) {
            uint32_t r2[N], nmod[N];
            C::get_n(nmod);
            mp_add<N>(r2, r, nmod);
            C::fmul(rm, r2, rr);
            C::fmul(lhs, rm, zz);
            match = mp_eq<N>(lhs, acc.X);
        }
    }
    return match;
}

// key (x, y big-endian) -> Montgomery form; false unless both coordinates < p and y^2 == x^3 - 3x + b
template <class C>
SBV_DEV bool load_key(uint32_t (&qxm)[C::N], uint32_t (&qym)[C::N], const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be, uint32_t idx) {
    constexpr int N = C::N;
    uint32_t x[N], y[N], rr[N], pmod[N];
    C::get_p(pmod);
    load_be<N>(x, qx_be + (size_t)idx * C::BYTES);
    load_be<N>(y, qy_be + (size_t)idx * C::BYTES);
    bool good = mp_lt<N>(x, pmod) && mp_lt<N>(y, pmod);
    C::get_rr_p(rr);
    C::fmul(qxm, x, rr);
    C::fmul(qym, y, rr);
    uint32_t lhs[N], rhs[N], t[N], b[N];
    C::fsqr(lhs, qym);
    C::fsqr(t, qxm);
    C::fmul(rhs, t, qxm);
    C::fsub(rhs, rhs, qxm); C::fsub(rhs, rhs, qxm); C::fsub(rhs, rhs, qxm);
    C::get_b(b);
    C::fadd(rhs, rhs, b);
    return good && mp_eq<N>(lhs, rhs);
}

// acc += u1*G from the fixed-base comb: GWINS complete points.  The next entry (a random gather from the
// table, an L2 hit for most entries) is in flight while the current one is added.
// FROM_INF: acc is the point at infinity on entry (k_gpart): window 0's entry is loaded into it (pt_seed) instead of
// added, and the loop adds windows 1..GWINS-1.
template <class C, bool FROM_INF = false>
SBV_DEV void add_u1G(Jac<C> &acc, const uint32_t *__restrict__ uw, uint32_t n, uint32_t idx, const uint4 *__restrict__ gtab) {
    constexpr int N = C::N;
    constexpr int EU4 = 2 * N / 4;
    constexpr int W0 = FROM_INF ? 1 : 0;  // first window added
    uint32_t one[N];
    C::get_one(one);
    uint32_t gx[N], gy[N];
    uint32_t gb = comb_digit_u1<C>(uw, n, idx, W0);
    load_affine<C>(gx, gy, gtab + (((size_t)W0 << C::GW) + gb) * EU4);
    if constexpr (FROM_INF) {
        uint32_t sx[N], sy[N];
        const uint32_t sb = comb_digit_u1<C>(uw, n, idx, 0);
        load_affine<C>(sx, sy, gtab + (size_t)sb * EU4);
        pt_seed<C>(acc, sx, sy, false, sb == 0);
    }
#pragma unroll 1
    for (int win = W0; win < C::GWINS; win++) {
        uint32_t ngx[N], ngy[N];
        uint32_t ngb = 0;
        if (win + 1 < C::GWINS) {
            ngb = comb_digit_u1<C>(uw, n, idx, win + 1);
            load_affine<C>(ngx, ngy, gtab + (((size_t)(win + 1) << C::GW) + ngb) * EU4);
        }
        pt_add<C, true>(acc, gx, gy, one, false, gb == 0);
        if (win + 1 < C::GWINS) { mp_copy<N>(gx, ngx); mp_copy<N>(gy, ngy); gb = ngb; }
    }
}

// ------------------------------------------------------------------------------------------------
// k_verify_coz — keys-per-item path with a 4-bit signed window over a COMMON-Z table of Q.
// The eight multiples k*Q are brought to one shared Z (Zc), so a table entry is 64 bytes: 2Q..8Q
// live in shared memory (448 B per thread, bank = lane), 1Q and Zc, Zc^2, Zc^3 in a coalesced global
// scratch (tscr[.][n]).  65 additions of 11M+3S.
// `list`/`count` (optional): the thread handles item list[t], t < *count — the items the key grouping
// (keygroup.cuh) left on this path.  Items whose key or (r, s) are invalid reject at once.
template <class C, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_verify_coz(uint32_t n, const uint8_t *__restrict__ qx_be, const uint8_t *__restrict__ qy_be,
                                                             const uint8_t *__restrict__ r_be, const uint32_t *__restrict__ uw,
                                                             const uint8_t *__restrict__ flags,
                                                             const uint4 *__restrict__ gtab, uint32_t *__restrict__ tscr,
                                                             uint8_t *__restrict__ ok_out, const uint32_t *__restrict__ list,
                                                             const uint32_t *__restrict__ count) {
    constexpr int N = C::N;
    constexpr int W = 4;
    constexpr int NWIN = Windows<32 * N, W>::COUNT;
    extern __shared__ uint32_t tab[];  // entries 2..8: [((k-2)*2 + coord)*N + limb][BLOCK]
    const uint32_t tid = threadIdx.x;
    const uint32_t t = blockIdx.x * BLOCK + tid;
    if (t >= (list ? __ldg(count) : n)) return;  // the table is thread-private: no block-wide barrier anywhere
    const uint32_t idx = list ? __ldg(list + t) : t;
#define TAB(k, c, w) tab[((((k) - 2) * 2 + (c)) * N + (w)) * BLOCK + tid]
#define SCR(w) tscr[(size_t)(w) * n + t]
    // scratch words: [0,2N) entry 1 (x, y) ; [2N,3N) Zc ; [3N,4N) Zc^2 ; [4N,5N) Zc^3 ; [5N, 12N) H_2..H_8
    uint32_t one[N];
    C::get_one(one);
    {
        uint32_t qxm[N], qym[N];
        const bool good = load_key<C>(qxm, qym, qx_be, qy_be, idx) && flags[idx] != 0;
        if (!good) { ok_out[idx] = 0; return; }
        // forward: T_k = k*Q in Jacobian; keep (X_k, Y_k) and the ratio H_k = Z_k / Z_{k-1}
        Jac<C> P;
        mp_copy<N>(P.X, qxm); mp_copy<N>(P.Y, qym); mp_copy<N>(P.Z, one);
        pt_double<C>(P);  // T_2, Z_2 = 2*y  (ratio to Z_1 = 1)
#pragma unroll
        for (int i = 0; i < N; i++) { TAB(2, 0, i) = P.X[i]; TAB(2, 1, i) = P.Y[i]; SCR(5 * N + i) = P.Z[i]; }
#pragma unroll 1
        for (int k = 3; k <= 8; k++) {
            uint32_t h[N];
            pt_madd_table<C>(P, qxm, qym, h);
#pragma unroll
            for (int i = 0; i < N; i++) { TAB(k, 0, i) = P.X[i]; TAB(k, 1, i) = P.Y[i]; SCR((5 + k - 2) * N + i) = h[i]; }
        }
        // common Z = Z_8
        {
            uint32_t z2[N], z3[N];
            C::fsqr(z2, P.Z);
            C::fmul(z3, z2, P.Z);
#pragma unroll
            for (int i = 0; i < N; i++) { SCR(2 * N + i) = P.Z[i]; SCR(3 * N + i) = z2[i]; SCR(4 * N + i) = z3[i]; }
        }
        // backward: c_j = Z_8 / Z_j = H_{j+1} * ... * H_8 ; (X_j, Y_j) *= (c_j^2, c_j^3)
        uint32_t cacc[N];
        mp_copy<N>(cacc, one);
#pragma unroll 1
        for (int j = 7; j >= 1; j--) {
            uint32_t h[N], c2[N], c3[N], xx[N], yy[N];
#pragma unroll
            for (int i = 0; i < N; i++) h[i] = SCR((5 + j + 1 - 2) * N + i);
            C::fmul(cacc, cacc, h);
            C::fsqr(c2, cacc);
            C::fmul(c3, c2, cacc);
            if (j >= 2) {
#pragma unroll
                for (int i = 0; i < N; i++) { xx[i] = TAB(j, 0, i); yy[i] = TAB(j, 1, i); }
            } else {
                mp_copy<N>(xx, qxm); mp_copy<N>(yy, qym);
            }
            C::fmul(xx, xx, c2);
            C::fmul(yy, yy, c3);
            if (j >= 2) {
#pragma unroll
                for (int i = 0; i < N; i++) { TAB(j, 0, i) = xx[i]; TAB(j, 1, i) = yy[i]; }
            } else {
#pragma unroll
                for (int i = 0; i < N; i++) { SCR(i) = xx[i]; SCR(N + i) = yy[i]; }
            }
        }
    }
    Jac<C> acc;
    mp_copy<N>(acc.X, one);
    mp_copy<N>(acc.Y, one);
#pragma unroll
    for (int i = 0; i < N; i++) acc.Z[i] = 0;

#pragma unroll 1
    for (int win = NWIN - 1; win >= 0; win--) {
        if (win != NWIN - 1) {
#pragma unroll 1
            for (int k = 0; k < W; k++) pt_double<C>(acc);
        }
        const int d = booth_digit_u2<C, W>(uw, n, idx, win);
        bool neg = d < 0, skip = d == 0;
        int e = neg ? -d : d;          // 0..8
        int es = e < 2 ? 2 : e;        // shared-memory slot actually read
        uint32_t x2[N], y2[N], zc[N], zc2[N], zc3[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            uint32_t sx = TAB(es, 0, i), sy = TAB(es, 1, i);
            uint32_t gx1 = SCR(i), gy1 = SCR(N + i);
            x2[i] = e == 1 ? gx1 : sx;
            y2[i] = e == 1 ? gy1 : sy;
            zc[i] = SCR(2 * N + i); zc2[i] = SCR(3 * N + i); zc3[i] = SCR(4 * N + i);
        }
        pt_add_m<C, 2>(acc, x2, y2, zc, zc2, zc3, neg, skip);
    }
    add_u1G<C>(acc, uw, n, idx, gtab);
#undef TAB
#undef SCR
    ok_out[idx] = final_check<C>(acc, r_be, idx) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// Per-key tables (keygroup.cuh builds both kinds).  The builder sees a table as NBASE bases 2^(STEP*i) * Q (a chain of
// doublings) and NCHAIN chains of ENT entries, the entries of a chain sharing one chain of Z ratios.
//
// Window table (registered keys; P-384 keys grouped inside a launch): KT[kid][win][e-1] = e * 2^(W*win) * Q_kid for e = 1..2^(W-1), affine Montgomery
// form.  u2*Q = sum over the NWIN Booth digits of u2: no doublings at all.
template <int BITS, int W>
struct KeyTab {
    static constexpr int NWIN = Windows<BITS, W>::COUNT;
    static constexpr int ENT = Windows<BITS, W>::ENTRIES;
    static constexpr int NBASE = NWIN, STEP = W, NCHAIN = NWIN;
    static constexpr size_t POINTS = (size_t)NWIN * ENT;  // affine points per key
};

// Comb table (P-256 keys grouped inside a launch; Lim–Lee, Hankerson–Menezes–Vanstone Alg. 3.44): 16 bases P_c = 2^(SPACING*c) * Q
// in BLOCKS = 2 blocks of TEETH = 8; a scalar is read as 16 rows of SPACING bits (row c = bits [SPACING*c, SPACING*(c+1))),
// and column j of the rows of block b is the mask m of entry T_b[m] = sum of P_(8b+t) over the set bits t of m.  u2*Q then
// takes SPACING - 1 doublings and 2 * SPACING additions (P-256: 15 and 32, P-384: 23 and 48).
// Layout: chain (b, hi) holds the 16 entries m = 16*hi + g in Gray-code order of the low nibble g (the order the builder
// walks them), so T_b[m] is slot (16*b + hi)*16 + k with gray(k) = g; the slot of m = 0 (hi = 0, k = 0) is never read.
template <class C>
struct CombTab {
    static constexpr int TEETH = 8, BLOCKS = 2, NBASE = TEETH * BLOCKS;
    static constexpr int SPACING = 32 * C::N / NBASE;       // 16 for P-256, 24 for P-384
    static constexpr int STEP = SPACING;
    static constexpr int NCHAIN = BLOCKS * 16, ENT = 16;  // (block, high nibble) x low nibble
    static constexpr size_t POINTS = (size_t)NCHAIN * ENT;  // 512 affine points per key: 32 KiB (P-256), 48 KiB (P-384)
    static_assert(SPACING * NBASE == 32 * C::N, "the rows cover the scalar exactly");
    SBV_DEV static uint32_t slot(int b, uint32_t m) {
        const uint32_t g = m & 15u;
        return ((uint32_t)b * 16u + (m >> 4)) * 16u + (g ^ (g >> 1) ^ (g >> 2) ^ (g >> 3));  // inverse Gray code of g
    }
};

// column j of block b of u2's comb: bit t = bit SPACING*(8b + t) + j of u2
template <class C>
SBV_DEV uint32_t comb_mask_u2(const uint32_t *__restrict__ uw, uint32_t n, uint32_t idx, int b, int j) {
    using CT = CombTab<C>;
    const uint32_t *u2 = uw + (size_t)C::N * n + idx;
    uint32_t m = 0;
#pragma unroll
    for (int t = 0; t < CT::TEETH; t++) {
        const int pos = CT::SPACING * (CT::TEETH * b + t) + j;
        m |= ((__ldg(u2 + (size_t)(pos >> 5) * n) >> (pos & 31)) & 1u) << t;
    }
    return m;
}

// Inl<C>: the same curve with the field multiplications inlined at every call site instead of called out of line —
// no argument marshalling and free scheduling across multiplications, at ~3 KB of code per site.  Only for loops
// with a single addition site (the fixed-base kernel below), which still fit the instruction cache.
template <class C>
struct Inl : C {
    SBV_DEV static void fmul(uint32_t (&r)[C::N], const uint32_t (&a)[C::N], const uint32_t (&b)[C::N]) { C::fmul_inline(r, a, b); }
    SBV_DEV static void fsqr(uint32_t (&r)[C::N], const uint32_t (&a)[C::N]) { C::fsqr_inline(r, a); }
};
template <class C, bool INL> struct PickArith { using type = C; };
template <class C> struct PickArith<C, true> { using type = Inl<C>; };

// k_gpart — the u1*G half of a fixed-base verification on its own: needs only the scalars, so the grouped pipeline runs
// it while the per-key tables are still being built; k_verify_comb (k_verify_kt<…, REG = false>) then closes with (starts
// from) the stored point.
// gacc: [3N][n] words (X, Y, Z of item idx at column idx).  The accumulator starts at infinity: window 0 is loaded, not added.
template <class C, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_gpart(uint32_t n, const uint32_t *__restrict__ uw, const uint4 *__restrict__ gtab,
                                                        uint32_t *__restrict__ gacc) {
    constexpr int N = C::N;
    const uint32_t idx = blockIdx.x * BLOCK + threadIdx.x;
    if (idx >= n) return;
    Jac<C> acc;
    add_u1G<C, true>(acc, uw, n, idx, gtab);
#pragma unroll
    for (int i = 0; i < N; i++) {
        gacc[(size_t)i * n + idx] = acc.X[i];
        gacc[(size_t)(N + i) * n + idx] = acc.Y[i];
        gacc[(size_t)(2 * N + i) * n + idx] = acc.Z[i];
    }
}

// REG = true: registered keys (sbv_set_keys): the key of item i is kidmap[slot[i]].
// REG = false: keys grouped on the fly: the key of item i is kidmap[i] (>= 0 for every listed item).
// gacc != NULL: the u1*G half was computed by k_gpart; only the key's windows remain.
// One loop over the NWIN windows of u2*Q and then the GWINS windows of u1*G: a single addition site, with the table
// entry of the next window (a random 64-byte gather) in flight while the current one is added.
template <class C, int W, int BLOCK, int MINB, bool REG, bool INL>
__global__ void __launch_bounds__(BLOCK, MINB) k_verify_kt(uint32_t n, const uint32_t *__restrict__ slot, const int32_t *__restrict__ kidmap,
                                                            uint32_t n_slots, const uint8_t *__restrict__ keyflags,
                                                            const uint8_t *__restrict__ r_be, const uint32_t *__restrict__ uw,
                                                            const uint8_t *__restrict__ flags, const uint4 *__restrict__ gtab,
                                                            const uint4 *__restrict__ ktab, uint8_t *__restrict__ ok_out,
                                                            const uint32_t *__restrict__ list, const uint32_t *__restrict__ count,
                                                            const uint32_t *__restrict__ gacc) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy
    constexpr int N = C::N;
    constexpr int EU4 = 2 * N / 4;  // uint4 per table entry
    using KT = KeyTab<32 * N, W>;
    const int TOTAL = gacc ? KT::NWIN : KT::NWIN + C::GWINS;
    const uint32_t t = blockIdx.x * BLOCK + threadIdx.x;
    if (t >= (list ? __ldg(count) : n)) return;
    const uint32_t idx = list ? __ldg(list + t) : t;
    bool good = flags[idx] != 0;
    int32_t kid;
    if (REG) {
        const uint32_t sl = slot[idx];
        kid = sl < n_slots ? kidmap[sl] : -1;
    } else {
        kid = kidmap[idx];
    }
    good = good && kid >= 0 && keyflags[kid < 0 ? 0 : kid] != 0;
    if (!good) { ok_out[idx] = 0; return; }
    const uint4 *kt = ktab + (size_t)kid * KT::POINTS * EU4;
    uint32_t one[N];
    C::get_one(one);
    Jac<A> acc;
    if (gacc) {
#pragma unroll
        for (int i = 0; i < N; i++) {
            acc.X[i] = __ldg(gacc + (size_t)i * n + idx);
            acc.Y[i] = __ldg(gacc + (size_t)(N + i) * n + idx);
            acc.Z[i] = __ldg(gacc + (size_t)(2 * N + i) * n + idx);
        }
    }
    // window w < NWIN: signed digit of u2 into the key's table; w >= NWIN: comb digit of u1 into the table of G
    auto fetch = [&](int w, uint32_t (&x)[N], uint32_t (&y)[N], bool &neg, bool &skip) {
        if (w < KT::NWIN) {
            const int d = booth_digit_u2<C, W>(uw, n, idx, w);
            const int e = d < 0 ? -d : d;
            load_affine<C>(x, y, kt + ((size_t)w * KT::ENT + (e ? e - 1 : 0)) * EU4);
            neg = d < 0; skip = d == 0;
        } else {
            const int g = w - KT::NWIN;
            const uint32_t b = comb_digit_u1<C>(uw, n, idx, g);
            load_affine<C>(x, y, gtab + (((size_t)g << C::GW) + b) * EU4);
            neg = false; skip = b == 0;
        }
    };
    uint32_t cx[N], cy[N];
    bool cneg, cskip;
    fetch(0, cx, cy, cneg, cskip);
    int w0 = 0;  // first window added
    if (!gacc) {  // the accumulator starts at infinity: window 0's entry is loaded, not added
        pt_seed<A>(acc, cx, cy, cneg, cskip);
        fetch(1, cx, cy, cneg, cskip);
        w0 = 1;
    }
#pragma unroll 1
    for (int w = w0; w < TOTAL; w++) {
        uint32_t nx[N], ny[N];
        bool nneg = false, nskip = true;
        if (w + 1 < TOTAL) fetch(w + 1, nx, ny, nneg, nskip);
        pt_add<A, true>(acc, cx, cy, one, cneg, cskip);
        if (w + 1 < TOTAL) { mp_copy<N>(cx, nx); mp_copy<N>(cy, ny); cneg = nneg; cskip = nskip; }
    }
    Jac<C> fin;
    mp_copy<N>(fin.X, acc.X); mp_copy<N>(fin.Y, acc.Y); mp_copy<N>(fin.Z, acc.Z);
    ok_out[idx] = final_check<C>(fin, r_be, idx) ? 1 : 0;
}

// k_verify_comb — keys grouped inside a launch: the key of item list[t] is kidmap[list[t]] (>= 0 for every listed item),
// its table a CombTab.  u2*Q column by column from the top: a doubling (none before the first column), then one table
// addition per block; then u1*G, after the last doubling: one general addition of k_gpart's point (gacc).
// One inlined addition site and one doubling site in one loop: the addition hands its exceptional case (accumulator ==
// entry) to the doubling site (pt_add_m<…, DEFER>) instead of carrying its own copy of the doubling, and the next table
// entry (a random 64-byte gather) is in flight while the current one is added.  The additions stay complete.  The first
// step's entry is loaded into the accumulator (pt_seed), so the loop adds steps 1..KADD-1.
template <class C, int BLOCK, int MINB, bool INL>
__global__ void __launch_bounds__(BLOCK, MINB) k_verify_comb(uint32_t n, const int32_t *__restrict__ kidmap, const uint8_t *__restrict__ keyflags,
                                                              const uint8_t *__restrict__ r_be, const uint32_t *__restrict__ uw,
                                                              const uint8_t *__restrict__ flags,
                                                              const uint4 *__restrict__ ktab, uint8_t *__restrict__ ok_out,
                                                              const uint32_t *__restrict__ list, const uint32_t *__restrict__ count,
                                                              const uint32_t *__restrict__ gacc) {
    using A = typename PickArith<C, INL>::type;  // arithmetic policy of the loop
    constexpr int N = C::N;
    constexpr int EU4 = 2 * N / 4;  // uint4 per table entry
    using CT = CombTab<C>;
    constexpr int KADD = CT::SPACING * CT::BLOCKS;  // key additions
    const uint32_t t = blockIdx.x * BLOCK + threadIdx.x;
    if (t >= __ldg(count)) return;
    const uint32_t idx = __ldg(list + t);
    const int32_t kid = kidmap[idx];
    const bool good = flags[idx] != 0 && kid >= 0 && keyflags[kid < 0 ? 0 : kid] != 0;
    if (!good) { ok_out[idx] = 0; return; }
    const uint4 *kt = ktab + (size_t)kid * CT::POINTS * EU4;
    uint32_t one[N];
    C::get_one(one);
    // step s: column SPACING-1 - s/2, block s%2 of u2's comb
    auto fetch = [&](int s, uint32_t (&x)[N], uint32_t (&y)[N], bool &skip) {
        const int b = s & 1;
        const uint32_t m = comb_mask_u2<C>(uw, n, idx, b, CT::SPACING - 1 - (s >> 1));
        load_affine<C>(x, y, kt + (size_t)CT::slot(b, m) * EU4);
        skip = m == 0;
    };
    uint32_t cx[N], cy[N];
    bool cskip;
    fetch(1, cx, cy, cskip);
    Jac<A> acc;
    {  // step 0 meets the accumulator at infinity: its entry is loaded, not added
        uint32_t sx[N], sy[N];
        bool sskip;
        fetch(0, sx, sy, sskip);
        pt_seed<A>(acc, sx, sy, false, sskip);
    }
    int s = 1, dbl = 0;  // dbl: doublings due before the addition of step s
#pragma unroll 1
    while (s < KADD || dbl) {
        if (dbl) {
            pt_double<A>(acc);
            dbl--;
            continue;
        }
        uint32_t nx[N], ny[N];
        bool nskip = true;
        if (s + 1 < KADD) fetch(s + 1, nx, ny, nskip);
        dbl = pt_add_m<A, 1, true>(acc, cx, cy, one, one, one, false, cskip) ? 1 : 0;  // acc == entry: the sum is 2 * acc
        s++;
        if (s < KADD && (s & 1) == 0) dbl++;  // next column
        if (s < KADD) { mp_copy<N>(cx, nx); mp_copy<N>(cy, ny); cskip = nskip; }
    }
    Jac<C> fin;
    mp_copy<N>(fin.X, acc.X); mp_copy<N>(fin.Y, acc.Y); mp_copy<N>(fin.Z, acc.Z);
    {  // the closing general addition (out-of-line multiplications: once per signature, outside the loop)
        Jac<C> g;
#pragma unroll
        for (int i = 0; i < N; i++) {
            g.X[i] = __ldg(gacc + (size_t)i * n + idx);
            g.Y[i] = __ldg(gacc + (size_t)(N + i) * n + idx);
            g.Z[i] = __ldg(gacc + (size_t)(2 * N + i) * n + idx);
        }
        pt_add<C, false>(fin, g.X, g.Y, g.Z, false, mp_is_zero<N>(g.Z));
    }
    ok_out[idx] = final_check<C>(fin, r_be, idx) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// k_verify_kt_warp — ONE SIGNATURE PER WARP, for small batches (latency path of the registered-key
// entry points).  The NWIN + GWINS table additions of a signature are independent, so each lane adds
// its two or three table points and the 32 partial sums are tree-reduced with warp shuffles (5 general
// additions).  Per signature this issues ~6x the instructions of the thread-per-signature kernel, but
// its dependent chain is 3 + 5 additions instead of NWIN + GWINS.  Chosen by the launcher when the batch
// cannot fill the machine anyway.
template <class C, int W>
__global__ void __launch_bounds__(128) k_verify_kt_warp(uint32_t n, const uint32_t *__restrict__ slot, const int32_t *__restrict__ slot2local,
                                                        uint32_t n_slots, const uint8_t *__restrict__ keyflags,
                                                        const uint8_t *__restrict__ r_be, const uint32_t *__restrict__ uw,
                                                        const uint8_t *__restrict__ flags,
                                                        const uint4 *__restrict__ gtab, const uint4 *__restrict__ ktab,
                                                        uint8_t *__restrict__ ok_out) {
    constexpr int N = C::N;
    constexpr int EU4 = 2 * N / 4;
    using KT = KeyTab<32 * N, W>;
    const uint32_t idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // signature = warp
    const uint32_t lane = threadIdx.x & 31;
    if (idx >= n) return;
    bool good = flags[idx] != 0;
    const uint32_t sl = slot[idx];
    int32_t local = sl < n_slots ? slot2local[sl] : -1;
    good = good && local >= 0;
    if (local < 0) local = 0;
    good = good && keyflags[local] != 0;
    const uint4 *kt = ktab + (size_t)local * KT::POINTS * EU4;
    uint32_t one[N];
    C::get_one(one);
    Jac<C> acc;
    mp_copy<N>(acc.X, one);
    mp_copy<N>(acc.Y, one);
#pragma unroll
    for (int i = 0; i < N; i++) acc.Z[i] = 0;
#pragma unroll 1
    for (int it = 0; it < (KT::NWIN + 31) / 32; it++) {  // u2 * Q_k : this lane's windows
        const int win = it * 32 + (int)lane;
        const bool live = win < KT::NWIN;
        const int d = live ? booth_digit_u2<C, W>(uw, n, idx, win) : 0;
        const int e = d < 0 ? -d : d;
        uint32_t x2[N], y2[N];
        load_affine<C>(x2, y2, kt + ((size_t)(live ? win : 0) * KT::ENT + (e ? e - 1 : 0)) * EU4);
        pt_add<C, true>(acc, x2, y2, one, d < 0, d == 0);
    }
#pragma unroll 1
    for (int it = 0; it < (C::GWINS + 31) / 32; it++) {  // u1 * G
        const int win = it * 32 + (int)lane;
        const bool live = win < C::GWINS;
        const uint32_t b = live ? comb_digit_u1<C>(uw, n, idx, win) : 0u;
        uint32_t x2[N], y2[N];
        load_affine<C>(x2, y2, gtab + (((size_t)(live ? win : 0) << C::GW) + b) * EU4);
        pt_add<C, true>(acc, x2, y2, one, false, b == 0);
    }
#pragma unroll 1
    for (int off = 16; off >= 1; off >>= 1) {  // tree reduction of the 32 partial sums
        uint32_t x2[N], y2[N], z2[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            x2[i] = __shfl_down_sync(0xffffffffu, acc.X[i], off);
            y2[i] = __shfl_down_sync(0xffffffffu, acc.Y[i], off);
            z2[i] = __shfl_down_sync(0xffffffffu, acc.Z[i], off);
        }
        pt_add<C, false>(acc, x2, y2, z2, false, mp_is_zero<N>(z2));
    }
    if (lane != 0) return;
    ok_out[idx] = (good && final_check<C>(acc, r_be, idx)) ? 1 : 0;
}

}  // namespace sbv
