// debug_ops.cuh — arithmetic-layer test operations shared by the GPU test hook (debug.cu, sbv_debug_op) and the
// CPU host simulation of the same headers (tools/hostsim).  Test infrastructure; not part of include/sbv.h.
// Operands are little-endian 32-bit limb arrays, 2N limbs per slot (unused limbs zero).
//
// op & 0xff: 0 fmul, 1 fadd, 2 fsub, 3 nmul, 4 f_inv, 5 doubling, 6 general add, 7 mixed add, 8 n_inv, 9 fsqr, 10 p_inv.
// Flags: DEBUG_INL runs the op with the inlined field multiplications of Inl<C> (the fixed-base kernels' arithmetic);
// DEBUG_NEG / DEBUG_SKIP are the `neg` / `skip` arguments of the additions (ops 6, 7).  For ops 5-7 an accumulator
// given as (0, 0) is the point at infinity (Z = 0).
#pragma once
#include "kernels.cuh"

namespace sbv {

constexpr int DEBUG_INL = 0x100, DEBUG_NEG = 0x200, DEBUG_SKIP = 0x400;

template <class C>
SBV_DEV void debug_op_item(int op, uint32_t i, const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, uint32_t *__restrict__ out) {
    constexpr int N = C::N;
    const bool neg = (op & DEBUG_NEG) != 0, skip = (op & DEBUG_SKIP) != 0;
    op &= 0xff;
    uint32_t x[N], y[N], u[N], v[N], r0[N], r1[N];
    for (int k = 0; k < N; k++) { x[k] = a[i * 2 * N + k]; y[k] = a[i * 2 * N + N + k]; u[k] = b[i * 2 * N + k]; v[k] = b[i * 2 * N + N + k]; r0[k] = 0; r1[k] = 0; }
    uint32_t rr[N], one[N], plain1[N];
    C::get_rr_p(rr); C::get_one(one);
    for (int k = 0; k < N; k++) plain1[k] = (k == 0);
    if (op == 0) C::fmul(r0, x, u);
    else if (op == 1) C::fadd(r0, x, u);
    else if (op == 2) C::fsub(r0, x, u);
    else if (op == 3) C::nmul(r0, x, u);
    else if (op == 4) f_inv<C>(r0, x);
    else if (op == 8) n_inv<C>(r0, x);
    else if (op == 10) p_inv<C>(r0, x);
    else if (op == 9) C::fsqr(r0, x);
    else if (op >= 5 && op <= 7) {
        // affine plain (x,y) [+ (u,v)] -> Montgomery Jacobian -> op -> affine plain
        Jac<C> P;
        const bool inf = mp_is_zero<N>(x) && mp_is_zero<N>(y);
        C::fmul(P.X, x, rr); C::fmul(P.Y, y, rr); mp_copy<N>(P.Z, one);
        if (inf) { mp_copy<N>(P.X, one); mp_copy<N>(P.Y, one); for (int k = 0; k < N; k++) P.Z[k] = 0; }
        uint32_t um[N], vm[N];
        C::fmul(um, u, rr); C::fmul(vm, v, rr);
        if (op == 5) pt_double<C>(P);
        else if (op == 6) {
            // general add with a non-trivial Z2: scale (u,v) by z=3 -> (9u, 27v, 3)
            uint32_t z[N], z2[N], z3[N], t[N];
            C::fadd(t, one, one); C::fadd(z, t, one);
            C::fsqr(z2, z); C::fmul(z3, z2, z);
            C::fmul(um, um, z2); C::fmul(vm, vm, z3);
            pt_double<C>(P);  // make Z1 non-trivial as well: P = 2*(x,y)
            pt_add<C, false>(P, um, vm, z, neg, skip);
        } else pt_add<C, true>(P, um, vm, one, neg, skip);
        if (mp_is_zero<N>(P.Z)) { for (int k = 0; k < N; k++) { r0[k] = 0; r1[k] = 0; } }
        else {
            uint32_t zi[N], zi2[N], zi3[N];
            f_inv<C>(zi, P.Z);
            C::fsqr(zi2, zi); C::fmul(zi3, zi2, zi);
            C::fmul(r0, P.X, zi2); C::fmul(r1, P.Y, zi3);
            C::fmul(r0, r0, plain1); C::fmul(r1, r1, plain1);  // out of Montgomery form
        }
    }
    for (int k = 0; k < N; k++) { out[i * 2 * N + k] = r0[k]; out[i * 2 * N + N + k] = r1[k]; }
}

// DEBUG_INL selects the arithmetic policy; the other bits go to debug_op_item
template <class C>
SBV_DEV void debug_op_dispatch(int op, uint32_t i, const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, uint32_t *__restrict__ out) {
    if (op & DEBUG_INL) debug_op_item<Inl<C>>(op & ~DEBUG_INL, i, a, b, out);
    else debug_op_item<C>(op, i, a, b, out);
}

}  // namespace sbv
