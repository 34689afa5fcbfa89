#include <cstring>
#include <vector>

#include "engine.h"
#include "debug_ops.cuh"
#include "ed25519_debug.cuh"
#include "rsa_debug.cuh"
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

namespace {
__global__ void k_debug_ed25519(int op, uint32_t n, const uint32_t *__restrict__ in, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ed_debug_dispatch(op, i, in, out);
}
}  // namespace

// Ed25519 arithmetic on device 0: op and the 24-word slots of in / out as in ed25519_debug.cuh.
extern "C" int sbv_debug_ed25519(sbv_engine *e, int op, size_t n, const uint32_t *in, uint32_t *out) {
    if (!e || op < ED_DBG_MUL || op > ED_DBG_REDUCE || !in || !out) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    const size_t bytes = n * ED_DEBUG_WORDS * 4;
    int rc = sbv_ensure_scratch(e, d, 2 * bytes + 1024);
    if (rc) return rc;
    uint32_t *din = (uint32_t *)d.d_scratch, *dout = din + n * ED_DEBUG_WORDS;
    CU(e, cudaMemcpyAsync(din, in, bytes, cudaMemcpyHostToDevice, d.stream));
    k_debug_ed25519<<<(uint32_t)((n + 63) / 64), 64, 0, d.stream>>>(op, (uint32_t)n, din, dout);
    CU(e, cudaGetLastError());
    CU(e, cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

namespace {
__global__ void k_debug_ed25519_point(int op, uint32_t n, const uint32_t *__restrict__ in, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ed_point_dispatch(op, i, in, out);
}
}  // namespace

// Ed25519 point ops on device 0: op (operation | ED_PT_* flags) and the ED_POINT_WORDS-word slots of in / out as in
// ed25519_debug.cuh.  SBV_ERR_ARG for an op or flag the dispatch does not run.
extern "C" int sbv_debug_ed25519_point(sbv_engine *e, int op, size_t n, const uint32_t *in, uint32_t *out) {
    if (!e || !ed_point_op_ok(op) || !in || !out || n > UINT32_MAX) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    const size_t bytes = n * ED_POINT_WORDS * 4;
    int rc = sbv_ensure_scratch(e, d, 2 * bytes + 1024);
    if (rc) return rc;
    uint32_t *din = (uint32_t *)d.d_scratch, *dout = din + n * ED_POINT_WORDS;
    CU(e, cudaMemcpyAsync(din, in, bytes, cudaMemcpyHostToDevice, d.stream));
    k_debug_ed25519_point<<<(uint32_t)((n + 63) / 64), 64, 0, d.stream>>>(op, (uint32_t)n, din, dout);
    CU(e, cudaGetLastError());
    CU(e, cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// The production SHA-512 kernel of Ed25519 on device 0: dig_out = the 64-byte digests of R || A || M (as SHA-512 outputs
// them), k_out = the 8 little-endian limbs of k = digest mod L per item.  msg_off are offsets into msgs (off[0] may be > 0).
extern "C" int sbv_debug_ed25519_sha512(sbv_engine *e, size_t n, const uint8_t *msgs, const uint64_t *msg_off, const uint8_t *sig,
                                        const uint8_t *pub, uint8_t *dig_out, uint32_t *k_out) {
    if (!e || !msgs || !msg_off || !sig || !pub || !dig_out || !k_out) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    const size_t mb = (msg_off[n] + 16 + 255) & ~(size_t)255, ob = ((n + 1) * 8 + 255) & ~(size_t)255;
    const size_t need = mb + ob + n * 64 + n * 32 + n * 64 + n * 32;
    int rc = sbv_ensure_scratch(e, d, need + 1024);
    if (rc) return rc;
    uint8_t *p = d.d_scratch;
    uint8_t *dm = p; p += mb;
    uint64_t *doff = (uint64_t *)p; p += ob;
    uint8_t *dsig = p; p += n * 64;
    uint8_t *dpub = p; p += n * 32;
    uint32_t *ddig = (uint32_t *)p; p += n * 64;
    uint32_t *dk = (uint32_t *)p;
    CU(e, cudaMemcpyAsync(dm, msgs, msg_off[n], cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(doff, msg_off, (n + 1) * 8, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dsig, sig, n * 64, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dpub, pub, n * 32, cudaMemcpyHostToDevice, d.stream));
    if ((rc = sbv_launch_ed_sha512_digest(e, n, dm, doff, dsig, dpub, dk, ddig, d.stream))) return rc;
    std::vector<uint32_t> dig(n * 16), kw(n * 8);
    CU(e, cudaMemcpyAsync(dig.data(), ddig, n * 64, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaMemcpyAsync(kw.data(), dk, n * 32, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    for (size_t i = 0; i < n; i++) {
        for (int w = 0; w < 16; w++)  // digest limbs are little-endian: back to bytes
            for (int b = 0; b < 4; b++) dig_out[i * 64 + 4 * w + b] = (uint8_t)(dig[i * 16 + w] >> (8 * b));
        for (int w = 0; w < 8; w++) k_out[i * 8 + w] = kw[(size_t)w * n + i];
    }
    return SBV_OK;
}

// The RSA arithmetic of rsa.cuh on device 0: op and the item layout of rsa_debug.cuh (a, b, mod, out: mod_bytes bytes per
// item; exp, aux: one word), k_rsa_debug in blocks of 128 threads as k_rsa_verify runs.  SBV_ERR_ARG, with nothing
// written, for a modulus size outside 256 / 384 / 512, an op outside 0-4, a null buffer or n >= 2^31.
extern "C" int sbv_debug_rsa(sbv_engine *e, uint32_t mod_bytes, int op, size_t n, const uint8_t *a, const uint8_t *b, const uint8_t *mod,
                             const uint32_t *exp, uint8_t *out, uint32_t *aux) {
    if (!e || !rsa_debug_args_ok(mod_bytes, op, n, a, b, mod, exp, out, aux)) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    const size_t bytes = n * mod_bytes, words = (n * 4 + 255) & ~(size_t)255;
    int rc = sbv_ensure_scratch(e, d, 4 * bytes + 2 * words + 1024);
    if (rc) return rc;
    uint8_t *p = d.d_scratch;
    uint8_t *da = p; p += bytes;
    uint8_t *db = p; p += bytes;
    uint8_t *dmod = p; p += bytes;
    uint8_t *dout = p; p += bytes;
    uint32_t *dexp = (uint32_t *)p; p += words;
    uint32_t *daux = (uint32_t *)p;
    CU(e, cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dmod, mod, bytes, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dexp, exp, n * 4, cudaMemcpyHostToDevice, d.stream));
    rsa_nl(mod_bytes, [&](auto nl) {
        k_rsa_debug<decltype(nl)::value><<<rsa_grid(n, RSA_GROUP), RSA_BLOCK, 0, d.stream>>>(op, (uint32_t)n, da, db, dmod, dexp, dout, daux);
    });
    CU(e, cudaGetLastError());
    CU(e, cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaMemcpyAsync(aux, daux, n * 4, cudaMemcpyDeviceToHost, d.stream));
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

// Copies entries [first, first + count) of the 8-bit window table of registered ECDSA slot `slot` on device 0
// (sbv_set_keys: entry win * 128 + e - 1 is e * 2^(8 win) * Q, affine Montgomery x then y, 2N limbs).  SBV_ERR_ARG for a
// slot that is not a key of `curve`, a key that got no table (off the curve, coordinate >= p) or a range outside the table.
extern "C" int sbv_debug_key_table(sbv_engine *e, uint8_t curve, uint32_t slot, size_t first, size_t count, uint32_t *out) {
    if (!e || curve > SBV_P384 || !out) return SBV_ERR_ARG;
    const CurveOps &ops = sbv_ops(curve);
    const size_t words = 2 * (size_t)ops.N, entries = ops.kt8->geom.ktab_words / words;
    if (first > entries || count > entries - first) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    if (slot >= d.n_slots || !d.slot2local[curve]) return SBV_ERR_ARG;
    CU(e, cudaSetDevice(d.ordinal));
    int32_t loc = -1;
    CU(e, cudaMemcpy(&loc, d.slot2local[curve] + slot, sizeof loc, cudaMemcpyDeviceToHost));
    if (loc < 0 || (uint32_t)loc >= d.n_local[curve]) return SBV_ERR_ARG;
    uint8_t flag = 0;
    CU(e, cudaMemcpy(&flag, d.keyflags[curve] + loc, 1, cudaMemcpyDeviceToHost));
    if (!flag) return SBV_ERR_ARG;
    CU(e, cudaMemcpyAsync(out, d.ktab[curve] + (size_t)loc * ops.kt8->geom.ktab_words + first * words, count * words * 4, cudaMemcpyDeviceToHost,
                          d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

namespace {
// The tables of a keys-per-item launch of scheme s over the n keys of a (and b: ECDSA qy, else nullptr), key_bytes per key
// in each, on device 0: the first half of the launch (sbv_launch_verify_begin: grouping with the engine's SBV_GROUP_*
// settings and the table construction), then the scratch set goes back.  For each of the m query items items[q] < n:
// status[q] = 0 and the key's table at out + q * (table words), as the verification kernel reads it; 1 when the key got
// no table (fewer items than the threshold, table slots used up, or a launch that does not group); 2 when it got a
// table slot but is not a valid key.
int grouped_tables(sbv_engine *e, const char *what, uint8_t scheme, size_t n, size_t key_bytes, const uint8_t *a, const uint8_t *b, size_t m,
                   const uint32_t *items, int32_t *status, uint32_t *out) {
    for (size_t q = 0; q < m; q++)
        if (items[q] >= n) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    const size_t words = sbv_group_ops(scheme).kt->geom.ktab_words, kb = (n * key_bytes + 255) & ~(size_t)255;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    int rc = sbv_ensure_scratch(e, d, 2 * kb + 1024);
    if (rc) return rc;
    uint8_t *da = d.d_scratch, *db = b ? d.d_scratch + kb : nullptr;
    CU(e, cudaMemcpyAsync(da, a, n * key_bytes, cudaMemcpyHostToDevice, d.stream));
    if (b) CU(e, cudaMemcpyAsync(db, b, n * key_bytes, cudaMemcpyHostToDevice, d.stream));
    VerifyLaunch vl;
    if ((rc = sbv_launch_verify_begin(e, d, scheme, n, da, db, d.stream, &vl))) return rc;
    Dev::Scratch *w = vl.w;
    uint32_t nkeys = 0;
    cudaError_t st = cudaSuccess;
    if (vl.grouping) {
        st = cudaStreamWaitEvent(d.stream, w->ev_tab, 0);
        if (st == cudaSuccess) st = cudaStreamSynchronize(d.stream);
        if (st == cudaSuccess) st = cudaMemcpy(&nkeys, (uint32_t *)w->zeroed, 4, cudaMemcpyDeviceToHost);  // counters[0]: may exceed the slots
    }
    const size_t kcap = vl.grouping ? w->keyflags.bytes : 0;  // bound for the key ids read back (they are < the launch's slots)
    for (size_t q = 0; q < m && st == cudaSuccess; q++) {
        status[q] = 1;
        if (!vl.grouping) continue;
        uint32_t r = 0;
        int32_t kid = -1;
        uint8_t flag = 0;
        st = cudaMemcpy(&r, (uint32_t *)w->rep + items[q], 4, cudaMemcpyDeviceToHost);
        if (st == cudaSuccess && r < n) st = cudaMemcpy(&kid, (int32_t *)w->keyid + r, 4, cudaMemcpyDeviceToHost);
        if (kid < 0 || (size_t)kid >= kcap || (uint32_t)kid >= nkeys) continue;
        if (st == cudaSuccess) st = cudaMemcpy(&flag, (uint8_t *)w->keyflags + kid, 1, cudaMemcpyDeviceToHost);
        if (st == cudaSuccess && flag)
            st = cudaMemcpy(out + q * words, (uint32_t *)w->ktab + (size_t)kid * words, words * 4, cudaMemcpyDeviceToHost);
        if (st == cudaSuccess) status[q] = flag ? 0 : 2;
    }
    if (st != cudaSuccess) return sbv_launch_verify_close(e, vl, d.stream, sbv_fail(e, SBV_ERR_CUDA, "%s: %s", what, cudaGetErrorString(st)));
    if ((rc = sbv_launch_verify_close(e, vl, d.stream, 0))) return rc;
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// Every k (8 little-endian limbs per item) is < L: the kernels only ever see reduced k, and their recoding of the top
// window assumes bit 255 clear.
bool k_below_l(size_t n, const uint32_t *k) {
    static const uint32_t L[8] = {0x5cf5d3ed, 0x5812631a, 0xa2f79cd6, 0x14def9de, 0, 0, 0, 0x10000000};
    for (size_t i = 0; i < n; i++) {
        int w = 7;
        while (w > 0 && k[i * 8 + w] == L[w]) w--;
        if (k[i * 8 + w] >= L[w]) return false;
    }
    return true;
}
}  // namespace

// The per-key tables of a keys-per-item launch of the n keys (qx, qy: BYTES each) on device 0, as grouped_tables reads
// them (P-256: CombTab, 512 entries in slot order; P-384: KeyTab<384, 5>, 77 x 16 entries; affine Montgomery x then y,
// 2N limbs each).
extern "C" int sbv_debug_grouped_key_table(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *qx, const uint8_t *qy, size_t m,
                                           const uint32_t *items, int32_t *status, uint32_t *out) {
    if (!e || curve > SBV_P384 || !qx || !qy || (m && (!items || !status || !out)) || n > UINT32_MAX) return SBV_ERR_ARG;
    return grouped_tables(e, "sbv_debug_grouped_key_table", curve, n, (size_t)sbv_ops(curve).bytes, qx, qy, m, items, status, out);
}

// Copies entries [first, first + count) of device 0's fixed-base table of B (k_ed_btab_init: entry win * 128 + j - 1 is
// j * 256^win * B as y + x, y - x, 2dxy, 24 limbs) to the host, building the table if no Ed25519 call has yet.
extern "C" int sbv_debug_ed25519_btab(sbv_engine *e, size_t first, size_t count, uint32_t *out) {
    if (!e || !out || first > SBV_ED_BTAB_ENTRIES || count > SBV_ED_BTAB_ENTRIES - first) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    int rc = sbv_ed_btab_ensure(e, d);
    if (rc) return rc;
    const size_t words = SBV_ED_BTAB_ENTRY_WORDS;
    CU(e, cudaMemcpyAsync(out, d.ed_btab + first * words, count * words * 4, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// The production Ed25519 verification kernel on device 0 with the caller's k in place of SHA-512(R || A || M) mod L, so
// that tests can choose it: k = 8 little-endian limbs per item, each < L (SBV_ERR_ARG otherwise: the kernel only ever sees
// reduced k, and its recoding of the top window assumes bit 255 clear).  sig: 64 bytes per item (R || S), pub: 32.
extern "C" int sbv_debug_ed25519_verify_k(sbv_engine *e, size_t n, const uint8_t *sig, const uint8_t *pub, const uint32_t *k, uint8_t *ok) {
    if (!e || !sig || !pub || !k || !ok || n > UINT32_MAX) return SBV_ERR_ARG;
    if (!k_below_l(n, k)) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    int rc = sbv_ed_btab_ensure(e, d);
    if (rc) return rc;
    const size_t okb = (n + 255) & ~(size_t)255;
    if ((rc = sbv_ensure_scratch(e, d, n * 64 + n * 32 + n * 32 + okb + 1024))) return rc;
    uint8_t *p = d.d_scratch;
    uint8_t *dsig = p; p += n * 64;
    uint8_t *dpub = p; p += n * 32;
    uint32_t *dk = (uint32_t *)p; p += n * 32;
    uint8_t *dok = p;
    std::vector<uint32_t> kw(n * 8);
    for (size_t i = 0; i < n; i++)
        for (int w = 0; w < 8; w++) kw[(size_t)w * n + i] = k[i * 8 + w];
    CU(e, cudaMemcpyAsync(dsig, sig, n * 64, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dpub, pub, n * 32, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dk, kw.data(), n * 32, cudaMemcpyHostToDevice, d.stream));
    if ((rc = sbv_launch_ed_verify_k(e, d, n, dsig, dpub, dk, dok, d.stream))) return rc;
    CU(e, cudaMemcpyAsync(ok, dok, n, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// Copies entries [first, first + count) of the table of registry slot `slot` on device 0 (sbv_ed25519_set_keys: entry
// win * 128 + j - 1 is j * 256^win * A as y + x, y - x, 2dxy, 24 limbs).  SBV_ERR_ARG for an unknown slot, a key that does
// not decode or a range outside the table.
extern "C" int sbv_debug_ed25519_ktab(sbv_engine *e, uint32_t slot, size_t first, size_t count, uint32_t *out) {
    if (!e || !out || first > SBV_ED_BTAB_ENTRIES || count > SBV_ED_BTAB_ENTRIES - first) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    if (slot >= d.ed_n_slots) return SBV_ERR_ARG;
    CU(e, cudaSetDevice(d.ordinal));
    int32_t loc = -1;
    CU(e, cudaMemcpy(&loc, d.ed_slot2local + slot, sizeof loc, cudaMemcpyDeviceToHost));
    if (loc < 0) return SBV_ERR_ARG;
    const size_t words = SBV_ED_BTAB_ENTRY_WORDS, per_key = SBV_ED_BTAB_ENTRIES * words;
    CU(e, cudaMemcpyAsync(out, d.ed_ktab + (size_t)loc * per_key + first * words, count * words * 4, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// The comb tables of a keys-per-item launch of the n keys of pub (32 bytes each) on device 0, as grouped_tables reads them
// (entry b * 255 + mask - 1 = the sum of 2^(16 (8b + t)) * A over the set bits t of mask, as y + x, y - x, 2dxy, 24
// limbs; 510 entries); status 2: the key does not decode.
extern "C" int sbv_debug_ed25519_comb_tab(sbv_engine *e, size_t n, const uint8_t *pub, size_t m, const uint32_t *items, int32_t *status,
                                          uint32_t *out) {
    if (!e || !pub || (m && (!items || !status || !out)) || n > UINT32_MAX) return SBV_ERR_ARG;
    return grouped_tables(e, "sbv_debug_ed25519_comb_tab", SBV_ED25519, n, 32, pub, nullptr, m, items, status, out);
}

// The comb kernel of grouped keys (k_ed_verify_comb) on device 0 with the caller's k in place of SHA-512(R || A || M) mod
// L: every distinct key of pub gets a comb table and every item takes the comb kernel.  k = 8 little-endian limbs per item,
// each < L (SBV_ERR_ARG otherwise); sig = R || S (64 bytes), pub = 32 bytes per item.
extern "C" int sbv_debug_ed25519_verify_comb_k(sbv_engine *e, size_t n, const uint8_t *sig, const uint8_t *pub, const uint32_t *k, uint8_t *ok) {
    if (!e || !sig || !pub || !k || !ok || n > UINT32_MAX) return SBV_ERR_ARG;
    if (!k_below_l(n, k)) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    int rc = sbv_ed_btab_ensure(e, d);
    if (rc) return rc;
    const size_t okb = (n + 255) & ~(size_t)255;
    if ((rc = sbv_ensure_scratch(e, d, n * 64 + n * 32 + n * 32 + okb + 1024))) return rc;
    uint8_t *p = d.d_scratch;
    uint8_t *dsig = p; p += n * 64;
    uint8_t *dpub = p; p += n * 32;
    uint32_t *dk = (uint32_t *)p; p += n * 32;
    uint8_t *dok = p;
    std::vector<uint32_t> kw(n * 8);
    for (size_t i = 0; i < n; i++)
        for (int w = 0; w < 8; w++) kw[(size_t)w * n + i] = k[i * 8 + w];
    CU(e, cudaMemcpyAsync(dsig, sig, n * 64, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dpub, pub, n * 32, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dk, kw.data(), n * 32, cudaMemcpyHostToDevice, d.stream));
    if ((rc = sbv_launch_ed_verify_comb_k(e, d, n, dsig, dpub, dk, dok, d.stream))) return rc;
    CU(e, cudaMemcpyAsync(ok, dok, n, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// The production registered-key kernel (k_ed_verify_keyed) on device 0 with the caller's k in place of SHA-512(R || A || M)
// mod L: k = 8 little-endian limbs per item, each < L (SBV_ERR_ARG otherwise), key_slot = registry slots, sig = R || S.
extern "C" int sbv_debug_ed25519_verify_registered_k(sbv_engine *e, size_t n, const uint32_t *key_slot, const uint8_t *sig, const uint32_t *k,
                                                     uint8_t *ok) {
    if (!e || !key_slot || !sig || !k || !ok || n > UINT32_MAX) return SBV_ERR_ARG;
    if (!k_below_l(n, k)) return SBV_ERR_ARG;
    if (n == 0) return SBV_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    int rc = sbv_ed_btab_ensure(e, d);
    if (rc) return rc;
    const size_t okb = (n + 255) & ~(size_t)255;
    if ((rc = sbv_ensure_scratch(e, d, n * 64 + n * 4 + n * 32 + okb + 1024))) return rc;
    uint8_t *p = d.d_scratch;
    uint8_t *dsig = p; p += n * 64;
    uint32_t *dk = (uint32_t *)p; p += n * 32;
    uint32_t *dslot = (uint32_t *)p; p += (n * 4 + 15) & ~(size_t)15;
    uint8_t *dok = p;
    std::vector<uint32_t> kw(n * 8);
    for (size_t i = 0; i < n; i++)
        for (int w = 0; w < 8; w++) kw[(size_t)w * n + i] = k[i * 8 + w];
    CU(e, cudaMemcpyAsync(dsig, sig, n * 64, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dk, kw.data(), n * 32, cudaMemcpyHostToDevice, d.stream));
    CU(e, cudaMemcpyAsync(dslot, key_slot, n * 4, cudaMemcpyHostToDevice, d.stream));
    if ((rc = sbv_launch_ed_verify_registered_k(e, d, n, dslot, dsig, dk, dok, d.stream))) return rc;
    CU(e, cudaMemcpyAsync(ok, dok, n, cudaMemcpyDeviceToHost, d.stream));
    CU(e, cudaStreamSynchronize(d.stream));
    return SBV_OK;
}

// The cached table of one key on device `device_index` (sbv_key_cache_reserve or _evicting): key = the exact key bytes of scheme s
// (qx || qy: 64 / 96 bytes; the 32-byte Ed25519 encoding).  Returns 1 with the table in out (the words of the scheme's
// per-launch table, as sbv_debug_grouped_key_table / sbv_debug_ed25519_comb_tab read it) when a READY slot holds the key,
// 0 when none does or no cache is reserved.  Drains the device first.
extern "C" int sbv_debug_key_cache_entry(sbv_engine *e, int device_index, uint8_t scheme, const uint8_t *key, uint32_t *out) {
    if (!e || scheme > SBV_ED25519 || !key || !out || device_index < 0 || device_index >= (int)e->devs.size()) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[device_index];
    const Dev::KeyCache &k = d.kc[scheme];
    if (!k.mem) return 0;
    const size_t kw = sbv_group_ops(scheme).key_words, slots = (size_t)k.map.smask + 1;
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, cudaDeviceSynchronize());
    if (k.evicting) {  // key_cache_assoc.cuh: way i is pool entry i
        std::vector<unsigned long long> st(k.capacity);
        std::vector<uint32_t> kv(k.capacity * kw);
        CU(e, cudaMemcpy(st.data(), k.amap.state, k.capacity * 8, cudaMemcpyDeviceToHost));
        CU(e, cudaMemcpy(kv.data(), k.amap.keys, k.capacity * kw * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < k.capacity; i++) {
            if ((st[i] & 3) != 2 || memcmp(&kv[i * kw], key, kw * 4) != 0) continue;
            CU(e, cudaMemcpy(out, k.amap.pool + i * k.tw4 * 4, k.tw4 * 16, cudaMemcpyDeviceToHost));
            return 1;
        }
        return 0;
    }
    std::vector<uint32_t> state(slots), keys(slots * kw);
    CU(e, cudaMemcpy(state.data(), k.map.state, slots * 4, cudaMemcpyDeviceToHost));
    CU(e, cudaMemcpy(keys.data(), k.map.keys, slots * kw * 4, cudaMemcpyDeviceToHost));
    for (size_t s = 0; s < slots; s++) {
        if ((state[s] & 3) != 2 || memcmp(&keys[s * kw], key, kw * 4) != 0) continue;  // low bits 2: KC_READY (key_cache.cuh)
        uint32_t at = 0;
        CU(e, cudaMemcpy(&at, k.map.pidx + s, 4, cudaMemcpyDeviceToHost));
        CU(e, cudaMemcpy(out, k.map.pool + (size_t)at * k.tw4 * 4, k.tw4 * 16, cudaMemcpyDeviceToHost));
        return 1;
    }
    return 0;
}

// The hash seed and set count of the evicting cache of scheme s on device `device_index` (key_cache_assoc.cuh: key w is in
// set umulhi(kc_hash(w, seed), sets)), so that a test can predict which keys compete for one set.  Returns 1 with out[0] =
// seed, out[1] = sets; 0 when no evicting cache is reserved.
extern "C" int sbv_debug_key_cache_sets(sbv_engine *e, int device_index, uint8_t scheme, uint32_t *out) {
    if (!e || scheme > SBV_ED25519 || !out || device_index < 0 || device_index >= (int)e->devs.size()) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    const Dev::KeyCache &k = e->devs[device_index].kc[scheme];
    if (!k.mem || !k.evicting) return 0;
    out[0] = k.amap.seed;
    out[1] = k.amap.sets;
    return 1;
}

// Copies the record of RSA registry slot `slot` on device 0 (sbv_rsa_set_keys; rsa_keyed.cuh): out[0..8) = {k, valid, ntop,
// n0', e, limb offset (2 words), 0}, then the K = k / 4 little-endian limbs of N and the K of R^2 mod N, 8 + 2K words (at
// most 264).  SBV_ERR_ARG for a slot outside the registry.
extern "C" int sbv_debug_rsa_key(sbv_engine *e, uint32_t slot, uint32_t *out) {
    if (!e || !out || e->devs.empty()) return SBV_ERR_ARG;
    std::shared_lock<std::shared_mutex> reg(e->registry_mu);
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    if (slot >= d.rsa_n_slots) return SBV_ERR_ARG;
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, cudaMemcpy(out, d.rsa_rec + 2 * (size_t)slot, 32, cudaMemcpyDeviceToHost));
    const uint64_t off = ((uint64_t)out[6] << 32) | out[5];
    CU(e, cudaMemcpy(out + 8, d.rsa_pool + off, (size_t)out[0] * 2, cudaMemcpyDeviceToHost));  // 2K words
    return SBV_OK;
}
