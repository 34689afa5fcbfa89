// engine.cu — host side of libsbv.so: the C ABI of include/sbv.h on top of the sm_90a kernels.
//
// One engine owns 1..8 devices of one box (single process), or is one RANK of a one-process-per-GPU deployment
// (sbv_comm_init_rank).  Every batch is sharded into contiguous ranges, one per device.  Every host-buffer entry point
// owns a lane (stream + buffers + pinned staging) per call, so up to SBV_LANES calls overlap; the per-launch scratch of
// the verify pipeline (pipeline.cu) is multi-buffered and event-guarded so launches on different streams overlap too.
// The only exchange between devices / ranks is the all-gather of packed verdict (and quorum) bitmasks, with NCCL
// (dlopen'd lazily).  No CPU fallback.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "engine.h"
#include "sha256.cuh"
#include "sha384.cuh"
#include "mixed_hash.cuh"
#include "quorum.cuh"
#include "shards.h"

using namespace sbv;

namespace {

int env_int(const char *name, int dflt) {
    const char *v = getenv(name);
    return v && *v ? atoi(v) : dflt;
}

size_t fbytes(uint8_t curve) { return curve == SBV_P256 ? 32 : 48; }

// a digest length the verify calls accept: whole 32-bit words, 4 to 64 bytes
bool digest_len_ok(uint8_t dl) { return dl != 0 && (dl & 3) == 0 && dl <= 64; }

bool is_pinned(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

__global__ void k_mad_probe(uint32_t *out, uint32_t iters) {
    uint32_t a = threadIdx.x * 2654435761u + 12345u, b = blockIdx.x * 40503u + 777u;
    uint64_t acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = a + i;
    for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = (uint64_t)a * (uint32_t)(b + i) + acc[i];  // IMAD.WIDE.U32
        a ^= (uint32_t)acc[3];
    }
    uint64_t s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s += acc[i];
    if (s == 0x1234567) out[0] = (uint32_t)s;
}

void buf_free(DevBuf &b) { if (b.p) cudaFree(b.p); b = DevBuf{}; }
void buf_free(PinBuf &b) { if (b.p) cudaFreeHost(b.p); b = PinBuf{}; }
// Replaces b's memory with `bytes` fresh bytes (its contents are not kept); on a fault b is left empty.
template <class Buf>
cudaError_t buf_regrow(Buf &b, size_t bytes) {
    buf_free(b);
    const cudaError_t err = std::is_base_of<PinBuf, Buf>::value ? cudaHostAlloc(&b.p, bytes, cudaHostAllocPortable) : cudaMalloc(&b.p, bytes);
    if (err == cudaSuccess) b.bytes = bytes; else b.p = nullptr;
    return err;
}

// Every buffer of lane ln, once: visit(buffer, need, alloc) with the bytes the call uses (need) and the bytes to allocate
// when the buffer must grow (alloc: the buffer's headroom rule).
template <class V>
void each_lane_buffer(Dev::Lane &ln, const LaneNeeds &s, V &&visit) {
    const size_t n = s.items, ni = n + n / 8 + 1024, o = s.offsets, oi = o + o / 8 + 1024;
    visit(ln.d_r, n * 48, ni * 48);
    visit(ln.d_s, n * 48, ni * 48);
    visit(ln.d_qx, n * 48, ni * 48);
    visit(ln.d_qy, n * 48, ni * 48);
    visit(ln.d_dig, n * 64, ni * 64);
    visit(ln.d_ok, n, ni);
    visit(ln.d_slot, n * 4, ni * 4);
    visit(ln.d_msgs, s.msg_bytes, s.msg_bytes + s.msg_bytes / 8 + 4096);
    visit(ln.d_off, o * 8, oi * 8);
    visit(ln.d_perm, o ? (o + 3 * 1024) * 4 : 0, (oi + 3 * 1024) * 4);
    visit(ln.h_pin, s.pinned, s.pinned + s.pinned / 4 + 4096);
    visit(ln.d_aux, s.aux, s.aux + s.aux / 4 + 4096);
    visit(ln.h_aux, s.aux, s.aux + s.aux / 4 + 4096);
    visit(ln.d_carve, s.carve, s.carve + s.carve / 8 + 4096);
}

// Frees every buffer, both streams and every event of lane ln; caller has set the device and drained it.
void lane_free(Dev::Lane &ln) {
    each_lane_buffer(ln, LaneNeeds{}, [](auto &b, size_t, size_t) { buf_free(b); });
    if (ln.stream) cudaStreamDestroy(ln.stream);
    if (ln.stream2) cudaStreamDestroy(ln.stream2);
    if (ln.ev_a) cudaEventDestroy(ln.ev_a);
    if (ln.ev_b) cudaEventDestroy(ln.ev_b);
    for (cudaEvent_t ev : ln.ev_chunk) if (ev) cudaEventDestroy(ev);
    ln = Dev::Lane{};
}

}  // namespace

int sbv_ensure_scratch(sbv_engine *e, Dev &d, size_t bytes) {
    if (bytes <= d.d_scratch.bytes) return 0;
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, buf_regrow(d.d_scratch, bytes + bytes / 4 + 4096));
    return 0;
}

int sbv_lane_acquire(sbv_engine *e) {
    std::unique_lock<std::mutex> lk(e->mu);
    int lane = -1;
    e->lane_cv.wait(lk, [&] {
        for (int i = 0; i < SBV_LANES; i++)
            if (!e->lane_busy[i]) { lane = i; return true; }
        return false;
    });
    e->lane_busy[lane] = true;
    return lane;
}
void sbv_lane_release(sbv_engine *e, int lane) {
    { std::lock_guard<std::mutex> lk(e->mu); e->lane_busy[lane] = false; }
    e->lane_cv.notify_one();
}
// Only the owner of the lane touches it, so no lock is needed here.
int sbv_lane_reserve(sbv_engine *e, Dev::Lane &ln, const LaneNeeds &needs) {
    if (!ln.stream) CU(e, cudaStreamCreateWithFlags(&ln.stream, cudaStreamNonBlocking));
    bool grows = false;
    each_lane_buffer(ln, needs, [&](DevBuf &b, size_t need, size_t) { grows = grows || need > b.bytes; });
    if (!grows) return 0;
    CU(e, cudaStreamSynchronize(ln.stream));
    if (ln.stream2) CU(e, cudaStreamSynchronize(ln.stream2));
    cudaError_t err = cudaSuccess;
    each_lane_buffer(ln, needs, [&](auto &b, size_t need, size_t alloc) {
        if (err == cudaSuccess && need > b.bytes) err = buf_regrow(b, alloc);
    });
    CU(e, err);
    return 0;
}
int sbv_lane_stream2(sbv_engine *e, Dev::Lane &ln) {
    if (ln.stream2) return 0;
    CU(e, cudaStreamCreateWithFlags(&ln.stream2, cudaStreamNonBlocking));
    CU(e, cudaEventCreateWithFlags(&ln.ev_a, cudaEventDisableTiming));
    CU(e, cudaEventCreateWithFlags(&ln.ev_b, cudaEventDisableTiming));
    return 0;
}
int sbv_launch_length_sort(sbv_engine *e, size_t n, const uint64_t *d_off, uint32_t *d_perm, cudaStream_t st, const uint32_t **perm) {
    *perm = nullptr;
    if (d_perm && n >= 2048) {  // sort by block count so that a warp's 32 messages have equal length
        uint32_t *hist = d_perm + n, *start = hist + SHA_BINS, *cursor = start + SHA_BINS;
        CU(e, cudaMemsetAsync(hist, 0, SHA_BINS * sizeof(uint32_t), st));
        k_sha_hist<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, d_off, hist);
        k_sha_scan<<<1, SHA_BINS, 0, st>>>(hist, start, cursor);
        k_sha_scatter<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, d_off, start, cursor, d_perm);
        e->launches += 3;
        *perm = d_perm;
    }
    return 0;
}
int sbv_launch_sha256(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                      cudaStream_t st) {
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_sha256<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_msgs, d_off, base, d_digest, perm);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
int sbv_launch_sha384(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                      cudaStream_t st) {
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_sha384<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_msgs, d_off, base, d_digest, perm);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
int sbv_launch_mix_alg(sbv_engine *e, size_t n, uint8_t *d_tag, uint8_t *d_alg, cudaStream_t st) {
    k_mix_alg<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, d_tag, d_alg);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
int sbv_launch_sha2_sel(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint32_t *d_idx,
                        const uint8_t *d_alg, uint32_t dlen, uint8_t *d_digest, uint32_t *d_perm, cudaStream_t st) {
    const uint32_t *perm = nullptr;
    int rc = sbv_launch_length_sort(e, n, d_off, d_perm, st, &perm);
    if (rc) return rc;
    k_sha2_sel<<<(uint32_t)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, d_msgs, d_off, base, d_idx, d_alg, dlen, d_digest, perm);
    e->launches += 1;
    CU(e, cudaGetLastError());
    return 0;
}
// H2D of a caller buffer on the lane's stream (or on st): direct when pinned, else through the lane's pinned staging area at offset
// `stage_off` (the caller sized it and does not reuse it until the stream has drained).
int sbv_lane_h2d(sbv_engine *e, Dev::Lane &ln, void *dst, const void *src, size_t bytes, size_t &stage_off, cudaStream_t st) {
    if (bytes == 0) return 0;
    if (!st) st = ln.stream;
    if (is_pinned(src)) {
        CU(e, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
    } else {
        if (stage_off + bytes > ln.h_pin.bytes) return fail(e, SBV_ERR_NOMEM, "pinned staging area too small (%zu + %zu > %zu)", stage_off, bytes, ln.h_pin.bytes);
        memcpy(ln.h_pin + stage_off, src, bytes);
        CU(e, cudaMemcpyAsync(dst, ln.h_pin + stage_off, bytes, cudaMemcpyHostToDevice, st));
        stage_off += (bytes + 255) & ~(size_t)255;
    }
    return 0;
}

namespace {

// ---- NCCL, loaded with dlopen only by multi-device / multi-rank engines ----
struct NcclUniqueId { char internal[128]; };
typedef int (*nccl_comm_init_all_t)(void **comms, int ndev, const int *devlist);
typedef int (*nccl_comm_init_rank_t)(void **comm, int nranks, NcclUniqueId id, int rank);
typedef int (*nccl_get_unique_id_t)(NcclUniqueId *id);
typedef int (*nccl_comm_destroy_t)(void *comm);
typedef int (*nccl_group_t)(void);
typedef int (*nccl_all_gather_t)(const void *send, void *recv, size_t count, int dtype, void *comm, cudaStream_t st);
typedef const char *(*nccl_err_t)(int);
struct NcclApi {
    void *lib = nullptr;
    nccl_comm_init_all_t comm_init_all = nullptr;
    nccl_comm_init_rank_t comm_init_rank = nullptr;
    nccl_get_unique_id_t get_unique_id = nullptr;
    nccl_comm_destroy_t comm_destroy = nullptr;
    nccl_group_t group_start = nullptr, group_end = nullptr;
    nccl_all_gather_t all_gather = nullptr;
    nccl_err_t err_string = nullptr;
} g_nccl;
std::mutex g_nccl_mu;
constexpr int NCCL_UINT32 = 3;  // ncclUint32

int nccl_load(sbv_engine *e) {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.lib) return 0;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
    if (!h) return fail(e, SBV_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
    g_nccl.comm_init_all = (nccl_comm_init_all_t)dlsym(h, "ncclCommInitAll");
    g_nccl.comm_init_rank = (nccl_comm_init_rank_t)dlsym(h, "ncclCommInitRank");
    g_nccl.get_unique_id = (nccl_get_unique_id_t)dlsym(h, "ncclGetUniqueId");
    g_nccl.comm_destroy = (nccl_comm_destroy_t)dlsym(h, "ncclCommDestroy");
    g_nccl.group_start = (nccl_group_t)dlsym(h, "ncclGroupStart");
    g_nccl.group_end = (nccl_group_t)dlsym(h, "ncclGroupEnd");
    g_nccl.all_gather = (nccl_all_gather_t)dlsym(h, "ncclAllGather");
    g_nccl.err_string = (nccl_err_t)dlsym(h, "ncclGetErrorString");
    if (!g_nccl.comm_init_all || !g_nccl.comm_init_rank || !g_nccl.get_unique_id || !g_nccl.comm_destroy || !g_nccl.group_start ||
        !g_nccl.group_end || !g_nccl.all_gather)
        return fail(e, SBV_ERR_NCCL, "libnccl lacks a required symbol");
    g_nccl.lib = h;
    return 0;
}
#define NC(e, call)                                                                                       \
    do {                                                                                                  \
        int _r = (call);                                                                                  \
        if (_r != 0)                                                                                      \
            return fail(e, SBV_ERR_NCCL, "%s failed: %s", #call, g_nccl.err_string ? g_nccl.err_string(_r) : "?"); \
    } while (0)

int sync_lane(sbv_engine *e, int lane) {
    for (Dev &d : e->devs) {
        if (!d.lanes[lane].stream) continue;
        CU(e, cudaSetDevice(d.ordinal));
        CU(e, cudaStreamSynchronize(d.lanes[lane].stream));
    }
    return 0;
}

// The verdicts of sbv_verify_batch and of the commit-vote calls leave the devices in two steps.  shard_out runs on device
// g's lane stream behind its verdicts d_ok (s.vr[g].n bytes) and reached flags d_rch (s.ir[g].n bytes, if there are
// instances).  A single device copies them to the host directly.  Several pack them (k_pack_bits) into device g's slot of
// its gather buffer gbuf (s.wp() * G words); then gather_unpack issues one grouped ncclAllGather (in place, on the lane
// streams), copies the whole buffer from device 0 into the lane's pinned mirror, drains the lane and unpacks on the host.
int shard_out(sbv_engine *e, Dev::Lane &ln, const Shards &s, int g, uint32_t *gbuf, const uint8_t *d_ok, const uint8_t *d_rch, uint8_t *ok,
              uint8_t *reached) {
    const size_t nv = s.vr[g].n, ni = s.ir.empty() ? 0 : s.ir[g].n;
    if (s.vr.size() == 1) {
        if (nv) CU(e, cudaMemcpyAsync(ok, d_ok, nv, cudaMemcpyDeviceToHost, ln.stream));
        if (ni) CU(e, cudaMemcpyAsync(reached, d_rch, ni, cudaMemcpyDeviceToHost, ln.stream));
        return 0;
    }
    uint32_t *mine = gbuf + s.wp() * g;
    CU(e, cudaMemsetAsync(mine, 0, s.wp() * 4, ln.stream));
    if (nv) {  // a grid of zero blocks is an invalid configuration
        k_pack_bits<<<(uint32_t)((nv + 255) / 256), 256, 0, ln.stream>>>((uint32_t)nv, d_ok, mine);
        e->launches += 1;
    }
    if (ni) {
        k_pack_bits<<<(uint32_t)((ni + 255) / 256), 256, 0, ln.stream>>>((uint32_t)ni, d_rch, mine + s.wv);
        e->launches += 1;
    }
    CU(e, cudaGetLastError());
    return 0;
}

int gather_unpack(sbv_engine *e, int lane, const Shards &s, const std::vector<uint32_t *> &gbuf, uint8_t *ok, uint8_t *reached) {
    const int G = (int)s.vr.size();
    const size_t wp = s.wp();
    if (G > 1) {
        {
            std::lock_guard<std::mutex> lk(e->mu);  // collectives of one communicator set must be issued in one order
            NC(e, g_nccl.group_start());
            for (int g = 0; g < G; g++)
                NC(e, g_nccl.all_gather(gbuf[g] + wp * g, gbuf[g], wp, NCCL_UINT32, e->nccl_comms[g], e->devs[g].lanes[lane].stream));
            NC(e, g_nccl.group_end());
        }
        Dev &d0 = e->devs[0];
        CU(e, cudaSetDevice(d0.ordinal));
        CU(e, cudaMemcpyAsync(d0.lanes[lane].h_aux, gbuf[0], wp * G * 4, cudaMemcpyDeviceToHost, d0.lanes[lane].stream));
    }
    int rc = sync_lane(e, lane);
    if (rc) return rc;
    if (G > 1) unpack_shards(s, (const uint32_t *)e->devs[0].lanes[lane].h_aux, ok, reached);
    return SBV_OK;
}

// The hash that turns the messages of an ECDSA call into its digests (e = their leftmost field bytes).
// (SHA-512 serves the RSA calls only.)  The values are the SBV_HASH_* tags.
enum class MsgHash : uint8_t { sha256, sha384, sha512 };
uint32_t hash_bytes(MsgHash h) { return h == MsgHash::sha512 ? 64u : h == MsgHash::sha384 ? 48u : 32u; }
int launch_hash(sbv_engine *e, MsgHash h, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                cudaStream_t st) {
    if (h == MsgHash::sha512) return sbv_launch_sha512(e, n, d_msgs, d_off, base, d_digest, d_perm, st);
    return h == MsgHash::sha384 ? sbv_launch_sha384(e, n, d_msgs, d_off, base, d_digest, d_perm, st)
                                : sbv_launch_sha256(e, n, d_msgs, d_off, base, d_digest, d_perm, st);
}

// One shard of a keys-per-item host-buffer call on device d's lane: what to verify and where it comes from.
struct BatchSrc {
    const uint8_t *r, *s, *qx, *qy;
    const uint8_t *digest;      // fixed-width digests, or nullptr: the digests are `hash` of the messages below
    uint8_t digest_len;
    const uint8_t *msgs;
    const uint64_t *msg_off;
    MsgHash hash = MsgHash::sha256;
};

// Stages items [lo, lo+cnt) and enqueues hashing (if asked for) and the verify pipeline; verdicts land in ln.d_ok (and the
// digests in ln.d_dig) in ln.stream order.  The KEYS go first, so that the grouping and the table construction run while
// the rest of the batch is still being copied.  A LARGE shard (>= chunk_items) then arrives in chunks on the lane's
// second stream while the lane's first stream hashes and verifies the chunks that are already there: the call costs
// max(upload, arithmetic) instead of their sum (C3: 1,048,576 requests of 256 B are 411 MB of upload).
// more / so_out: the caller's own needs of the lane (the pinned bytes and aux area of the quorum columns, or a gather
// buffer), reserved with ours; the caller stages its arrays behind ours in the lane's pinned area.
int stage_and_verify(sbv_engine *e, Dev &d, Dev::Lane &ln, uint8_t curve, size_t lo, size_t cnt, const BatchSrc &b, const LaneNeeds &more = {},
                     size_t *so_out = nullptr) {
    const size_t L = fbytes(curve);
    const bool hashing = b.digest == nullptr;
    const uint32_t dlen = hashing ? hash_bytes(b.hash) : b.digest_len;
    CU(e, cudaSetDevice(d.ordinal));
    const uint64_t base = hashing ? b.msg_off[lo] : 0, bytes = hashing ? b.msg_off[lo + cnt] - base : 0;
    int chunks = 1;
    if (e->chunk_items > 0 && cnt >= (size_t)e->chunk_items) {  // at least two chunks, nominally chunk_items each
        chunks = (int)std::min<size_t>(std::max<size_t>(cnt / (size_t)e->chunk_items, 2), SBV_MAX_CHUNKS);
    }
    const size_t per = (((cnt + chunks - 1) / chunks) + 255) & ~(size_t)255;   // items per chunk
    LaneNeeds need = more;
    need.items = cnt;
    need.pinned += cnt * (4 * L + dlen + 1) + bytes + (cnt + 1) * 8 + (size_t)(4 * chunks + 8) * 256;
    if (hashing) need.msgs(bytes, cnt);
    int rc = sbv_lane_reserve(e, ln, need);
    if (rc) return rc;
    cudaStream_t up = ln.stream;   // the stream the rest of the batch is uploaded on
    if (chunks > 1) {
        if (int rc2 = sbv_lane_stream2(e, ln)) return rc2;
        for (int c = 0; c < chunks; c++)
            if (!ln.ev_chunk[c]) CU(e, cudaEventCreateWithFlags(&ln.ev_chunk[c], cudaEventDisableTiming));
        up = ln.stream2;
    }
    size_t so = 0;
    if ((rc = sbv_lane_h2d(e, ln, ln.d_qx, b.qx + lo * L, cnt * L, so))) return rc;
    if ((rc = sbv_lane_h2d(e, ln, ln.d_qy, b.qy + lo * L, cnt * L, so))) return rc;
    VerifyLaunch vl;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        if ((rc = sbv_launch_verify_begin(e, d, curve, cnt, ln.d_qx, ln.d_qy, ln.stream, &vl, chunks))) return rc;
    }
    auto abandon = [&](int code) {  // a fault between the halves: hand the scratch set back (the caller fail-stops anyway)
        std::lock_guard<std::mutex> lk(e->mu);
        return sbv_launch_verify_close(e, vl, ln.stream, code);
    };
    for (int c = 0; c < chunks; c++) {
        const size_t clo = (size_t)c * per < cnt ? (size_t)c * per : cnt, cn = cnt - clo < per ? cnt - clo : per;
        const size_t g = lo + clo;   // first item of the chunk in the caller's arrays
        if (hashing && cn) {
            const uint64_t o = b.msg_off[g] - base, len = b.msg_off[g + cn] - b.msg_off[g];
            rc = sbv_lane_h2d(e, ln, ln.d_msgs + o, b.msgs + b.msg_off[g], len, so, up);
            if (!rc) rc = sbv_lane_h2d(e, ln, ln.d_off + clo, b.msg_off + g, (cn + 1) * 8, so, up);
        } else if (cn) {
            rc = sbv_lane_h2d(e, ln, ln.d_dig + clo * dlen, b.digest + g * dlen, cn * dlen, so, up);
        }
        if (!rc) rc = sbv_lane_h2d(e, ln, ln.d_r + clo * L, b.r + g * L, cn * L, so, up);
        if (!rc) rc = sbv_lane_h2d(e, ln, ln.d_s + clo * L, b.s + g * L, cn * L, so, up);
        if (rc) return abandon(rc);
        if (chunks > 1) {
            cudaError_t ce = cudaEventRecord(ln.ev_chunk[c], up);
            if (ce == cudaSuccess) ce = cudaStreamWaitEvent(ln.stream, ln.ev_chunk[c], 0);
            if (ce != cudaSuccess) return abandon(sbv_fail(e, SBV_ERR_CUDA, "chunk event: %s", cudaGetErrorString(ce)));
        }
        if (hashing && cn && (rc = launch_hash(e, b.hash, cn, ln.d_msgs, ln.d_off + clo, base, ln.d_dig + clo * dlen, ln.d_perm + clo, ln.stream)))
            return abandon(rc);
        std::lock_guard<std::mutex> lk(e->mu);
        rc = sbv_launch_verify_chunk(e, d, vl, c, clo, cn, c == chunks - 1, ln.d_r, ln.d_s, ln.d_dig, dlen, ln.d_ok, ln.stream);
        if (rc) return sbv_launch_verify_close(e, vl, ln.stream, rc);
    }
    if (so_out) *so_out = so;
    return 0;
}

}  // namespace

// ================================================================================================
extern "C" {

int sbv_create(const int *device_ordinals, int n_devices, sbv_engine **out) {
    if (!out || n_devices < 1 || n_devices > 8) return SBV_ERR_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count < n_devices) return SBV_ERR_CUDA;
    sbv_engine *e = new sbv_engine();
    e->keyed_warp_limit = env_int("SBV_KEYED_WARP_LIMIT", 2048);
    e->group_threshold = env_int("SBV_GROUP_THRESHOLD", 16);
    e->group_max_keys = env_int("SBV_GROUP_MAX_KEYS", 8192);
    e->group_min_batch = env_int("SBV_GROUP_MIN_BATCH", 0);
    e->chunk_items = env_int("SBV_CHUNK_ITEMS", 262144);
    {
        // per-engine hash seed: an adversary who picks the keys of a batch cannot aim at the probe sequence
        uint64_t t = (uint64_t)(uintptr_t)e;
        FILE *f = fopen("/dev/urandom", "rb");
        if (f) { if (fread(&t, sizeof t, 1, f) != 1) t ^= 0x9e3779b97f4a7c15ull; fclose(f); }
        e->hash_seed = (uint32_t)(t ^ (t >> 32)) | 1u;
    }
    e->devs.resize(n_devices);
    for (int g = 0; g < n_devices; g++) {
        Dev &d = e->devs[g];
        d.ordinal = device_ordinals ? device_ordinals[g] : g;
        cudaError_t st = cudaSetDevice(d.ordinal);
        if (st == cudaSuccess) st = cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking);
        if (st == cudaSuccess && sbv_init_gtables(e, d) != 0) st = cudaErrorUnknown;
        if (st != cudaSuccess) {
            fprintf(stderr, "sbv_create: device %d: %s (%s)\n", d.ordinal, cudaGetErrorString(st), e->err.c_str());
            sbv_destroy(e);
            return SBV_ERR_CUDA;
        }
    }
    if (n_devices > 1) {
        std::vector<int> ords;
        for (Dev &d : e->devs) ords.push_back(d.ordinal);
        e->nccl_comms.assign(n_devices, nullptr);
        if (nccl_load(e) != 0 || g_nccl.comm_init_all(e->nccl_comms.data(), n_devices, ords.data()) != 0) {
            fprintf(stderr, "sbv_create: NCCL initialisation failed: %s\n", e->err.c_str());
            e->nccl_comms.clear();
            sbv_destroy(e);
            return SBV_ERR_NCCL;
        }
    }
    *out = e;
    return SBV_OK;
}

void sbv_destroy(sbv_engine *e) {
    if (!e) return;
    for (Dev &d : e->devs) {
        cudaSetDevice(d.ordinal);
        cudaDeviceSynchronize();
    }
    for (void *c : e->nccl_comms) if (c && g_nccl.comm_destroy) g_nccl.comm_destroy(c);
    for (void *c : e->rank_comms) if (c && g_nccl.comm_destroy) g_nccl.comm_destroy(c);
    for (auto &hi : e->rank_hi) {
        if (hi.st) cudaStreamDestroy(hi.st);
        if (hi.in) cudaEventDestroy(hi.in);
        if (hi.out) cudaEventDestroy(hi.out);
    }
    for (Dev &d : e->devs) {
        cudaSetDevice(d.ordinal);
        void *ptrs[] = {d.gtab[0], d.gtab[1], d.ed_btab};
        for (void *p : ptrs) if (p) cudaFree(p);
        buf_free(d.d_scratch);
        sbv_scratch_free(d);
        sbv_keys_free(d);
        sbv_ed_keys_free(d);
        sbv_rsa_keys_free(d);
        sbv_key_cache_free(d);
        for (auto &ln : d.lanes) lane_free(ln);
        for (cudaEvent_t ev : d.prof_events) cudaEventDestroy(ev);
        if (d.stream) cudaStreamDestroy(d.stream);
    }
    delete e;
}

// Copies the description of the last fault into a thread-local buffer: valid until this thread's next call.
const char *sbv_last_error(const sbv_engine *e) {
    static thread_local std::string copy;
    if (!e) return "null engine";
    sbv_engine *m = const_cast<sbv_engine *>(e);
    std::lock_guard<std::mutex> lk(m->err_mu);
    copy = m->err;
    return copy.c_str();
}
int sbv_device_count(const sbv_engine *e) { return e ? (int)e->devs.size() : 0; }
uint64_t sbv_kernel_launches(const sbv_engine *e) { return e ? e->launches.load() : 0; }

void sbv_compute_quorum(uint64_t n, uint32_t *q, uint32_t *f) {
    // f = (n-1)/3 ; q = ceil((n+f+1)/2) — util.go:183-187, exact in integers
    uint64_t ff = n ? (n - 1) / 3 : 0;
    if (f) *f = (uint32_t)ff;
    if (q) *q = (uint32_t)((n + ff + 2) / 2);
}

int sbv_verify_batch_device(sbv_engine *e, int device_index, uint8_t curve, size_t n, const uint8_t *d_r,
                            const uint8_t *d_s, const uint8_t *d_qx, const uint8_t *d_qy, const uint8_t *d_digest,
                            uint8_t digest_len, uint8_t *d_ok, void *cuda_stream) {
    if (!e || curve > SBV_P384 || device_index < 0 || device_index >= (int)e->devs.size() || digest_len == 0)
        return fail(e, SBV_ERR_ARG, "sbv_verify_batch_device: bad argument");
    if (n == 0) return SBV_OK;
    if (n > 0x7fffffffu || (digest_len & 3) || digest_len > 64) return fail(e, SBV_ERR_ARG, "n too large or digest_len not a multiple of 4");
    if (!d_r || !d_s || !d_qx || !d_qy || !d_digest || !d_ok) return fail(e, SBV_ERR_ARG, "null buffer");
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[device_index];
    CU(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = (cudaStream_t)cuda_stream;  // NULL = the legacy default stream
    return sbv_launch_verify(e, d, curve, n, d_r, d_s, d_qx, d_qy, d_digest, digest_len, d_ok, st);
}

int sbv_verify_batch(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx,
                     const uint8_t *qy, const uint8_t *digest, uint8_t digest_len, uint8_t *ok) {
    if (!e || curve > SBV_P384 || !digest_len_ok(digest_len)) return fail(e, SBV_ERR_ARG, "sbv_verify_batch: bad argument");
    if (n == 0) return SBV_OK;
    if (!r || !s || !qx || !qy || !digest || !ok) return fail(e, SBV_ERR_ARG, "null buffer");
    if (n > 0x7fffffffu) return fail(e, SBV_ERR_ARG, "n too large");
    const int G = (int)e->devs.size();
    const Shards sh = batch_shards(n, G);
    std::vector<uint32_t *> gbuf(G);
    // A call owns one lane (stream + buffers) on every device; the engine lock is held only while
    // kernels are enqueued, so other host threads overlap their copies and kernels with ours.
    LaneGuard guard(e);
    const int lane = guard.lane;
    for (int g = 0; g < G; g++) {
        Dev &d = e->devs[g];
        Dev::Lane &ln = d.lanes[lane];
        const Range v = sh.vr[g];
        LaneNeeds gather;  // the aux area holds the gather buffer
        gather.aux = G > 1 ? sh.wp() * G * 4 : 0;
        CU(e, cudaSetDevice(d.ordinal));
        int rc = v.n ? stage_and_verify(e, d, ln, curve, v.lo, v.n, BatchSrc{r, s, qx, qy, digest, digest_len, nullptr, nullptr}, gather)
                     : sbv_lane_reserve(e, ln, gather);
        if (rc) return rc;
        gbuf[g] = (uint32_t *)ln.d_aux;
        if ((rc = shard_out(e, ln, sh, g, gbuf[g], ln.d_ok, nullptr, ok, nullptr))) return rc;
    }
    return gather_unpack(e, lane, sh, gbuf, ok, nullptr);
}

// ---- one process per GPU: this engine is one rank of an N-rank job ------------------------------------------
int sbv_comm_unique_id(uint8_t *id128) {
    if (!id128) return SBV_ERR_ARG;
    if (nccl_load(nullptr) != 0) return SBV_ERR_NCCL;
    NcclUniqueId id;
    if (g_nccl.get_unique_id(&id) != 0) return SBV_ERR_NCCL;
    memcpy(id128, id.internal, 128);
    return SBV_OK;
}

// Adds one CHANNEL (an NCCL communicator over all ranks) and returns its index (>= 0) — call it once per concurrent
// caller thread, with a fresh id each time, in the same order on every rank.
int sbv_comm_init_rank(sbv_engine *e, const uint8_t *id128, int nranks, int rank) {
    if (!e || !id128 || nranks < 1 || rank < 0 || rank >= nranks || e->devs.size() != 1)
        return fail(e, SBV_ERR_ARG, "sbv_comm_init_rank: bad argument (needs a single-device engine)");
    if (!e->rank_comms.empty() && (e->nranks != nranks || e->rank != rank)) return fail(e, SBV_ERR_ARG, "sbv_comm_init_rank: rank / nranks changed");
    if (int rc = nccl_load(e)) return rc;
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    NcclUniqueId id;
    memcpy(id.internal, id128, 128);
    void *comm = nullptr;
    NC(e, g_nccl.comm_init_rank(&comm, nranks, id, rank));
    sbv_engine::ChannelHi hi;
    int lo_p = 0, hi_p = 0;
    CU(e, cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p));
    CU(e, cudaStreamCreateWithPriority(&hi.st, cudaStreamNonBlocking, hi_p));
    CU(e, cudaEventCreateWithFlags(&hi.in, cudaEventDisableTiming));
    CU(e, cudaEventCreateWithFlags(&hi.out, cudaEventDisableTiming));
    std::lock_guard<std::mutex> lk(e->mu);
    e->rank_comms.push_back(comm);
    e->rank_hi.push_back(hi);
    e->rank = rank;
    e->nranks = nranks;
    return (int)e->rank_comms.size() - 1;
}

int sbv_comm_ranks(const sbv_engine *e) { return e ? e->nranks : 0; }

// Packs n verdict bytes on the device into a bitmask and all-gathers the masks of all ranks over `channel`:
// d_mask_all[rank * words_per_rank + w], words_per_rank = ceil(n / 32) (every rank passes the same n).
// Enqueued on cuda_stream behind whatever produced d_ok; not synchronised.
int sbv_gather_verdicts_device(sbv_engine *e, int channel, const uint8_t *d_ok, size_t n, uint32_t *d_mask_all, void *cuda_stream) {
    if (!e || e->devs.size() != 1 || !d_ok || !d_mask_all || n == 0 || n > 0x7fffffffu) return fail(e, SBV_ERR_ARG, "sbv_gather_verdicts_device: bad argument");
    Dev &d = e->devs[0];
    CU(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const size_t wp = (n + 31) / 32;
    uint32_t *mine = d_mask_all + wp * (size_t)e->rank;
    if (e->nranks > 1 && (channel < 0 || channel >= (int)e->rank_comms.size())) return fail(e, SBV_ERR_NCCL, "no such channel: call sbv_comm_init_rank first");
    const bool fork = e->nranks > 1;
    cudaStream_t gs = st;
    if (fork) {  // the exchange runs on the channel's high-priority stream, between two events on the caller's stream
        const sbv_engine::ChannelHi &hi = e->rank_hi[channel];
        CU(e, cudaEventRecord(hi.in, st));
        CU(e, cudaStreamWaitEvent(hi.st, hi.in, 0));
        gs = hi.st;
    }
    k_pack_bits<<<(uint32_t)((n + 255) / 256), 256, 0, gs>>>((uint32_t)n, d_ok, mine);
    e->launches += 1;
    CU(e, cudaGetLastError());
    if (fork) {
        const sbv_engine::ChannelHi &hi = e->rank_hi[channel];
        NC(e, g_nccl.all_gather(mine, d_mask_all, wp, NCCL_UINT32, e->rank_comms[channel], gs));
        CU(e, cudaEventRecord(hi.out, gs));
        CU(e, cudaStreamWaitEvent(st, hi.out, 0));
    }
    return SBV_OK;
}

// All-gather of `words` 32-bit words per rank (already on the device): d_all[rank * words + w].  The sender's words
// must sit at d_all + rank * words (in place).  Used for the per-instance `reached` bitmask of the quorum path.
int sbv_gather_words_device(sbv_engine *e, int channel, uint32_t *d_all, size_t words, void *cuda_stream) {
    if (!e || e->devs.size() != 1 || !d_all || words == 0) return fail(e, SBV_ERR_ARG, "sbv_gather_words_device: bad argument");
    if (e->nranks == 1) return SBV_OK;
    if (channel < 0 || channel >= (int)e->rank_comms.size()) return fail(e, SBV_ERR_NCCL, "no such channel: call sbv_comm_init_rank first");
    CU(e, cudaSetDevice(e->devs[0].ordinal));
    NC(e, g_nccl.all_gather(d_all + words * (size_t)e->rank, d_all, words, NCCL_UINT32, e->rank_comms[channel], (cudaStream_t)cuda_stream));
    return SBV_OK;
}

// Host-buffer form for a rank: this rank's n items are verified, its verdict bytes go to ok (n bytes) and the packed
// masks of ALL ranks to mask_all (nranks * ceil(n/32) words).  Every rank calls it with the same n, and the calls of
// one channel are issued in the same order on every rank.
int sbv_verify_batch_ranked(sbv_engine *e, int channel, uint8_t curve, size_t n, const uint8_t *r, const uint8_t *s, const uint8_t *qx,
                            const uint8_t *qy, const uint8_t *digest, uint8_t digest_len, uint8_t *ok, uint32_t *mask_all) {
    if (!e || curve > SBV_P384 || !digest_len_ok(digest_len) || e->devs.size() != 1)
        return fail(e, SBV_ERR_ARG, "sbv_verify_batch_ranked: bad argument");
    if (n == 0 || n > 0x7fffffffu) return fail(e, SBV_ERR_ARG, "n must be in [1, 2^31)");
    if (!r || !s || !qx || !qy || !digest || !ok || !mask_all) return fail(e, SBV_ERR_ARG, "null buffer");
    LaneGuard guard(e);
    const int lane = guard.lane;
    Dev &d = e->devs[0];
    Dev::Lane &ln = d.lanes[lane];
    const size_t wp = (n + 31) / 32;
    LaneNeeds masks;  // the aux area holds the masks of all ranks
    masks.aux = wp * (size_t)e->nranks * 4;
    int rc = stage_and_verify(e, d, ln, curve, 0, n, BatchSrc{r, s, qx, qy, digest, digest_len, nullptr, nullptr}, masks);
    if (rc) return rc;
    CU(e, cudaMemcpyAsync(ok, ln.d_ok, n, cudaMemcpyDeviceToHost, ln.stream));
    if ((rc = sbv_gather_verdicts_device(e, channel, ln.d_ok, n, (uint32_t *)ln.d_aux, ln.stream))) return rc;
    CU(e, cudaMemcpyAsync(mask_all, ln.d_aux, wp * (size_t)e->nranks * 4, cudaMemcpyDeviceToHost, ln.stream));
    return sync_lane(e, lane);
}

void *sbv_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void sbv_host_free(void *p) { if (p) cudaFreeHost(p); }

double sbv_probe_mad_rate(sbv_engine *e) {
    if (!e) return 0.0;
    std::lock_guard<std::mutex> lk(e->mu);
    Dev &d = e->devs[0];
    if (cudaSetDevice(d.ordinal) != cudaSuccess) return 0.0;
    if (sbv_ensure_scratch(e, d, 4096)) return 0.0;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, d.ordinal);
    const uint32_t iters = 4096;
    const int blocks = prop.multiProcessorCount * 8, threads = 256;
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    k_mad_probe<<<blocks, threads, 0, d.stream>>>((uint32_t *)d.d_scratch, 64);
    float best = 1e30f;
    for (int rep = 0; rep < 5; rep++) {
        cudaEventRecord(a, d.stream);
        k_mad_probe<<<blocks, threads, 0, d.stream>>>((uint32_t *)d.d_scratch, iters);
        cudaEventRecord(b, d.stream);
        if (cudaStreamSynchronize(d.stream) != cudaSuccess) return 0.0;
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        if (ms < best) best = ms;
    }
    e->launches += 6;
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    double macs = (double)blocks * threads * (double)iters * 8.0;
    return macs / (best * 1e-3);
}

}  // extern "C"

#include "engine_more.inc"
#include "engine_rsa.inc"

// ---- profiling hooks (bench.py's roofline leg): CUDA-event timing inside every verify launch ----
extern "C" {

int sbv_profile_enable(sbv_engine *e, int on) {
    if (!e) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    e->profiling = on != 0;
    for (Dev &d : e->devs) d.prof_used = 0;
    return SBV_OK;
}

// Sums the recorded intervals (all devices), then resets: prep_ms = start .. end of k_prep (includes the key grouping),
// verify_ms = the verification kernels alone (k_gpart + k_verify_kt when keys were grouped, k_verify_coz otherwise).
// The caller must have synchronised the streams it used.
int sbv_profile_read(sbv_engine *e, double *prep_ms, double *verify_ms, uint64_t *n_launches) {
    if (!e) return SBV_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    double p = 0, v = 0;
    uint64_t cnt = 0;
    for (Dev &d : e->devs) {
        CU(e, cudaSetDevice(d.ordinal));
        for (size_t i = 0; i + 4 < d.prof_used && i + 4 < d.prof_events.size(); i += 5) {
            float a = 0, b = 0, g = 0;
            CU(e, cudaEventSynchronize(d.prof_events[i + 3]));
            CU(e, cudaEventElapsedTime(&a, d.prof_events[i], d.prof_events[i + 1]));
            CU(e, cudaEventElapsedTime(&b, d.prof_events[i + 2], d.prof_events[i + 3]));
            CU(e, cudaEventElapsedTime(&g, d.prof_events[i + 1], d.prof_events[i + 4]));  // k_gpart (0 without the split)
            p += a; v += b + g; cnt++;
        }
        d.prof_used = 0;
    }
    if (prep_ms) *prep_ms = p;
    if (verify_ms) *verify_ms = v;
    if (n_launches) *n_launches = cnt;
    return SBV_OK;
}

}  // extern "C"
