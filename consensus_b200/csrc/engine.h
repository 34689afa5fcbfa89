// engine.h — shared host-side state of libsbv.so (one engine = 1..8 devices of one box).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdint>
#include <condition_variable>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <vector>

#include "../../include/sbv.h"
#include "ops.h"

constexpr int SBV_LANES = 6;    // concurrent host-buffer calls per engine
constexpr int SBV_SCRATCH = 8;  // scratch sets per device (> SBV_LANES + 1: a launch may be held open per lane)
constexpr int SBV_MAX_CHUNKS = 32;  // a large host-buffer batch is uploaded and verified in at most this many chunks

// A device buffer with the bytes allocated for it; reads as a T *.
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
};
template <class T>
struct DevArray : DevBuf {
    operator T *() const { return static_cast<T *>(p); }
};

struct Dev {
    int ordinal = 0;
    cudaStream_t stream = nullptr;
    uint32_t *gtab[2] = {nullptr, nullptr};
    uint32_t *ed_btab = nullptr;  // fixed-base table of the Ed25519 base point, built on the device's first Ed25519 call
    // Per-launch workspace of the verify pipeline.  A launch takes the next set and first waits for the event of
    // that set's previous user, so launches on different streams overlap without sharing mutable state.
    // The buffers are sized, grown and freed from one list (pipeline.cu: each_buffer).
    struct Scratch {
        DevArray<uint32_t> uw;      // k_prep output: u1, u2 word-major [2N][n]
        DevArray<uint8_t> flags;    // r, s range verdicts
        DevArray<uint32_t> tscr;    // k_verify_coz per-signature scratch: 12N words, word-major
        DevArray<uint32_t> gacc;    // k_gpart -> fixed-base kernel: u1*G of every item (Jacobian, 3N words, word-major)
        // key grouping
        uint32_t hsize = 0;
        DevArray<uint32_t> htab, rep, keylist, klist, glist;
        DevArray<uint32_t> zeroed;  // one memset: counters[4], kcnt[n], then counters[4] per chunk
        DevArray<int32_t> keyid, item_kid;
        // per-key tables of the launch
        DevArray<uint32_t> bases, hs, ztop, pref, ktab;
        DevArray<uint8_t> keyflags;
        cudaStream_t s_tab = nullptr, s_gen = nullptr;  // table construction / generic kernel run beside the main stream
        cudaEvent_t done = nullptr, ev_group = nullptr, ev_prep = nullptr, ev_tab = nullptr, ev_gen = nullptr;
        bool used = false;
        bool open = false;  // taken by a launch whose second half has not been enqueued yet
    } ws[SBV_SCRATCH];
    unsigned ws_next = 0;
    // Per-call lanes of the host-buffer entry points: own stream, input/verdict buffers and pinned staging, so that
    // SBV_LANES host threads can have a call in flight each (H2D / kernels / D2H of one overlap the others').
    struct Lane {
        cudaStream_t stream = nullptr;
        size_t cap = 0;
        uint8_t *d_r = nullptr, *d_s = nullptr, *d_qx = nullptr, *d_qy = nullptr, *d_dig = nullptr, *d_ok = nullptr;
        uint32_t *d_slot = nullptr;
        uint8_t *d_msgs = nullptr;
        uint64_t *d_off = nullptr;
        uint32_t *d_perm = nullptr;  // off_cap entries + 3 * 1024 words of sort state
        size_t msg_cap = 0, off_cap = 0;
        uint8_t *h_pin = nullptr;
        size_t h_pin_cap = 0;
        // small device scratch (quorum inputs / counts, packed verdict masks) and its pinned mirror
        uint8_t *d_aux = nullptr, *h_aux = nullptr;
        size_t aux_cap = 0;
        // second stream of the call (mixed-curve batches run their two pipelines side by side)
        cudaStream_t stream2 = nullptr;
        cudaEvent_t ev_a = nullptr, ev_b = nullptr;
        cudaEvent_t ev_chunk[SBV_MAX_CHUNKS] = {};  // "chunk c has arrived" (recorded on stream2, the upload stream of a chunked call)
        // device scratch of a mixed ECDSA / Ed25519 shard (inst_mixed.cu: sbv_mix_carve)
        uint8_t *d_mix = nullptr;
        size_t mix_cap = 0;
        // device scratch of an RSA shard (engine_rsa.inc: rsa_carve)
        uint8_t *d_rsa = nullptr;
        size_t rsa_cap = 0;
    } lanes[SBV_LANES];
    // generic scratch of the entry points that serialise on the engine lock
    uint8_t *d_scratch = nullptr;
    size_t scratch_cap = 0;
    // registered keys (sbv_set_keys): per-curve tables (8-bit signed windows), validity flags, slot -> table index
    uint32_t *ktab[2] = {nullptr, nullptr};
    uint8_t *keyflags[2] = {nullptr, nullptr};
    int32_t *slot2local[2] = {nullptr, nullptr};
    uint32_t n_slots = 0, n_local[2] = {0, 0};
    // registered Ed25519 keys (sbv_ed25519_set_keys): the registered bytes of every slot (32 each), slot -> table index
    // (-1: the key does not decode) and one fixed-base table per decodable key (ed25519_keyed.cuh)
    uint8_t *ed_kpub = nullptr;
    int32_t *ed_slot2local = nullptr;
    uint32_t *ed_ktab = nullptr;
    uint32_t ed_n_slots = 0, ed_n_local = 0;
    // the opt-in cache of grouped-key tables across launches (sbv_key_cache_reserve), per scheme tag: one allocation holding
    // the pool, the counters, the map (key_cache.cuh) and one launch area per scratch set (2 + SBV_GROUP_MAX_KEYS words:
    // the lookup's miss and hit counts and the renumbered keylist of the launch holding that set).  An evicting cache
    // (sbv_key_cache_reserve_evicting) holds the set-associative map of key_cache_assoc.cuh instead, and stamps every
    // grouped launch with the next value of `stamp` (taken under e->mu).
    struct KeyCache {
        void *mem = nullptr;
        bool evicting = false;
        KcMap map{};
        KcaMap amap{};
        unsigned long long stamp = 0;
        size_t capacity = 0;  // tables (evicting: rounded up to a multiple of KCA_WAYS)
        uint32_t *lk = nullptr;
        size_t lk_words = 0;
        size_t tw4 = 0;  // 16-byte words per table
    } kc[3];
    // profiling: event quadruples per verify launch (start, after prep, before / after the dominant kernel)
    std::vector<cudaEvent_t> prof_events;
    size_t prof_used = 0;
};

struct sbv_engine {
    std::vector<Dev> devs;
    std::mutex mu;       // kernel enqueue + workspace growth
    std::mutex err_mu;   // last-error string
    // the Ed25519 registry: sbv_ed25519_set_keys holds it exclusively, sbv_ed25519_verify_registered shared for the
    // enqueue of all its shards, so every shard of one call reads the same registry (taken before mu, never inside it)
    std::shared_mutex ed_reg_mu;
    std::condition_variable lane_cv;
    bool lane_busy[SBV_LANES] = {};
    std::string err;
    std::atomic<uint64_t> launches{0};
    int keyed_warp_limit = 2048;   // registered-key batches up to this size use one warp per signature (SBV_KEYED_WARP_LIMIT)
    int group_threshold = 16;      // a key gets a table when it occurs at least this often in a batch (SBV_GROUP_THRESHOLD; 0 = never)
    int group_max_keys = 8192;     // table slots per launch (SBV_GROUP_MAX_KEYS)
    int group_min_batch = 0;       // launches smaller than this skip the grouping (SBV_GROUP_MIN_BATCH)
    int chunk_items = 262144;      // host-buffer shards of >= this many items are uploaded and verified in >= 2 chunks of nominally this size (SBV_CHUNK_ITEMS; 0 = never)
    uint32_t hash_seed = 0x9e3779b9u;
    bool profiling = false;
    // NCCL (loaded lazily with dlopen so single-device, single-rank users never touch it)
    void *nccl_lib = nullptr;
    std::vector<void *> nccl_comms;  // one per device of a multi-device engine
    // one-process-per-GPU deployments: this engine is rank `rank` of `nranks`.  One communicator per CHANNEL: the
    // collectives of a channel must be issued in the same order on every rank, so concurrent host threads take one each.
    std::vector<void *> rank_comms;
    // per channel: a high-priority stream for the pack + all-gather of a step (fork / join with two events), so that the
    // exchange is dispatched ahead of the pending blocks of other lanes' verification kernels
    struct ChannelHi { cudaStream_t st = nullptr; cudaEvent_t in = nullptr, out = nullptr; };
    std::vector<ChannelHi> rank_hi;
    int rank = 0, nranks = 1;
    // key registry
    uint64_t verification_seq = 0;
    std::vector<uint64_t> key_ids;
    std::vector<uint8_t> key_curve;
    std::vector<uint8_t> key_xy;
};

inline int sbv_fail(sbv_engine *e, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (e) {
        std::lock_guard<std::mutex> lk(e->err_mu);
        e->err = buf;
    }
    return code;
}
#define fail sbv_fail

#define CU(e, call)                                                                                   \
    do {                                                                                              \
        cudaError_t _st = (call);                                                                     \
        if (_st != cudaSuccess)                                                                       \
            return sbv_fail(e, SBV_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_st), \
                            __FILE__, __LINE__);                                                      \
    } while (0)

constexpr size_t SBV_NO_PROFILE = ~(size_t)0;

// one keys-per-item launch between its two halves (pipeline.cu)
struct VerifyLaunch {
    Dev::Scratch *w = nullptr;  // nullptr: no scratch set held (n = 0, or an Ed25519 launch that does not group)
    // first of the launch's five profiling events in d.prof_events (SBV_NO_PROFILE: none).  An index, resolved under
    // e->mu at each use: another thread's launch may grow the vector while this one is held open between its halves.
    size_t ev = SBV_NO_PROFILE;
    const uint8_t *d_qx = nullptr, *d_qy = nullptr;
    size_t n = 0;
    uint8_t scheme = 0;
    bool grouping = false;
    int chunks = 1;   // the second half comes in this many chunks (sbv_launch_verify_chunk)
};

// ---- pipeline.cu: the verify pipelines (device pointers in, verdict bytes out; enqueue only, no sync) ----
// keys-per-item: k_prep, key grouping, per-key tables for repeated keys, fixed-base kernel + generic kernel for the rest
int sbv_launch_verify(sbv_engine *e, Dev &d, uint8_t curve, size_t n, const uint8_t *d_r, const uint8_t *d_s, const uint8_t *d_qx,
                      const uint8_t *d_qy, const uint8_t *d_dig, uint32_t dlen, uint8_t *d_ok, cudaStream_t st);
// The first half of a keys-per-item launch of n items of scheme s (keys as GroupOps takes them): a scratch set, the
// grouping of the keys with the engine's SBV_GROUP_* settings on st and the tables of the grouped keys on the set's side
// stream, ending in ev_tab.  every_key: every distinct key gets a table slot whatever the settings (a test hook's launch).
// An ECDSA launch always holds a scratch set (its per-item buffers) and takes its profiling events here.
int sbv_launch_verify_begin(sbv_engine *e, Dev &d, uint8_t scheme, size_t n, const uint8_t *d_qx, const uint8_t *d_qy, cudaStream_t st, VerifyLaunch *vl,
                            int chunks = 1, bool every_key = false);
// Hands the scratch set back: waits for the generic kernel on the second side stream, and with rc != 0 (a fault before the
// join) for the tables too, then records the set's `done` event.  Returns rc, or a fault of its own.
int sbv_launch_verify_close(sbv_engine *e, const VerifyLaunch &vl, cudaStream_t st, int rc);
// second half for items [lo, lo + cn) of chunk c (the pointers are those of the WHOLE batch; a launch of one chunk has
// c = 0, lo = 0, cn = n); `last` closes the launch
int sbv_launch_verify_chunk(sbv_engine *e, Dev &d, const VerifyLaunch &vl, int c, size_t lo, size_t cn, bool last, const uint8_t *d_r, const uint8_t *d_s,
                            const uint8_t *d_dig, uint32_t dlen, uint8_t *d_ok, cudaStream_t st);
// registered keys (sbv_set_keys)
int sbv_launch_keyed(sbv_engine *e, Dev &d, uint8_t curve, size_t n, const uint32_t *d_slot, const uint8_t *d_r, const uint8_t *d_s,
                     const uint8_t *d_dig, uint32_t dlen, uint8_t *d_ok, cudaStream_t st);
// the next scratch set of device d for a launch of n items (N words per coordinate; 0: none of the ECDSA per-item buffers)
// with kcap keys of table geometry q (nullptr: no grouping); the launch must record the set's `done` event on st
int sbv_take_scratch(sbv_engine *e, Dev &d, size_t N, const KtGeom *q, size_t n, size_t kcap, cudaStream_t st, Dev::Scratch **out);
int sbv_init_gtables(sbv_engine *e, Dev &d);
int sbv_keys_build(sbv_engine *e, Dev &d);  // (re)builds the per-key tables of the registry
void sbv_keys_free(Dev &d);
void sbv_scratch_free(Dev &d);
// ---- key_cache.cu: the grouped-key cache ----
void sbv_key_cache_free(Dev &d);  // caller has drained the device
// the launch area of scratch set w in the cache of scheme s for a launch of kcap table slots, or nullptr when none is
// reserved (or kcap exceeds SBV_GROUP_MAX_KEYS, as only a test hook's launch can); caller holds e->mu
uint32_t *sbv_key_cache_area(Dev &d, int s, const Dev::Scratch *w, size_t kcap);
// ---- inst_ed25519.cu: Ed25519 (enqueue only, no sync) ----
int sbv_ed_btab_ensure(sbv_engine *e, Dev &d);  // caller holds e->mu and has set the device
// k = SHA-512(R || A || M) mod L into d_k (word-major, 8n words), then the verdicts into d_ok.  d_sig: 64n bytes (R || S),
// d_pub: 32n bytes, d_perm: n + 3072 words of scratch.  The table of B must exist (sbv_ed_btab_ensure).  Keys whose 32
// bytes occur at least group_threshold times get a comb table built in the launch (ed25519_comb.cuh), over a scratch
// set; caller holds e->mu.
int sbv_launch_ed25519(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint8_t *d_sig,
                       const uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st);
// test hooks (caller holds e->mu; the table of B must exist):
// k_ed_verify_comb over every item with the caller's k (word-major [8][n], every k < L); every distinct key gets a table
int sbv_launch_ed_verify_comb_k(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_sig, const uint8_t *d_pub, const uint32_t *d_k, uint8_t *d_ok,
                                cudaStream_t st);
int sbv_launch_ed_sha512_digest(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, const uint8_t *d_sig, const uint8_t *d_pub,
                                uint32_t *d_k, uint32_t *d_dig, cudaStream_t st);
// test hook: k_ed_verify with the caller's k (word-major [8][n], every k < L); the table of B must exist
int sbv_launch_ed_verify_k(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_sig, const uint8_t *d_pub, const uint32_t *d_k, uint8_t *d_ok,
                           cudaStream_t st);
// registered Ed25519 keys.  sbv_ed_keys_build: caller holds e->mu; waits for the device to drain, frees the old registry of
// device d and builds one from the n keys of pub (host, 32 bytes each); a fault leaves d's registry empty.
int sbv_ed_keys_build(sbv_engine *e, Dev &d, size_t n, const uint8_t *pub);
void sbv_ed_keys_free(Dev &d);
// k_ed_key_gather (registered bytes of each item's slot into d_pub, 32n bytes), SHA-512 into d_k, then k_ed_verify_keyed.
// Caller holds e->mu (the registry is read at enqueue time); the table of B must exist.
int sbv_launch_ed25519_registered(sbv_engine *e, Dev &d, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint32_t *d_slot,
                                  const uint8_t *d_sig, uint8_t *d_pub, uint32_t *d_k, uint32_t *d_perm, uint8_t *d_ok, cudaStream_t st);
// test hook: k_ed_verify_keyed with the caller's k (word-major [8][n], every k < L); caller holds e->mu
int sbv_launch_ed_verify_registered_k(sbv_engine *e, Dev &d, size_t n, const uint32_t *d_slot, const uint8_t *d_sig, const uint32_t *d_k, uint8_t *d_ok,
                                      cudaStream_t st);
// ---- inst_mixed.cu: mixed ECDSA / Ed25519 shards (mixed.cuh; family f = scheme tag f) ----
// The device scratch of a shard of n items, m[f] of family f and `bytes` message bytes, carved from one buffer: the
// uploaded tags, slots (or, keys per item, 96-byte key rows) and 96-byte signature rows, the tile prefixes of the split,
// the shared message buffer of the three families, and per family the compacted arrays and the scratch of its pipeline.
// A registered shard has no key arrays (key96, qx, qy are null); a keys-per-item shard has no slots.  alg: the SHA-384 flag
// of each item (mixed_hash.cuh: k_mix_alg), carved only for a shard that holds SHA-384 items.
struct MixBufs {
    uint8_t *tag, *sig96, *key96, *alg;
    uint32_t *slot_in, *tile_cnt;
    uint64_t *tile_bytes;
    uint8_t *blob;
    uint32_t *idx[3], *slot[3], *perm[3];
    uint8_t *r[3], *s[3], *ok[3], *dig[3], *pub[3];  // dig: the ECDSA e (32 bytes per item, 48 for a P-384 family with
                                                       // SHA-384 items) or k (Ed25519); pub: Ed25519 only
    uint8_t *qx[3], *qy[3];                            // keys per item, ECDSA only
    uint64_t *off[3];
};
// base == nullptr only sizes; returns the bytes the carve takes.  keys: a keys-per-item shard (sbv_mixed_verify_batch).
// m384 (may be null): the SHA-384 items of the P-256 and P-384 families; when either is nonzero the carve adds alg.
size_t sbv_mix_carve(uint8_t *base, size_t n, const uint32_t m[3], uint64_t bytes, bool keys, MixBufs *out, const uint32_t *m384 = nullptr);
// the split of a staged shard (b.tag, b.slot_in or b.key96, b.sig96, messages at d_msgs with offsets d_off from base) into
// the families
int sbv_launch_mix_split(sbv_engine *e, const MixBufs &b, size_t n, const uint32_t m[3], const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base,
                         cudaStream_t st);
// the family verdicts b.ok[f] back into item order in d_ok
int sbv_launch_mix_ok(sbv_engine *e, const MixBufs &b, size_t n, const uint32_t m[3], uint8_t *d_ok, cudaStream_t st);

// shape of the table of B (ed25519_verify.cuh: ED_BWINS x ED_BENT entries of ED_BWORDS words; checked in inst_ed25519.cu)
constexpr size_t SBV_ED_BTAB_ENTRIES = 32 * 128, SBV_ED_BTAB_ENTRY_WORDS = 24;

// ---- engine.cu helpers shared with the other translation units ----
int sbv_lane_acquire(sbv_engine *e);            // blocks until a lane index is free; returns it
void sbv_lane_release(sbv_engine *e, int lane);
int sbv_lane_ensure(sbv_engine *e, Dev &d, Dev::Lane &ln, size_t n, size_t pinned_bytes);
int sbv_lane_ensure_msgs(sbv_engine *e, Dev::Lane &ln, size_t bytes, size_t n_off);
int sbv_lane_ensure_aux(sbv_engine *e, Dev::Lane &ln, size_t bytes);
int sbv_lane_ensure_mix(sbv_engine *e, Dev::Lane &ln, size_t bytes);
int sbv_lane_ensure_rsa(sbv_engine *e, Dev::Lane &ln, size_t bytes);
int sbv_lane_stream2(sbv_engine *e, Dev::Lane &ln);  // creates the lane's second stream and its two events on first use
// d_perm: n + 3072 words of scratch (may be null: no length sort)
int sbv_launch_sha256(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                      cudaStream_t st);
// the same with SHA-384: 48 bytes per message into d_digest
int sbv_launch_sha384(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                      cudaStream_t st);
// ---- inst_rsa.cu: RSA (enqueue only, no sync) ----
// the same with SHA-512 (sha512_batch.cuh: k_sha512): 64 bytes per message into d_digest
int sbv_launch_sha512(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, uint8_t *d_digest, uint32_t *d_perm,
                      cudaStream_t st);
// k_rsa_verify over n items of mod_bytes (256, 384 or 512) bytes each: d_sig and d_mod n * mod_bytes bytes (big-endian),
// d_exp n words, d_digest n * hLen bytes (hash 0 / 1 / 2: SHA-256 / SHA-384 / SHA-512), verdicts into d_ok.  Every pointer
// 4-byte aligned.
int sbv_launch_rsa(sbv_engine *e, uint32_t mod_bytes, uint8_t hash, size_t n, const uint8_t *d_sig, const uint8_t *d_mod, const uint32_t *d_exp,
                   const uint8_t *d_digest, uint8_t *d_ok, cudaStream_t st);
// mixed_hash.cuh: k_mix_alg over the n uploaded tags of a mixed shard (tags 3 and 4 to their family, flags into d_alg)
int sbv_launch_mix_alg(sbv_engine *e, size_t n, uint8_t *d_tag, uint8_t *d_alg, cudaStream_t st);
// mixed_hash.cuh: k_sha2_sel over the n items of one family (d_idx: their shard indices, d_alg: the shard's flags), dlen
// bytes of e per item into d_digest, behind the block-count sort of sbv_launch_sha256
int sbv_launch_sha2_sel(sbv_engine *e, size_t n, const uint8_t *d_msgs, const uint64_t *d_off, uint64_t base, const uint32_t *d_idx,
                        const uint8_t *d_alg, uint32_t dlen, uint8_t *d_digest, uint32_t *d_perm, cudaStream_t st);
// the block-count sort of the SHA-256 launch on its own: *perm = the permutation in d_perm, or nullptr below 2048 items
int sbv_launch_length_sort(sbv_engine *e, size_t n, const uint64_t *d_off, uint32_t *d_perm, cudaStream_t st, const uint32_t **perm);
int sbv_lane_h2d(sbv_engine *e, Dev::Lane &ln, void *dst, const void *src, size_t bytes, size_t &stage_off, cudaStream_t st = nullptr);
int sbv_ensure_scratch(sbv_engine *e, Dev &d, size_t bytes);

// A host-buffer call owns one lane on every device for its duration.  On every exit path — faults included — the
// lane's streams are drained before the lane is handed to the next caller, so no copy into the caller's buffers or out
// of the lane's staging area is still in flight when the call returns (cgo contract of sbv.h).
struct LaneGuard {
    sbv_engine *e;
    int lane;
    explicit LaneGuard(sbv_engine *eng) : e(eng), lane(sbv_lane_acquire(eng)) {}
    ~LaneGuard() {
        for (Dev &d : e->devs) {
            if (!d.lanes[lane].stream) continue;
            cudaSetDevice(d.ordinal);
            if (d.lanes[lane].stream2) cudaStreamSynchronize(d.lanes[lane].stream2);
            cudaStreamSynchronize(d.lanes[lane].stream);
        }
        sbv_lane_release(e, lane);
    }
    LaneGuard(const LaneGuard &) = delete;
    LaneGuard &operator=(const LaneGuard &) = delete;
};
