// pipeline.cu — the verify pipelines of libsbv.so: which kernels run for a batch, on which streams, over which scratch.
//
// Keys-per-item batch (sbv_verify_batch*, sbv_hash_verify_batch, sbv_verify_mixed):
//
//          ├──────────────── begin (every scheme) ─────┤
//   st     memsets  k_kg_insert  k_kg_assign ─┬─ k_prep  k_kg_route ─┬─ k_gpart ──────────────────────────────────┬─ (wait tables) k_verify_comb ─ (wait generic) ─ done
//   s_tab                                     └─ k_kt_bases2  k_comb_affine  k_comb_fill_warp  k_kt_inv  k_comb_final ─┘
//   s_gen                                                             └─ k_verify_coz (keys without a table) ──────────────────────────────────┘
//
// Keys that occur at least `group_threshold` times in the batch get a fixed-base table built on the spot (keygroup.cuh: a
// comb for P-256, 5-bit windows for P-384) and their signatures take the fixed-base kernel; the rest take the generic kernel.  The scalar preparation
// (latency-bound: one inversion chain) runs beside the table construction (latency-bound: one doubling chain).
// A large host-buffer batch runs the part after the table fork chunk by chunk, as its chunks arrive.
// Registered keys (sbv_set_keys) skip the grouping: their tables were built at registration.
// With a key cache reserved (sbv_key_cache_reserve), k_kc_lookup runs after k_kg_assign on st and k_kc_insert after
// the table construction on s_tab (key_cache.cuh): the build then makes only the tables the cache does not hold.  An
// evicting cache (sbv_key_cache_reserve_evicting) runs k_kca_lookup and k_kca_insert in the same places
// (key_cache_assoc.cuh).
// The first half up to the fork and the table construction is one function for P-256, P-384 and Ed25519 (verify_begin),
// driven by the scheme's entry of the grouping table (ops.h: GroupOps); Ed25519's second half is in inst_ed25519.cu.
#include "engine.h"

namespace {

uint32_t hash_slots(size_t n) {  // open-addressing table of the key grouping: a power of two >= 2n
    uint32_t h = 1;
    while (h < 2 * n) h <<= 1;
    return h;
}

// A launch of n items of a curve with N words per coordinate, kcap keys of which get a table with geometry q
struct ScratchDims {
    size_t N = 0, n = 0, kcap = 0;
    KtGeom q{};
};

// Every per-launch buffer of scratch set x, once: visit(buffer, need, alloc) with the bytes the launch uses (need) and
// the bytes to allocate when the buffer must grow (alloc: headroom, so that a slowly growing batch size does not
// reallocate every call).
template <class V>
void each_buffer(Dev::Scratch &x, const ScratchDims &s, V &&visit) {
    const size_t N = s.N, n = s.n, k = s.kcap, ni = n + n / 8 + 1024, kc = k + k / 8 + 16;
    const bool g = k > 0;
    const KtGeom &q = s.q;
    visit(x.uw, 2 * N * n * 4, 2 * N * ni * 4);
    visit(x.flags, n, ni);
    visit(x.tscr, 12 * N * n * 4, 12 * N * ni * 4);
    visit(x.gacc, g ? 3 * N * n * 4 : 0, 3 * N * ni * 4);
    visit(x.htab, g ? (size_t)hash_slots(n) * 4 : 0, (size_t)hash_slots(ni) * 4);
    visit(x.rep, g ? n * 4 : 0, ni * 4);
    visit(x.klist, g ? n * 4 : 0, ni * 4);
    visit(x.glist, g ? n * 4 : 0, ni * 4);
    visit(x.zeroed, g ? (n + 4 + 4 * SBV_MAX_CHUNKS) * 4 : 0, (ni + 4 + 4 * SBV_MAX_CHUNKS) * 4);
    visit(x.keyid, g ? n * 4 : 0, ni * 4);
    visit(x.item_kid, g ? n * 4 : 0, ni * 4);
    visit(x.keylist, k * 4, kc * 4);
    visit(x.keyflags, k, kc);
    visit(x.bases, q.bases_words * k * 4, q.bases_words * kc * 4);
    visit(x.hs, q.hs_words * k * 4, q.hs_words * kc * 4);
    visit(x.ztop, q.ztop_words * k * 4, q.ztop_words * kc * 4);
    visit(x.pref, q.ztop_words * k * 4, q.ztop_words * kc * 4);
    visit(x.ktab, q.ktab_words * k * 4, q.ktab_words * kc * 4);
}

}  // namespace

// Takes the next scratch set of device d for a launch on stream st: waits (on the stream) for the set's previous user
// and grows the buffers to n items with N words per coordinate / kcap keys of table geometry q (growth drains the
// previous user on the host first).  A buffer never shrinks, so the sets fit the largest launch of either family.
int sbv_take_scratch(sbv_engine *e, Dev &d, size_t N, const KtGeom *q, size_t n, size_t kcap, cudaStream_t st, Dev::Scratch **out) {
    // round robin over the sets that are not held open between the two halves of a host-buffer launch (at most
    // SBV_LANES < SBV_SCRATCH of them at any time)
    int idx = (int)(d.ws_next++ % SBV_SCRATCH);
    for (int tries = 0; tries < SBV_SCRATCH && d.ws[idx].open; tries++) idx = (int)(d.ws_next++ % SBV_SCRATCH);
    if (d.ws[idx].open) return sbv_fail(e, SBV_ERR_ARG, "no free scratch set (more launches held open than lanes?)");
    Dev::Scratch &w = d.ws[idx];
    if (!w.done) {
        // The events and side streams of EVERY set are created now: a set first taken in the middle of a steady stream of
        // launches would otherwise stop to create streams there (measured: 2 - 40 ms at the head of a timed region).
        // The table-construction stream runs at high priority: its few, latency-bound blocks are dispatched ahead of the
        // pending blocks of other launches' verification kernels.
        int lo_p = 0, hi_p = 0;
        CU(e, cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p));
        for (int j = 0; j < SBV_SCRATCH; j++) {
            Dev::Scratch &x = d.ws[j];
            if (x.done) continue;
            CU(e, cudaEventCreateWithFlags(&x.done, cudaEventDisableTiming));
            CU(e, cudaEventCreateWithFlags(&x.ev_group, cudaEventDisableTiming));
            CU(e, cudaEventCreateWithFlags(&x.ev_prep, cudaEventDisableTiming));
            CU(e, cudaEventCreateWithFlags(&x.ev_tab, cudaEventDisableTiming));
            CU(e, cudaEventCreateWithFlags(&x.ev_gen, cudaEventDisableTiming));
            CU(e, cudaStreamCreateWithPriority(&x.s_tab, cudaStreamNonBlocking, hi_p));
            CU(e, cudaStreamCreateWithFlags(&x.s_gen, cudaStreamNonBlocking));
        }
    }
    const ScratchDims dims{N, n, kcap, q ? *q : KtGeom{}};
    bool grows = false;
    each_buffer(w, dims, [&](DevBuf &b, size_t need, size_t) { grows = grows || need > b.bytes; });
    if (grows) {
        // Grow EVERY scratch set of the device now, not just this one: otherwise the first launch on each of the other sets
        // would stop to allocate in the middle of a steady stream of launches (cudaMalloc of hundreds of MB synchronises).
        for (int j = 0; j < SBV_SCRATCH; j++) {
            Dev::Scratch &x = d.ws[j];
            if (x.open && &x != &w) continue;  // held by a launch between its halves: it grows when it is next taken
            if (x.used && x.done) CU(e, cudaEventSynchronize(x.done));  // nothing may still be using the buffers we are about to free
            cudaError_t err = cudaSuccess;
            each_buffer(x, dims, [&](DevBuf &b, size_t need, size_t alloc) {
                if (err != cudaSuccess || need <= b.bytes) return;
                if (b.p) cudaFree(b.p);
                b = DevBuf{};
                err = cudaMalloc(&b.p, alloc);
                if (err == cudaSuccess) b.bytes = alloc;
            });
            CU(e, err);
        }
    }
    w.hsize = hash_slots(n);
    if (w.used) CU(e, cudaStreamWaitEvent(st, w.done, 0));
    w.used = true;
    *out = &w;
    return 0;
}

namespace {

// The index of five fresh profiling events of device d (SBV_NO_PROFILE: profiling is off).  Growing the vector moves
// its elements, so a launch keeps the index and takes a pointer only under e->mu (prof_at).
size_t prof_take(sbv_engine *e, Dev &d) {
    if (!e->profiling) return SBV_NO_PROFILE;
    if (d.prof_used + 5 > d.prof_events.size()) {
        size_t old = d.prof_events.size();
        d.prof_events.resize(old + 128);
        for (size_t i = old; i < d.prof_events.size(); i++)
            if (cudaEventCreate(&d.prof_events[i]) != cudaSuccess) { d.prof_events.resize(i); return SBV_NO_PROFILE; }
    }
    size_t ev = d.prof_used;
    d.prof_used += 5;  // start, after prep, before / after the fixed-base (or generic) kernel, after k_gpart
    return ev;
}

cudaEvent_t *prof_at(Dev &d, size_t ev) { return ev == SBV_NO_PROFILE ? nullptr : &d.prof_events[ev]; }

}  // namespace

void sbv_scratch_free(Dev &d) {
    for (auto &w : d.ws) {
        each_buffer(w, ScratchDims{}, [](DevBuf &b, size_t, size_t) { if (b.p) cudaFree(b.p); });
        cudaEvent_t evs[] = {w.done, w.ev_group, w.ev_prep, w.ev_tab, w.ev_gen};
        for (cudaEvent_t ev : evs) if (ev) cudaEventDestroy(ev);
        if (w.s_tab) cudaStreamDestroy(w.s_tab);
        if (w.s_gen) cudaStreamDestroy(w.s_gen);
        w = Dev::Scratch{};
    }
}

int sbv_init_gtables(sbv_engine *e, Dev &d) {
    for (int c = 0; c < 2; c++) {
        const CurveOps &ops = sbv_ops(c);
        CU(e, cudaMalloc(&d.gtab[c], ops.gtab_entries * 2 * ops.N * 4));  // P-256: 64 MiB, mostly held by the 50 MB L2
        CU(e, ops.gtable_init(d.gtab[c], d.stream));
    }
    e->launches += 2;
    CU(e, cudaStreamSynchronize(d.stream));
    return 0;
}

// The keys-per-item pipeline in two halves, so that a host-buffer call can upload the keys first and let the grouping
// and the table construction (the latency-bound part) run while the rest of the batch is still on its way:
//   begin : scratch set, key grouping on st, table construction on the set's side stream   (needs the keys)
//   ECDSA chunk : k_prep, routing, generic kernel on the second side stream, k_gpart, fixed-base kernel, join
//                 (needs r, s, digest), once per chunk of the batch
//   Ed25519 (inst_ed25519.cu) : routing, SHA-512, generic kernel on the second side stream, comb kernel, join
namespace {
// Table slots of a keys-per-item launch of n items; 0: the launch does not group (SBV_GROUP_THRESHOLD = 0, fewer items
// than the threshold or than SBV_GROUP_MIN_BATCH, or SBV_GROUP_MAX_KEYS <= 0).
size_t group_slots(const sbv_engine *e, size_t n) {
    const size_t T = e->group_threshold > 0 ? (size_t)e->group_threshold : 0;
    if (T == 0 || n < T || n < (size_t)e->group_min_batch || e->group_max_keys <= 0) return 0;
    return std::min(n / T, (size_t)e->group_max_keys);
}

int verify_begin(sbv_engine *e, Dev &d, uint8_t scheme, size_t n, const uint8_t *d_qx, const uint8_t *d_qy, cudaStream_t st, VerifyLaunch *vl,
                 int chunks, bool every_key) {
    *vl = VerifyLaunch{};
    if (n == 0) return 0;
    if (chunks < 1 || chunks > SBV_MAX_CHUNKS) return sbv_fail(e, SBV_ERR_ARG, "bad chunk count %d", chunks);
    const GroupOps &g = sbv_group_ops(scheme);
    const bool ecdsa = scheme != SBV_ED25519;
    const size_t N = ecdsa ? (size_t)sbv_ops(scheme).N : 0, kcap = every_key ? n : group_slots(e, n);
    if (kcap == 0 && !ecdsa) return 0;  // an Ed25519 launch that does not group holds no scratch set
    Dev::Scratch *w = nullptr;
    if (int rc = sbv_take_scratch(e, d, N, kcap ? &g.kt->geom : nullptr, n, kcap, st, &w)) return rc;
    w->open = true;  // until the launch records the set's `done` event
    vl->w = w; vl->scheme = scheme; vl->n = n; vl->grouping = kcap > 0; vl->d_qx = d_qx; vl->d_qy = d_qy; vl->chunks = chunks;
    if (ecdsa) {  // sbv_profile_read reports the ECDSA launches
        vl->ev = prof_take(e, d);
        if (cudaEvent_t *ev = prof_at(d, vl->ev)) CU(e, cudaEventRecord(ev[0], st));
    }
    if (!kcap) return 0;
    const uint32_t T = every_key ? 1 : (uint32_t)e->group_threshold;
    uint32_t *counters = w->zeroed, *kcnt = w->zeroed + 4;
    CU(e, cudaMemsetAsync(w->htab, 0xff, (size_t)w->hsize * 4, st));
    CU(e, cudaMemsetAsync(w->zeroed, 0, (n + 4 + 4 * (size_t)chunks) * 4, st));
    CU(e, g.group((uint32_t)n, d_qx, d_qy, e->hash_seed, w->hsize - 1, w->htab, w->rep, kcnt, T, (uint32_t)kcap, w->keyid, w->keylist, counters, st));
    // with a key cache: the lookup renumbers the keys (misses first), copies the hits' tables, and the build makes the misses
    // (an evicting cache: the same with the launch's stamp, key_cache_assoc.cuh)
    Dev::KeyCache &kc = d.kc[scheme];
    uint32_t *lk = sbv_key_cache_area(d, scheme, w, kcap);
    const unsigned long long now = lk && kc.evicting ? ++kc.stamp : 0;
    if (lk) {
        CU(e, cudaMemsetAsync(lk, 0, 8, st));
        if (kc.evicting)
            CU(e, g.evict_lookup(counters, (uint32_t)kcap, w->keylist, d_qx, d_qy, kc.amap, now, (uint32_t)kc.tw4, w->keyid, lk, w->keyflags, w->ktab, st));
        else
            CU(e, g.cache_lookup(counters, (uint32_t)kcap, w->keylist, d_qx, d_qy, kc.map, (uint32_t)kc.tw4, w->keyid, lk, w->keyflags, w->ktab, st));
    }
    CU(e, cudaEventRecord(w->ev_group, st));
    CU(e, cudaStreamWaitEvent(w->s_tab, w->ev_group, 0));
    CU(e, g.kt->build(lk ? lk : counters, (uint32_t)kcap, lk ? lk + 2 : w->keylist, d_qx, d_qy, w->bases, w->hs, w->ztop, w->pref, w->ktab, w->keyflags,
                      w->s_tab));
    if (lk && kc.evicting) CU(e, g.evict_insert((uint32_t)kcap, lk, d_qx, d_qy, kc.amap, now, (uint32_t)kc.tw4, w->keyflags, w->ktab, w->s_tab));
    else if (lk) CU(e, g.cache_insert((uint32_t)kcap, lk, d_qx, d_qy, kc.map, (uint32_t)kc.tw4, w->keyflags, w->ktab, w->s_tab));
    CU(e, cudaEventRecord(w->ev_tab, w->s_tab));
    e->launches += 2 + g.build_launches + (lk ? 2 : 0);  // grouping + table construction (+ cache lookup and insert)
    return 0;
}
}  // namespace

// A fault after the scratch set was taken hands it back here, so that no caller leaves it held open.
int sbv_launch_verify_begin(sbv_engine *e, Dev &d, uint8_t scheme, size_t n, const uint8_t *d_qx, const uint8_t *d_qy, cudaStream_t st,
                            VerifyLaunch *vl, int chunks, bool every_key) {
    const int rc = verify_begin(e, d, scheme, n, d_qx, d_qy, st, vl, chunks, every_key);
    if (rc) {
        sbv_launch_verify_close(e, *vl, st, rc);
        *vl = VerifyLaunch{};
    }
    return rc;
}

// One chunk of a launch: the items [lo, lo + cn) are a batch of their own as far as the per-item arrays go (every one
// of them is word-major with the batch size as its stride, so the chunk's slice is the contiguous block at `words per item *
// lo`); what the chunks share is the grouping (hash table, rep, key ids) and the key tables.
int sbv_launch_verify_chunk(sbv_engine *e, Dev &d, const VerifyLaunch &vl, int c, size_t lo, size_t cn, bool last, const uint8_t *d_r, const uint8_t *d_s,
                            const uint8_t *d_dig, uint32_t dlen, uint8_t *d_ok, cudaStream_t st) {
    if (vl.n == 0) return 0;
    Dev::Scratch *w = vl.w;
    if (c < 0 || c >= vl.chunks || lo + cn > vl.n) return sbv_fail(e, SBV_ERR_ARG, "bad chunk");
    const CurveOps &ops = sbv_ops(vl.scheme);
    const GroupedKtOps *kt = ops.grouped;
    const size_t N = (size_t)ops.N, L = (size_t)ops.bytes;
    const uint32_t nn = (uint32_t)cn;
    const uint32_t *gtab = d.gtab[vl.scheme];
    // The profile of a launch is that of its last chunk.  A chunked launch starts it again there (nothing of the first
    // half overlaps the last chunk); a launch of one chunk keeps the start of its first half, so the grouping counts as prep.
    cudaEvent_t *ev = last ? prof_at(d, vl.ev) : nullptr;
    if (ev && vl.chunks > 1) CU(e, cudaEventRecord(ev[0], st));
    uint32_t *uw = w->uw + 2 * N * lo, *tscr = w->tscr + 12 * N * lo;
    uint8_t *flags = w->flags + lo;
    const uint8_t *r = d_r + lo * L;
    if (cn) {
        CU(e, ops.prep(nn, r, d_s + lo * L, d_dig + lo * dlen, dlen, uw, flags, st));
        e->launches += 1;
    }
    if (!vl.grouping) {
        if (ev) { CU(e, cudaEventRecord(ev[1], st)); CU(e, cudaEventRecord(ev[4], st)); CU(e, cudaEventRecord(ev[2], st)); }
        if (cn) {
            CU(e, ops.coz(nn, vl.d_qx + lo * L, vl.d_qy + lo * L, r, uw, flags, gtab, tscr, d_ok + lo, nullptr, nullptr, st));
            e->launches += 1;
        }
        if (ev) CU(e, cudaEventRecord(ev[3], st));
    } else if (cn) {
        uint32_t *cc = w->zeroed + 4 + vl.n + 4 * (size_t)c;   // this chunk's counters (zeroed by the first half)
        uint32_t *klist = w->klist + lo, *glist = w->glist + lo, *gacc = w->gacc + 3 * N * lo;
        CU(e, ops.route(nn, w->rep + lo, w->keyid, w->item_kid + lo, klist, glist, cc, st));
        if (ev) CU(e, cudaEventRecord(ev[1], st));
        CU(e, cudaEventRecord(w->ev_prep, st));
        CU(e, cudaStreamWaitEvent(w->s_gen, w->ev_prep, 0));
        CU(e, ops.coz(nn, vl.d_qx + lo * L, vl.d_qy + lo * L, r, uw, flags, gtab, tscr, d_ok + lo, glist, cc + 2, w->s_gen));
        CU(e, cudaEventRecord(w->ev_gen, w->s_gen));
        // the u1*G half needs no table: it runs while the tables are still being built
        CU(e, ops.gpart(nn, uw, gtab, gacc, st));
        if (ev) CU(e, cudaEventRecord(ev[4], st));
        if (c == 0) CU(e, cudaStreamWaitEvent(st, w->ev_tab, 0));
        if (ev) CU(e, cudaEventRecord(ev[2], st));
        CU(e, kt->verify(nn, w->item_kid + lo, w->keyflags, r, uw, flags, gtab, w->ktab, d_ok + lo, klist, cc + 1, gacc, st));
        if (ev) CU(e, cudaEventRecord(ev[3], st));
        CU(e, cudaStreamWaitEvent(st, w->ev_gen, 0));
        e->launches += 4;
    } else if (ev) {
        CU(e, cudaEventRecord(ev[1], st)); CU(e, cudaEventRecord(ev[4], st)); CU(e, cudaEventRecord(ev[2], st)); CU(e, cudaEventRecord(ev[3], st));
    }
    if (last) {
        CU(e, cudaEventRecord(w->done, st));
        w->open = false;
    }
    return 0;
}

// On success and after a fault alike, the set goes back only behind everything the launch enqueued on its side streams.
int sbv_launch_verify_close(sbv_engine *e, const VerifyLaunch &vl, cudaStream_t st, int rc) {
    Dev::Scratch *w = vl.w;
    if (!w || !w->open) return rc;
    if (rc && vl.grouping) cudaStreamWaitEvent(st, w->ev_tab, 0);
    // the generic kernel (a never-recorded event is a no-op)
    const cudaError_t a = cudaStreamWaitEvent(st, w->ev_gen, 0), b = cudaEventRecord(w->done, st);
    w->open = false;
    if (rc) return rc;
    CU(e, a);
    CU(e, b);
    return 0;
}

int sbv_launch_verify(sbv_engine *e, Dev &d, uint8_t curve, size_t n, const uint8_t *d_r, const uint8_t *d_s, const uint8_t *d_qx,
                      const uint8_t *d_qy, const uint8_t *d_dig, uint32_t dlen, uint8_t *d_ok, cudaStream_t st) {
    VerifyLaunch vl;
    if (int rc = sbv_launch_verify_begin(e, d, curve, n, d_qx, d_qy, st, &vl)) return rc;
    return sbv_launch_verify_chunk(e, d, vl, 0, 0, n, true, d_r, d_s, d_dig, dlen, d_ok, st);
}

// ---- registered keys ----------------------------------------------------------------------------------------
void sbv_keys_free(Dev &d) {
    for (int c = 0; c < 2; c++) {
        if (d.ktab[c]) cudaFree(d.ktab[c]);
        if (d.keyflags[c]) cudaFree(d.keyflags[c]);
        if (d.slot2local[c]) cudaFree(d.slot2local[c]);
        d.ktab[c] = nullptr; d.keyflags[c] = nullptr; d.slot2local[c] = nullptr; d.n_local[c] = 0;
    }
    d.n_slots = 0;
}

// Consenter keys are configuration (they change only with a reconfiguration, i.e. a new VerificationSequence —
// /root/reference/pkg/api/dependencies.go:65-66): one table per key with 8-bit signed windows, built by the doubling,
// inversion and conversion kernels the on-the-fly path uses (a few milliseconds for a thousand keys).
int sbv_keys_build(sbv_engine *e, Dev &d) {
    CU(e, cudaSetDevice(d.ordinal));
    CU(e, cudaDeviceSynchronize());  // no launch on any lane may still read the old tables
    sbv_keys_free(d);
    const size_t n = e->key_ids.size();
    d.n_slots = (uint32_t)n;
    if (n == 0) return 0;
    for (int c = 0; c < 2; c++) {
        const CurveOps &ops = sbv_ops(c);
        const KtOps *kt = ops.kt8;
        const size_t L = (size_t)ops.bytes;
        std::vector<int32_t> map(n, -1);
        std::vector<uint8_t> kx, ky;
        uint32_t cnt = 0;
        for (size_t i = 0; i < n; i++) {
            if (e->key_curve[i] != c) continue;
            const uint8_t *x = &e->key_xy[96 * i], *y = x + 48;
            bool fits = true;
            for (size_t b = 0; b < 48 - L; b++) if (x[b] || y[b]) fits = false;
            if (!fits) continue;  // value >= 2^(8L): not a valid key for this curve -> slot stays unmapped (rejects)
            map[i] = (int32_t)cnt++;
            kx.insert(kx.end(), x + (48 - L), x + 48);
            ky.insert(ky.end(), y + (48 - L), y + 48);
        }
        CU(e, cudaMalloc(&d.slot2local[c], n * sizeof(int32_t)));
        CU(e, cudaMemcpyAsync(d.slot2local[c], map.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, d.stream));
        d.n_local[c] = cnt;
        if (cnt == 0) { CU(e, cudaStreamSynchronize(d.stream)); continue; }
        CU(e, cudaMalloc(&d.ktab[c], kt->geom.ktab_words * cnt * 4));
        CU(e, cudaMalloc(&d.keyflags[c], cnt));
        uint8_t *d_kx = nullptr, *d_ky = nullptr;
        uint32_t *tmp = nullptr, *d_cnt = nullptr;
        const size_t tmp_words = (kt->geom.bases_words + kt->geom.hs_words + 2 * kt->geom.ztop_words) * cnt;
        CU(e, cudaMalloc(&d_kx, kx.size()));
        CU(e, cudaMalloc(&d_ky, ky.size()));
        CU(e, cudaMalloc(&tmp, tmp_words * 4));
        CU(e, cudaMalloc(&d_cnt, 4));
        CU(e, cudaMemcpyAsync(d_kx, kx.data(), kx.size(), cudaMemcpyHostToDevice, d.stream));
        CU(e, cudaMemcpyAsync(d_ky, ky.data(), ky.size(), cudaMemcpyHostToDevice, d.stream));
        CU(e, cudaMemcpyAsync(d_cnt, &cnt, 4, cudaMemcpyHostToDevice, d.stream));
        uint32_t *bases = tmp, *hs = bases + kt->geom.bases_words * cnt, *ztop = hs + kt->geom.hs_words * cnt, *pref = ztop + kt->geom.ztop_words * cnt;
        cudaError_t st = kt->build(d_cnt, cnt, nullptr, d_kx, d_ky, bases, hs, ztop, pref, d.ktab[c], d.keyflags[c], d.stream);
        e->launches += 4;
        if (st == cudaSuccess) st = cudaStreamSynchronize(d.stream);
        cudaFree(d_kx); cudaFree(d_ky); cudaFree(tmp); cudaFree(d_cnt);
        CU(e, st);
    }
    return 0;
}

int sbv_launch_keyed(sbv_engine *e, Dev &d, uint8_t curve, size_t n, const uint32_t *d_slot, const uint8_t *d_r, const uint8_t *d_s,
                     const uint8_t *d_dig, uint32_t dlen, uint8_t *d_ok, cudaStream_t st) {
    if (n == 0) return 0;
    if (d.n_local[curve] == 0) {  // no registered key of this curve: every item rejects
        CU(e, cudaMemsetAsync(d_ok, 0, n, st));
        return 0;
    }
    const CurveOps &ops = sbv_ops(curve);
    const RegisteredKtOps *kt = ops.kt8;
    const uint32_t nn = (uint32_t)n;
    Dev::Scratch *w = nullptr;
    if (int rc = sbv_take_scratch(e, d, (size_t)ops.N, nullptr, n, 0, st, &w)) return rc;
    cudaEvent_t *ev = prof_at(d, prof_take(e, d));
    if (ev) CU(e, cudaEventRecord(ev[0], st));
    CU(e, ops.prep(nn, d_r, d_s, d_dig, dlen, w->uw, w->flags, st));
    if (ev) { CU(e, cudaEventRecord(ev[1], st)); CU(e, cudaEventRecord(ev[4], st)); CU(e, cudaEventRecord(ev[2], st)); }
    const int warp = nn <= (uint32_t)e->keyed_warp_limit ? 1 : 0;  // small batch: one signature per warp (latency path)
    CU(e, kt->verify(nn, d_slot, d.slot2local[curve], d.n_slots, d.keyflags[curve], d_r, w->uw, w->flags, d.gtab[curve], d.ktab[curve], d_ok, warp,
                     st));
    if (ev) CU(e, cudaEventRecord(ev[3], st));
    CU(e, cudaEventRecord(w->done, st));
    e->launches += 2;
    return 0;
}
