"""Mixed batches with ECDSA items over SHA-384 through the C ABI: one sbv_mixed384_* call against the per-family
composition, alternated call by call in one run.

    python tools/mixed384_bench.py [--instances 4096] [--steps 20] [--warmup 5]

(a) The C4 shape with a consenter set of 16 that signs with every tag: 4 P-256 / SHA-256, 3 P-256 / SHA-384, 1 P-384 /
    SHA-256, 2 P-384 / SHA-384 and 6 Ed25519 (Q = 11, threshold Q - 1).  Every consenter votes once per instance plus two
    repeated votes per instance, some with a signer that is not their sender (tests/mixed384_cases.vote_stream).  One
    sbv_mixed384_verify_quorum call against the family calls (sbv_hash_verify_registered and
    sbv_hash384_verify_registered per curve, sbv_ed25519_verify_registered), a host scatter of their verdicts and
    sbv_quorum.
(b) Flush-sized batches of 16, 256 and 2,048 items with tags 0 to 4 drawn at random: one sbv_mixed384_verify_registered
    call against the five family calls and the host scatter that a per-scheme, per-hash Verifier makes.
Inputs and outputs live in pinned host memory (sbv_host_alloc); the family arms get their per-family arrays ready-made,
so their marshalling is not timed.  Every timed call's outputs are checked against OpenSSL and
oracle.ecdsa_ref.count_commit_votes_batch.
(c) A separate torch.profiler run on 16,384 P-256 items, half over SHA-256 and half over SHA-384: k_mix_alg and
    k_sha2_sel inside sbv_mixed384_verify_registered against k_sha256 + k_sha384 of the two family calls, with the two
    hashes interleaved at random (both inside most warps) and in two runs (warps of one hash).
The card's name and power limit are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

C4_TAGS = [0] * 4 + [3] * 3 + [1] + [4] * 2 + [2] * 6
PROFILED = ("k_mix_alg", "k_sha2_sel", "k_sha256", "k_sha384")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-items", type=int, default=16384)
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import mixed384_cases as mc
    from ed25519_quorum_bench import power_limit_w
    from oracle import ecdsa_ref

    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    eng = sbv.Engine(devices=[0])
    bufs = []
    vp = C.c_void_p

    def pinned(a):
        a = np.ascontiguousarray(a)
        ptr = lib.sbv_host_alloc(C.c_size_t(max(a.nbytes, 1)))
        if not ptr:
            raise sbv.EngineFault("sbv_host_alloc failed")
        bufs.append(ptr)
        view = np.ctypeslib.as_array((C.c_uint8 * max(a.nbytes, 1)).from_address(ptr))[: a.nbytes].view(a.dtype).reshape(a.shape)
        view[...] = a
        return ptr, view

    def families(cp):
        """Pinned per-(curve, hash) arrays of the composition arms: (tag, idx, n, msgs, off, slot, r|sig, s, ok) per tag present."""
        out = []
        for t in range(5):
            idx = np.flatnonzero(cp["scheme"] == t)
            if idx.size == 0:
                continue
            m, o = mc.gather(cp["msgs"], cp["off"], idx)
            w = 64 if t == mc.ED else mc.L[mc.CURVE[t]]
            r = pinned(cp["sig96"][idx, :w])[0]
            s = pinned(cp["sig96"][idx, w:2 * w])[0] if t != mc.ED else None
            out.append((t, idx, idx.size, pinned(m)[0], pinned(o)[0], pinned(cp["key_slot"][idx])[0], r, s, pinned(np.zeros(idx.size, np.uint8))))
        return out

    def run_families(fams, ok):
        for t, idx, k, m, o, slot, r, s, (okp, okv) in fams:
            if t == mc.ED:
                eng._check(lib.sbv_ed25519_verify_registered(eng._h, C.c_size_t(k), vp(m), vp(o), vp(slot), vp(r), vp(okp)), "sbv_ed25519_verify_registered")
            else:
                fn = "sbv_hash384_verify_registered" if t >= mc.P256_SHA384 else "sbv_hash_verify_registered"
                eng._check(getattr(lib, fn)(eng._h, C.c_uint8(mc.CURVE[t]), C.c_size_t(k), vp(m), vp(o), vp(slot), vp(r), vp(s), vp(okp)), fn)
            ok[idx] = okv

    def alternate(arms, check):
        for _ in range(args.warmup):
            for f in arms.values():
                f()
        times, good = {a: [] for a in arms}, True
        names = list(arms)
        for step in range(args.steps):
            for a in (names if step % 2 == 0 else names[::-1]):
                t0 = time.perf_counter()
                arms[a]()
                times[a].append(time.perf_counter() - t0)
                good &= check()
        return times, good

    def consenter_slots(reg, tags):
        slots, seen = [], {0: 0, 1: 0, 2: 0}
        for t in tags:
            c = mc.CURVE.get(t, mc.ED)
            own = np.flatnonzero(reg["ecdsa_curve"] == c) if c != mc.ED else np.arange(reg["ed_pub"].shape[0])
            slots.append(own[seen[c] % own.size])
            seen[c] += 1
        return np.array(slots, np.uint32)

    res = {"metric": "mixed384_commit_votes_per_s", "unit": "votes/s", "steps": args.steps, "warmup": args.warmup}
    try:
        # (a) the C4 shape
        reg = mc.registries(n256=7, n384=3, n_ed=6, seed=2026)
        scheme, who, inst, sender, signer, dm = mc.vote_stream(C4_TAGS, args.instances, seed=2026)
        st = mc.make_corpus(scheme, reg, seed=2026, lo=200, hi=400, corrupt=1 / 16, key_slot=consenter_slots(reg, C4_TAGS)[who])
        q, _ = sbv.compute_quorum(len(C4_TAGS))
        thr = q - 1
        I = args.instances
        self_id = np.zeros(I, np.uint16)
        want_ok = mc.expected_ok(st, reg)
        want_cnt, want_rch = ecdsa_ref.count_commit_votes_batch(inst, sender, signer, dm, want_ok, I, thr, self_id)
        want_cnt, want_rch = np.asarray(want_cnt, np.uint32), np.asarray(want_rch, np.uint8)
        n = inst.size
        mc.set_keys(eng, reg)
        cols = dict(st, instance=inst, sender=sender, signer=signer, digest_match=dm, self_id=self_id)
        p = {k: pinned(cols[k])[0] for k in ("scheme", "msgs", "off", "key_slot", "sig96", "instance", "sender", "signer", "digest_match", "self_id")}
        ok_p, ok = pinned(np.zeros(n, np.uint8))
        cnt_p, cnt = pinned(np.zeros(I, np.uint32))
        rch_p, rch = pinned(np.zeros(I, np.uint8))
        fams = families(st)

        def one_call():
            eng.mixed384_verify_quorum_ptr(n, p["scheme"], p["msgs"], p["off"], p["key_slot"], p["sig96"], p["instance"], p["sender"], p["signer"],
                                           p["digest_match"], I, p["self_id"], thr, ok_p, cnt_p, rch_p)

        def composition():
            run_families(fams, ok)
            eng._check(lib.sbv_quorum(eng._h, C.c_size_t(n), vp(p["instance"]), vp(p["sender"]), vp(p["signer"]), vp(p["digest_match"]),
                                      vp(ok_p), C.c_size_t(I), vp(p["self_id"]), C.c_uint32(thr), vp(cnt_p), vp(rch_p)), "sbv_quorum")

        def check_a():
            good = np.array_equal(ok, want_ok) and np.array_equal(cnt, want_cnt) and np.array_equal(rch, want_rch)
            ok[:] = 2
            cnt[:] = 0xFFFFFFFF
            rch[:] = 2
            return bool(good)

        times, good = alternate({"one_call": one_call, "composition": composition}, check_a)
        m1, m2 = float(np.median(times["one_call"])), float(np.median(times["composition"]))
        res.update(value=n / m1, votes=n, instances=I, threshold=thr, tags_per_vote=np.bincount(scheme, minlength=5).tolist(),
                   c4_one_call_median_ms=m1 * 1e3, c4_one_call_best_ms=min(times["one_call"]) * 1e3,
                   c4_composition_median_ms=m2 * 1e3, c4_composition_best_ms=min(times["composition"]) * 1e3,
                   c4_one_call_mvotes_per_s=n / m1 / 1e6, c4_composition_mvotes_per_s=n / m2 / 1e6, c4_outputs_match_oracle=good)
        all_good = good

        # (b) flush-sized batches, tags 0 to 4 at random
        breg = mc.registries(n256=8, n384=8, n_ed=8, seed=2027)
        mc.set_keys(eng, breg)
        for size in (16, 256, 2048):
            tag = np.random.default_rng(size).integers(0, 5, size).astype(np.uint8)
            cp = mc.make_corpus(tag, breg, seed=size, lo=64, hi=320, corrupt=1 / 16)
            wok = mc.expected_ok(cp, breg)
            pb = {k: pinned(cp[k])[0] for k in ("scheme", "msgs", "off", "key_slot", "sig96")}
            okb_p, okb = pinned(np.zeros(size, np.uint8))
            fb = families(cp)
            arms = {"one_call": lambda: eng.mixed384_verify_registered_ptr(size, pb["scheme"], pb["msgs"], pb["off"], pb["key_slot"], pb["sig96"], okb_p),
                    "family_calls": lambda: run_families(fb, okb)}

            def check_b():
                good = bool(np.array_equal(okb, wok))
                okb[:] = 2
                return good

            times, good = alternate(arms, check_b)
            all_good &= good
            for a in arms:
                res[f"b{size}_{a}_median_us"] = float(np.median(times[a])) * 1e6
                res[f"b{size}_{a}_best_us"] = min(times[a]) * 1e6
            res[f"b{size}_outputs_match_oracle"] = good

        # (c) kernel times on one P-256 family of both hashes
        from torch.profiler import ProfilerActivity, profile
        N = args.profile_items
        for layout in ("interleaved", "runs"):
            tag = np.random.default_rng(7).integers(0, 2, N).astype(np.uint8) * 3 if layout == "interleaved" else np.repeat(np.array([0, 3], np.uint8), N // 2)
            cp = mc.make_corpus(tag, breg, seed=N, lo=64, hi=320, corrupt=1 / 16)
            wok = mc.expected_ok(cp, breg)
            fb = families(cp)
            okc = np.zeros(N, np.uint8)
            got = eng.mixed384_verify_registered(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"])
            run_families(fb, okc)
            all_good &= bool(np.array_equal(got, wok) and np.array_equal(okc, wok))
            for arm, f in (("one_call", lambda: eng.mixed384_verify_registered(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"])),
                           ("family_calls", lambda: run_families(fb, okc))):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        f()
                    torch.cuda.synchronize()
                for ev in prof.key_averages():
                    for name in PROFILED:
                        if re.search(r"\b" + name + r"\b", ev.key):
                            t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per launch
                            res[f"p{N}_{layout}_{arm}_{name}_us"] = round(float(t), 1)
                            res[f"p{N}_{layout}_{arm}_{name}_launches"] = int(ev.count)
    finally:
        eng.close()
        for ptr in bufs:
            lib.sbv_host_free(C.c_void_p(ptr))
    res["outputs_match_oracle"] = bool(all_good)
    res["device"] = torch.cuda.get_device_properties(0).name
    res["power_limit_w"] = power_limit_w()
    print(json.dumps(res))
    return 0 if all_good else 1


if __name__ == "__main__":
    sys.exit(main())
