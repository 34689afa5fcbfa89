"""Mixed ECDSA / Ed25519 batches through the C ABI: one sbv_mixed_* call against the per-family composition, alternated
call by call in one run.

    python tools/mixed_bench.py [--steps 20] [--warmup 5]

(a) The C4 shape with a mixed consenter set of 16 (7 P-256, 2 P-384, 7 Ed25519; Q = 11, threshold Q - 1): 17,476
    instances x 15 votes + 4 inert votes = 262,144 votes with Byzantine votes (tests/mixed_cases.make_votes).  One
    sbv_mixed_verify_quorum call against the family calls (sbv_hash_verify_registered per curve,
    sbv_ed25519_verify_registered), a host scatter of their verdicts and sbv_quorum.
(b) Flush-sized batches of 16, 256 and 2,048 items, half P-256 and half Ed25519, interleaved: one
    sbv_mixed_verify_registered call against the two family calls and the host scatter that a per-scheme Verifier makes.
Inputs and outputs live in pinned host memory (sbv_host_alloc); the family arms get their per-family arrays ready-made,
so their marshalling is not timed.  Every timed call's outputs are checked against OpenSSL and
oracle.ecdsa_ref.count_commit_votes_batch.  Kernel times of the split / scatter kernels come from a separate
torch.profiler run; the card's name and power limit are read in the same run.  Prints one JSON line.
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

KERNELS = ("k_mix_count", "k_mix_scan", "k_mix_split", "k_mix_compact", "k_mix_ok", "k_sha256", "k_ed_sha512", "k_ed_verify_keyed")
C4_SCHEMES = [0] * 7 + [1] * 2 + [2] * 7


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=17476)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import mixed_cases as mc
    from ed25519_quorum_bench import power_limit_w

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
        """Pinned per-family arrays of the composition arms: (tag, idx, n, msgs, off, slot, r|sig, s, ok) per family present."""
        out = []
        for c in (0, 1, 2):
            idx = np.flatnonzero(cp["scheme"] == c)
            if idx.size == 0:
                continue
            m, o = mc.gather(cp["msgs"], cp["off"], idx)
            w = 64 if c == 2 else mc.L[c]
            r = pinned(cp["sig96"][idx, :w])[0]
            s = pinned(cp["sig96"][idx, w:2 * w])[0] if c != 2 else None
            out.append((c, idx, idx.size, pinned(m)[0], pinned(o)[0], pinned(cp["key_slot"][idx])[0], r, s, pinned(np.zeros(idx.size, np.uint8))))
        return out

    def run_families(fams, ok):
        for c, idx, k, m, o, slot, r, s, (okp, okv) in fams:
            if c == 2:
                eng._check(lib.sbv_ed25519_verify_registered(eng._h, C.c_size_t(k), vp(m), vp(o), vp(slot), vp(r), vp(okp)), "sbv_ed25519_verify_registered")
            else:
                eng._check(lib.sbv_hash_verify_registered(eng._h, C.c_uint8(c), C.c_size_t(k), vp(m), vp(o), vp(slot), vp(r), vp(s), vp(okp)),
                           "sbv_hash_verify_registered")
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

    res = {"metric": "mixed_commit_votes_per_s", "unit": "votes/s", "steps": args.steps, "warmup": args.warmup}
    try:
        # (a) the C4 shape
        st, reg = mc.make_votes(args.instances, C4_SCHEMES, seed=2026, pad=4)
        q, _ = sbv.compute_quorum(len(C4_SCHEMES))
        thr = q - 1
        want = mc.expected_votes(st, reg, thr)
        n, I = st["instance"].size, st["n_instances"]
        eng.set_keys(reg["ecdsa_curve"], reg["ecdsa_xy"])
        eng.ed25519_set_keys(reg["ed_pub"])
        p = {k: pinned(st[k])[0] for k in ("scheme", "msgs", "off", "key_slot", "sig96", "instance", "sender", "signer", "digest_match", "self_id")}
        ok_p, ok = pinned(np.zeros(n, np.uint8))
        cnt_p, cnt = pinned(np.zeros(I, np.uint32))
        rch_p, rch = pinned(np.zeros(I, np.uint8))
        fams = families(st)

        def one_call():
            eng.mixed_verify_quorum_ptr(n, p["scheme"], p["msgs"], p["off"], p["key_slot"], p["sig96"], p["instance"], p["sender"], p["signer"],
                                        p["digest_match"], I, p["self_id"], thr, ok_p, cnt_p, rch_p)

        def composition():
            run_families(fams, ok)
            eng._check(lib.sbv_quorum(eng._h, C.c_size_t(n), vp(p["instance"]), vp(p["sender"]), vp(p["signer"]), vp(p["digest_match"]),
                                      vp(ok_p), C.c_size_t(I), vp(p["self_id"]), C.c_uint32(thr), vp(cnt_p), vp(rch_p)), "sbv_quorum")

        def check_a():
            good = np.array_equal(ok, want[0]) and np.array_equal(cnt, want[1]) and np.array_equal(rch, want[2])
            ok[:] = 2
            cnt[:] = 0xFFFFFFFF
            rch[:] = 2
            return bool(good)

        times, good = alternate({"one_call": one_call, "composition": composition}, check_a)
        m1, m2 = float(np.median(times["one_call"])), float(np.median(times["composition"]))
        res.update(value=n / m1, votes=n, instances=I, threshold=thr, c4_one_call_median_ms=m1 * 1e3, c4_one_call_best_ms=min(times["one_call"]) * 1e3,
                   c4_composition_median_ms=m2 * 1e3, c4_composition_best_ms=min(times["composition"]) * 1e3,
                   c4_one_call_mvotes_per_s=n / m1 / 1e6, c4_composition_mvotes_per_s=n / m2 / 1e6, c4_outputs_match_oracle=good)
        all_good = good

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                one_call()
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            for name in KERNELS:
                if re.search(r"\b" + name + r"\b", ev.key):
                    t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per launch
                    res[f"c4_{name}_us"] = round(float(t), 1)

        # (b) flush-sized batches, half P-256 and half Ed25519
        breg = mc.registries(n256=8, n384=1, n_ed=8, seed=2027)
        eng.set_keys(breg["ecdsa_curve"], breg["ecdsa_xy"])
        eng.ed25519_set_keys(breg["ed_pub"])
        for size in (16, 256, 2048):
            tag = np.tile(np.array([0, 2], np.uint8), size // 2)
            cp = mc.make_corpus(tag, breg, seed=size, lo=64, hi=320)
            wok = mc.expected_ok(cp, breg["ecdsa_curve"], breg["ecdsa_xy"], breg["ed_pub"])
            pb = {k: pinned(cp[k])[0] for k in ("scheme", "msgs", "off", "key_slot", "sig96")}
            okb_p, okb = pinned(np.zeros(size, np.uint8))
            fb = families(cp)
            arms = {"one_call": lambda: eng.mixed_verify_registered_ptr(size, pb["scheme"], pb["msgs"], pb["off"], pb["key_slot"], pb["sig96"], okb_p),
                    "two_calls": lambda: run_families(fb, okb)}

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
