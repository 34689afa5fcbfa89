"""RSA commit votes through the C ABI: sbv_rsa_verify_quorum (one call) against the two-call form (per key size
sbv_rsa_hash_verify_registered over that size's votes, the verdicts put back in vote order on the host, then sbv_quorum),
alternated call by call in one run, for two consenter sets.

    python tools/rsa_quorum_bench.py [--instances 17476] [--pad 4] [--steps 20] [--warmup 3] [--sets mixed all2048]

The default is the C4 shape: N = 16 consenters (Q = 11, threshold Q - 1), 17,476 instances x 15 votes + 4 inert votes =
262,144 votes, up to f Byzantine votes per instance, SHA-256, PKCS #1 v1.5 (tests/rsa_quorum_cases.py).  `mixed` is ten
2048-bit, four 3072-bit and two 4096-bit consenter keys, `all2048` sixteen 2048-bit keys.  Inputs and outputs live in
pinned host memory (sbv_host_alloc); the two-call form gets its per-size inputs already split and packed (the caller's
host work of splitting the wire votes is not timed), so it is timed from its first call to the end of sbv_quorum.  Every
timed call's ok / valid_count / reached are checked against oracle_rsa.ref and oracle.ecdsa_ref.count_commit_votes_batch.
Kernel times of the one call, and the kernel, host-to-device and device-to-host copy time of each form, come from
torch.profiler runs of their own; the card's name and power limit are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KERNELS = ("k_sha256", "k_mix_count", "k_mix_scan", "k_rsa_split", "k_mix_compact", "k_rsa_verify_reg", "k_mix_ok", "k_quorum_count",
           "k_quorum_reached")


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def bench_set(sbv, lib, eng, torch, name, sizes, args):
    import rsa_quorum_cases as q

    cons = q.Consenters(sizes)
    st = q.pack(q.make_stream(cons, args.instances, seed=2026, pad=args.pad))
    q_, _ = sbv.compute_quorum(cons.n)
    thr = q_ - 1
    want = q.expected(cons.reg, st, thr)
    n, I = st["instance"].size, st["n_instances"]
    mb, mods, exp = cons.arrays()
    eng.rsa_set_keys(mb, mods, exp)
    bufs = []

    def pinned(a):
        a = np.ascontiguousarray(a)
        ptr = lib.sbv_host_alloc(C.c_size_t(max(a.nbytes, 1)))
        if not ptr:
            raise sbv.EngineFault("sbv_host_alloc failed")
        bufs.append(ptr)
        view = np.ctypeslib.as_array((C.c_uint8 * max(a.nbytes, 1)).from_address(ptr))[: a.nbytes].view(a.dtype).reshape(a.shape)
        view[...] = a
        return ptr, view

    kern = {}
    try:
        cols = ("msgs", "off", "key_slot", "sig", "sig_off", "instance", "sender", "signer", "digest_match", "self_id")
        p = {k: pinned(st[k])[0] for k in cols}
        ok_p, ok = pinned(np.zeros(n, np.uint8))
        cnt_p, cnt = pinned(np.zeros(I, np.uint32))
        rch_p, rch = pinned(np.zeros(I, np.uint8))
        # the two-call form's inputs: per size, the votes of that signature length packed in fixed k-byte rows
        lens = np.diff(st["sig_off"].astype(np.int64))
        fam = []
        for k in q.SIZES:
            idx = np.flatnonzero(lens == k)
            if not idx.size:
                continue
            msgs, off = q.blob([st["msgs_l"][i] for i in idx])
            sig = np.frombuffer(b"".join(st["sigs_l"][i] for i in idx), np.uint8)
            fam.append((k, idx, pinned(msgs)[0], pinned(off)[0], pinned(st["key_slot"][idx])[0], pinned(sig)[0], *pinned(np.zeros(idx.size, np.uint8))))
        vp = C.c_void_p

        def one_call():
            eng.rsa_verify_quorum_ptr(st["hash"], n, *(p[c] for c in cols[:9]), I, p["self_id"], thr, ok_p, cnt_p, rch_p)

        def two_calls():
            for k, idx, m_p, o_p, s_p, g_p, f_okp, f_ok in fam:
                eng.rsa_hash_verify_registered_ptr(k, st["hash"], idx.size, m_p, o_p, s_p, g_p, 0, f_okp)
            ok[:] = 0
            for k, idx, m_p, o_p, s_p, g_p, f_okp, f_ok in fam:
                ok[idx] = f_ok
            eng._check(lib.sbv_quorum(eng._h, C.c_size_t(n), vp(p["instance"]), vp(p["sender"]), vp(p["signer"]), vp(p["digest_match"]),
                                      vp(ok_p), C.c_size_t(I), vp(p["self_id"]), C.c_uint32(thr), vp(cnt_p), vp(rch_p)), "sbv_quorum")

        arms = {"one_call": one_call, "two_calls": two_calls}
        for _ in range(args.warmup):
            for f in arms.values():
                f()
        times, outputs_ok = {a: [] for a in arms}, True
        for step in range(args.steps):
            for a in (("one_call", "two_calls") if step % 2 == 0 else ("two_calls", "one_call")):
                ok[:] = 2
                cnt[:] = 0xFFFFFFFF
                rch[:] = 2
                t0 = time.perf_counter()
                arms[a]()
                times[a].append(time.perf_counter() - t0)
                outputs_ok &= bool(np.array_equal(ok, want[0]) and np.array_equal(cnt, want[1]) and np.array_equal(rch, want[2]))
        from torch.profiler import ProfilerActivity, profile
        reps = 3
        for a, f in arms.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    f()
                torch.cuda.synchronize()
            busy = {"kernels": 0.0, "h2d": 0.0, "d2h": 0.0}
            for ev in prof.key_averages():
                t = float(getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)) / reps
                cat = "h2d" if "HtoD" in ev.key else "d2h" if "DtoH" in ev.key else None if "Memset" in ev.key or "Memcpy" in ev.key else "kernels"
                if cat:
                    busy[cat] += t
                for kname in KERNELS if a == "one_call" else ():
                    if re.search(r"\b" + kname + r"\b", ev.key):
                        kern[kname + "_us_per_call"] = round(kern.get(kname + "_us_per_call", 0.0) + t, 1)
            for cat, t in busy.items():
                kern[f"{a}_{cat}_us_per_call"] = round(t, 1)
    finally:
        for ptr in bufs:
            lib.sbv_host_free(C.c_void_p(ptr))
    med1, med2 = float(np.median(times["one_call"])), float(np.median(times["two_calls"]))
    split = sum(kern.get(k + "_us_per_call", 0.0) for k in ("k_mix_count", "k_mix_scan", "k_rsa_split", "k_mix_compact", "k_mix_ok"))
    return {
        "set": name, "votes": n, "instances": I, "consenters": cons.n, "key_bytes": list(sizes), "threshold": thr,
        "one_call_median_ms": round(med1 * 1e3, 3), "one_call_best_ms": round(min(times["one_call"]) * 1e3, 3),
        "one_call_mvotes_per_s": round(n / med1 / 1e6, 3),
        "two_calls_median_ms": round(med2 * 1e3, 3), "two_calls_best_ms": round(min(times["two_calls"]) * 1e3, 3),
        "two_calls_mvotes_per_s": round(n / med2 / 1e6, 3),
        "split_kernels_us_per_call": round(split, 1), **kern,
        "accepts": int(want[0].sum()), "reached": int(want[2].sum()), "outputs_match_oracle": bool(outputs_ok),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=17476)
    ap.add_argument("--pad", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sets", nargs="+", default=["mixed", "all2048"], choices=["mixed", "all2048"])
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import rsa_quorum_cases as q

    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    eng = sbv.Engine(devices=[0])
    try:
        sets = {"mixed": q.MIXED, "all2048": q.ALL_2048}
        results = [bench_set(sbv, lib, eng, torch, s, sets[s], args) for s in args.sets]
    finally:
        eng.close()
    res = {
        "metric": "rsa_commit_votes_per_s",
        "value": results[0]["votes"] * 1e3 / results[0]["one_call_median_ms"],
        "unit": "votes/s",
        "steps": args.steps, "warmup": args.warmup,
        "sets": results,
        "outputs_match_oracle": all(r["outputs_match_oracle"] for r in results),
        "device": torch.cuda.get_device_properties(0).name,
        "power_limit_w": power_limit_w(),
    }
    print(json.dumps(res))
    return 0 if res["outputs_match_oracle"] else 1


if __name__ == "__main__":
    sys.exit(main())
