"""Ed25519 commit votes through the C ABI: sbv_ed25519_verify_quorum (one call) against the two-call form
(sbv_ed25519_verify_registered, then sbv_quorum over the verdicts), alternated call by call in one run.

    python tools/ed25519_quorum_bench.py [--instances 17476] [--consenters 16] [--pad 4] [--steps 20] [--warmup 5]

The default is the C4 shape: N = 16 consenters (Q = 11, threshold Q - 1), 17,476 instances x 15 votes + 4 inert votes =
262,144 votes, up to f Byzantine votes per instance (oracle_ed25519.votes).  Inputs and outputs live in pinned host
memory (sbv_host_alloc).  Every timed call's ok / valid_count / reached are checked against OpenSSL and
oracle.ecdsa_ref.count_commit_votes_batch.  Kernel times come from a separate torch.profiler run; the card's name and
power limit are read in the same run.  Prints one JSON line.
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

KERNELS = ("k_ed_key_gather", "k_ed_sha512", "k_ed_verify_keyed", "k_quorum_count", "k_quorum_reached")


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=17476)
    ap.add_argument("--consenters", type=int, default=16)
    ap.add_argument("--pad", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    from oracle_ed25519 import votes

    st = votes.make_stream(args.instances, args.consenters, seed=2026, pad=args.pad)
    q, _ = sbv.compute_quorum(args.consenters)
    thr = q - 1
    want = votes.expected(st, thr)
    n, I = st["instance"].size, st["n_instances"]
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    eng = sbv.Engine(devices=[0])
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

    try:
        p = {k: pinned(st[k])[0] for k in ("msgs", "off", "key_slot", "sig", "instance", "sender", "signer", "digest_match", "self_id")}
        ok_p, ok = pinned(np.zeros(n, np.uint8))
        cnt_p, cnt = pinned(np.zeros(I, np.uint32))
        rch_p, rch = pinned(np.zeros(I, np.uint8))
        eng.ed25519_set_keys(st["pub"])
        vp = C.c_void_p

        def one_call():
            eng.ed25519_verify_quorum_ptr(n, p["msgs"], p["off"], p["key_slot"], p["sig"], p["instance"], p["sender"], p["signer"],
                                          p["digest_match"], I, p["self_id"], thr, ok_p, cnt_p, rch_p)

        def two_calls():
            eng.ed25519_verify_registered_ptr(n, p["msgs"], p["off"], p["key_slot"], p["sig"], ok_p)
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
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                for f in arms.values():
                    f()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            for name in KERNELS:
                if re.search(r"\b" + name + r"\b", ev.key):
                    t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per call
                    kern[name + "_us"] = round(float(t), 1)
    finally:
        eng.close()
        for ptr in bufs:
            lib.sbv_host_free(C.c_void_p(ptr))
    med1, med2 = float(np.median(times["one_call"])), float(np.median(times["two_calls"]))
    res = {
        "metric": "ed25519_commit_votes_per_s",
        "value": n / med1,
        "unit": "votes/s",
        "votes": n, "instances": I, "consenters": args.consenters, "threshold": thr, "steps": args.steps, "warmup": args.warmup,
        "one_call_median_ms": med1 * 1e3,
        "one_call_best_ms": min(times["one_call"]) * 1e3,
        "one_call_mvotes_per_s": n / med1 / 1e6,
        "two_calls_median_ms": med2 * 1e3,
        "two_calls_best_ms": min(times["two_calls"]) * 1e3,
        "two_calls_mvotes_per_s": n / med2 / 1e6,
        **kern,
        "accepts": int(want[0].sum()),
        "reached": int(want[2].sum()),
        "outputs_match_oracle": bool(outputs_ok),
        "device": torch.cuda.get_device_properties(0).name,
        "power_limit_w": power_limit_w(),
    }
    print(json.dumps(res))
    return 0 if res["outputs_match_oracle"] else 1


if __name__ == "__main__":
    sys.exit(main())
