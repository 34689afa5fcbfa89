"""Ed25519 throughput through the C ABI, three arms timed in the same run and alternated step by step:
  per_item          sbv_ed25519_verify_batch (keys per item) on an engine with the default grouping: keys that repeat
                    at least SBV_GROUP_THRESHOLD (16) times in the batch get a comb table built in the launch
  per_item_generic  the same call on a second engine with SBV_GROUP_THRESHOLD=0: every item takes k_ed_verify
  registered        sbv_ed25519_verify_registered (the corpus's distinct keys registered with sbv_ed25519_set_keys, items
                    by slot); left out above 4,096 distinct keys (the registry would hold 384 KiB per key)
and the OpenSSL CPU arm measured in the same run.

    python tools/ed25519_bench.py [--n 65536] [--keys 1024] [--msg-len 256] [--steps 20] [--warmup 5]

--keys equal to --n makes every key distinct.  Inputs live in pinned host memory (sbv_host_alloc); each timed call
uploads them, hashes, verifies and returns the verdicts.  Kernel times (k_ed_sha512, k_ed_verify, k_ed_verify_comb, the
grouping and comb construction kernels, k_ed_key_gather, k_ed_verify_keyed) come from a separate torch.profiler run;
sbv_ed25519_set_keys is timed on its first and second call.  Prints one JSON line with the card's name and power limit;
the verdicts of every timed call are checked against the oracle.
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


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--keys", type=int, default=1024)
    ap.add_argument("--msg-len", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import oracle_ed25519 as oe
    from oracle_ed25519 import corpus

    c = corpus.make_corpus(args.n, seed=2024, n_keys=args.keys, fixed_len=args.msg_len, crafted_max=64)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    eng = sbv.Engine(devices=[0])
    old = os.environ.get("SBV_GROUP_THRESHOLD")
    os.environ["SBV_GROUP_THRESHOLD"] = "0"
    try:
        eng_gen = sbv.Engine(devices=[0])
    finally:
        if old is None:
            os.environ.pop("SBV_GROUP_THRESHOLD", None)
        else:
            os.environ["SBV_GROUP_THRESHOLD"] = old
    bufs = []

    def pinned(a):
        a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        ptr = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
        if not ptr:
            raise sbv.EngineFault("sbv_host_alloc failed")
        bufs.append(ptr)
        np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(ptr))[:] = a
        return ptr

    n = args.n
    keys, slot = np.unique(c["pub"], axis=0, return_inverse=True)
    slot = slot.reshape(-1).astype(np.uint32)
    m, o, s, p, ok = pinned(c["msgs"]), pinned(c["off"]), pinned(c["sig"]), pinned(c["pub"]), pinned(np.zeros(n, np.uint8))
    sl = pinned(slot)
    okv = np.ctypeslib.as_array((C.c_uint8 * n).from_address(ok))
    registered = keys.shape[0] <= 4096
    try:
        set_keys_ms = []
        for _ in range(2 if registered else 0):  # the first call on a fresh engine also loads the kernels; the second replaces a full registry
            t0 = time.perf_counter()
            eng.ed25519_set_keys(keys)
            set_keys_ms.append((time.perf_counter() - t0) * 1e3)
        arms = {"per_item": lambda: eng.ed25519_verify_batch_ptr(n, m, o, s, p, ok),
                "per_item_generic": lambda: eng_gen.ed25519_verify_batch_ptr(n, m, o, s, p, ok)}
        if registered:
            arms["registered"] = lambda: eng.ed25519_verify_registered_ptr(n, m, o, sl, s, ok)
        for _ in range(args.warmup):
            for f in arms.values():
                f()
        times, verdicts_ok = {a: [] for a in arms}, True
        order = list(arms)
        for step in range(args.steps):
            for a in order[step % len(order):] + order[:step % len(order)]:
                okv[:] = 2
                t0 = time.perf_counter()
                arms[a]()
                times[a].append(time.perf_counter() - t0)
                verdicts_ok &= bool(np.array_equal(okv, want))
        from torch.profiler import ProfilerActivity, profile
        kern = {}
        for a, f in arms.items():  # one profile per arm: k_ed_verify runs in both per-item arms, over different lists
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    f()
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                for name in ("k_ed_sha512", "k_ed_verify", "k_ed_verify_comb", "k_kg_insert", "k_kg_assign", "k_kg_route", "k_edc_bases",
                             "k_edc_fill", "k_edc_inv", "k_edc_final", "k_ed_key_gather", "k_ed_verify_keyed"):
                    if re.search(r"\b" + name + r"\b", ev.key):
                        t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per call
                        kern[f"{a}_{name}_us"] = round(float(t), 1)
            verdicts_ok &= bool(np.array_equal(okv, want))
    finally:
        eng.close()
        eng_gen.close()
        for ptr in bufs:
            lib.sbv_host_free(C.c_void_p(ptr))
    cores = oe.ncores()
    cpu_s, cpu_ok = oe.bench_verify(c["msgs"], c["off"], c["sig"], c["pub"], nthreads=cores)
    med = float(np.median(times["per_item"]))
    med_gen = float(np.median(times["per_item_generic"]))
    med_reg = float(np.median(times["registered"])) if registered else None
    props = torch.cuda.get_device_properties(0)
    res = {
        "metric": "ed25519_verifies_per_s",
        "value": n / med,
        "unit": "verifies/s",
        "n": n, "keys": args.keys, "msg_len": args.msg_len, "steps": args.steps, "warmup": args.warmup,
        "median_call_ms": med * 1e3,
        "best_call_ms": min(times["per_item"]) * 1e3,
        "per_item_generic_verifies_per_s": n / med_gen,
        "per_item_generic_median_call_ms": med_gen * 1e3,
        "per_item_generic_best_call_ms": min(times["per_item_generic"]) * 1e3,
        "grouped_over_generic": med_gen / med,
        "registered_verifies_per_s": n / med_reg if registered else None,
        "registered_median_call_ms": med_reg * 1e3 if registered else None,
        "registered_best_call_ms": min(times["registered"]) * 1e3 if registered else None,
        "distinct_keys": int(keys.shape[0]),
        "set_keys_first_ms": round(set_keys_ms[0], 2) if registered else None,
        "set_keys_second_ms": round(set_keys_ms[1], 2) if registered else None,
        **kern,
        "cpu_openssl_verifies_per_s": n / cpu_s,
        "cpu_cores": cores,
        "gpu_over_cpu": (n / med) / (n / cpu_s),
        "accepts": int(want.sum()),
        "verdicts_match_oracle": bool(verdicts_ok and np.array_equal(cpu_ok, want)),
        "device": props.name,
        "power_limit_w": power_limit_w(),
    }
    print(json.dumps(res))
    return 0 if res["verdicts_match_oracle"] else 1


if __name__ == "__main__":
    sys.exit(main())
