"""Keys-per-item calls with the grouped-key cache (sbv_key_cache_reserve) against the same calls without it, alternated in
one run.

    python tools/key_cache_bench.py [--steps 20] [--warmup 5] [--threads 6]

Workloads (the shapes of bench.py's keys-per-item steps, seeded):
  p256   sbv_verify_batch, 65,536 P-256 items over 1,024 keys (every key repeats ~64 times: all of them are grouped)
  p384   the same on P-384
  ed     sbv_ed25519_verify_batch, 65,536 items of 256-byte messages over 1,024 keys
Two engines on device 0: one with a cache big enough for every key (warmed, so every grouped key hits), one without.
For each workload and engine:
  isolated   one call at a time from pinned host memory (sbv_host_alloc): median and best wall time per call
  steady     `threads` host threads, each issuing calls back to back through the host-buffer entry points, the two
             engines alternating block by block: items per second over the whole block
Every call's verdicts are checked against OpenSSL.  The card's name and power limit are read in the same run.  Prints one
JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--threads", type=int, default=6)
    ap.add_argument("--calls", type=int, default=8, help="calls per thread in a steady block")
    ap.add_argument("--blocks", type=int, default=4, help="steady blocks per engine")
    ap.add_argument("--items", type=int, default=65536)
    ap.add_argument("--keys", type=int, default=1024)
    ap.add_argument("--only", nargs="*", default=["p256", "p384", "ed"])
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import oracle
    import oracle_ed25519
    from ed25519_quorum_bench import power_limit_w
    from oracle import corpus
    from oracle_ed25519 import corpus as edcorpus

    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
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

    n, K = args.items, args.keys
    engines = {"cached": sbv.Engine(devices=[0]), "uncached": sbv.Engine(devices=[0])}
    engines["cached"].key_cache_reserve(K, K, K)
    res = {"metric": "key_cache_isolated_speedup", "unit": "x", "items": n, "keys": K, "steps": args.steps, "warmup": args.warmup,
           "threads": args.threads}
    all_good = True
    try:
        for wl in args.only:
            if wl in ("p256", "p384"):
                curve = oracle.P256 if wl == "p256" else oracle.P384
                b = corpus.make_batch(curve, n=n, K=K, seed=911 + curve)
                want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
                ptrs = [pinned(b[k])[0] for k in ("r", "s", "qx", "qy", "digest")]
                dlen = b["digest"].shape[1] if b["digest"].ndim == 2 else b["digest"].size // n

                def call(eng, ok_ptr, curve=curve, ptrs=ptrs, dlen=dlen):
                    eng._check(lib.sbv_verify_batch(eng._h, C.c_uint8(curve), C.c_size_t(n), *(vp(p) for p in ptrs), C.c_uint8(dlen), vp(ok_ptr)),
                               "sbv_verify_batch")
            else:
                c = edcorpus.make_corpus(n, seed=2024, n_keys=K, fixed_len=256, crafted_max=64)
                want = oracle_ed25519.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
                ptrs = [pinned(c[k])[0] for k in ("msgs", "off", "sig", "pub")]

                def call(eng, ok_ptr, ptrs=ptrs):
                    eng._check(lib.sbv_ed25519_verify_batch(eng._h, C.c_size_t(n), *(vp(p) for p in ptrs), vp(ok_ptr)), "sbv_ed25519_verify_batch")

            outs = [pinned(np.zeros(n, np.uint8)) for _ in range(args.threads)]

            def check(view):
                good = bool(np.array_equal(view, want))
                view[:] = 2
                return good

            # isolated calls, alternating the engines call by call
            names = list(engines)
            for _ in range(args.warmup):
                for name in names:
                    call(engines[name], outs[0][0])
            times = {name: [] for name in names}
            for step in range(args.steps):
                for name in (names if step % 2 == 0 else names[::-1]):
                    t0 = time.perf_counter()
                    call(engines[name], outs[0][0])
                    times[name].append(time.perf_counter() - t0)
                    all_good &= check(outs[0][1])
            for name in names:
                res[f"{wl}_{name}_isolated_median_ms"] = round(float(np.median(times[name])) * 1e3, 3)
                res[f"{wl}_{name}_isolated_best_ms"] = round(min(times[name]) * 1e3, 3)
            res[f"{wl}_isolated_speedup"] = round(res[f"{wl}_uncached_isolated_median_ms"] / res[f"{wl}_cached_isolated_median_ms"], 3)

            # steady throughput: blocks of `threads` x `calls` calls, the engines alternating block by block
            rates = {name: [] for name in names}
            errors = []

            def worker(eng, t):
                try:
                    for _ in range(args.calls):
                        call(eng, outs[t][0])
                except Exception as ex:  # noqa: BLE001
                    errors.append(ex)

            for blk in range(2 * args.blocks + 2):
                name = names[blk % 2]
                th = [threading.Thread(target=worker, args=(engines[name], t)) for t in range(args.threads)]
                t0 = time.perf_counter()
                for x in th:
                    x.start()
                for x in th:
                    x.join()
                dt = time.perf_counter() - t0
                if errors:
                    raise errors[0]
                for t in range(args.threads):
                    all_good &= check(outs[t][1])
                if blk >= 2:  # the first block of each engine warms its lanes and scratch sets
                    rates[name].append(args.threads * args.calls * n / dt)
            for name in names:
                res[f"{wl}_{name}_steady_items_per_s"] = round(float(np.median(rates[name])))
                res[f"{wl}_{name}_steady_spread"] = [round(min(rates[name])), round(max(rates[name]))]
            res[f"{wl}_steady_speedup"] = round(res[f"{wl}_cached_steady_items_per_s"] / res[f"{wl}_uncached_steady_items_per_s"], 3)
        for s, tag in ((oracle.P256, "p256"), (oracle.P384, "p384"), (2, "ed")):
            res[f"{tag}_cache_stats"] = engines["cached"].key_cache_stats(s)
        if "p256" in args.only:
            res["value"] = res["p256_isolated_speedup"]
    finally:
        for eng in engines.values():
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
