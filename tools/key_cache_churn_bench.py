"""The grouped-key cache under churn: keys-per-item P-256 calls whose keys come from a client population larger than the
cache, with no cache, the fill-once cache (sbv_key_cache_reserve) and the evicting cache (sbv_key_cache_reserve_evicting),
alternated in one run.

    python tools/key_cache_churn_bench.py [--steps 12] [--warmup 4] [--threads 6] [--caps 1024 4096]

Workload: sbv_verify_batch calls of 65,536 items.  The key of each item is drawn from `clients` keys (16,384) with Zipf
weights (rank r has weight 1 / r^zipf), and the popularity drifts: call i ranks the clients starting `drift * i` places
further along, so the hot clients of the first calls leave and new ones arrive, as a deployment's clients do.  Keys of
roughly the 500 most popular ranks occur 16 times or more in a call and are grouped.  Signatures come from a bank of
`bank` signed digests per client (a sixteenth of them corrupted), so every item's verdict is known and checked.

For each capacity and engine:
  hit rate   hits / (hits + misses) over the timed isolated calls (sbv_key_cache_stats_ex)
  isolated   one call at a time, the engines alternating call by call over the same sequence: median and best ms
  steady     `threads` host threads issuing calls back to back over the sequence, the engines alternating block by block:
             items per second
and the warm workload of key_cache_bench.py (65,536 items over 1,024 keys, every key hit) with the fill-once cache (1,024
tables) and the evicting cache (4,096 ways, so that no set overflows) beside no cache: what pinning and stamping cost when
everything hits.  Every verdict of every call is
checked.  The card's name and power limit are read in the same run.  Prints one JSON line.
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
    ap.add_argument("--steps", type=int, default=12, help="timed calls per engine and capacity")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--threads", type=int, default=6)
    ap.add_argument("--blocks", type=int, default=3, help="steady blocks per engine")
    ap.add_argument("--items", type=int, default=65536)
    ap.add_argument("--clients", type=int, default=16384)
    ap.add_argument("--zipf", type=float, default=1.0)
    ap.add_argument("--drift", type=int, default=64, help="clients the popularity ranking moves per call")
    ap.add_argument("--bank", type=int, default=4, help="signed digests per client")
    ap.add_argument("--caps", type=int, nargs="*", default=[1024, 4096])
    ap.add_argument("--warm-ways", type=int, default=4096, help="ways of the evicting cache in the all-hit workload")
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import oracle
    from ed25519_quorum_bench import power_limit_w
    from oracle import corpus

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

    P256, n, Kc, B = oracle.P256, args.items, args.clients, args.bank
    # the bank: B signed digests per client, a sixteenth corrupted; entry j = client j % Kc, digest j // Kc
    d, kxy = corpus.make_keys(P256, Kc, 2101)
    key_idx = (np.arange(Kc * B) % Kc).astype(np.uint32)
    bdig = corpus.make_digests(Kc * B, 2102)
    br, bs = oracle.sign_batch(P256, d, key_idx, bdig, corpus._blocks(2103, Kc * B, 32, b"k"))
    br[::16, 7] ^= 1
    bwant = oracle.verify_batch(P256, br, bs, kxy[key_idx, :32], kxy[key_idx, 32:], bdig)

    rng = np.random.default_rng(2104)
    w = 1.0 / np.arange(1, Kc + 1) ** args.zipf
    w /= w.sum()
    total = args.warmup + args.steps
    calls = []  # (pointers, verdicts) of call i
    for i in range(total):
        client = (rng.choice(Kc, n, p=w) + args.drift * i) % Kc
        j = client + Kc * rng.integers(0, B, n)
        arrs = (br[j], bs[j], kxy[client, :32], kxy[client, 32:], bdig[j])
        calls.append(([pinned(a)[0] for a in arrs], bwant[j]))
    grouped = [int((np.bincount((rng.choice(Kc, n, p=w)), minlength=Kc) >= 16).sum()) for _ in range(4)]

    outs = [pinned(np.zeros(n, np.uint8)) for _ in range(args.threads)]
    all_good = True

    def call(eng, i, t=0):
        ptrs, _ = calls[i]
        eng._check(lib.sbv_verify_batch(eng._h, C.c_uint8(P256), C.c_size_t(n), *(vp(p) for p in ptrs), C.c_uint8(32), vp(outs[t][0])),
                   "sbv_verify_batch")

    def check(i, t=0):
        view = outs[t][1]
        good = bool(np.array_equal(view, calls[i][1]))
        view[:] = 2
        return good

    res = {"metric": "key_cache_churn", "unit": "hit rate / ms / items per s", "items": n, "clients": Kc, "zipf": args.zipf,
           "drift": args.drift, "grouped_keys_per_call": int(np.median(grouped)), "steps": args.steps, "warmup": args.warmup,
           "threads": args.threads}
    engines = {"none": sbv.Engine(devices=[0]), "fill_once": sbv.Engine(devices=[0]), "evicting": sbv.Engine(devices=[0])}
    names = list(engines)
    try:
        for cap in args.caps:
            engines["fill_once"].key_cache_reserve(cap, 0, 0)
            engines["evicting"].key_cache_reserve_evicting(cap, 0, 0)
            tag = f"cap{cap}"
            times = {name: [] for name in names}
            base = {}
            for i in range(total):
                if i == args.warmup:
                    base = {name: engines[name].key_cache_stats_ex(P256) for name in names[1:]}
                for name in (names if i % 2 == 0 else names[::-1]):
                    t0 = time.perf_counter()
                    call(engines[name], i)
                    dt = time.perf_counter() - t0
                    all_good &= check(i)
                    if i >= args.warmup:
                        times[name].append(dt)
            for name in names:
                res[f"{tag}_{name}_isolated_median_ms"] = round(float(np.median(times[name])) * 1e3, 3)
                res[f"{tag}_{name}_isolated_best_ms"] = round(min(times[name]) * 1e3, 3)
            for name in names[1:]:
                st = engines[name].key_cache_stats_ex(P256)
                h, m = st["hits"] - base[name]["hits"], st["misses"] - base[name]["misses"]
                res[f"{tag}_{name}_hit_rate"] = round(h / max(h + m, 1), 4)
                res[f"{tag}_{name}_stats"] = st

            rates = {name: [] for name in names}
            errors = []

            def worker(eng, t):
                try:
                    for k in range(len(calls)):
                        i = (k + 3 * t) % len(calls)
                        call(eng, i, t)
                        if not check(i, t):
                            errors.append(f"verdicts of call {i}")
                except Exception as ex:  # noqa: BLE001
                    errors.append(ex)

            for blk in range(len(names) * (args.blocks + 1)):
                name = names[blk % len(names)]
                th = [threading.Thread(target=worker, args=(engines[name], t)) for t in range(args.threads)]
                t0 = time.perf_counter()
                for x in th:
                    x.start()
                for x in th:
                    x.join()
                dt = time.perf_counter() - t0
                if errors:
                    all_good = False
                    if not isinstance(errors[0], str):
                        raise errors[0]
                if blk >= len(names):  # the first block of each engine warms its lanes and scratch sets
                    rates[name].append(args.threads * len(calls) * n / dt)
            for name in names:
                res[f"{tag}_{name}_steady_items_per_s"] = round(float(np.median(rates[name])))
                res[f"{tag}_{name}_steady_spread"] = [round(min(rates[name])), round(max(rates[name]))]

        # every key hit: key_cache_bench.py's P-256 workload, both caches warmed
        b = corpus.make_batch(P256, n=n, K=1024, seed=911 + P256)
        want = oracle.verify_batch(P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
        calls[:] = [([pinned(b[k])[0] for k in ("r", "s", "qx", "qy", "digest")], want)]
        engines["fill_once"].key_cache_reserve(1024, 0, 0)
        # 1,024 keys fall into the sets unevenly, and the keys past 16 in a set miss in every call (each miss rebuilds a
        # table, which is not what this measures): 4,096 ways (256 sets) hold all of them (the stats show it)
        engines["evicting"].key_cache_reserve_evicting(args.warm_ways, 0, 0)
        for _ in range(args.warmup):
            for name in names:
                call(engines[name], 0)
                all_good &= check(0)
        times = {name: [] for name in names}
        for step in range(2 * args.steps):
            for name in (names if step % 2 == 0 else names[::-1]):
                t0 = time.perf_counter()
                call(engines[name], 0)
                times[name].append(time.perf_counter() - t0)
                all_good &= check(0)
        for name in names:
            res[f"warm1024_{name}_isolated_median_ms"] = round(float(np.median(times[name])) * 1e3, 3)
            res[f"warm1024_{name}_isolated_spread_ms"] = [round(min(times[name]) * 1e3, 3), round(max(times[name]) * 1e3, 3)]
        for name in names[1:]:
            res[f"warm1024_{name}_stats"] = engines[name].key_cache_stats_ex(P256)
        res["value"] = res.get(f"cap{args.caps[0]}_evicting_hit_rate") if args.caps else None
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
