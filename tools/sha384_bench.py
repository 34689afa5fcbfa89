"""SHA-384 against SHA-256 on the fused ECDSA calls, through the C ABI, alternated call by call in one run.

    python tools/sha384_bench.py [--steps 20] [--warmup 5]
    python tools/sha384_bench.py --profile      # k_sha384 against k_sha256 kernel time (torch.profiler), nothing timed

Corpus: 65,536 P-384 items, 256-byte messages, 1,024 keys, seeded.  Every item is signed twice with the same nonce, once
over SHA-384(M) and once over SHA-256(M), so that both arms verify the same messages and accept the same items.
  keys per item   sbv_hash384_verify_batch      against sbv_hash_verify_batch
  registered      sbv_hash384_verify_registered against sbv_hash_verify_registered (the 1,024 keys registered)
Inputs and outputs live in pinned host memory (sbv_host_alloc).  Every timed call's verdicts are checked against
OpenSSL.  The card's name and power limit are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

P384 = 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--items", type=int, default=65536)
    ap.add_argument("--keys", type=int, default=1024)
    ap.add_argument("--profile", action="store_true", help="profile the two hash kernels instead of timing the calls")
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import oracle
    from ed25519_quorum_bench import power_limit_w
    from oracle import corpus

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

    n, K = args.items, args.keys
    d, kxy = corpus.make_keys(P384, K, seed=384)
    msgs, off = corpus.make_requests(n, seed=385, fixed_len=256)
    key_idx = (np.random.default_rng(386).integers(0, K, n)).astype(np.uint32)
    k = np.random.default_rng(387).integers(0, 256, (n, 48), dtype=np.uint8)
    m = [msgs[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]
    d384 = np.frombuffer(b"".join(hashlib.sha384(x).digest() for x in m), np.uint8).reshape(n, 48)
    d256 = np.frombuffer(b"".join(hashlib.sha256(x).digest() for x in m), np.uint8).reshape(n, 32)
    qx, qy = kxy[key_idx, :48].copy(), kxy[key_idx, 48:].copy()
    sig = {h: oracle.sign_batch(P384, d, key_idx, dig, k) for h, dig in (("sha384", d384), ("sha256", d256))}
    for i in range(0, n, 16):  # 1/16 of the items reject in both arms
        for h in sig:
            sig[h][1][i, 47] ^= 1
    want = oracle.verify_batch(P384, sig["sha384"][0], sig["sha384"][1], qx, qy, d384)
    assert np.array_equal(want, oracle.verify_batch(P384, sig["sha256"][0], sig["sha256"][1], qx, qy, d256))
    eng.set_keys(np.full(K, P384, np.uint8), kxy.reshape(K, 2, 48))

    pm, po, pqx, pqy = pinned(msgs)[0], pinned(off)[0], pinned(qx)[0], pinned(qy)[0]
    pslot = pinned(key_idx)[0]
    prs = {h: (pinned(r)[0], pinned(s)[0]) for h, (r, s) in sig.items()}
    ok_p, ok = pinned(np.zeros(n, np.uint8))
    dig_p, _ = pinned(np.zeros(n * 48, np.uint8))
    N = C.c_size_t(n)
    c = C.c_uint8(P384)
    fn = {"sha384": (lib.sbv_hash384_verify_batch, lib.sbv_hash384_verify_registered, lib.sbv_sha384_batch),
          "sha256": (lib.sbv_hash_verify_batch, lib.sbv_hash_verify_registered, lib.sbv_sha256_batch)}

    def batch(h):
        r, s = prs[h]
        eng._check(fn[h][0](eng._h, c, N, vp(pm), vp(po), vp(r), vp(s), vp(pqx), vp(pqy), None, vp(ok_p)), h + " verify_batch")

    def registered(h):
        r, s = prs[h]
        eng._check(fn[h][1](eng._h, c, N, vp(pm), vp(po), vp(pslot), vp(r), vp(s), vp(ok_p)), h + " verify_registered")

    def check():
        good = bool(np.array_equal(ok, want))
        ok[:] = 2
        return good

    res = {"metric": "sha384_verify_items_per_s", "unit": "items/s", "items": n, "keys": K, "msg_bytes": 256}
    all_good = True
    try:
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            for h in fn:
                eng._check(fn[h][2](eng._h, N, vp(pm), vp(po), vp(dig_p)), h)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    for h in fn:
                        eng._check(fn[h][2](eng._h, N, vp(pm), vp(po), vp(dig_p)), h)
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                for name in ("k_sha384", "k_sha256"):
                    if re.search(r"\b" + name + r"\b", ev.key):
                        t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per launch
                        res[f"{name}_us"] = round(float(t), 1)
                        res[f"{name}_launches"] = int(ev.count)
            if "k_sha384_us" in res and "k_sha256_us" in res:
                res["k_sha384_over_k_sha256"] = round(res["k_sha384_us"] / res["k_sha256_us"], 2)
        else:
            res.update(steps=args.steps, warmup=args.warmup)
            for tag, call in (("batch", batch), ("registered", registered)):
                for _ in range(args.warmup):
                    for h in fn:
                        call(h)
                times = {h: [] for h in fn}
                names = list(fn)
                for step in range(args.steps):
                    for h in (names if step % 2 == 0 else names[::-1]):
                        t0 = time.perf_counter()
                        call(h)
                        times[h].append(time.perf_counter() - t0)
                        all_good &= check()
                for h in fn:
                    res[f"{tag}_{h}_median_ms"] = round(float(np.median(times[h])) * 1e3, 3)
                    res[f"{tag}_{h}_best_ms"] = round(min(times[h]) * 1e3, 3)
                res[f"{tag}_sha384_over_sha256"] = round(res[f"{tag}_sha384_median_ms"] / res[f"{tag}_sha256_median_ms"], 3)
            res["value"] = n / (res["batch_sha384_median_ms"] * 1e-3)
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
