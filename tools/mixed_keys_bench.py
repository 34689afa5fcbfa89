"""Mixed ECDSA / Ed25519 batches with the key of each item through the C ABI: one sbv_mixed_verify_batch call against the
per-family composition, alternated call by call in one run.

    python tools/mixed_keys_bench.py [--steps 20] [--warmup 5]
    python tools/mixed_keys_bench.py --profile      # kernel times of one 65,536-item call (torch.profiler), nothing timed

Shapes: flush-sized batches of 16, 256 and 2,048 items, half P-256 and half Ed25519, interleaved, over 8 keys per scheme
(a Verifier's flush of client requests); and 65,536 items, half P-256 and half Ed25519, interleaved, over 1,024 keys per
scheme with 256-byte messages.
  one_call     sbv_mixed_verify_batch
  composition  sbv_hash_verify_batch for the P-256 items, sbv_ed25519_verify_batch for the Ed25519 items, on per-family
               arrays prepared beforehand (their marshalling is not timed), and the host scatter of their verdicts
Inputs and outputs live in pinned host memory (sbv_host_alloc).  Every timed call's outputs are checked against
OpenSSL.  The card's name and power limit are read in the same run.  Prints one JSON line.
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

KERNELS = ("k_mix_count", "k_mix_scan", "k_mix_split", "k_mix_compact", "k_mix_ok", "k_sha256", "k_ed_sha512", "k_ed_verify", "k_ed_verify_comb",
           "k_kg_insert", "k_kg_assign", "k_kg_route")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--large", type=int, default=65536)
    ap.add_argument("--profile", action="store_true", help="profile the kernels of one large call instead of timing")
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    import mixed_keys_cases as mk
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

    def shape(size, keys, lens, seed):
        """A corpus of `size` items, P-256 and Ed25519 interleaved, its pinned call arrays and its composition arms."""
        pools = mk.key_pools(k256=keys, k384=0, k_ed=keys, seed=seed)
        tag = np.tile(np.array([mk.P256, mk.ED], np.uint8), size // 2)
        cp = mk.make_corpus(tag, pools, seed=seed, lens=lens(size), corrupt=1 / 16)
        want = mk.expected_ok(cp)
        p = {k: pinned(cp[k])[0] for k in ("scheme", "msgs", "off", "sig96", "key96")}
        ok_p, ok = pinned(np.zeros(size, np.uint8))
        fams = []
        for c in (mk.P256, mk.ED):
            idx, m, o, sig, key = mk.family_arrays(cp, c)
            fams.append((c, idx, pinned(m)[0], pinned(o)[0], [pinned(a)[0] for a in sig], [pinned(a)[0] for a in key], pinned(np.zeros(idx.size, np.uint8))))

        def one_call():
            eng.mixed_verify_batch_ptr(size, p["scheme"], p["msgs"], p["off"], p["sig96"], p["key96"], ok_p)

        def composition():
            for c, idx, m, o, sig, key, (okp, okv) in fams:
                k = C.c_size_t(idx.size)
                if c == mk.ED:
                    eng._check(lib.sbv_ed25519_verify_batch(eng._h, k, vp(m), vp(o), vp(sig[0]), vp(key[0]), vp(okp)), "sbv_ed25519_verify_batch")
                else:
                    eng._check(lib.sbv_hash_verify_batch(eng._h, C.c_uint8(c), k, vp(m), vp(o), vp(sig[0]), vp(sig[1]), vp(key[0]), vp(key[1]), None,
                                                         vp(okp)), "sbv_hash_verify_batch")
                ok[idx] = okv

        def check():
            good = bool(np.array_equal(ok, want))
            ok[:] = 2
            return good

        return {"one_call": one_call, "composition": composition}, check

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

    big_lens = lambda n: np.full(n, 256)
    res = {"metric": "mixed_keys_items_per_s", "unit": "items/s"}
    all_good = True
    try:
        if args.profile:
            arms, check = shape(args.large, 1024, big_lens, 2029)
            for _ in range(3):
                arms["one_call"]()
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arms["one_call"]()
                torch.cuda.synchronize()
            all_good = check()
            for ev in prof.key_averages():
                for name in KERNELS:
                    if re.search(r"\b" + name + r"\b", ev.key):
                        t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per launch
                        res[f"{name}_us"] = round(float(t), 1)
                        res[f"{name}_launches"] = int(ev.count)
            res["profile_items"] = args.large
        else:
            res.update(steps=args.steps, warmup=args.warmup)
            for size, keys, lens, seed, tag in ((16, 8, None, 16, "b16"), (256, 8, None, 256, "b256"), (2048, 8, None, 2048, "b2048"),
                                                (args.large, 1024, big_lens, 2028, "large")):
                lens_fn = lens or (lambda n, s=seed: np.random.default_rng(s).integers(64, 321, n))
                arms, check = shape(size, keys, lens_fn, seed)
                times, good = alternate(arms, check)
                all_good &= good
                for a in arms:
                    res[f"{tag}_{a}_median_us"] = round(float(np.median(times[a])) * 1e6, 1)
                    res[f"{tag}_{a}_best_us"] = round(min(times[a]) * 1e6, 1)
                res[f"{tag}_outputs_match_oracle"] = good
            res["large_items"] = args.large
            res["value"] = args.large / (res["large_one_call_median_us"] * 1e-6)
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
