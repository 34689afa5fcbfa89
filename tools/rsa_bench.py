"""RSA PKCS #1 v1.5 verification through the C ABI (sbv_rsa_hash_verify_batch), per modulus size, against OpenSSL on every
core.

    python tools/rsa_bench.py [--steps 20] [--warmup 3] [--sizes 256 384 512]
    python tools/rsa_bench.py --profile      # k_rsa_verify / k_sha256 kernel times (torch.profiler), nothing timed

Workload per size: 65,536 items over 1,024 key rows, 256-byte messages, SHA-256, e = 65537.  The keys come from OpenSSL
(--distinct-keys of them per size, default 16, each filling 1,024 / 16 of the key rows), the signatures from OpenSSL too:
1,024 distinct signed messages, tiled to the item count, every seventh one with a flipped message byte.  The RSA path
does no key grouping, so the device work of an item does not depend on how often its key repeats.  Inputs and outputs
live in pinned host memory (sbv_host_alloc); every timed call's verdicts are checked.  Reported per size: the median and
best call time and verifies/s, the wide MADs per verify from the algorithm and their share of sbv_probe_mad_rate, and
OpenSSL verifies/s on all usable cores (each worker parses a key once and reuses it, as a Verifier keeps its clients'
parsed certificates; with 16 distinct keys that reuse is kinder to the CPU's caches than 1,024 would be).  The card's
name and power limit are read in the same run.  Prints one JSON line.
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
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def mont_products(k: int, e: int = 65537) -> int:
    """Montgomery products of one verify (rsa.cuh): five squarings for R^2, S -> S*R, one squaring per bit of e below its
    top bit and one multiplication per further set bit, and the product by 1 that leaves EM."""
    return 5 + 1 + (e.bit_length() - 1) + (bin(e).count("1") - 1) + 1


def mads_per_verify(k: int, e: int = 65537) -> int:
    """A product is K rows of a_i * b and q * N over K limbs: 2 K^2 wide MADs (K = k / 4).  The doublings of the R^2 setup
    (no multiplications) are not counted."""
    K = k // 4
    return mont_products(k, e) * 2 * K * K


def _keys(bits, count):
    from cryptography.hazmat.primitives.asymmetric import rsa
    return [rsa.generate_private_key(public_exponent=65537, key_size=bits) for _ in range(count)]


def _sign(args):
    from cryptography.hazmat.primitives import hashes, serialization
    from cryptography.hazmat.primitives.asymmetric import padding
    pem, msgs = args
    key = serialization.load_pem_private_key(pem, password=None)
    return [key.sign(m, padding.PKCS1v15(), hashes.SHA256()) for m in msgs]


def _cpu_verify(args):
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding, rsa
    items = args
    cache, good = {}, 0
    t0 = time.perf_counter()
    for n, m, s in items:
        pub = cache.get(n)
        if pub is None:
            pub = cache[n] = rsa.RSAPublicNumbers(65537, n).public_key()
        try:
            pub.verify(s, m, padding.PKCS1v15(), hashes.SHA256())
            good += 1
        except InvalidSignature:
            pass
    return good, time.perf_counter() - t0


def corpus(k, items, key_rows, distinct, msg_len, seed, pool):
    from cryptography.hazmat.primitives import serialization
    rng = np.random.default_rng(seed)
    keys = _keys(8 * k, distinct)
    nints = [kk.public_key().public_numbers().n for kk in keys]
    uniq = 1024
    msgs = [rng.integers(0, 256, msg_len, dtype=np.uint8).tobytes() for _ in range(uniq)]
    row = np.arange(uniq) % key_rows  # key row of each distinct message
    owner = row % distinct
    pems = [kk.private_bytes(serialization.Encoding.PEM, serialization.PrivateFormat.PKCS8, serialization.NoEncryption()) for kk in keys]
    sigs = [None] * uniq
    jobs = [(pems[d], [msgs[i] for i in range(uniq) if owner[i] == d]) for d in range(distinct)]
    for d, out in enumerate(pool.map(_sign, jobs)):
        for i, s in zip([i for i in range(uniq) if owner[i] == d], out):
            sigs[i] = s
    idx = np.arange(items) % uniq
    m = [bytearray(msgs[i]) for i in idx]
    want = np.ones(items, np.uint8)
    for j in range(0, items, 7):
        m[j][j % msg_len] ^= 1
        want[j] = 0
    off = np.arange(items + 1, dtype=np.uint64) * msg_len
    return dict(msgs=np.frombuffer(b"".join(m), np.uint8), off=off, sig=np.frombuffer(b"".join(sigs[i] for i in idx), np.uint8),
                mod=np.frombuffer(b"".join(nints[owner[i]].to_bytes(k, "big") for i in idx), np.uint8),
                exp=np.full(items, 65537, np.uint32), want=want, cpu=[(nints[owner[i]], bytes(m[j]), sigs[i]) for j, i in enumerate(idx)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--items", type=int, default=65536)
    ap.add_argument("--keys", type=int, default=1024, help="key rows")
    ap.add_argument("--distinct-keys", type=int, default=16)
    ap.add_argument("--msg-len", type=int, default=256)
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 384, 512])
    ap.add_argument("--cpu-items", type=int, default=16384, help="items of the OpenSSL arm (0: skip it)")
    ap.add_argument("--profile", action="store_true", help="kernel times from torch.profiler instead of timing the calls")
    args = ap.parse_args()

    import torch

    import consensus_b200 as sbv
    from ed25519_quorum_bench import power_limit_w

    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    vp = C.c_void_p
    ncpu = len(os.sched_getaffinity(0))
    res = {"metric": "rsa_verifies_per_s", "unit": "verifies/s", "items": args.items, "key_rows": args.keys, "distinct_keys": args.distinct_keys,
           "msg_bytes": args.msg_len, "hash": "SHA-256", "e": 65537, "cpu_cores": ncpu}
    all_good = True
    eng = sbv.Engine(n_devices=1)
    res["mad_rate_per_s"] = eng.probe_mad_rate()
    try:
        with ProcessPoolExecutor(ncpu) as pool:
            for k in args.sizes:
                c = corpus(k, args.items, args.keys, args.distinct_keys, args.msg_len, seed=k, pool=pool)
                n = args.items
                arrays = [c["msgs"], c["off"], c["sig"], c["mod"], c["exp"], np.zeros(n, np.uint8)]
                bufs = []
                try:
                    views = []
                    for a in arrays:
                        p = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
                        assert p
                        bufs.append(p)
                        v = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(p))
                        v[:] = a.view(np.uint8).reshape(-1)
                        views.append(v)
                    ok = views[5]

                    def call():
                        eng.rsa_hash_verify_batch_ptr(k, sbv.SHA256, n, *bufs[:5], 0, bufs[5])

                    def check():
                        good = bool(np.array_equal(ok, c["want"]))
                        ok[:] = 2
                        return good

                    tag = f"k{k}"
                    res[f"{tag}_mont_products"] = mont_products(k)
                    res[f"{tag}_wide_mads_per_verify"] = mads_per_verify(k)
                    if args.profile:
                        from torch.profiler import ProfilerActivity, profile
                        call()
                        all_good &= check()
                        torch.cuda.synchronize()
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            for _ in range(5):
                                call()
                                all_good &= check()
                            torch.cuda.synchronize()
                        for ev in prof.key_averages():
                            for name in ("k_rsa_verify", "k_sha256"):
                                if re.search(r"\b" + name + r"\b", ev.key):
                                    t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per launch
                                    res[f"{tag}_{name}_us"] = round(float(t), 1)
                                    res[f"{tag}_{name}_launches"] = int(ev.count)
                        if f"{tag}_k_rsa_verify_us" in res:
                            kt = res[f"{tag}_k_rsa_verify_us"] * 1e-6
                            res[f"{tag}_kernel_verifies_per_s"] = round(n / kt)
                            res[f"{tag}_kernel_mad_share"] = round(n * mads_per_verify(k) / kt / res["mad_rate_per_s"], 3)
                    else:
                        for _ in range(args.warmup):
                            call()
                            all_good &= check()
                        times = []
                        for _ in range(args.steps):
                            t0 = time.perf_counter()
                            call()
                            times.append(time.perf_counter() - t0)
                            all_good &= check()
                        med = float(np.median(times))
                        res[f"{tag}_median_ms"] = round(med * 1e3, 3)
                        res[f"{tag}_best_ms"] = round(min(times) * 1e3, 3)
                        res[f"{tag}_verifies_per_s"] = round(n / med)
                        res[f"{tag}_call_mad_share"] = round(n * mads_per_verify(k) / med / res["mad_rate_per_s"], 3)
                        if args.cpu_items:
                            items = c["cpu"][:args.cpu_items]
                            parts = [items[i::ncpu] for i in range(ncpu)]
                            t0 = time.perf_counter()
                            out = list(pool.map(_cpu_verify, parts))
                            wall = time.perf_counter() - t0
                            good = sum(o[0] for o in out)
                            all_good &= good == int(c["want"][:len(items)].sum())
                            res[f"{tag}_openssl_verifies_per_s"] = round(len(items) / wall)
                finally:
                    for p in bufs:
                        lib.sbv_host_free(C.c_void_p(p))
    finally:
        eng.close()
    if not args.profile and f"k{args.sizes[0]}_verifies_per_s" in res:
        res["value"] = res[f"k{args.sizes[0]}_verifies_per_s"]
    res["outputs_match_expected"] = bool(all_good)
    res["device"] = torch.cuda.get_device_properties(0).name
    res["power_limit_w"] = power_limit_w()
    print(json.dumps(res))
    return 0 if all_good else 1


if __name__ == "__main__":
    sys.exit(main())
