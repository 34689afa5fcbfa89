"""RSA verification through the C ABI (sbv_rsa_hash_verify_batch, or sbv_rsa_pss_hash_verify_batch with --padding pss; with
--keys registered their registered-key forms), per modulus size, against OpenSSL on every core.

    python tools/rsa_bench.py [--steps 20] [--warmup 3] [--sizes 256 384 512]
    python tools/rsa_bench.py --padding pss [--salt-len -1]   # RSA-PSS, MGF1-SHA-256; salt_len as sbv.h (-1: 32 bytes)
    python tools/rsa_bench.py --padding both  # PKCS #1 v1.5 and PSS over the same keys and messages, calls alternated
    python tools/rsa_bench.py --profile      # k_rsa_verify / k_rsa_em / k_rsa_pss / k_sha256 kernel times (torch.profiler)
    python tools/rsa_bench.py --keys both --padding both  # keys per item and registered keys (sbv_rsa_set_keys), alternated

Workload per size: 65,536 items over 1,024 key rows, 256-byte messages, SHA-256, e = 65537.  The keys come from OpenSSL
(--distinct-keys of them per size, default 16, each filling 1,024 / 16 of the key rows), the signatures from OpenSSL too:
1,024 distinct signed messages, tiled to the item count, every seventh one with a flipped message byte.  The RSA path
does no key grouping, so the device work of an item does not depend on how often its key repeats.  Inputs and outputs
live in pinned host memory (sbv_host_alloc); every timed call's verdicts are checked.  Reported per size: the median and
best call time and verifies/s, the wide MADs per verify from the algorithm and their share of sbv_probe_mad_rate, and
OpenSSL verifies/s on all usable cores (each worker parses a key once and reuses it, as a Verifier keeps its clients'
parsed certificates; with 16 distinct keys that reuse is kinder to the CPU's caches than 1,024 would be).  The card's
name, power limit and maximum SM clock are read in the same run.  Prints one JSON line.  With --padding pss the keys are signed with
RSA-PSS (salt of --salt-len bytes, hLen for -1 and auto) and the keys are reported with a _pss suffix; with both, each size
reports both, the two calls alternating step by step, and the ratio pss / pkcs1 of their median times.  With --keys
registered the --distinct-keys keys of each size are registered once (sbv_rsa_set_keys, its time reported as set_keys_ms)
and the calls take a slot per item instead of a modulus and an exponent; those results carry a _reg suffix.  With --keys
both the two forms alternate within each step, for every padding, and each size reports the ratio registered / per-item of
the median call times (reg_over_per_item_time, pss_reg_over_per_item_time).
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def mont_products(k: int, e: int = 65537, registered: bool = False) -> int:
    """Montgomery products of one verify (rsa.cuh): five squarings for R^2 (keys per item only: a registered key's R^2 is
    built by sbv_rsa_set_keys), S -> S*R, one squaring per bit of e below its top bit and one multiplication per further
    set bit, and the product by 1 that leaves EM."""
    return (0 if registered else 5) + 1 + (e.bit_length() - 1) + (bin(e).count("1") - 1) + 1


def mads_per_verify(k: int, e: int = 65537, registered: bool = False) -> int:
    """A product is K rows of a_i * b and q * N over K limbs: 2 K^2 wide MADs (K = k / 4).  The doublings of the R^2 setup
    (no multiplications) are not counted."""
    K = k // 4
    return mont_products(k, e, registered) * 2 * K * K


def _keys(bits, count):
    from cryptography.hazmat.primitives.asymmetric import rsa
    return [rsa.generate_private_key(public_exponent=65537, key_size=bits) for _ in range(count)]


def _padding(pad, salt_len):
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding
    if pad == "pkcs1":
        return padding.PKCS1v15()
    return padding.PSS(mgf=padding.MGF1(hashes.SHA256()), salt_length=salt_len if salt_len > 0 else padding.PSS.DIGEST_LENGTH)


def _sign(args):
    from cryptography.hazmat.primitives import hashes, serialization
    pem, msgs, pad, salt_len = args
    key = serialization.load_pem_private_key(pem, password=None)
    return [key.sign(m, _padding(pad, salt_len), hashes.SHA256()) for m in msgs]


def _cpu_verify(args):
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import rsa
    items, pad, salt_len = args
    cache, good = {}, 0
    t0 = time.perf_counter()
    for n, m, s in items:
        pub = cache.get(n)
        if pub is None:
            pub = cache[n] = rsa.RSAPublicNumbers(65537, n).public_key()
        try:
            pub.verify(s, m, _padding(pad, salt_len), hashes.SHA256())
            good += 1
        except InvalidSignature:
            pass
    return good, time.perf_counter() - t0


def corpus(k, items, key_rows, distinct, msg_len, seed, pool, pads=("pkcs1",), salt_len=-1):
    """The items of one size, signed under each padding of pads (sig_<pad>, cpu_<pad>) over the same keys and messages."""
    from cryptography.hazmat.primitives import serialization
    rng = np.random.default_rng(seed)
    keys = _keys(8 * k, distinct)
    nints = [kk.public_key().public_numbers().n for kk in keys]
    uniq = 1024
    msgs = [rng.integers(0, 256, msg_len, dtype=np.uint8).tobytes() for _ in range(uniq)]
    row = np.arange(uniq) % key_rows  # key row of each distinct message
    owner = row % distinct
    pems = [kk.private_bytes(serialization.Encoding.PEM, serialization.PrivateFormat.PKCS8, serialization.NoEncryption()) for kk in keys]
    sigs = {}
    for pad in pads:
        sigs[pad] = [None] * uniq
        jobs = [(pems[d], [msgs[i] for i in range(uniq) if owner[i] == d], pad, salt_len) for d in range(distinct)]
        for d, out in enumerate(pool.map(_sign, jobs)):
            for i, s in zip([i for i in range(uniq) if owner[i] == d], out):
                sigs[pad][i] = s
    idx = np.arange(items) % uniq
    m = [bytearray(msgs[i]) for i in idx]
    want = np.ones(items, np.uint8)
    for j in range(0, items, 7):
        m[j][j % msg_len] ^= 1
        want[j] = 0
    off = np.arange(items + 1, dtype=np.uint64) * msg_len
    out = dict(msgs=np.frombuffer(b"".join(m), np.uint8), off=off, mod=np.frombuffer(b"".join(nints[owner[i]].to_bytes(k, "big") for i in idx), np.uint8),
               exp=np.full(items, 65537, np.uint32), want=want, slot=owner[idx].astype(np.uint32),
               reg_mod=np.frombuffer(b"".join(n.to_bytes(k, "big") for n in nints), np.uint8))
    for pad in pads:
        out[f"sig_{pad}"] = np.frombuffer(b"".join(sigs[pad][i] for i in idx), np.uint8)
        out[f"cpu_{pad}"] = [(nints[owner[i]], bytes(m[j]), sigs[pad][i]) for j, i in enumerate(idx)]
    return out


def key_form(v):
    """--keys: the key form.  An integer was the key-row count before the key forms existed: point to --key-rows."""
    if v.isdigit():
        raise argparse.ArgumentTypeError(f"--keys {v}: the key-row count is --key-rows; --keys takes per-item, registered or both")
    if v not in ("per-item", "registered", "both"):
        raise argparse.ArgumentTypeError(f"--keys {v}: choose per-item, registered or both")
    return v


def max_sm_clock_mhz():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--items", type=int, default=65536)
    ap.add_argument("--key-rows", type=int, default=1024, help="key rows")
    ap.add_argument("--distinct-keys", type=int, default=16)
    ap.add_argument("--msg-len", type=int, default=256)
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 384, 512])
    ap.add_argument("--cpu-items", type=int, default=16384, help="items of the OpenSSL arm (0: skip it)")
    ap.add_argument("--profile", action="store_true", help="kernel times from torch.profiler instead of timing the calls")
    ap.add_argument("--padding", choices=("pkcs1", "pss", "both"), default="pkcs1")
    ap.add_argument("--salt-len", type=int, default=-1, help="salt_len of the PSS calls (-1: equals hash, 0: auto, > 0: exact)")
    ap.add_argument("--keys", type=key_form, default="per-item", metavar="{per-item,registered,both}",
                    help="keys carried per item, registered once (sbv_rsa_set_keys), or both alternated")
    args = ap.parse_args()
    pads = ("pkcs1", "pss") if args.padding == "both" else (args.padding,)
    forms = ("per-item", "registered") if args.keys == "both" else (args.keys,)

    import torch

    import consensus_b200 as sbv
    from ed25519_quorum_bench import power_limit_w

    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    vp = C.c_void_p
    ncpu = len(os.sched_getaffinity(0))
    res = {"metric": "rsa_verifies_per_s", "unit": "verifies/s", "items": args.items, "key_rows": args.key_rows, "distinct_keys": args.distinct_keys,
           "msg_bytes": args.msg_len, "hash": "SHA-256", "e": 65537, "cpu_cores": ncpu, "padding": args.padding, "keys": args.keys}
    if args.padding != "pkcs1":
        res["salt_len"] = args.salt_len
    all_good = True
    eng = sbv.Engine(n_devices=1)
    res["mad_rate_per_s"] = eng.probe_mad_rate()
    try:
        with ProcessPoolExecutor(ncpu) as pool:
            for k in args.sizes:
                c = corpus(k, args.items, args.key_rows, args.distinct_keys, args.msg_len, seed=k, pool=pool, pads=pads, salt_len=args.salt_len)
                n = args.items
                tag = f"k{k}"
                if "registered" in forms:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    eng.rsa_set_keys(np.full(args.distinct_keys, k, np.uint32), c["reg_mod"], np.full(args.distinct_keys, 65537, np.uint32))
                    res[f"{tag}_set_keys_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
                arrays = [c["msgs"], c["off"], c["mod"], c["exp"], np.zeros(n, np.uint8), c["slot"]] + [c[f"sig_{p}"] for p in pads]
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
                    ok = views[4]
                    sigbuf = dict(zip(pads, bufs[6:]))
                    runs = [(pad, form) for pad in pads for form in forms]  # alternated within each step

                    def call(pad, form):
                        if form == "registered" and pad == "pss":
                            eng.rsa_pss_hash_verify_registered_ptr(k, sbv.SHA256, args.salt_len, n, bufs[0], bufs[1], bufs[5], sigbuf[pad], 0, bufs[4])
                        elif form == "registered":
                            eng.rsa_hash_verify_registered_ptr(k, sbv.SHA256, n, bufs[0], bufs[1], bufs[5], sigbuf[pad], 0, bufs[4])
                        elif pad == "pss":
                            eng.rsa_pss_hash_verify_batch_ptr(k, sbv.SHA256, args.salt_len, n, bufs[0], bufs[1], sigbuf[pad], bufs[2], bufs[3], 0, bufs[4])
                        else:
                            eng.rsa_hash_verify_batch_ptr(k, sbv.SHA256, n, bufs[0], bufs[1], sigbuf[pad], bufs[2], bufs[3], 0, bufs[4])

                    def check():
                        good = bool(np.array_equal(ok, c["want"]))
                        ok[:] = 2
                        return good

                    res[f"{tag}_mont_products"] = mont_products(k)
                    res[f"{tag}_wide_mads_per_verify"] = mads_per_verify(k)
                    if "registered" in forms:
                        res[f"{tag}_reg_mont_products"] = mont_products(k, registered=True)
                    if args.profile:
                        from torch.profiler import ProfilerActivity, profile
                        for pad, form in runs:
                            call(pad, form)
                            all_good &= check()
                        torch.cuda.synchronize()
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            for _ in range(5):
                                for pad, form in runs:
                                    call(pad, form)
                                    all_good &= check()
                            torch.cuda.synchronize()
                        for ev in prof.key_averages():
                            for name in ("k_rsa_verify", "k_rsa_em", "k_rsa_pss", "k_rsa_verify_reg", "k_rsa_em_reg", "k_rsa_pss_reg", "k_sha256"):
                                if re.search(r"\b" + name + r"\b", ev.key):
                                    t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per launch
                                    res[f"{tag}_{name}_us"] = round(float(t), 1)
                                    res[f"{tag}_{name}_launches"] = int(ev.count)
                        for name, reg in (("k_rsa_verify", False), ("k_rsa_verify_reg", True)):
                            if f"{tag}_{name}_us" in res:
                                kt = res[f"{tag}_{name}_us"] * 1e-6
                                sfx = "_reg" if reg else ""
                                res[f"{tag}{sfx}_kernel_verifies_per_s"] = round(n / kt)
                                res[f"{tag}{sfx}_kernel_mad_share"] = round(n * mads_per_verify(k, registered=reg) / kt / res["mad_rate_per_s"], 3)
                    else:
                        for _ in range(args.warmup):
                            for pad, form in runs:
                                call(pad, form)
                                all_good &= check()
                        times = {r: [] for r in runs}
                        for _ in range(args.steps):
                            for r in runs:  # alternated: every padding and key form sees the same state of the card
                                t0 = time.perf_counter()
                                call(*r)
                                times[r].append(time.perf_counter() - t0)
                                all_good &= check()
                        for pad, form in runs:
                            sfx = ("" if pad == "pkcs1" else "_pss") + ("_reg" if form == "registered" else "")
                            med = float(np.median(times[(pad, form)]))
                            res[f"{tag}{sfx}_median_ms"] = round(med * 1e3, 3)
                            res[f"{tag}{sfx}_best_ms"] = round(min(times[(pad, form)]) * 1e3, 3)
                            res[f"{tag}{sfx}_verifies_per_s"] = round(n / med)
                            res[f"{tag}{sfx}_call_mad_share"] = round(n * mads_per_verify(k, registered=form == "registered") / med / res["mad_rate_per_s"], 3)
                            if args.cpu_items and form == forms[0]:  # OpenSSL once per padding
                                sfx = "" if pad == "pkcs1" else "_pss"
                                items = c[f"cpu_{pad}"][:args.cpu_items]
                                parts = [(items[i::ncpu], pad, args.salt_len) for i in range(ncpu)]
                                t0 = time.perf_counter()
                                out = list(pool.map(_cpu_verify, parts))
                                wall = time.perf_counter() - t0
                                good = sum(o[0] for o in out)
                                all_good &= good == int(c["want"][:len(items)].sum())
                                res[f"{tag}{sfx}_openssl_verifies_per_s"] = round(len(items) / wall)
                        r0 = "_reg" if forms == ("registered",) else ""
                        if len(pads) == 2:
                            res[f"{tag}{r0}_pss_over_pkcs1_time"] = round(res[f"{tag}_pss{r0}_median_ms"] / res[f"{tag}{r0}_median_ms"], 4)
                        if len(forms) == 2:
                            for pad in pads:
                                p = "" if pad == "pkcs1" else "pss_"
                                pp = "" if pad == "pkcs1" else "_pss"
                                res[f"{tag}_{p}reg_over_per_item_time"] = round(res[f"{tag}{pp}_reg_median_ms"] / res[f"{tag}{pp}_median_ms"], 4)
                finally:
                    for p in bufs:
                        lib.sbv_host_free(C.c_void_p(p))
    finally:
        eng.close()
    first = f"k{args.sizes[0]}" + ("_pss" if args.padding == "pss" else "") + ("_reg" if args.keys == "registered" else "") + "_verifies_per_s"
    if not args.profile and first in res:
        res["value"] = res[first]
    res["outputs_match_expected"] = bool(all_good)
    res["device"] = torch.cuda.get_device_properties(0).name
    res["power_limit_w"] = power_limit_w()
    res["max_sm_clock_mhz"] = max_sm_clock_mhz()
    print(json.dumps(res))
    return 0 if all_good else 1


if __name__ == "__main__":
    sys.exit(main())
