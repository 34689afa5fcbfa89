"""Per-kernel device times of the grouped P-256 step under torch.profiler: the benchmark's batch (65,536 signatures over
1,024 keys, seed 1) through sbv_verify_batch on device buffers, one step at a time (each step ends in a synchronise,
so the kernels of a step do not overlap those of the next).  Nothing else is timed: throughput comes from bench.py.

    python tools/grouped_kernel_profile.py [--steps 20] [--warmup 5]

Prints one JSON line: the average µs per call of every sbv kernel the step launches (k_gpart, k_verify_comb, the table
kernels, ...), the card's name and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import consensus_b200 as sbv
    import oracle
    from oracle import corpus

    n = 65536
    b = corpus.make_batch(oracle.P256, n=n, K=1024, seed=1)
    dev = torch.device("cuda", 0)
    d = {k: torch.from_numpy(np.ascontiguousarray(b[k])).to(dev) for k in ("r", "s", "qx", "qy", "digest")}
    ok = torch.zeros(n, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    with sbv.Engine(devices=[0]) as eng:
        def step():
            eng.verify_batch_device(sbv.P256, n, d["r"].data_ptr(), d["s"].data_ptr(), d["qx"].data_ptr(), d["qy"].data_ptr(),
                                    d["digest"].data_ptr(), 32, ok.data_ptr(), stream=stream)
            torch.cuda.synchronize()
        for _ in range(args.warmup):
            step()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
        kern = {}
        for ev in prof.key_averages():
            m = re.search(r"\b(k_\w+)[<(]", ev.key)
            if m:
                name = m.group(1)
                while name in kern:  # two instantiations of one template
                    name += "'"
                t = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)  # average µs per call
                kern[name] = {"us_per_call": round(float(t), 1), "calls": int(ev.count)}
    print(json.dumps({"workload": "grouped P-256 step, 65,536 signatures over 1,024 keys (bench.py's batch)", "steps": args.steps,
                      "kernels": kern, "card": card()}))


if __name__ == "__main__":
    main()
