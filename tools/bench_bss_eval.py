"""Time BSS-eval (sdr_bss_eval) on the GPU against the fp64 numpy restatement on every host core.

Batches of 4 s @ 8 kHz, 2 sources, 512-tap filters, as the reference's WHAMR! evaluation scores them.  GPU: CUDA
events around each call after a warm-up, the median of --reps calls per batch size.  CPU: tests/bss_oracle.py's
bss_eval over --cpu-items items in a process pool of os.cpu_count() workers, wall clock.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

import sudo_rm_rf_b200 as P          # noqa: E402
from bss_oracle import bss_eval      # noqa: E402

S, T, F = 2, 32000, 512


def item(seed):
    rng = np.random.default_rng(seed)
    refs = rng.standard_normal((S, T))
    ests = (np.eye(S) + 0.2 * rng.standard_normal((S, S))) @ refs + 0.1 * rng.standard_normal((S, T))
    return refs.astype(np.float32), ests.astype(np.float32)


def cpu_one(seed):
    refs, ests = item(seed)
    return bss_eval(refs.astype(np.float64), ests.astype(np.float64), True, F)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16,64,256")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-items", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bss_eval needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = {}
    for B in (int(b) for b in args.batches.split(",")):
        data = [item(b) for b in range(B)]
        r = torch.from_numpy(np.stack([d[0] for d in data])).to(dev)
        e = torch.from_numpy(np.stack([d[1] for d in data])).to(dev)
        times = []
        with torch.no_grad():
            P.bss_eval_sources(r, e)
            torch.cuda.synchronize()
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                P.bss_eval_sources(r, e)
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
        med = float(np.median(times))
        gpu[B] = {"median_ms": round(med, 3), "ms_per_item": round(med / B, 4)}
    workers = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ProcessPoolExecutor(workers) as pool:
        list(pool.map(cpu_one, range(args.cpu_items)))
    cpu_s = time.perf_counter() - t0
    props = torch.cuda.get_device_properties(dev)
    print(json.dumps({"metric": "bss_eval_sources", "S": S, "T": T, "F": F, "gpu": props.name, "gpu_batches": gpu,
                      "cpu_workers": workers, "cpu_items": args.cpu_items,
                      "cpu_ms_per_item": round(1000 * cpu_s / args.cpu_items, 2)}))


if __name__ == "__main__":
    main()
