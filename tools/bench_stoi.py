"""Time STOI (sdr_stoi) on the GPU against the fp64 numpy restatement on every host core, and pystoi if installed.

Batches of 4 s @ 8 kHz, 2 sources, with the mixture scored as well (asteroid's stoi and input_stoi), as the
reference's WHAMR! evaluation scores them.  GPU: CUDA events around each call after a warm-up, the median of --reps
calls per batch size; the card's name and power limit are read in the same run.  CPU: tests/stoi_oracle.py's stoi for
the estimate and the mixture of each source over --cpu-items items in a process pool of os.cpu_count() workers, wall
clock.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

import sudo_rm_rf_b200 as P          # noqa: E402
import stoi_oracle                   # noqa: E402

S, FS, T = 2, 8000, 32000


def item(seed):
    rng = np.random.default_rng(seed)
    refs = rng.standard_normal((S, T))
    refs[:, T // 4:T // 3] *= 1e-3
    ests = (np.eye(S) + 0.2 * rng.standard_normal((S, S))) @ refs + 0.1 * rng.standard_normal((S, T))
    mix = refs.sum(0) + 0.05 * rng.standard_normal(T)
    return refs.astype(np.float32), ests.astype(np.float32), mix.astype(np.float32)


def cpu_one(args):
    seed, fn = args
    refs, ests, mix = (a.astype(np.float64) for a in item(seed))
    return [(fn(refs[j], ests[j], FS), fn(refs[j], mix, FS)) for j in range(S)]


def cpu_rate(fn, items):
    workers = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ProcessPoolExecutor(workers) as pool:
        list(pool.map(cpu_one, [(i, fn) for i in range(items)]))
    return workers, round(1000 * (time.perf_counter() - t0) / items, 2)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16,64,256")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-items", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stoi needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = {}
    for B in (int(b) for b in args.batches.split(",")):
        data = [item(b) for b in range(B)]
        r, e, m = (torch.from_numpy(np.stack([d[k] for d in data])).to(dev) for k in range(3))
        times = []
        with torch.no_grad():
            P.stoi(r, e, FS, mixture=m)
            torch.cuda.synchronize()
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                P.stoi(r, e, FS, mixture=m)
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
        med = float(np.median(times))
        gpu[B] = {"median_ms": round(med, 3), "ms_per_item": round(med / B, 4)}
    props = torch.cuda.get_device_properties(dev)
    result = {"metric": "stoi", "S": S, "T": T, "fs": FS, "mixture": True, "gpu": props.name,
              "power_limit": power_limit(), "gpu_batches": gpu}
    workers, ms = cpu_rate(stoi_oracle.stoi, args.cpu_items)
    result.update({"cpu_workers": workers, "cpu_items": args.cpu_items, "oracle_cpu_ms_per_item": ms})
    try:
        import pystoi
        result["pystoi_cpu_ms_per_item"] = cpu_rate(pystoi.stoi, args.cpu_items)[1]
    except ImportError:
        result["pystoi_cpu_ms_per_item"] = None
    print(json.dumps(result))


if __name__ == "__main__":
    main()
