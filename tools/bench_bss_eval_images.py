"""Time BSS-eval of source images (sdr_bss_eval_images, sdr_bss_eval_images_framewise) on the GPU, and the fp64 numpy
restatement per item.

Cases: two stereo sources (S = 2, C = 2), F = 512, 4 s at 8 kHz at batch 1 and 256; one hour of the same at 8 kHz in
30 s windows every 15 s (239 windows).  The signals are held as a stereo model returns them, [B, S, C, T], and passed
as the [B, S, T, C] views bss_eval_images reads without a copy.  GPU: CUDA events around each call after a warm-up,
the median of --reps calls.  CPU: tests/bss_images_oracle.py on --cpu-items items of 4 s, one spawned process per host
core, all started before the clock; wall clock, reported per item.  The card's name and power limit are read in the
same run; without a CUDA device every GPU number is "not measured".  Prints one JSON line per case."""
import argparse
import json
import multiprocessing as mp
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

import sudo_rm_rf_b200 as P                    # noqa: E402
from bss_images_oracle import bss_eval_images  # noqa: E402

FS, S, C, F = 8000, 2, 2, 512
W, H = 30 * FS, 15 * FS
CASES = {"4s_8k_b1": (1, 4, False), "4s_8k_b256": (256, 4, False), "1h_8k_framewise": (1, 3600, True)}
NOT_MEASURED = "not measured"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def ready(_):
    time.sleep(0.5)


def cpu_item(seed):
    rng = np.random.default_rng(seed)
    T = 4 * FS
    refs = rng.standard_normal((S, T, C)).astype(np.float32).astype(np.float64)
    ests = refs[::-1] + 0.1 * rng.standard_normal((S, T, C))
    return bss_eval_images(refs, ests.astype(np.float32).astype(np.float64), True, F)


def gpu_case(B, seconds, windows, reps):
    dev = torch.device("cuda:0")
    T = seconds * FS
    g = torch.Generator(dev).manual_seed(B * T)
    refs = torch.randn(B, S, C, T, device=dev, generator=g)
    ests = 0.3 * torch.randn(B, S, C, T, device=dev, generator=g) + refs.flip(1)
    refs, ests = refs.transpose(-1, -2), ests.transpose(-1, -2)

    def call():
        if windows:
            return P.bss_eval_images_framewise(refs, ests, W, H, False, F)
        return P.bss_eval_images(refs, ests, True, F)
    times = []
    with torch.no_grad():
        call()
        torch.cuda.synchronize()
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
    n = B * (P.bss_eval.window_count(T, W, H) if windows else 1)
    med = float(np.median(times))
    return {"items": n, "median_ms": round(med, 3), "ms_per_item": round(med / n, 4),
            "spread_ms": [round(min(times), 3), round(max(times), 3)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cpu-items", type=int, default=8, help="0: skip the host restatement")
    args = ap.parse_args()
    gpu = torch.cuda.is_available()
    info = {"gpu": torch.cuda.get_device_properties(0).name if gpu else NOT_MEASURED,
            "card": (card() or NOT_MEASURED) if gpu else NOT_MEASURED}
    for name, (B, seconds, windows) in CASES.items():
        res = gpu_case(B, seconds, windows, args.reps) if gpu else {"median_ms": NOT_MEASURED}
        print(json.dumps({"metric": "bss_eval_images" + ("_framewise" if windows else ""), "case": name, "S": S,
                          "C": C, "F": F, "B": B, "seconds": seconds, **({"window": W, "hop": H} if windows else {}),
                          **info, **res}), flush=True)
    if args.cpu_items < 1:
        return
    workers = os.cpu_count() or 1
    with ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as pool:   # the parent holds CUDA
        list(pool.map(ready, range(workers)))       # every worker started (and its imports done) before the clock
        t0 = time.perf_counter()
        list(pool.map(cpu_item, range(args.cpu_items)))
        cpu_s = time.perf_counter() - t0
    print(json.dumps({"metric": "bss_eval_images", "case": "fp64_numpy_restatement", "S": S, "C": C, "F": F,
                      "seconds": 4, "cpu_workers": workers, "cpu_items": args.cpu_items,
                      "cpu_ms_per_item": round(1000 * cpu_s / args.cpu_items, 1)}))


if __name__ == "__main__":
    main()
