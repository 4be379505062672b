"""Time BSS-eval v4 (sdr_bss_eval_v4, museval's v4) on the GPU, and the fp64 numpy restatement per track.

Cases, all with one-second windows and hops and F = 512 (museval's defaults), 4-minute tracks: four mono stems
(S = 4, C = 1) at 44.1 kHz and at 8 kHz, batch 1 and batch 8; stereo vocals and accompaniment (S = 2, C = 2) at
44.1 kHz, batch 1.  GPU: CUDA events around each call after a warm-up, the median of --reps calls; and, in a separate
profiled call, the correlation pass's kernel time (bss_corr_kernel and bss_fold_kernel), reported with the achieved
fp64 FMA rate against its arithmetic count, R (2 R) F n FMAs per track.  CPU: tests/bss_v4_oracle.py on --cpu-tracks
four-stem tracks of --cpu-seconds at 44.1 kHz, one spawned process per host core, all started before the clock; wall
clock, reported per track and scaled to 4 minutes.  The card's name and power limit are read in the same run; without
a CUDA device every GPU number is "not measured".  Prints one JSON line per case."""
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
from bss_v4_oracle import bss_eval_v4          # noqa: E402

F, SECONDS = 512, 240
CASES = {"4mono_44k_b1": (4, 1, 44100, 1), "4mono_44k_b8": (4, 1, 44100, 8), "4mono_8k_b1": (4, 1, 8000, 1),
         "4mono_8k_b8": (4, 1, 8000, 8), "stereo_voc_acc_44k_b1": (2, 2, 44100, 1)}
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


def cpu_track(args):
    seed, seconds = args
    rng = np.random.default_rng(seed)
    T = seconds * 44100
    refs = rng.standard_normal((4, T, 1)).astype(np.float32).astype(np.float64)
    ests = refs + 0.3 * rng.standard_normal((4, T, 1))
    return bss_eval_v4(refs, ests.astype(np.float32).astype(np.float64), 44100, 44100, False, F)


def corr_kernel_ms(call):
    """Device time of the correlation pass's kernels in one profiled call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages()
             if "bss_corr_kernel" in e.key or "bss_fold_kernel" in e.key)
    return us / 1000.0


def gpu_case(S, C, fs, B, reps):
    dev = torch.device("cuda:0")
    T = SECONDS * fs
    g = torch.Generator(dev).manual_seed(S * C * fs + B)
    refs = torch.randn(B, S, C, T, device=dev, generator=g)
    ests = 0.3 * torch.randn(B, S, C, T, device=dev, generator=g) + refs
    refs, ests = refs.transpose(-1, -2), ests.transpose(-1, -2)

    def call():
        return P.bss_eval_v4(refs, ests, fs, fs, False, F)
    times = []
    with torch.no_grad():
        out = call()
        torch.cuda.synchronize()
        finite = bool(torch.isfinite(out[0]).all())
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        corr_ms = corr_kernel_ms(call)
    R = S * C
    fma = float(B) * R * 2 * R * F * T
    med = float(np.median(times))
    return {"windows": B * ((T - fs) // fs + 1), "all_finite": finite, "median_ms": round(med, 3),
            "ms_per_track": round(med / B, 3), "spread_ms": [round(min(times), 3), round(max(times), 3)],
            "corr_pass_ms": round(corr_ms, 3), "corr_fma": fma,
            "corr_fp64_tflops": round(2 * fma / (corr_ms * 1e-3) / 1e12, 2) if corr_ms > 0 else NOT_MEASURED}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-tracks", type=int, default=8, help="0: skip the host restatement")
    ap.add_argument("--cpu-seconds", type=int, default=30)
    args = ap.parse_args()
    gpu = torch.cuda.is_available()
    info = {"gpu": torch.cuda.get_device_properties(0).name if gpu else NOT_MEASURED,
            "card": (card() or NOT_MEASURED) if gpu else NOT_MEASURED}
    for name, (S, C, fs, B) in CASES.items():
        res = gpu_case(S, C, fs, B, args.reps) if gpu else {"median_ms": NOT_MEASURED}
        print(json.dumps({"metric": "bss_eval_v4", "case": name, "S": S, "C": C, "F": F, "B": B, "fs": fs,
                          "seconds": SECONDS, "window": fs, "hop": fs, **info, **res}), flush=True)
    if args.cpu_tracks < 1:
        return
    workers = os.cpu_count() or 1
    with ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as pool:   # the parent holds CUDA
        list(pool.map(ready, range(workers)))       # every worker started (and its imports done) before the clock
        t0 = time.perf_counter()
        list(pool.map(cpu_track, [(i, args.cpu_seconds) for i in range(args.cpu_tracks)]))
        cpu_s = time.perf_counter() - t0
    per = cpu_s / args.cpu_tracks
    print(json.dumps({"metric": "bss_eval_v4", "case": "fp64_numpy_restatement", "S": 4, "C": 1, "F": F,
                      "fs": 44100, "seconds": args.cpu_seconds, "cpu_workers": workers, "cpu_tracks": args.cpu_tracks,
                      "cpu_s_per_track": round(per, 2),
                      "cpu_s_per_4min_track_scaled": round(per * SECONDS / args.cpu_seconds, 1)}))


if __name__ == "__main__":
    main()
