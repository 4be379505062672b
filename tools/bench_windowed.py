"""Time windowed separation (``separate_long``) of long recordings on the GPU.

Two workloads, 4 s windows every 2 s, 32 windows per batch, the README recipe per window (``normalize=True``):
  - improved U16/512 (bench.py's improved_u16_512 model) on one hour at 8 kHz;
  - improved U36/4096 (bench.py's improved_u36_4096_16k model) on ten minutes at 16 kHz, which the whole-clip forward
    refuses (more than 2^31 encoder elements).
Weights are the oracle's seeded initialisation and the mixture is seeded noise: the time does not depend on either.
Default run: one warm-up call, then the median wall time of --reps calls (host clock around a call that ends in a
device synchronise), the real-time factor (audio seconds per second of compute) and torch's peak allocated memory
during a timed call; the card's name and power limit are read in the same run.  --profile instead runs one call
under torch.profiler and reports the share of device time each kernel family takes.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import sudo_rm_rf_b200 as P                 # noqa: E402
from sudo_rm_rf_b200 import _engine          # noqa: E402
from sudo_rm_rf_b200 import _native as N     # noqa: E402
from oracle import sudormrf_oracle as O     # noqa: E402

WORKLOADS = {
    "improved_u16_512_1h_8k": dict(fs=8000, seconds=3600, kw=dict(
        out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5,
        enc_kernel_size=21, enc_num_basis=512, num_sources=2)),
    "improved_u36_4096_10min_16k": dict(fs=16000, seconds=600, kw=dict(
        out_channels=512, in_channels=512, num_blocks=36, upsampling_depth=6,
        enc_kernel_size=21, enc_num_basis=4096, num_sources=2)),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def family(name):
    if "window_" in name:
        return "windowed (gather, align, scan, overlap-add, carry)"
    return "model forward"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--max-windows", type=int, default=32)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_windowed needs a CUDA device")
    dev = torch.device("cuda:0")
    result = {"metric": "separate_long", "gpu": torch.cuda.get_device_properties(dev).name, "card": card(),
              "max_windows": args.max_windows, "workloads": {}}
    for name in args.workloads.split(","):
        w = WORKLOADS[name]
        fs = w["fs"]
        T, W, H = w["seconds"] * fs, 4 * fs, 2 * fs
        model = P.SuDORMRF(**w["kw"])
        model.load_state_dict(O.make_state_dict(O.Config(variant="improved", **w["kw"]), seed=0, perturbed=False))
        model = model.to(dev).eval()
        x = torch.randn(1, 1, T, generator=torch.Generator().manual_seed(0)).to(dev)
        row = {"T": T, "fs": fs, "window": W, "hop": H, "windows": 1 + -(-(T - W) // H)}
        with torch.no_grad():
            # what one forward over the whole clip would need (0: refused), from the size query alone
            ws = N.lib().sdr_separate_workspace_bytes(C.byref(_engine.make_config(model)), 1, T)
            row["whole_clip_workspace_gb"] = round(ws / 2 ** 30, 2) if ws else "refused"
            run = lambda: model.separate_long(x, W, H, max_windows=args.max_windows)   # noqa: E731
            run()
            torch.cuda.synchronize()
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run()
                    torch.cuda.synchronize()
                shares, total = {}, 0.0
                for e in prof.key_averages():
                    t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                    if t <= 0:
                        continue
                    shares[family(e.key)] = shares.get(family(e.key), 0.0) + t
                    total += t
                    if "window_" in e.key:
                        row.setdefault("windowed_kernels_ms", {})[e.key.split("(")[0]] = round(t / 1000, 3)
                row["device_ms"] = round(total / 1000, 1)
                row["shares"] = {k: round(v / total, 5) for k, v in shares.items()}
            else:
                times = []
                for _ in range(args.reps):
                    torch.cuda.reset_peak_memory_stats(dev)
                    t0 = time.perf_counter()
                    out = run()
                    torch.cuda.synchronize()
                    times.append(time.perf_counter() - t0)
                    row["peak_allocated_gb"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 3)
                    del out
                med = sorted(times)[len(times) // 2]
                row.update({"seconds": round(med, 3), "all_seconds": [round(t, 3) for t in times],
                            "real_time_factor": round(w["seconds"] / med, 1),
                            "input_output_gb": round(T * (1 + w["kw"]["num_sources"]) * 4 / 2 ** 30, 3)})
        result["workloads"][name] = row
        del model, x
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
