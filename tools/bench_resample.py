"""Time polyphase resampling (``resample_poly``) on the GPU, and its share of a separation at another rate.

Workloads: one hour of mono audio at 48 -> 8, 8 -> 48, 44.1 -> 8, 8 -> 44.1 and 44.1 -> 16 kHz, and 256 rows of 4 s
at 44.1 -> 8 kHz.  Each is timed with CUDA events over --reps calls after --warmup calls; the achieved rate counts the
algorithmic bytes (4 per input sample plus 4 per output sample) against the H100 SXM's 3.35 TB/s.  scipy's
``resample_poly`` on the same input (fp64, one host thread) is timed once per workload (--no-scipy skips it).
Then ``separate_long`` of improved U16/512 (bench_windowed.py's model; 4 s windows every 2 s, 32 per batch) on one
hour at 44.1 kHz through the model at 8 kHz, next to the same call on the 8 kHz recording: the difference is the
resampling's share.  The card's name and power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import sudo_rm_rf_b200 as P                 # noqa: E402
from oracle import sudormrf_oracle as O     # noqa: E402

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {                                # (input rate, output rate, rows, seconds)
    "1h_48k_to_8k": (48000, 8000, 1, 3600),
    "1h_8k_to_48k": (8000, 48000, 1, 3600),
    "1h_44k1_to_8k": (44100, 8000, 1, 3600),
    "1h_8k_to_44k1": (8000, 44100, 1, 3600),
    "1h_44k1_to_16k": (44100, 16000, 1, 3600),
    "256x4s_44k1_to_8k": (44100, 8000, 256, 4),
}
U16_512 = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
               enc_num_basis=512, num_sources=2)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def events_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return sorted(times)[len(times) // 2], times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-scipy", action="store_true")
    ap.add_argument("--no-separate", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample needs a CUDA device")
    dev = torch.device("cuda:0")
    result = {"metric": "resample_poly", "gpu": torch.cuda.get_device_properties(dev).name, "card": card(),
              "workloads": {}}
    for name in args.workloads.split(","):
        fs_in, fs_out, rows, seconds = WORKLOADS[name]
        T = fs_in * seconds
        x = torch.randn(rows, T, generator=torch.Generator().manual_seed(0)).to(dev)
        out = P.resample_poly(x, fs_out, fs_in)
        med, times = events_ms(lambda: P.resample_poly(x, fs_out, fs_in), args.warmup, args.reps)
        nbytes = 4 * (x.numel() + out.numel())
        row = {"rows": rows, "T": T, "outputs": out.numel(), "ms": round(med, 3),
               "min_max_ms": [round(min(times), 3), round(max(times), 3)],
               "gb_per_s": round(nbytes / (med * 1e-3) / 1e9, 1),
               "share_of_3_35_tb_s": round(nbytes / (med * 1e-3) / HBM_BYTES_PER_S, 3)}
        if not args.no_scipy:
            import scipy.signal as ss
            xh = x.cpu().numpy().astype(np.float64)
            t0 = time.perf_counter()
            ss.resample_poly(xh, fs_out, fs_in, axis=-1)
            row["scipy_host_s"] = round(time.perf_counter() - t0, 2)
            del xh
        result["workloads"][name] = row
        del x, out
        torch.cuda.empty_cache()
    if not args.no_separate:
        model = P.SuDORMRF(**U16_512)
        model.load_state_dict(O.make_state_dict(O.Config(variant="improved", **U16_512), seed=0, perturbed=False))
        model = model.to(dev).eval()
        W, H = 4 * 8000, 2 * 8000
        x44 = torch.randn(1, 1, 3600 * 44100, generator=torch.Generator().manual_seed(1)).to(dev)
        x8 = P.resample_poly(x44, 8000, 44100)
        row = {}
        with torch.no_grad():
            for key, fn in (("separate_long_1h_8k_s", lambda: model.separate_long(x8, W, H)),
                            ("separate_long_1h_44k1_via_8k_s",
                             lambda: model.separate_long(x44, W, H, sample_rate=44100, model_rate=8000))):
                fn()
                torch.cuda.synchronize()
                times = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times.append(time.perf_counter() - t0)
                row[key] = round(sorted(times)[1], 3)
        row["resampling_share"] = round(1 - row["separate_long_1h_8k_s"] / row["separate_long_1h_44k1_via_8k_s"], 4)
        result["separate_long_u16_512"] = row
    print(json.dumps(result))


if __name__ == "__main__":
    main()
