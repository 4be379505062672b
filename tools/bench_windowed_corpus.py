"""Time windowed separation of a corpus of recordings of different lengths on the GPU: ``separate_long_corpus``, whose
windows share batches across recordings, against a loop of ``separate_long`` over the same corpus.

Workload: improved U16/512 (bench.py's improved_u16_512 model), --recordings recordings with lengths drawn uniformly
from --min-s .. --max-s seconds at 8 kHz (seeded), 4 s windows every 2 s, --max-windows windows per batch, the README
recipe per window (``normalize=True``).  Weights are the oracle's seeded initialisation and the audio seeded noise:
the time does not depend on either.  One warm-up of each path, then --reps timed calls of each, alternating; each call
is timed with CUDA events on the current stream and ends in a device synchronise.  Reports the median time,
recordings per second, the real-time factor (audio seconds per second of compute) and torch's peak allocated memory
during a timed call of each path, with the card's name and power limit read in the same run, and the largest
difference between the two paths' outputs.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import sudo_rm_rf_b200 as P                 # noqa: E402
from sudo_rm_rf_b200 import windowed         # noqa: E402
from oracle import sudormrf_oracle as O     # noqa: E402

KW = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21, enc_num_basis=512,
          num_sources=2)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn):
    """(result, milliseconds, peak allocated bytes above what was allocated before the call)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    return out, start.elapsed_time(end), torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=200)
    ap.add_argument("--min-s", type=float, default=5.0)
    ap.add_argument("--max-s", type=float, default=60.0)
    ap.add_argument("--fs", type=int, default=8000)
    ap.add_argument("--window-s", type=float, default=4.0)
    ap.add_argument("--hop-s", type=float, default=2.0)
    ap.add_argument("--max-windows", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_windowed_corpus.py measures on the GPU and needs a CUDA device")
    dev = torch.device("cuda:0")
    W, H = int(a.window_s * a.fs), int(a.hop_s * a.fs)
    gen = torch.Generator().manual_seed(0)
    lengths = (a.min_s + (a.max_s - a.min_s) * torch.rand(a.recordings, generator=gen)).mul(a.fs).long().tolist()
    wavs = [torch.randn(T, generator=gen).to(dev) for T in lengths]
    m = P.SuDORMRF(**KW)
    m.load_state_dict(O.make_state_dict(O.Config(variant="improved", **KW), seed=0))
    m = m.to(dev).eval()

    def corpus():
        return windowed.separate_long_corpus(m, wavs, W, H, max_windows=a.max_windows)

    def loop():
        return [windowed.separate_long(m, w[None], W, H, max_windows=a.max_windows)[0] for w in wavs]

    runs = {"corpus": corpus, "loop": loop}
    times, peaks, outs = {k: [] for k in runs}, {k: 0 for k in runs}, {}
    with torch.no_grad():
        for k, fn in runs.items():
            fn()                                            # warm-up: workspaces, kernels, allocator
        for _ in range(a.reps):
            for k, fn in runs.items():
                outs[k], ms, peak = timed(fn)
                times[k].append(ms)
                peaks[k] = max(peaks[k], peak)
        diff = max(float((c - l).abs().max() / l.abs().max().clamp_min(1e-30))
                   for c, l in zip(outs["corpus"], outs["loop"]))
    audio_s = sum(lengths) / a.fs
    windows = sum(windowed.window_plan(T, W, H)[0] for T in lengths)
    res = dict(metric="windowed_corpus", model="improved_u16_512", card=card(), fs=a.fs, window=W, hop=H,
               recordings=a.recordings, audio_s=round(audio_s, 1), windows=windows, max_windows=a.max_windows,
               reps=a.reps, max_rel_diff_corpus_vs_loop=diff)
    for k in runs:
        ms = statistics.median(times[k])
        res[k] = dict(median_ms=round(ms, 2), min_ms=round(min(times[k]), 2), max_ms=round(max(times[k]), 2),
                      recordings_per_s=round(a.recordings / (ms / 1e3), 1),
                      real_time_factor=round(audio_s / (ms / 1e3), 1), peak_allocated_gb=round(peaks[k] / 1e9, 3))
    res["speedup"] = round(res["loop"]["median_ms"] / res["corpus"]["median_ms"], 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
