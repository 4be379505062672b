"""Time streaming at another sample rate (DESIGN.md section 7h) on the GPU.

1. ``ResampleStream`` steps with 10 ms chunks, 44.1 -> 8 kHz and 8 -> 44.1 kHz, for 1 and 256 slots.
2. The default causal model (``CausalSuDORMRF()``) stepped through ``ResampledStream`` for 256 slots with 10 ms chunks
   at 44.1 kHz, against the plain ``CausalStream`` step at 8 kHz on the same 10 ms.
3. The windowed U16/512 (bench.py's improved_u16_512, 4 s windows every 2 s) through ``ResampledStream`` for 256 slots
   with 2 s chunks at 44.1 kHz, against the plain ``WindowedStream`` step at 8 kHz.

Every time is the median of per-step CUDA-event times after warm-up.  Weights are the oracle's seeded initialisation
and the audio seeded noise: the times depend on neither.  The card's name and power limit are read in the same run.
Prints one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import sudo_rm_rf_b200 as P                 # noqa: E402
from oracle import sudormrf_oracle as O     # noqa: E402

U16 = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
           enc_num_basis=512, num_sources=2)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def median(xs):
    return sorted(xs)[len(xs) // 2]


def time_steps(step, chunks, steps, warmup):
    """Median ms of `steps` calls of step(chunk), each timed by its own pair of CUDA events, after `warmup` calls."""
    for j in range(warmup):
        step(chunks[j % len(chunks)])
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for j, (a, b) in enumerate(evs):
        a.record()
        step(chunks[j % len(chunks)])
        b.record()
    torch.cuda.synchronize()
    return median([a.elapsed_time(b) for a, b in evs])


def noise(shape, n=4):
    g = torch.Generator(device="cuda").manual_seed(0)
    return [torch.randn(shape, generator=g, device="cuda") for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample_stream needs a CUDA device")
    dev = torch.device("cuda:0")
    info = dict(gpu=torch.cuda.get_device_properties(dev).name, power=card())

    def emit(**kw):
        print(json.dumps(dict(kw, **info)), flush=True)

    with torch.no_grad():
        for sr, mr in ((44100, 8000), (8000, 44100)):
            C = sr // 100
            for B in (1, 256):
                st = P.ResampleStream(B, 1, C, mr, sr)
                out = torch.empty(B, 1, st.out_samples, device=dev)
                ms = time_steps(lambda x: st.step(x, out=out), noise((B, 1, C)), args.steps, args.warmup)
                emit(what="ResampleStream.step", rates=f"{sr}->{mr}", slots=B, chunk_ms=10, step_ms=ms)

        causal = P.CausalSuDORMRF().to(dev).eval()
        B = 256
        st = causal.stream(B, 441, sample_rate=44100, model_rate=8000)
        out = torch.empty(B, 2, 441, device=dev)
        ms = time_steps(lambda x: st.step(x, out=out), noise((B, 1, 441)), args.steps, args.warmup)
        plain = causal.stream(B, 80)
        out8 = torch.empty(B, 2, 80, device=dev)
        ms8 = time_steps(lambda x: plain.step(x, out=out8), noise((B, 1, 80)), args.steps, args.warmup)
        emit(what="causal default, 10 ms chunks", slots=B, step_ms_44k1=ms, step_ms_8k=ms8, latency=st.latency)
        del st, plain, causal

        model = P.SuDORMRF(**U16)
        model.load_state_dict(O.make_state_dict(O.Config(variant="improved", **U16), seed=0, perturbed=False))
        model = model.to(dev).eval()
        st = model.stream_windows(B, 88200, 32000, 16000, sample_rate=44100, model_rate=8000)
        out = torch.empty(B, 2, 88200, device=dev)
        steps = max(5, args.steps // 5)
        ms = time_steps(lambda x: st.step(x, out=out), noise((B, 1, 88200), 2), steps, args.warmup)
        del st, out
        plain = model.stream_windows(B, 16000, 32000, 16000)
        out8 = torch.empty(B, 2, 16000, device=dev)
        ms8 = time_steps(lambda x: plain.step(x, out=out8), noise((B, 1, 16000), 2), steps, args.warmup)
        emit(what="windowed U16/512, 2 s chunks", slots=B, step_ms_44k1=ms, step_ms_8k=ms8,
             realtime_streams_44k1=B * 2000.0 / ms)


if __name__ == "__main__":
    main()
