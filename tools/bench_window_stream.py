"""Time windowed streams (``model.stream_windows``, DESIGN.md section 7f) on the GPU.

Two models at 8 kHz, 4 s windows every 2 s, 2 s chunks (q = 1), the README recipe per window (``normalize=True``):
improved U16/512 (bench.py's improved_u16_512) and GroupComm U8/512 (bench.py's groupcomm_u8_512, with mixture
consistency, its separate() default).  For every slot count B it reports the median step time by CUDA events, eager
and replayed from a CUDA graph, after warm-up; the real-time factor (chunk seconds per step second), the number of
real-time streams that factor allows (B times it), and torch's peak allocated memory over the steps.  Next to it, on
the same audio (B recordings of --seconds each), ``separate_long``'s audio seconds per second, with at most 256
windows per forward (``max_windows = max(1, 256 // B)``) so that its workspace stays bounded.  Weights are the
oracle's seeded initialisation and the audio is seeded noise: the times do not depend on either.  The card's name and
power limit are read in the same run.  Prints one JSON line per (model, B)."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import sudo_rm_rf_b200 as P                 # noqa: E402
from oracle import sudormrf_oracle as O     # noqa: E402

MODELS = {
    "improved_u16_512": (P.SuDORMRF, "improved", dict(
        out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5,
        enc_kernel_size=21, enc_num_basis=512, num_sources=2)),
    "groupcomm_u8_512": (P.GroupCommSudoRmRf, "groupcomm", dict(
        out_channels=256, in_channels=512, num_blocks=8, upsampling_depth=5,
        enc_kernel_size=21, enc_num_basis=512, num_sources=2, group_size=16)),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def median(xs):
    return sorted(xs)[len(xs) // 2]


def time_steps(fn, steps):
    """Median ms of `steps` calls of fn(j), each timed by its own pair of CUDA events."""
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for j, (a, b) in enumerate(evs):
        a.record()
        fn(j)
        b.record()
    torch.cuda.synchronize()
    return median([a.elapsed_time(b) for a, b in evs])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--batches", default="1,32,256")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seconds", type=int, default=60, help="length of each recording separate_long is timed on")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_window_stream needs a CUDA device")
    dev = torch.device("cuda:0")
    fs, W, H = 8000, 32000, 16000
    C = H
    gpu, power = torch.cuda.get_device_properties(dev).name, card()
    for name in args.models.split(","):
        cls, variant, kw = MODELS[name]
        model = cls(**kw)
        model.load_state_dict(O.make_state_dict(O.Config(variant=variant, **kw), seed=0, perturbed=False))
        model = model.to(dev).eval()
        for B in (int(b) for b in args.batches.split(",")):
            n = args.warmup + args.steps
            x = torch.randn(B, 1, args.seconds * fs, generator=torch.Generator().manual_seed(B)).to(dev)
            chunks = x[..., :n * C].reshape(B, 1, n, C).permute(2, 0, 1, 3).contiguous()
            row = {"metric": "window_stream_step", "model": name, "gpu": gpu, "card": power, "fs": fs, "window": W,
                   "hop": H, "chunk": C, "B": B}
            with torch.no_grad():
                st = model.stream_windows(B, C, W, H)
                out = torch.empty(B, 2, C, device=dev)
                for j in range(args.warmup):
                    st.step(chunks[j], out=out)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                eager = time_steps(lambda j: st.step(chunks[args.warmup + j], out=out), args.steps)
                row["peak_allocated_gb"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 3)
                buf = torch.empty_like(chunks[0])
                buf.copy_(chunks[0])
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    st.step(buf, out=out)
                for _ in range(args.warmup):
                    graph.replay()
                graphed = time_steps(lambda j: graph.replay(), args.steps)
                del graph
                step = min(eager, graphed)
                rtf = C / fs / (step / 1000)
                row.update({"step_ms_eager": round(eager, 3), "step_ms_graph": round(graphed, 3),
                            "real_time_factor": round(rtf, 1), "real_time_streams": int(B * rtf)})
                mw = max(1, 256 // B)
                model.separate_long(x, W, H, max_windows=mw)    # warm
                torch.cuda.synchronize()
                times = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    model.separate_long(x, W, H, max_windows=mw)
                    torch.cuda.synchronize()
                    times.append(time.perf_counter() - t0)
                row["separate_long_audio_s_per_s"] = round(B * args.seconds / median(times), 1)
            print(json.dumps(row), flush=True)
            del st, x, chunks
            torch.cuda.empty_cache()
        del model


if __name__ == "__main__":
    main()
