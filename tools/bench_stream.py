"""Streaming throughput of the default CausalSuDORMRF (U16, Ci 512, D 4, 8 kHz).

For each (slots B, chunk C): one step captured in a CUDA graph and replayed, each replay timed with CUDA events; the
median of --steps replays after --warmup.  Prints one JSON line per configuration with the step time, the real-time
factor (chunk duration / step time) and the number of concurrent real-time streams (B x that factor); the stream
stage kernel alone against its byte model; the offline forward at B = 32 x 4 s for comparison; the card and its
power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import sudo_rm_rf_b200 as P  # noqa: E402
from sudo_rm_rf_b200 import _native as N  # noqa: E402
from oracle import sudormrf_oracle as O  # noqa: E402

HBM_TBPS = 3.35
SR = 8000

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=300)
ap.add_argument("--warmup", type=int, default=30)
ap.add_argument("--slots", default="1,16,256")
ap.add_argument("--chunks", default="80,320")
a = ap.parse_args()

dev = torch.device("cuda")
kw = dict(in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=512, num_sources=2)
cfg = O.Config(variant="causal", **kw)
sd = O.make_state_dict(cfg, seed=0)
model = P.CausalSuDORMRF(**kw)
model.load_state_dict(sd)
model = model.to(dev).eval()
lib = N.lib()

try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
except Exception:
    smi = "?"
print(json.dumps({"device": torch.cuda.get_device_name(), "nvidia_smi_name_powerlimit_sm": smi}), flush=True)


def median_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for s, e in ev:
        s.record(); fn(); e.record()
    torch.cuda.synchronize()
    t = sorted(s.elapsed_time(e) for s, e in ev)
    return t[len(t) // 2]


# offline reference point: model(x) at B = 32 x 4 s
x_off = torch.randn(32, 1, 32000, device=dev)
with torch.no_grad():
    off_ms = median_ms(lambda: model(x_off), 20, 3)
offline_aps = 32 * 4.0 / (off_ms / 1e3)
print(json.dumps({"offline": "B=32 x 4 s", "ms": round(off_ms, 3), "audio_s_per_s": round(offline_aps, 1)}), flush=True)
del x_off

D, Ci, U = kw["upsampling_depth"], kw["in_channels"], kw["num_blocks"]
for B in [int(v) for v in a.slots.split(",")]:
    for Cn in [int(v) for v in a.chunks.split(",")]:
        s = model.stream(B, Cn)
        inp = torch.randn(B, 1, Cn, device=dev)
        out = torch.empty(B, 2, Cn, device=dev)
        with torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                s.step(inp, out=out)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                s.step(inp, out=out)
        step_ms = median_ms(g.replay, a.steps, a.warmup)
        rtf = (Cn / SR) / (step_ms / 1e3)

        # the stream stage kernel alone at this shape
        F = Cn // cfg.hop
        y = torch.randn(Ci, B * F, device=dev)
        m = torch.empty_like(y)
        hist = torch.zeros(B, D, 10, Ci, device=dev)
        ws = [model.sm[0].spp_dw[d].conv.weight.detach() for d in range(D)]
        bs = [model.sm[0].spp_dw[d].conv.bias.detach() for d in range(D)]
        sl = [model.sm[0].spp_dw[d].act.weight.detach() for d in range(D)]
        ptrs = lambda ts: (C.c_void_p * len(ts))(*[C.c_void_p(t.data_ptr()) for t in ts])
        pw, pb, ps = ptrs(ws), ptrs(bs), ptrs(sl)
        slope_in = model.sm[0].proj_1x1.act.weight.detach()
        sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        stage = lambda: N.check(lib.sdr_causal_stream_stage(
            C.c_void_p(y.data_ptr()), C.c_void_p(slope_in.data_ptr()), pw, pb, ps, C.c_void_p(hist.data_ptr()),
            C.c_void_p(m.data_ptr()), D, B, Ci, F, sp), "stage")
        stage_ms = median_ms(stage, a.steps, a.warmup)
        nbytes = 4 * (2 * Ci * B * F + 2 * B * D * 10 * Ci)
        print(json.dumps({
            "slots": B, "chunk_samples": Cn, "chunk_ms": 1e3 * Cn / SR, "step_ms": round(step_ms, 4),
            "real_time_factor": round(rtf, 1), "realtime_streams": round(B * rtf, 1),
            "streamed_audio_s_per_s": round(B * rtf, 1), "offline_audio_s_per_s": round(offline_aps, 1),
            "stage_us": round(stage_ms * 1e3, 2), "stage_MB": round(nbytes / 1e6, 3),
            "stage_frac_hbm": round(nbytes / (stage_ms / 1e3) / (HBM_TBPS * 1e12), 3),
            "launches_per_step": lib.sdr_stream_launch_count(C.byref(P._engine.make_config(model)), B, Cn)}), flush=True)
        del s, g, y, m, hist
        torch.cuda.empty_cache()
