"""Times the depthwise stage of one U-ConvBlock two ways at the benchmark workloads' shapes, alternating them:

  pair   sdr_depthwise_pyramid + sdr_merge_pyramid: z_0 and R_1 .. R_{D-1} are written to HBM and read back
  fused  sdr_depthwise_pyramid_fused (what the forward runs): statistics pass over y, solve, merge pass over y

Both merge in place over y, as the forward does.  y is restored and the L2 flushed (256 MiB write) before every
timed run; times are CUDA events on the launching stream, the median over --reps.  Bytes are the fp32 tensors each
way must move (the row statistics and the merge table are under 0.2 % and left out); the fraction is of the H100
SXM data sheet's 3.35 TB/s.  Prints one JSON line per workload, after one with the GPU's name and power limit.

    python tools/time_depthwise_stage.py [--reps 20] [--workloads improved_u16_512,...]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import bench  # noqa: E402
from sudo_rm_rf_b200 import _native as N  # noqa: E402

HBM_GBPS = 3350.0
CONFIGS = {   # workload -> the name BASELINE.md gives it
    "improved_u16_512": "cfg 2", "improved_u36_2048": "cfg 3", "groupcomm_u8_512": "cfg 4",
    "improved_u36_4096_16k": "cfg 5", "original_u16_512": "original",
}

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--workloads", default=",".join(CONFIGS))
args = ap.parse_args()

assert torch.cuda.is_available(), "needs a CUDA device"
dev = torch.device("cuda")
lib = N.lib()
st = torch.cuda.current_stream()
sp = C.c_void_p(st.cuda_stream)
P = lambda t: C.c_void_p(t.data_ptr())
arr = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": smi, "library": N.LIB_PATH}), flush=True)


def stage(workload):
    w = bench.WORKLOADS[workload]
    kw = w["kw"]
    G = kw.get("group_size", 1) if w["variant"] == "groupcomm" else 1
    S, Ci, L, D = w["B"] * G, kw["in_channels"] // G, bench.algorithmic_model(w)["L"], kw["upsampling_depth"]
    nb = lib.sdr_pyramid_scratch_bytes(S, Ci, D, L)
    assert nb > 0, (workload, "the pyramid does not take this shape")
    g = torch.Generator(device=dev).manual_seed(0)
    y0 = torch.randn(S, Ci, L, device=dev, generator=g)
    y = torch.empty_like(y0)
    xd = y0.double().reshape(S, -1)
    stats_y = torch.stack([xd.sum(1), (xd * xd).sum(1)], 1).contiguous()
    del xd
    ones, zeros = torch.ones(Ci, device=dev), torch.zeros(Ci, device=dev)
    slope = torch.full((Ci,), 0.25, device=dev) if w["variant"] == "original" else torch.full((1,), 0.25, device=dev)
    nin = N.SdrNormIn(stats_y.data_ptr(), ones.data_ptr(), zeros.data_ptr(), slope.data_ptr(), float(Ci * L),
                      1 if slope.numel() > 1 else 0)
    ws = [torch.randn(Ci, 5, device=dev, generator=g) * 0.4 for _ in range(D)]
    bs = [torch.randn(Ci, device=dev, generator=g) * 0.1 for _ in range(D)]
    gs, bes = [ones] * D, [zeros] * D
    zs = [torch.empty(S, Ci, L >> d, device=dev) for d in range(D)]
    scratch = torch.zeros(nb, dtype=torch.uint8, device=dev)
    st0 = torch.zeros(S, 2, dtype=torch.float64, device=dev)
    stm = torch.zeros(S, 2, dtype=torch.float64, device=dev)

    def pair():
        N.check(lib.sdr_depthwise_pyramid(P(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), P(st0),
                                          P(scratch), D, S, Ci, L, sp), "sdr_depthwise_pyramid")
        N.check(lib.sdr_merge_pyramid(arr(zs), P(scratch), D, P(y), P(stm), S, Ci, L, sp), "sdr_merge_pyramid")

    def fused():
        N.check(lib.sdr_depthwise_pyramid_fused(P(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), P(y), P(st0),
                                                P(stm), P(scratch), D, S, Ci, L, sp), "sdr_depthwise_pyramid_fused")

    def run(fn):
        y.copy_(y0)
        st0.zero_()
        stm.zero_()
        flush.fill_(1)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(st)
        fn()
        e.record(st)
        torch.cuda.synchronize()
        return s.elapsed_time(e)

    run(pair)
    m_pair = y.clone()
    run(fused)
    diff = float((m_pair - y).abs().max() / m_pair.abs().max())
    del m_pair
    times = {"pair": [], "fused": []}
    for _ in range(args.reps):                         # alternating: drift and neighbours hit both alike
        for name, fn in (("pair", pair), ("fused", fused)):
            times[name].append(run(fn))
    tensor = 4.0 * S * Ci * L
    levels = sum(2.0 ** -d for d in range(D))          # z_0 + R_1 .. R_{D-1}, in units of one [S, Ci, L] tensor
    moved = {"pair": tensor * (2 + 2 * levels), "fused": tensor * 3}
    out = {"workload": workload, "config": CONFIGS.get(workload, ""), "samples": S, "C": Ci, "L": L, "D": D,
           "m_rel_diff": diff}
    for name, ms in times.items():
        t = sorted(ms)[len(ms) // 2]
        out[name] = {"us": round(1e3 * t, 1), "MB": round(moved[name] / 1e6, 1),
                     "GBps": round(moved[name] / t / 1e6, 1), "frac_hbm": round(moved[name] / t / 1e6 / HBM_GBPS, 3)}
    out["fused_over_pair"] = round(out["fused"]["us"] / out["pair"]["us"], 3)
    print(json.dumps(out), flush=True)


for wl in args.workloads.split(","):
    stage(wl)
    torch.cuda.empty_cache()
