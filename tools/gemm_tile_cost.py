"""Splits the wgmma GEMM's time into a per-tile cost E and a per-k-block cost c.

Times ``sdr_pointwise_mma`` at the shapes of bench.py's flagship workload (Improved U16/512, 32 x 4 s at 8 kHz:
L = 3200, 32 samples) in each epilogue mode, with K swept and M, L and the batch fixed, so every point runs the same
tiles.  A persistent CTA runs ceil(tiles / CTAs) tiles on the critical path, so

    t = tiles_per_cta * (E + KB * c),     KB = K / 64

and a least-squares line through (KB, t / tiles_per_cta) gives E (epilogue, tile switch, pipeline fill and drain) and
c (one k-block of the main loop).  CUDA events around each launch, L2 flushed before it, median of --reps runs.
Prints one JSON line with the card's name, power limit and median SM clock sampled while the timings ran.
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from sudo_rm_rf_b200 import _native as N  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=30, help="timed launches per point (median)")
ap.add_argument("--ks", default="64,128,256,512,1024")
ap.add_argument("--samples", type=int, default=32)
ap.add_argument("--L", type=int, default=3200)
a = ap.parse_args()
assert a.reps >= 20, "the median needs at least 20 runs"
KS = [int(k) for k in a.ks.split(",")]
L, S = a.L, a.samples
NB = 512                       # encoder basis = the mask GEMM's gate channels

# mode: (M, bias, statistics out, operand transform, epilogue)
MODES = {
    "proj": (512, True, True, "norm", "bias"),               # proj_1x1: bias + statistics
    "res_conv": (256, True, False, "norm_prelu", "res"),     # + residual in place, PReLU(GlobLN) operand
    "mask": (2 * NB, True, False, "prelu", "gate"),          # ReLU(.) * gate
    "decoder": (42, False, False, "none", "plain"),          # plain; 42 rows padded to one 128-wide tile
}

dev = torch.device("cuda")
lib = N.lib()
st = torch.cuda.current_stream()
sp = C.c_void_p(st.cuda_stream)
P = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
sms = torch.cuda.get_device_properties(dev).multi_processor_count


def smi_target():
    uuid = getattr(torch.cuda.get_device_properties(dev), "uuid", None)
    return ["-i", "GPU-" + str(uuid)] if uuid is not None else []


def stats_of(x):
    xd = x.double().reshape(x.shape[0], -1)
    return torch.stack([xd.sum(1), (xd * xd).sum(1)], 1).contiguous()


def time_point(mode, K):
    M, has_bias, stats, act, epi = MODES[mode]
    g = torch.Generator(device=dev).manual_seed(K)
    x = torch.randn(S, K, L, device=dev, generator=g)
    W = torch.randn(M, K, device=dev, generator=g) / K ** 0.5
    bias = torch.randn(M, device=dev, generator=g) if has_bias else None
    sin = stats_of(x)
    gamma, beta = torch.ones(K, device=dev), torch.zeros(K, device=dev)
    slope = torch.full((1,), 0.25, device=dev)
    if act == "none":
        nin = N.SdrNormIn(0, 0, 0, 0, 1.0)
    elif act == "prelu":
        nin = N.SdrNormIn(0, 0, 0, slope.data_ptr(), 1.0)
    else:
        nin = N.SdrNormIn(sin.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                          slope.data_ptr() if act == "norm_prelu" else 0, float(K * L))
    y = torch.randn(S, M, L, device=dev, generator=g)
    res = y if epi == "res" else None                  # in place, as res_conv's skip connection runs
    gate = torch.randn(S, NB, L, device=dev, generator=g) if epi == "gate" else None
    sto = torch.zeros(S, 2, dtype=torch.float64, device=dev) if stats else None
    wpk = torch.empty(lib.sdr_pointwise_mma_packed_bytes(M, K), dtype=torch.uint8, device=dev)
    N.check(lib.sdr_pointwise_mma_pack(P(W), M, K, P(wpk), sp))

    def run():
        N.check(lib.sdr_pointwise_mma(P(x), C.byref(nin), P(wpk), P(bias), P(res), P(gate),
                                      NB if epi == "gate" else 0, P(y), P(sto), S, M, K, L,
                                      1 if epi == "gate" else 0, sp))

    for _ in range(3):
        run()
    ms = []
    for _ in range(a.reps):
        flush.fill_(1)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(st); run(); e.record(st)
        torch.cuda.synchronize()
        ms.append(s.elapsed_time(e))
    return float(np.median(ms)) * 1e3


def main():
    smi = subprocess.run(["nvidia-smi", *smi_target(), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    clk = subprocess.Popen(["nvidia-smi", *smi_target(), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                            "-lms", "200"], stdout=subprocess.PIPE, text=True)
    out = {}
    try:
        for mode, (M, *_rest) in MODES.items():
            tiles = S * math.ceil(L / 128) * math.ceil(M / 128)
            per_cta = math.ceil(tiles / min(tiles, sms))
            pts = [(K, time_point(mode, K)) for K in KS]
            kb = np.array([K / 64 for K, _ in pts])
            per_tile = np.array([us for _, us in pts]) / per_cta
            c, E = np.polyfit(kb, per_tile, 1)
            fit = E + c * kb
            out[mode] = {"M": M, "tiles": tiles, "tiles_per_cta": per_cta, "E_us": round(float(E), 3),
                         "c_us": round(float(c), 3),
                         "max_fit_residual_us": round(float(np.abs(per_tile - fit).max() * per_cta), 1),
                         "us": {str(K): round(us, 1) for K, us in pts}}
    finally:
        clk.terminate()
        samples_mhz = clk.communicate()[0].split()
    clocks = [float(v) for v in samples_mhz if v.replace(".", "", 1).isdigit()]
    print(json.dumps({"card": smi[0], "power_limit": smi[1],
                      "sm_clock_MHz_median": float(np.median(clocks)) if clocks else None,
                      "samples": S, "L": L, "ctas": sms, "reps": a.reps, "lib": os.path.basename(N.LIB_PATH),
                      "modes": out}), flush=True)


if __name__ == "__main__":
    main()
