"""Times each hot-path kernel alone at a benchmark workload's shapes (CUDA events on
the launching stream, L2 flushed between launches) and prints achieved algorithmic GB/s."""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import bench  # noqa: E402
from sudo_rm_rf_b200 import _native as N  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="improved_u16_512")
ap.add_argument("--batch", type=int, default=0)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--only", default="")
a = ap.parse_args()
w = bench.WORKLOADS[a.workload]
kw = w["kw"]
B = a.batch or w["B"]
gc = w["variant"] == "groupcomm"
G = kw.get("group_size", 1) if gc else 1
am = bench.algorithmic_model(w)
L, D = am["L"], kw["upsampling_depth"]
S, Co, Ci, NB = B * G, kw["out_channels"] // G, kw["in_channels"] // G, kw["enc_num_basis"]
dev = torch.device("cuda")
lib = N.lib()
peak, _ = bench.load_peaks()
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
st = torch.cuda.current_stream()
sp = C.c_void_p(st.cuda_stream)
P = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)


def stats_of(x):
    xd = x.double().reshape(x.shape[0], -1)
    return torch.stack([xd.sum(1), (xd * xd).sum(1)], 1).contiguous()


def timeit(name, fn, nbytes, flops=0.0):
    if a.only and a.only not in name:
        return
    for _ in range(2):
        fn()
    ms = []
    for _ in range(a.reps):
        flush.fill_(1)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(st); fn(); e.record(st)
        torch.cuda.synchronize()
        ms.append(s.elapsed_time(e))
    t = sorted(ms)[len(ms) // 2]
    print(json.dumps({"kernel": name, "ms": round(t, 4), "alg_MB": round(nbytes / 1e6, 1),
                      "GBps": round(nbytes / t / 1e6, 1), "frac_hbm": round(nbytes / t / 1e6 / peak, 3),
                      "TFLOPs": round(flops / t / 1e9, 1)}), flush=True)


# per-box normaliser: device-to-device copy bandwidth (same definition as MEASURED_PEAKS.json) + clocks
import subprocess
_a = torch.empty(1 << 30, dtype=torch.uint8, device=dev); _b = torch.empty_like(_a)
for _ in range(3): _b.copy_(_a)
best = 1e9
for _ in range(10):
    s_, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s_.record(st); _b.copy_(_a); e_.record(st); torch.cuda.synchronize()
    best = min(best, s_.elapsed_time(e_))
try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.mem,power.draw,temperature.gpu,uuid",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
except Exception:
    smi = "?"
print(json.dumps({"box_copy_GBps": round(2 * (1 << 30) / best / 1e6, 1), "peak_file_GBps": peak, "nvidia_smi": smi}), flush=True)
del _a, _b

ones = lambda n: torch.ones(n, device=dev)
zeros = lambda n: torch.zeros(n, device=dev)
slope = torch.full((1,), 0.25, device=dev)


def pointwise(name, M, K, mode, samples=S):
    x = torch.randn(samples, K, L, device=dev)
    Wt = torch.randn(M, K, device=dev) / K ** 0.5
    bias = torch.randn(M, device=dev)
    stt = stats_of(x)
    nin = N.SdrNormIn(stt.data_ptr(), ones(K).data_ptr(), zeros(K).data_ptr(),
                      slope.data_ptr() if mode == "res" else 0, float(K * L))
    if mode in ("plain", "dec"):
        nin = N.SdrNormIn(0, 0, 0, 0, 1.0)
    if mode == "dec":                  # the decoder GEMM: no bias, no statistics
        bias = None
    y = torch.randn(samples, M, L, device=dev)
    sto = torch.zeros(samples, 2, dtype=torch.float64, device=dev)
    gate = torch.randn(samples, NB, L, device=dev) if mode == "mask" else None
    res = y if mode == "res" else None
    epi = 1 if mode == "mask" else 0
    keep = [x, Wt, bias, stt, y, sto, gate]
    nb = 4 * L * samples * (K + M + (M if mode == "res" else 0) + (M if mode == "mask" else 0))
    fl = 2.0 * M * K * L * samples
    nbytes = lib.sdr_pointwise_mma_packed_bytes(M, K)
    if nbytes:
        wpk = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        N.check(lib.sdr_pointwise_mma_pack(P(Wt), M, K, P(wpk), sp))
        keep.append(wpk)
        timeit(name + " [wgmma]", lambda: N.check(lib.sdr_pointwise_mma(
            P(x), C.byref(nin), P(wpk), P(bias), P(res), P(gate), NB, P(y),
            P(sto) if mode == "plain" else P(None), samples, M, K, L, epi, sp)), nb, fl)
    timeit(name + " [ffma]", lambda: N.check(lib.sdr_pointwise(
        P(x), C.byref(nin), P(Wt), P(bias), P(res), P(gate), NB, P(y),
        P(sto) if mode == "plain" else P(None), samples, M, K, L, epi, sp)), nb, fl)
    return keep


pointwise("proj_1x1", Ci, Co, "plain")
pointwise("res_conv+skip", Co, Ci, "res")
pointwise("bottleneck", kw["out_channels"], NB, "norm", samples=B)
pointwise("mask_net", kw["num_sources"] * NB, kw["out_channels"], "mask", samples=B)
pointwise("decoder", kw["num_sources"] * kw["enc_kernel_size"], kw["num_sources"] * NB, "dec", samples=B)

# depthwise levels
for d in range(D):
    Lin = L >> max(d - 1, 0)
    stride = 1 if d == 0 else 2
    x = torch.randn(S, Ci, Lin, device=dev)
    stt = stats_of(x)
    nin = N.SdrNormIn(stt.data_ptr(), ones(Ci).data_ptr(), zeros(Ci).data_ptr(),
                      slope.data_ptr() if d == 0 else 0, float(Ci * Lin))
    w5 = torch.randn(Ci, 5, device=dev)
    b5 = torch.randn(Ci, device=dev)
    Lout = (Lin - 1) // stride + 1
    y = torch.empty(S, Ci, Lout, device=dev)
    sto = torch.zeros(S, 2, dtype=torch.float64, device=dev)
    timeit(f"depthwise level {d} (stride {stride})", lambda: N.check(lib.sdr_depthwise(
        P(x), C.byref(nin), P(w5), P(b5), P(y), P(sto), S, Ci, Lin, stride, sp)),
        4 * S * Ci * (Lin + Lout))

# merge
zs = [torch.randn(S, Ci, L >> d, device=dev) for d in range(D)]
sts = [stats_of(z) for z in zs]
g1, b0 = ones(Ci), zeros(Ci)
fins = (N.SdrNormIn * D)(*[N.SdrNormIn(sts[d].data_ptr(), g1.data_ptr(), b0.data_ptr(), 0,
                                       float(Ci * (L >> d))) for d in range(D)])
zp = (C.c_void_p * D)(*[z.data_ptr() for z in zs])
m = torch.empty(S, Ci, L, device=dev)
sto = torch.zeros(S, 2, dtype=torch.float64, device=dev)
timeit("merge", lambda: N.check(lib.sdr_merge(zp, fins, D, P(m), P(sto), S, Ci, L, sp)),
       4 * S * Ci * (L + sum(L >> d for d in range(D))))

# encoder
wav = torch.rand(B, 1, w["T"], device=dev)
we = torch.randn(NB, 1, kw["enc_kernel_size"], device=dev)
enc = torch.empty(B, NB, L, device=dev)
sto = torch.zeros(B, 2, dtype=torch.float64, device=dev)
timeit("encoder", lambda: N.check(lib.sdr_encoder(P(wav), P(we), P(enc), P(sto), B, 1, w["T"], NB,
                                                  kw["enc_kernel_size"], L, sp)),
       4 * B * (w["T"] + NB * L), 2.0 * kw["enc_kernel_size"] * NB * L * B)
