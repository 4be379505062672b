"""Training-step throughput of the improved SuDORMRF on the native path against stock PyTorch.

One step is the runners' (run_improved_sudormrf.py): forward, PIT over the pairwise negative SI-SDR, backward.  It is
timed with CUDA events after --warmup steps; the median of --steps is reported with mixtures/s and the peak memory
of the step.  The comparator runs the oracle's op sequence (the reference's forward as plain torch ops) in fp32 eager
CUDA autograd on the same GPU.  Three implementations: `native` (native model, the loss as eager torch ops),
`native+native_loss` (native model, PITLossWrapper(PairwiseNegSDR("sisdr")) of sudo_rm_rf_b200.sisdr) and
`eager_fp32`.  Then the loss alone, forward plus backward on fixed estimates: the native loss against the reference's
op sequence (PairwiseNegSDR's [B, S, S, T] tensors, PITLossWrapper's einsum) in fp32 eager CUDA autograd.
Prints the card and its power limit, read in the same run, then one JSON line per (model, batch, implementation)
and per (loss shape, implementation).  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import sudo_rm_rf_b200 as P  # noqa: E402
from sudo_rm_rf_b200 import sisdr as S  # noqa: E402
from oracle import sudormrf_oracle as O  # noqa: E402

MODELS = {
    "U16/512": dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
                    enc_num_basis=512, num_sources=2),
    "U36/2048": dict(out_channels=512, in_channels=512, num_blocks=36, upsampling_depth=6, enc_kernel_size=21,
                     enc_num_basis=2048, num_sources=2),
}


def pit_loss(y, tgt):
    best, _ = O.pit_from_pairwise(O.pairwise_neg_sdr(y, tgt))
    return best.mean()


NATIVE_LOSS = S.PITLossWrapper(S.PairwiseNegSDR("sisdr"), pit_from="pw_mtx")
EAGER_LOSS = S.PITLossWrapper(lambda e, t: O.pairwise_neg_sdr(e, t, "sisdr"), pit_from="pw_mtx")


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2], torch.cuda.max_memory_allocated() / 2 ** 30


def run(name, B, impl, steps, warmup, T=32000):
    kw = MODELS[name]
    cfg = O.Config(variant="improved", **kw)
    sd = O.make_state_dict(cfg, seed=0)
    gen = torch.Generator().manual_seed(1)
    tgt = torch.randn(B, 2, T, generator=gen).cuda()
    x = tgt.sum(1, keepdim=True)
    if impl in ("native", "native+native_loss"):
        m = P.SuDORMRF(**kw)
        m.load_state_dict(sd)
        m = m.cuda().train().enable_training()
        loss_fn = pit_loss if impl == "native" else NATIVE_LOSS

        def step():
            m.zero_grad(set_to_none=True)
            loss_fn(m(x), tgt).backward()
    else:
        params = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
        O.prelu1 = lambda v, slope: F.prelu(v, slope.reshape(1))      # nn.PReLU, as the reference

        def step():
            for p in params.values():
                p.grad = None
            pit_loss(O.forward(cfg, params, x), tgt).backward()
    torch.cuda.empty_cache()
    ms, peak = time_steps(step, steps, warmup)
    return {"model": name, "B": B, "T": T, "impl": impl, "step_ms": round(ms, 3),
            "mixtures_per_s": round(B / ms * 1e3, 2), "peak_gib": round(peak, 2)}


def run_loss(B, Sn, T, impl, steps, warmup):
    gen = torch.Generator().manual_seed(2)
    tgt = torch.randn(B, Sn, T, generator=gen).cuda()
    est = (tgt.flip(1) + 0.3 * torch.randn(B, Sn, T, generator=gen).cuda()).requires_grad_(True)
    loss_fn = NATIVE_LOSS if impl == "native" else EAGER_LOSS

    def step():
        est.grad = None
        loss_fn(est, tgt).backward()
    torch.cuda.empty_cache()
    ms, peak = time_steps(step, steps, warmup)
    return {"loss": "PIT(PairwiseNegSDR('sisdr'))", "B": B, "S": Sn, "T": T, "impl": impl, "fwd_bwd_ms": round(ms, 4),
            "peak_gib": round(peak, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--big-batches", default="16,8,4,2,1", help="U36/2048 batches tried, largest first")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print(json.dumps({"card": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip().splitlines()[:1]}))
    for B in (4, 32):
        for impl in ("native", "native+native_loss", "eager_fp32"):
            try:
                print(json.dumps(run("U16/512", B, impl, a.steps, a.warmup)), flush=True)
            except torch.cuda.OutOfMemoryError:
                print(json.dumps({"model": "U16/512", "B": B, "impl": impl, "error": "out of memory"}), flush=True)
            torch.cuda.empty_cache()
    for impl in ("native", "native+native_loss", "eager_fp32"):
        for B in [int(b) for b in a.big_batches.split(",")]:
            try:
                print(json.dumps(run("U36/2048", B, impl, a.steps, a.warmup)), flush=True)
                break
            except torch.cuda.OutOfMemoryError:
                torch.cuda.empty_cache()
                continue
    for B, Sn, T in ((4, 2, 32000), (32, 2, 32000), (4, 4, 160000)):
        for impl in ("native", "eager_fp32"):
            print(json.dumps(run_loss(B, Sn, T, impl, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
