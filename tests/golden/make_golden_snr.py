"""Golden fixtures for the FUSS training step after the model, generated from the UNMODIFIED reference on the CPU in
fp64.  Needs a checkout of the original sudo_rm_rf repository, named by SUDO_RM_RF_REFERENCE:

    SUDO_RM_RF_REFERENCE=/path/to/sudo_rm_rf python tests/golden/make_golden_snr.py

``prepost_snr_zero_refs.npz`` holds, per case:
* ``snr``: ``PermInvariantSNRwithZeroRefs`` (dnn/losses/snr.py:13-142) for 1..4 sources with every flag combination,
  non-default ``inactivity_threshold`` and ``eps``, degenerate items (a silent target, a target below -40 dB, an
  all-silent item, two identical estimates) and both crops.  Stored: the inputs, the returned value, the best
  permutations and the autograd gradient with respect to ``pr_batch`` of ``sum(value * w)`` (``w`` is stored too).
* ``mc``: ``mixture_consistency.apply`` (experiments/utils/mixture_consistency.py:14-36) for both weight types, with
  the autograd gradients of ``sum(out * g)`` with respect to both inputs.
The inputs are fp32 values (stored as fp32, computed on in fp64); every result is stored in fp64.  The signals are
short: the restatement's arithmetic does not depend on the length, and the file stays small.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ["SUDO_RM_RF_REFERENCE"])
warnings.filterwarnings("ignore")

import sudo_rm_rf.dnn.losses.snr as ref_snr                                 # noqa: E402
import sudo_rm_rf.dnn.experiments.utils.mixture_consistency as ref_mc     # noqa: E402

D = torch.float64


def signals(S, B, T, g, Tp=None):
    """Targets with different powers, estimates a permuted, noisy, scaled copy of them."""
    Tp = T if Tp is None else Tp
    n = max(T, Tp)
    tgt = torch.randn(B, S, n, generator=g, dtype=D) * (0.2 + torch.rand(B, S, 1, generator=g, dtype=D)) + 0.05
    est = torch.stack([tgt[b, torch.randperm(S, generator=g)] for b in range(B)])
    est = est * 0.8 + torch.randn(B, S, n, generator=g, dtype=D) * torch.logspace(-2, -0.3, B, dtype=D).view(B, 1, 1)
    return f32(est[:, :, :Tp].contiguous()), f32(tgt[:, :, :T].contiguous())


def f32(x):
    """fp64 tensor of fp32-representable values, so the stored fp32 inputs are exactly what the reference ran on."""
    return x.float().double()


def snr_cases():
    g = torch.Generator().manual_seed(9090)
    cases = []
    for S, B, T in ((1, 2, 19), (2, 2, 23), (3, 3, 20), (4, 2, 24)):
        for zero_mean in (False, True):
            for backward_loss in (False, True):
                for individual in (False, True):
                    est, tgt = signals(S, B, T, g)
                    cases.append(dict(S=S, zero_mean=zero_mean, backward_loss=backward_loss, individual=individual,
                                      thr=-40., eps=1e-9, name="flags", est=est, tgt=tgt))
    for thr, eps in ((-20., 1e-9), (-60., 1e-6), (-40., 0.0), (-10., 1e-3)):
        est, tgt = signals(4, 4, 24, g)
        tgt[0, 3] *= 0.03                                                # -30 dB: inactive at -20 and -10 only
        cases.append(dict(S=4, zero_mean=False, backward_loss=True, individual=True, thr=thr, eps=eps,
                          name=f"thr{thr:g}_eps{eps:g}", est=est, tgt=tgt))
    for S in (2, 3, 4):
        for zero_mean in (False, True):
            est, tgt = signals(S, 4, 20, g)
            tgt[0, 0] = 0.0                                              # a silent target
            tgt[1, S - 1] *= 1e-3                                        # a target 60 dB below the rest
            tgt[2] = 0.0                                                 # an all-silent item: num_active = 0
            est[3, 1] = est[3, 0]                                        # two identical estimates
            cases.append(dict(S=S, zero_mean=zero_mean, backward_loss=True, individual=True, thr=-40., eps=1e-9,
                              name="degenerate", est=est, tgt=tgt))
    for S, T, Tp in ((3, 20, 25), (4, 24, 19), (2, 20, 21)):
        for zero_mean in (False, True):
            est, tgt = signals(S, 3, T, g, Tp)
            cases.append(dict(S=S, zero_mean=zero_mean, backward_loss=True, individual=False, thr=-40., eps=1e-9,
                              name="crop", est=est, tgt=tgt))
    return cases


def make():
    arrays, metas = {}, []
    g = torch.Generator().manual_seed(77)
    for ci, c in enumerate(snr_cases()):
        est = f32(c.pop("est")).requires_grad_(True)              # after the edits above: fp32 values again
        tgt = f32(c.pop("tgt"))
        fn = ref_snr.PermInvariantSNRwithZeroRefs(zero_mean=c["zero_mean"], n_sources=c["S"],
                                                  backward_loss=c["backward_loss"], inactivity_threshold=c["thr"],
                                                  return_individual_results=c["individual"])
        value, perms = fn(est, tgt, eps=c["eps"], return_best_permutation=True)
        w = f32(torch.rand(value.shape, generator=g, dtype=D) + 0.5)
        (value * w).sum().backward()
        k = f"snr{ci}/"
        arrays.update({k + "est": est.detach().float().numpy(), k + "tgt": tgt.float().numpy(),
                       k + "value": value.detach().numpy(), k + "perms": perms.numpy(), k + "w": w.float().numpy(),
                       k + "grad": est.grad.numpy()})
        metas.append(c)
        print(f"snr{ci} {c['name']} S={c['S']}: value={value.detach().numpy().round(3)}")
    mc = []
    for mi, (S, B, T, kind) in enumerate(((1, 2, 20, "uniform"), (2, 3, 21, "uniform"), (3, 2, 17, "uniform"),
                                          (4, 3, 24, "uniform"), (1, 2, 20, "magsq"), (2, 3, 21, "magsq"),
                                          (3, 2, 17, "magsq"), (4, 3, 24, "magsq"))):
        est = f32(torch.randn(B, S, T, generator=g, dtype=D) * torch.rand(B, S, 1, generator=g, dtype=D)).requires_grad_(True)
        mix = f32(torch.randn(B, 1, T, generator=g, dtype=D)).requires_grad_(True)
        gout = f32(torch.randn(B, S, T, generator=g, dtype=D))
        out = ref_mc.apply(est, mix, kind)
        (out * gout).sum().backward()
        k = f"mc{mi}/"
        arrays.update({k + "est": est.detach().float().numpy(), k + "mix": mix.detach().float().numpy(),
                       k + "g": gout.float().numpy(),
                       k + "out": out.detach().numpy(), k + "grad_est": est.grad.numpy(),
                       k + "grad_mix": mix.grad.numpy()})
        mc.append(dict(S=S, B=B, T=T, kind=kind))
    arrays["meta"] = np.frombuffer(json.dumps(dict(snr=metas, mc=mc, torch=torch.__version__)).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "prepost_snr_zero_refs.npz")
    np.savez_compressed(path, **arrays)
    print(f"{len(metas)} snr cases, {len(mc)} mc cases -> {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    make()
