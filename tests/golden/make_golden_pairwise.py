"""Golden fixtures for the improved model's training loss, generated from the UNMODIFIED reference on the CPU in fp64.
Needs a checkout of the original sudo_rm_rf repository, named by SUDO_RM_RF_REFERENCE:

    SUDO_RM_RF_REFERENCE=/path/to/sudo_rm_rf python tests/golden/make_golden_pairwise.py

``prepost_pairwise_grad.npz`` holds, per case, ``PairwiseNegSDR`` (dnn/losses/sisdr.py:372-457) and
``PITLossWrapper(..., pit_from='pw_mtx')`` (sisdr.py:197-369) on top of it, for every sdr_type and (zero_mean, take_log)
combination, 1..4 sources and short odd lengths, and for degenerate items (a silent target, a constant estimate row, an
estimate equal to its target).  Stored: the inputs, the pairwise matrix and the autograd gradient with respect to
``est_targets`` of ``sum(pw * w)`` (``w`` is stored too), the wrapper's loss and its gradient.
The inputs are fp32 values (stored as fp32, computed on in fp64); every result is stored in fp64.
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

import sudo_rm_rf.dnn.losses.sisdr as ref_sisdr                             # noqa: E402

D = torch.float64
TYPES = ("snr", "sisdr", "sdsdr")
FLAGS = ((False, False), (False, True), (True, False), (True, True))


def f32(x):
    """fp64 tensor of fp32-representable values, so the stored fp32 inputs are exactly what the reference ran on."""
    return x.float().double()


def signals(S, B, T, g):
    """Targets with different powers and a DC offset, estimates a permuted, noisy, scaled copy of them."""
    tgt = torch.randn(B, S, T, generator=g, dtype=D) * (0.2 + torch.rand(B, S, 1, generator=g, dtype=D)) + 0.05
    est = torch.stack([tgt[b, torch.randperm(S, generator=g)] for b in range(B)])
    est = est * 0.8 + torch.randn(B, S, T, generator=g, dtype=D) * torch.logspace(-2, -0.3, B, dtype=D).view(B, 1, 1)
    return f32(est), f32(tgt)


def cases():
    g = torch.Generator().manual_seed(4242)
    out = []
    for sdr_type in TYPES:
        for zero_mean, take_log in FLAGS:
            for S, B, T in ((1, 2, 17), (2, 3, 19), (3, 2, 21), (4, 2, 23)):
                est, tgt = signals(S, B, T, g)
                out.append(dict(name="flags", sdr_type=sdr_type, zero_mean=zero_mean, take_log=take_log, S=S,
                                est=est, tgt=tgt))
            est, tgt = signals(3, 3, 25, g)
            tgt[0, 0] = 0.0                                                  # a silent target
            est[1, 1] = 0.375                                                # a constant estimate row
            est[2, 2] = tgt[2, 2]                                            # an estimate equal to its target
            out.append(dict(name="degenerate", sdr_type=sdr_type, zero_mean=zero_mean, take_log=take_log, S=3,
                            est=est, tgt=tgt))
    return out


def make():
    arrays, metas = {}, []
    g = torch.Generator().manual_seed(99)
    for ci, c in enumerate(cases()):
        est, tgt = c.pop("est"), c.pop("tgt")
        fn = ref_sisdr.PairwiseNegSDR(c["sdr_type"], zero_mean=c["zero_mean"], take_log=c["take_log"])
        e = est.clone().requires_grad_(True)
        pw = fn(e, tgt)
        w = f32(torch.rand(pw.shape, generator=g, dtype=D) + 0.5)
        (pw * w).sum().backward()
        e2 = est.clone().requires_grad_(True)
        loss = ref_sisdr.PITLossWrapper(fn, pit_from="pw_mtx")(e2, tgt)
        loss.backward()
        k = f"c{ci}/"
        arrays.update({k + "est": est.float().numpy(), k + "tgt": tgt.float().numpy(), k + "w": w.float().numpy(),
                       k + "pw": pw.detach().numpy(), k + "grad": e.grad.numpy(),
                       k + "pit_loss": loss.detach().numpy(), k + "pit_grad": e2.grad.numpy()})
        metas.append(c)
        print(f"c{ci} {c['name']} {c['sdr_type']} zm={c['zero_mean']} log={c['take_log']} S={c['S']}: "
              f"loss={float(loss):.4f}")
    arrays["meta"] = np.frombuffer(json.dumps(dict(cases=metas, torch=torch.__version__)).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "prepost_pairwise_grad.npz")
    np.savez_compressed(path, **arrays)
    print(f"{len(metas)} cases -> {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    make()
