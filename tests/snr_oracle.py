"""fp64-capable, autograd-differentiable restatement of ``PermInvariantSNRwithZeroRefs.forward`` (the FUSS training
loss, dnn/losses/snr.py:38-116 of the reference), written from its formulas.  Pinned to the unmodified reference by
``tests/golden/make_golden_snr.py`` (tests/test_snr_cpu.py), and the checker of the native loss on the GPU
(tests/test_gpu_snr.py)."""
import itertools

import torch


def snr_zero_refs(pr, tgt, zero_mean=False, inactivity_threshold=-40., eps=1e-9):
    """backward_loss=False, return_individual_results=True: returns (best [B], index of the best permutation [B]) with
    the permutations in itertools.permutations(range(S)) order (snr.py:31-32), differentiable with respect to pr."""
    n = min(pr.shape[-1], tgt.shape[-1])                                  # snr.py:39-42
    pr, tgt = pr[:, :, :n], tgt[:, :, :n]
    if zero_mean:                                                         # snr.py:44-48
        pr = pr - pr.mean(-1, keepdim=True)
        tgt = tgt - tgt.mean(-1, keepdim=True)

    def dot(a, b):                                                        # snr.py:52-53
        return torch.sum(a * b, dim=-1, keepdim=True)

    S = pr.shape[1]
    mix = tgt.sum(-2, keepdim=True)                                       # snr.py:86-97
    mix_pow = dot(mix, mix)
    tgt_pow = dot(tgt, tgt)
    active = (10. * torch.log10(tgt_pow / (mix_pow + eps))).ge(inactivity_threshold)
    stab = 0.001 * (active * tgt_pow + (~active) * mix_pow.repeat(1, S, 1))
    num_active = active.sum([-2, -1]).unsqueeze(-1)
    nom = tgt_pow + eps                                                   # snr.py:62-68
    cols = []
    for perm in itertools.permutations(range(S)):                         # snr.py:100-106
        err = pr[:, list(perm), :] - tgt
        cols.append(10. * active * torch.log10(nom / (dot(err, err) + stab + eps) + eps))
    return torch.max(torch.cat(cols, -1).sum(-2) * num_active, -1)       # snr.py:108-109
