"""H100-native mirror of ``sudo_rm_rf/dnn/experiments/utils/mixture_consistency.py``."""
import ctypes as C

import torch

from . import _native as N


def apply(pr_batch, input_mixture, mix_weights_type='uniform'):
    """Mixture consistency (mixture_consistency.py:14-36).

    pr_batch [B, S, T], input_mixture [B, 1, T] -> pr_batch + w * (mixture - sum_s pr_batch),
    w = 1/S ('uniform') or the normalised mean power of each estimate ('magsq').
    """
    if mix_weights_type not in ('uniform', 'magsq'):
        raise ValueError('Invalid mixture consistency weight type: {}'.format(mix_weights_type))
    if pr_batch.dim() != 3 or input_mixture.dim() != 3 or input_mixture.shape[1] != 1 \
            or input_mixture.shape[0] != pr_batch.shape[0] \
            or input_mixture.shape[2] != pr_batch.shape[2]:
        raise RuntimeError("expected pr_batch [B,S,T] and input_mixture [B,1,T]")
    if not (pr_batch.is_cuda and input_mixture.is_cuda):
        raise RuntimeError("sudo_rm_rf_b200.mixture_consistency runs on CUDA tensors only")
    lib = N.lib()
    est = pr_batch.detach().to(torch.float32).contiguous()
    mix = input_mixture.detach().to(torch.float32).contiguous()
    B, S, T = est.shape
    out = torch.empty_like(est)
    with torch.cuda.device(est.device):
        scratch = torch.empty(B * S, dtype=torch.float64, device=est.device) \
            if mix_weights_type == 'magsq' else None
        N.check(lib.sdr_mixture_consistency(
            C.c_void_p(est.data_ptr()), C.c_void_p(mix.data_ptr()), C.c_void_p(out.data_ptr()),
            B, S, T, 1 if mix_weights_type == 'magsq' else 0,
            C.c_void_p(scratch.data_ptr() if scratch is not None else 0),
            C.c_void_p(torch.cuda.current_stream(est.device).cuda_stream)),
            "sdr_mixture_consistency")
    return out
