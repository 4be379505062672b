"""H100-native mirror of ``sudo_rm_rf/dnn/experiments/utils/mixture_consistency.py``."""
import torch
from torch.autograd.function import once_differentiable

from . import _native as N


def _project(est, mix, magsq):
    """sdr_mixture_consistency on fp32 contiguous [B, S, T] / [B, 1, T] -> a new fp32 tensor (no graph)."""
    lib = N.lib()
    B, S, T = est.shape
    out = torch.empty_like(est)
    with torch.cuda.device(est.device):
        scratch = torch.empty(B * S, dtype=torch.float64, device=est.device) if magsq else None
        N.check(lib.sdr_mixture_consistency(N.ptr(est), N.ptr(mix), N.ptr(out), B, S, T, 1 if magsq else 0,
                                            N.ptr(scratch), N.stream(est.device)), "sdr_mixture_consistency")
    return out


class _Consistency(torch.autograd.Function):
    """Forward: the same sdr_mixture_consistency call (bitwise the no-grad result).  Backward:
    sdr_mixture_consistency_backward, gradients in the inputs' dtypes."""

    @staticmethod
    def forward(ctx, pr_batch, input_mixture, magsq):
        est = pr_batch.detach().to(torch.float32).contiguous()
        mix = input_mixture.detach().to(torch.float32).contiguous()
        ctx.magsq = magsq
        ctx.dtypes = (pr_batch.dtype, input_mixture.dtype)
        ctx.save_for_backward(est, mix)
        return _project(est, mix, magsq)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        est, mix = ctx.saved_tensors
        lib = N.lib()
        B, S, T = est.shape
        dev = est.device
        g = grad_out.to(torch.float32).contiguous()
        want_mix = ctx.needs_input_grad[1]
        with torch.cuda.device(dev):
            nbytes = lib.sdr_mixture_consistency_backward_scratch_bytes(B, S, T, 1 if ctx.magsq else 0)
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
            grad_est = torch.empty_like(est)
            grad_mix = torch.empty_like(mix) if want_mix else None
            N.check(lib.sdr_mixture_consistency_backward(
                N.ptr(est), N.ptr(mix), N.ptr(g), N.ptr(grad_est), N.ptr(grad_mix), B, S, T, 1 if ctx.magsq else 0,
                N.ptr(scratch), N.stream(dev)), "sdr_mixture_consistency_backward")
        return (grad_est.to(ctx.dtypes[0]) if ctx.needs_input_grad[0] else None,
                grad_mix.to(ctx.dtypes[1]) if want_mix else None, None)


def apply(pr_batch, input_mixture, mix_weights_type='uniform'):
    """Mixture consistency (mixture_consistency.py:14-36).

    pr_batch [B, S, T], input_mixture [B, 1, T] -> pr_batch + w * (mixture - sum_s pr_batch),
    w = 1/S ('uniform') or the normalised mean power of each estimate ('magsq').  With grad mode on and an input that
    requires grad the result carries a ``grad_fn`` (the projection is differentiable, as in the reference); otherwise
    it is a plain fp32 tensor.
    """
    if mix_weights_type not in ('uniform', 'magsq'):
        raise ValueError('Invalid mixture consistency weight type: {}'.format(mix_weights_type))
    if pr_batch.dim() != 3 or input_mixture.dim() != 3 or input_mixture.shape[1] != 1 \
            or input_mixture.shape[0] != pr_batch.shape[0] \
            or input_mixture.shape[2] != pr_batch.shape[2]:
        raise RuntimeError("expected pr_batch [B,S,T] and input_mixture [B,1,T]")
    if not (pr_batch.is_cuda and input_mixture.is_cuda):
        raise RuntimeError("sudo_rm_rf_b200.mixture_consistency runs on CUDA tensors only")
    magsq = mix_weights_type == 'magsq'
    if torch.is_grad_enabled() and (pr_batch.requires_grad or input_mixture.requires_grad):
        return _Consistency.apply(pr_batch, input_mixture, magsq)
    return _project(pr_batch.detach().to(torch.float32).contiguous(),
                    input_mixture.detach().to(torch.float32).contiguous(), magsq)
