"""H100-native mirror of ``PermInvariantSNRwithZeroRefs`` in ``sudo_rm_rf/dnn/losses/snr.py``.

The FUSS runner's training loss (run_fuss_separation.py:257-259).  The class keeps the reference's constructor
arguments, ``forward`` signature and return conventions (snr.py:13-142).  Unlike the SI-SDR metrics in ``sisdr.py``
it is differentiable with respect to ``pr_batch``: one fp64 Gram pass and a per-item permutation search
(``sdr_snr_zero_refs``) in the forward, one elementwise kernel (``sdr_snr_zero_refs_backward``) in the backward.
Neither synchronises with the host, so a training step that uses the loss can be captured in a CUDA graph.
"""
import ctypes as C
import itertools

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _native as N


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _forward(est, tgt, zero_mean, threshold, eps):
    """-> (best [B] fp32, permutation index [B] int32, backward coefficients) of fp32 contiguous [B, S, T] inputs."""
    lib = N.lib()
    B, S, T = est.shape
    dev = est.device
    with torch.cuda.device(dev):
        scratch = torch.empty(lib.sdr_snr_zero_refs_scratch_bytes(B, S, T), dtype=torch.uint8, device=dev)
        coef = torch.empty(lib.sdr_snr_zero_refs_coef_bytes(B, S), dtype=torch.uint8, device=dev)
        best = torch.empty(B, dtype=torch.float32, device=dev)
        perm = torch.empty(B, dtype=torch.int32, device=dev)
        N.check(lib.sdr_snr_zero_refs(
            C.c_void_p(est.data_ptr()), C.c_void_p(tgt.data_ptr()), C.c_void_p(best.data_ptr()),
            C.c_void_p(perm.data_ptr()), C.c_void_p(coef.data_ptr()), B, S, T, 1 if zero_mean else 0,
            float(threshold), float(eps), C.c_void_p(scratch.data_ptr()), _stream(dev)), "sdr_snr_zero_refs")
    return best, perm, coef


class _SNRZeroRefs(torch.autograd.Function):
    """best [B] as a function of pr_batch; the permutation index is returned alongside, without a gradient."""

    @staticmethod
    def forward(ctx, pr_batch, est, tgt, zero_mean, threshold, eps):
        best, perm, coef = _forward(est, tgt, zero_mean, threshold, eps)
        ctx.save_for_backward(est, tgt, coef)
        ctx.shape, ctx.dtype = pr_batch.shape, pr_batch.dtype
        ctx.mark_non_differentiable(perm)
        return best, perm

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_best, _grad_perm):
        est, tgt, coef = ctx.saved_tensors
        B, S, T = est.shape
        dev = est.device
        g = grad_best.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            grad = torch.empty(ctx.shape, dtype=torch.float32, device=dev)
            N.check(N.lib().sdr_snr_zero_refs_backward(
                C.c_void_p(est.data_ptr()), C.c_void_p(tgt.data_ptr()), C.c_void_p(coef.data_ptr()),
                C.c_void_p(g.data_ptr()), C.c_void_p(grad.data_ptr()), B, S, T, ctx.shape[-1], _stream(dev)),
                "sdr_snr_zero_refs_backward")
        return grad.to(ctx.dtype), None, None, None, None, None


class PermInvariantSNRwithZeroRefs(nn.Module):
    """Permutation-invariant SNR with compensation for silent references (snr.py:13-142).

    Per item and permutation: the targets whose power is at least ``inactivity_threshold`` dB below the mixture's are
    inactive and weigh 0, the denominators carry a stabiliser of 1e-3 of the target's (active) or the mixture's
    (inactive) power, and the score is the number of active targets times the sum of the per-source SNRs.  Returns
    the best score (negated with ``backward_loss``), its batch mean unless ``return_individual_results``, and
    optionally the best permutations ``[B, n_sources]``.  Gradients flow to ``pr_batch`` only.  1..4 sources."""

    def __init__(self, zero_mean=False, n_sources=None, backward_loss=True, inactivity_threshold=-40.,
                 return_individual_results=False):
        super().__init__()
        self.perform_zero_mean = zero_mean
        self.backward_loss = backward_loss
        self.permutations = list(itertools.permutations(torch.arange(n_sources)))
        self.permutations_tensor = torch.LongTensor(self.permutations)
        self.n_sources = n_sources
        self.inactivity_threshold = inactivity_threshold
        self.return_individual_results = return_individual_results

    def forward(self, pr_batch, t_batch, eps=1e-9, return_best_permutation=False):
        """pr_batch, t_batch ``[B, n_sources, T]`` (the longer one is cropped to the shorter, snr.py:38-42)."""
        if pr_batch.dim() != 3 or t_batch.dim() != 3 or pr_batch.shape[:2] != t_batch.shape[:2] \
                or pr_batch.shape[1] != self.n_sources:
            raise RuntimeError("expected pr_batch and t_batch of shape [B, n_sources, T]")
        if not 1 <= self.n_sources <= 4:
            raise N.NativeError("sdr_snr_zero_refs supports 1..4 sources")
        if t_batch.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("PermInvariantSNRwithZeroRefs computes the gradient with respect to pr_batch only: "
                               "pass a t_batch that does not require grad (e.g. `t_batch.detach()`)")
        if not (pr_batch.is_cuda and t_batch.is_cuda):
            raise RuntimeError("sudo_rm_rf_b200.snr runs on CUDA tensors only (no CPU path)")
        if pr_batch.shape[0] == 0 or min(pr_batch.shape[-1], t_batch.shape[-1]) == 0:
            raise RuntimeError("empty batch or zero-length signals")
        dev = pr_batch.device
        min_len = min(pr_batch.shape[-1], t_batch.shape[-1])
        est = pr_batch.detach()[:, :, :min_len].to(torch.float32).contiguous()
        tgt = t_batch.detach()[:, :, :min_len].to(device=dev, dtype=torch.float32).contiguous()
        if torch.is_grad_enabled() and pr_batch.requires_grad:
            best, perm = _SNRZeroRefs.apply(pr_batch, est, tgt, self.perform_zero_mean,
                                            self.inactivity_threshold, eps)
        else:
            best, perm, _ = _forward(est, tgt, self.perform_zero_mean, self.inactivity_threshold, eps)
        result = best if self.return_individual_results else best.mean()
        if self.backward_loss:
            result = -result
        if return_best_permutation:
            return result, self.permutations_tensor.to(dev)[perm.long()]
        return result
