"""H100-native mirror of the losses and metrics in ``sudo_rm_rf/dnn/losses/sisdr.py``.

``PermInvariantSISDR`` keeps the reference's constructor arguments, ``forward``
signature and return conventions (sisdr.py:66-194), but it is the *metric* the
validation loops compute right after ``model(...)``
(run_improved_sudormrf.py:82-85,201-205): inference only, no autograd.  The
arithmetic (one fp64 Gram pass over the batch + a permutation search per item)
runs in ``libsudormrf_b200.so`` (``sdr_pit_sisdr``).  ``StabilizedPermInvSISDRMetric``
is metric-only as well.

``PITLossWrapper(PairwiseNegSDR("sisdr"), pit_from="pw_mtx")`` is the training loss of
run_improved_sudormrf.py:64-66.  ``PairwiseNegSDR`` is differentiable with respect to
``est_targets``: one fp64 Gram pass (``sdr_pairwise_neg_sdr_train``) in the forward, one
elementwise kernel (``sdr_pairwise_neg_sdr_backward``) in the backward, neither of which
synchronises with the host, so a training step that uses the loss can be captured in a CUDA graph.
"""
import itertools

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _native as N

_PERMS = {}


def _perms(n_src, device):
    """itertools.permutations(range(n_src)) as a long tensor on `device`, made once per (n_src, device): building it
    on every call is a pageable host-to-device copy, which a CUDA graph cannot capture."""
    key = (n_src, device)
    if key not in _PERMS:
        _PERMS[key] = torch.tensor(list(itertools.permutations(range(n_src))), dtype=torch.long, device=device)
    return _PERMS[key]


def _result(metric, best, perm, return_best_permutation):
    """The reference metrics' return conventions: the best score per item (``return_individual_results``) or its batch
    mean, negated with ``backward_loss``, and optionally the best permutations ``[B, n_sources]``."""
    result = best if metric.return_individual_results else best.mean()
    if metric.backward_loss:
        result = -result
    if return_best_permutation:
        return result, metric.permutations_tensor.to(best.device)[perm.long()]
    return result


class PermInvariantSISDR(nn.Module):
    """Permutation-invariant SI-SDR / SI-SDRi of a batch of estimates (sisdr.py:66-194)."""

    def __init__(self, batch_size=None, zero_mean=False, n_sources=None, backward_loss=True,
                 improvement=False, return_individual_results=False):
        super().__init__()
        self.bs = batch_size
        self.perform_zero_mean = zero_mean
        self.backward_loss = backward_loss
        self.permutations = list(itertools.permutations(torch.arange(n_sources)))
        self.permutations_tensor = torch.LongTensor(self.permutations)
        self.improvement = improvement
        self.n_sources = n_sources
        self.return_individual_results = return_individual_results

    def forward(self, pr_batch, t_batch, eps=1e-9, initial_mixtures=None,
                return_best_permutation=False):
        """pr_batch, t_batch ``[B, n_sources, T]``; initial_mixtures ``[B, 1, T]`` (SI-SDRi only).
        Returns what the reference returns: the (negated if ``backward_loss``) best SI-SDR(i), per
        item if ``return_individual_results`` else its batch mean, and optionally the best
        permutations ``[B, n_sources]``."""
        if pr_batch.dim() != 3 or t_batch.dim() != 3 or pr_batch.shape[:2] != t_batch.shape[:2] \
                or pr_batch.shape[1] != self.n_sources:
            raise RuntimeError("expected pr_batch and t_batch of shape [B, n_sources, T]")
        if not (pr_batch.is_cuda and t_batch.is_cuda):
            raise RuntimeError("sudo_rm_rf_b200.sisdr runs on CUDA tensors only (no CPU path)")
        if torch.is_grad_enabled() and (pr_batch.requires_grad or t_batch.requires_grad):
            raise RuntimeError("sudo_rm_rf_b200.sisdr is the evaluation metric only (no autograd): "
                               "wrap the call in torch.no_grad()")
        if self.improvement and initial_mixtures is None:
            raise RuntimeError("improvement=True needs initial_mixtures")
        # normalize_input (sisdr.py:95-112): crop everything to the shortest length
        min_len = min(pr_batch.shape[-1], t_batch.shape[-1])
        if initial_mixtures is not None:
            min_len = min(min_len, initial_mixtures.shape[-1])
        dev = pr_batch.device
        est = pr_batch.detach()[:, :, :min_len].to(torch.float32).contiguous()
        tgt = t_batch.detach()[:, :, :min_len].to(device=dev, dtype=torch.float32).contiguous()
        mix = None
        if initial_mixtures is not None:
            if initial_mixtures.dim() != 3 or initial_mixtures.shape[1] != 1 \
                    or initial_mixtures.shape[0] != est.shape[0]:
                raise RuntimeError("expected initial_mixtures of shape [B, 1, T]")
            mix = initial_mixtures.detach()[:, :, :min_len].to(device=dev, dtype=torch.float32).contiguous()
        B, S, T = est.shape
        lib = N.lib()
        nbytes = lib.sdr_pit_sisdr_scratch_bytes(B, S)
        if nbytes == 0:
            raise N.NativeError("sdr_pit_sisdr supports 1..4 sources")
        with torch.cuda.device(dev):
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            best = torch.empty(B, dtype=torch.float32, device=dev)
            perm = torch.empty(B, dtype=torch.int32, device=dev)
            N.check(lib.sdr_pit_sisdr(
                N.ptr(est), N.ptr(tgt), N.ptr(mix if self.improvement else None), N.ptr(best), N.ptr(perm), B, S, T,
                1 if self.perform_zero_mean else 0, 1 if self.improvement else 0, float(eps),
                N.ptr(scratch), N.stream(dev)), "sdr_pit_sisdr")
        return _result(self, best, perm, return_best_permutation)


class StabilizedPermInvSISDRMetric(nn.Module):
    """Stabilised permutation-invariant SI-SDR(i) with more estimated than actual sources (sisdr.py:460-591), the
    validation metric of ``run_fuss_separation.py:111-131``: same constructor, ``forward`` signature and return
    conventions as the reference class.  Metric only (no autograd); one fp64 Gram pass + an assignment search per item
    in ``libsudormrf_b200.so`` (``sdr_stabilized_sisdr``).  Up to 4 estimated sources."""

    def __init__(self, zero_mean=False, single_source=False, n_estimated_sources=None, n_actual_sources=None,
                 backward_loss=True, improvement=False, return_individual_results=False):
        super().__init__()
        self.perform_zero_mean = zero_mean
        self.backward_loss = backward_loss
        self.improvement = improvement
        self.n_estimated_sources = n_estimated_sources
        self.n_actual_sources = n_actual_sources
        assert self.n_estimated_sources >= self.n_actual_sources, (
            'Estimates need to be at least: {} but got: {}'.format(
                self.n_actual_sources, self.n_estimated_sources))
        self.permutations = list(itertools.permutations(
            torch.arange(self.n_estimated_sources), r=self.n_actual_sources))
        self.permutations_tensor = torch.LongTensor(self.permutations)
        self.return_individual_results = return_individual_results
        self.single_source = single_source
        if self.single_source:
            assert self.n_actual_sources == 1

    def forward(self, pr_batch, t_batch, eps=1e-9, return_best_permutation=False):
        """pr_batch ``[B, rows, T]``, t_batch ``[B, n_actual, T]``.  Without ``single_source`` the first
        ``n_estimated_sources`` rows are scored and any further rows are ignored, as in the reference; with it, every
        row is summed into the one estimate."""
        if pr_batch.dim() != 3 or t_batch.dim() != 3 or pr_batch.shape[0] != t_batch.shape[0] \
                or pr_batch.shape[-1] != t_batch.shape[-1]:
            raise RuntimeError("expected pr_batch [B, n_estimated, T] and t_batch [B, n_actual, T]")
        if t_batch.shape[1] != self.n_actual_sources:
            raise RuntimeError(f"expected {self.n_actual_sources} actual sources, got {t_batch.shape[1]}")   # sisdr.py:521
        if not self.single_source and pr_batch.shape[1] < self.n_estimated_sources:
            raise RuntimeError(f"expected at least {self.n_estimated_sources} estimated sources, got {pr_batch.shape[1]}")
        if self.single_source and self.n_estimated_sources != 1:
            raise RuntimeError("single_source sums the estimates into one: construct the metric with "
                               "n_estimated_sources=1 (the reference's permutation table indexes the summed tensor)")
        if not (pr_batch.is_cuda and t_batch.is_cuda):
            raise RuntimeError("sudo_rm_rf_b200.sisdr runs on CUDA tensors only (no CPU path)")
        if torch.is_grad_enabled() and (pr_batch.requires_grad or t_batch.requires_grad):
            raise RuntimeError("sudo_rm_rf_b200.sisdr is the evaluation metric only (no autograd): "
                               "wrap the call in torch.no_grad()")
        dev = pr_batch.device
        if not self.single_source:
            # the assignments index rows 0 .. n_estimated - 1 only (sisdr.py:490-492,526-527): run_fuss_separation.py
            # scores its one-source set with n_estimated_sources=1 on every output row of the model
            pr_batch = pr_batch[:, :self.n_estimated_sources]
        est = pr_batch.detach().to(torch.float32).contiguous()
        tgt = t_batch.detach().to(device=dev, dtype=torch.float32).contiguous()
        B, rows, T = est.shape
        lib = N.lib()
        nbytes = lib.sdr_stabilized_sisdr_scratch_bytes(B, self.n_estimated_sources, self.n_actual_sources)
        if nbytes == 0:
            raise N.NativeError("sdr_stabilized_sisdr supports 1 <= n_actual <= n_estimated <= 4 sources")
        with torch.cuda.device(dev):
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            best = torch.empty(B, dtype=torch.float32, device=dev)
            perm = torch.empty(B, dtype=torch.int32, device=dev)
            N.check(lib.sdr_stabilized_sisdr(
                N.ptr(est), N.ptr(tgt), N.ptr(best), N.ptr(perm), B, rows, self.n_estimated_sources,
                self.n_actual_sources, T,
                1 if self.perform_zero_mean else 0, 1 if self.improvement else 0, float(eps),
                N.ptr(scratch), N.stream(dev)), "sdr_stabilized_sisdr")
        return _result(self, best, perm, return_best_permutation)


class _PairwiseNegSDR(torch.autograd.Function):
    """The [B, S, S] pairwise losses as a function of est_targets (fp32 contiguous copies est, tgt are passed along)."""

    @staticmethod
    def forward(ctx, est_targets, est, tgt, sdr_type, zero_mean, take_log):
        lib = N.lib()
        B, S, T = est.shape
        dev = est.device
        with torch.cuda.device(dev):
            scratch = torch.empty(lib.sdr_pairwise_neg_sdr_train_scratch_bytes(B, S, T), dtype=torch.uint8, device=dev)
            coef = torch.empty(lib.sdr_pairwise_neg_sdr_coef_bytes(B, S), dtype=torch.uint8, device=dev)
            out = torch.empty((B, S, S), dtype=torch.float32, device=dev)
            N.check(lib.sdr_pairwise_neg_sdr_train(
                N.ptr(est), N.ptr(tgt), N.ptr(out), N.ptr(coef), B, S, T, sdr_type, 1 if zero_mean else 0,
                1 if take_log else 0,
                N.ptr(scratch), N.stream(dev)), "sdr_pairwise_neg_sdr_train")
        ctx.save_for_backward(est, tgt, coef)
        ctx.dtype = est_targets.dtype
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        est, tgt, coef = ctx.saved_tensors
        B, S, T = est.shape
        dev = est.device
        g = grad_out.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            grad = torch.empty((B, S, T), dtype=torch.float32, device=dev)
            N.check(N.lib().sdr_pairwise_neg_sdr_backward(
                N.ptr(est), N.ptr(tgt), N.ptr(coef), N.ptr(g), N.ptr(grad), B, S, T, N.stream(dev)),
                "sdr_pairwise_neg_sdr_backward")
        return grad.to(ctx.dtype), None, None, None, None, None


class PairwiseNegSDR(nn.Module):
    """Pairwise negative SNR / SI-SDR / SD-SDR on a batch (sisdr.py:372-457): same constructor and ``forward``
    as the reference class; returns ``[batch, n_src, n_src]`` fp32 with ``[b, i, j] = -sdr(estimate i, target j)``.
    The arithmetic is one fp64 Gram pass in ``libsudormrf_b200.so``.  With grad mode on and ``est_targets`` requiring
    grad the result is differentiable with respect to ``est_targets`` (the gradient comes back in its dtype; fp16,
    bf16 and fp64 inputs are computed on in fp32), its Gram sums are added in a fixed order, and a forward and a
    backward are bitwise reproducible.  Gradients with respect to ``targets`` are not computed: ``targets`` that
    require grad are refused.  1..4 sources."""
    _TYPES = {"snr": 0, "sisdr": 1, "sdsdr": 2}

    def __init__(self, sdr_type, zero_mean=True, take_log=True):
        super().__init__()
        assert sdr_type in ["snr", "sisdr", "sdsdr"]
        self.sdr_type = sdr_type
        self.zero_mean = zero_mean
        self.take_log = take_log

    def forward(self, est_targets, targets):
        assert targets.size() == est_targets.size()
        if est_targets.dim() != 3:
            raise RuntimeError("expected est_targets and targets of shape [batch, n_src, time]")
        if not 1 <= est_targets.shape[1] <= 4:
            raise N.NativeError("sdr_pairwise_neg_sdr supports 1..4 sources")
        if torch.is_grad_enabled() and targets.requires_grad:
            raise RuntimeError("PairwiseNegSDR computes the gradient with respect to est_targets only: "
                               "pass targets that do not require grad (e.g. `targets.detach()`)")
        if not (est_targets.is_cuda and targets.is_cuda):
            raise RuntimeError("sudo_rm_rf_b200.sisdr runs on CUDA tensors only (no CPU path)")
        dev = est_targets.device
        est = est_targets.detach().to(torch.float32).contiguous()
        tgt = targets.detach().to(device=dev, dtype=torch.float32).contiguous()
        if torch.is_grad_enabled() and est_targets.requires_grad:
            return _PairwiseNegSDR.apply(est_targets, est, tgt, self._TYPES[self.sdr_type], self.zero_mean,
                                         self.take_log)
        B, S, T = est.shape
        lib = N.lib()
        nbytes = lib.sdr_pit_sisdr_scratch_bytes(B, S)
        if nbytes == 0:
            raise N.NativeError("sdr_pairwise_neg_sdr supports 1..4 sources")
        with torch.cuda.device(dev):
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            out = torch.empty((B, S, S), dtype=torch.float32, device=dev)
            N.check(lib.sdr_pairwise_neg_sdr(
                N.ptr(est), N.ptr(tgt), N.ptr(out), B, S, T,
                self._TYPES[self.sdr_type], 1 if self.zero_mean else 0, 1 if self.take_log else 0,
                N.ptr(scratch), N.stream(dev)), "sdr_pairwise_neg_sdr")
        return out


class PITLossWrapper(nn.Module):
    """Permutation-invariant wrapper (sisdr.py:197-369): same constructor, ``forward`` signature and return
    conventions as the reference class.  The pairwise matrix comes from ``loss_func`` (``PairwiseNegSDR`` above for
    ``pit_from='pw_mtx'``); the search over the n_src! permutations works on that ``[batch, n_src, n_src]`` tensor
    with a handful of tiny torch ops, exactly as the reference does (host logic, not a hot path), and gradients flow
    through them to whatever ``loss_func`` differentiates.  The permutation table is made once per (n_src, device),
    so a training step through ``PairwiseNegSDR`` and ``pit_from='pw_mtx'`` can be captured in a CUDA graph.  The
    reference's copy calls ``best_perm_from_perm_avg_loss`` / ``reorder_source`` without defining them (``pit_from='perm_avg'`` and
    ``return_est=True`` raise there); the two helpers below follow the asteroid definitions the file was copied from."""

    def __init__(self, loss_func, pit_from="pw_mtx", perm_reduce=None):
        super().__init__()
        self.loss_func = loss_func
        self.pit_from = pit_from
        self.perm_reduce = perm_reduce
        if self.pit_from not in ["pw_mtx", "pw_pt", "perm_avg"]:
            raise ValueError("Unsupported loss function type for now. Expected"
                             "one of [`pw_mtx`, `pw_pt`, `perm_avg`]")

    def forward(self, est_targets, targets, return_est=False, reduce_kwargs=None, **kwargs):
        n_src = targets.shape[1]
        assert n_src < 10, f"Expected source axis along dim 1, found {n_src}"
        if self.pit_from == "pw_mtx":
            pw_losses = self.loss_func(est_targets, targets, **kwargs)
        elif self.pit_from == "pw_pt":
            pw_losses = self.get_pw_losses(self.loss_func, est_targets, targets, **kwargs)
        else:
            min_loss, min_loss_idx = self.best_perm_from_perm_avg_loss(self.loss_func, est_targets, targets, **kwargs)
            mean_loss = torch.mean(min_loss)
            if not return_est:
                return mean_loss
            return mean_loss, self.reorder_source(est_targets, n_src, min_loss_idx)
        assert pw_losses.ndim == 3, "Something went wrong with the loss function, please read the docs."
        assert pw_losses.shape[0] == targets.shape[0], "PIT loss needs same batch dim as input"
        reduce_kwargs = reduce_kwargs if reduce_kwargs is not None else dict()
        min_loss, min_loss_idx = self.find_best_perm(pw_losses, n_src, perm_reduce=self.perm_reduce, **reduce_kwargs)
        mean_loss = torch.mean(min_loss)
        if not return_est:
            return mean_loss
        return mean_loss, self.reorder_source(est_targets, n_src, min_loss_idx)

    @staticmethod
    def get_pw_losses(loss_func, est_targets, targets, **kwargs):
        batch_size, n_src = targets.shape[:2]
        pw = targets.new_empty(batch_size, n_src, n_src)
        for ei, est_src in enumerate(est_targets.transpose(0, 1)):
            for ti, target_src in enumerate(targets.transpose(0, 1)):
                pw[:, ei, ti] = loss_func(est_src, target_src, **kwargs)
        return pw

    @staticmethod
    def find_best_perm(pair_wise_losses, n_src, perm_reduce=None, **kwargs):
        pwl = pair_wise_losses.transpose(-1, -2)             # dim 1: sources, dim 2: estimates
        perms = _perms(n_src, pwl.device)
        idx = torch.unsqueeze(perms, 2)
        if perm_reduce is None:
            one_hot = pwl.new_zeros((*perms.size(), n_src)).scatter_(2, idx, 1)
            loss_set = torch.einsum("bij,pij->bp", [pwl, one_hot]) / n_src
        else:
            pwl_set = pwl[:, torch.arange(n_src), idx.squeeze(-1)]
            loss_set = perm_reduce(pwl_set, **kwargs)
        min_loss_idx = torch.argmin(loss_set, dim=1)
        min_loss, _ = torch.min(loss_set, dim=1, keepdim=True)
        return min_loss, min_loss_idx

    @staticmethod
    def best_perm_from_perm_avg_loss(loss_func, est_targets, targets, **kwargs):
        n_src = targets.shape[1]
        perms = list(itertools.permutations(range(n_src)))
        loss_set = torch.stack([loss_func(est_targets[:, perm], targets, **kwargs) for perm in perms], dim=1)
        min_loss, min_loss_idx = torch.min(loss_set, dim=1, keepdim=True)
        return min_loss, min_loss_idx[:, 0]

    @staticmethod
    def reorder_source(source, n_src, min_loss_idx):
        perms = _perms(n_src, source.device)
        min_loss_perm = torch.index_select(perms, dim=0, index=min_loss_idx)
        return torch.stack([torch.index_select(s, 0, b) for s, b in zip(source, min_loss_perm)])
