"""Autograd through the native path of the improved SuDORMRF (``enable_training()``).

``_NativeTrain`` is one ``torch.autograd.Function`` whose inputs are the mixture and every parameter in
``state_dict`` order, so ``nn.DataParallel``'s broadcast routes each replica's parameter gradients back to the
master.  Its forward is ``sdr_forward_train`` (the inference forward's kernels, plus a copy of the block inputs, the
encoder output and the statistics into a per-call ``saved`` buffer); its backward is ``sdr_backward``, which
recomputes each block's internals from its saved input and writes every parameter gradient.  The gradient with
respect to the mixture is not built, and double backward is not supported.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch.autograd.function import once_differentiable

from . import _engine
from . import _native as N


def wants_autograd(model, wav: torch.Tensor) -> bool:
    """True when ``model(wav)`` has to be differentiable: training enabled, grad mode on, a parameter requires grad."""
    if not getattr(model, "native_training", False) or not torch.is_grad_enabled():
        return False
    return any(_engine._fetch(model, n).requires_grad for n in _engine._probe_names(model)) or \
        bool(getattr(wav, "requires_grad", False))


def _check(model, cfg, wav: torch.Tensor) -> torch.Tensor:
    if wav.requires_grad:
        raise RuntimeError("sudo_rm_rf_b200 training computes parameter gradients only: the gradient with respect "
                           "to the mixture is not built, so pass a mixture that does not require grad "
                           "(e.g. `mixture.detach()`).")
    _engine._check_mixture(cfg, wav)
    return wav.to(torch.float32).contiguous()


class _NativeTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, cfg, wav, *params):
        lib = N.lib()
        device = wav.device
        B, _, T = wav.shape
        unsupported = "configuration not supported by the training path"
        saved_bytes = lib.sdr_train_saved_bytes(C.byref(cfg), B, T)
        if saved_bytes == 0:
            raise N.NativeError(unsupported)
        # per call, so that several forwards before one backward keep their own activations
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device=device)
        out = torch.empty((B, cfg.num_sources, T), dtype=torch.float32, device=device)

        def enqueue(packed, ws):
            N.check(lib.sdr_forward_train(C.byref(cfg), N.ptr(packed), N.ptr(wav), N.ptr(out), B, T, N.ptr(saved),
                                          saved.numel(), N.ptr(ws), ws.numel(), N.stream(device)), "sdr_forward_train")
        packed = _engine._call_shared(model, cfg, device, lib.sdr_workspace_bytes(C.byref(cfg), B, T), unsupported,
                                      enqueue)
        ctx.cfg = cfg
        ctx.packed = packed          # the weights this forward ran with, whatever a later forward packs
        ctx.saved = saved
        # the parameters go through save_for_backward so that an in-place update before backward raises
        ctx.save_for_backward(wav, *params)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        lib = N.lib()
        wav, *params = ctx.saved_tensors
        cfg = ctx.cfg
        device = wav.device
        B, _, T = wav.shape
        g = grad_out.to(torch.float32).contiguous()
        with torch.cuda.device(device):
            ws_bytes = lib.sdr_backward_workspace_bytes(C.byref(cfg), B, T)
            if ws_bytes == 0:
                raise N.NativeError("configuration not supported by the training path")
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            numel = [p.numel() for p in params]
            flat = torch.empty(sum(numel), dtype=torch.float32, device=device)
            N.check(lib.sdr_backward(C.byref(cfg), N.ptr(ctx.packed), N.ptr(wav), N.ptr(ctx.saved), N.ptr(g),
                                     N.ptr(flat), B, T, N.ptr(ws), ws.numel(), N.stream(device)), "sdr_backward")
        ctx.saved = None
        grads = []
        for p, part in zip(params, flat.split(numel)):
            grads.append(part.view(p.shape).to(p.dtype) if ctx.needs_input_grad[3 + len(grads)] else None)
        return (None, None, None, *grads)


def forward(model, wav: torch.Tensor) -> torch.Tensor:
    """Differentiable ``model(wav)`` on the native path: [B, 1, T] -> [B, S, T] fp32 with a ``grad_fn``."""
    cfg = _engine.make_config(model)
    x = _check(model, cfg, wav)
    if cfg.variant != 0:
        raise NotImplementedError("native training covers the improved SuDORMRF only")
    params = [_engine._fetch(model, n) for n in _engine.state_dict_names(cfg)]
    return _NativeTrain.apply(model, cfg, x, *params)
