"""Chunk-by-chunk inference of ``CausalSuDORMRF`` (variant 2 of ``include/sudormrf_b200.h``).

Every convolution of the causal model is causally masked and it has no normalisation layers, so a stream that
carries a small state per slot (the last input samples, the last inputs of every depthwise level, the pending
overlap-add sums) produces exactly what ``model(x)`` produces on the concatenated audio, delayed by
``hop = enc_kernel_size // 2`` samples::

    cat(step(x_0), ..., step(x_{n-1}))[..., hop:] == model(x)[..., :n*C - hop]
    flush() == model(x)[..., n*C - hop:n*C]          when n*C is a multiple of hop * 2**upsampling_depth

A step costs the same whatever has been streamed before.  The other variants normalise over the whole clip and
cannot be streamed.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Iterable, Optional

import torch

from . import _engine
from . import _native as N

MAX_SLOTS = 65535            # slots per step (one grid row per slot, include/sudormrf_b200.h)
MAX_CHUNK_FRAMES = 4096      # encoder frames per slot and step, i.e. chunk_samples <= 4096 * hop


class SlotStream:
    """What every stream of ``batch_size`` independent slots shares: its device, and the CUDA stream of the last call
    on its buffers, which a call on another stream waits for on the device."""

    def __init__(self, device: torch.device, batch_size: int):
        self.device = device
        self.batch_size = batch_size
        self._order = _engine._Order()      # the stream of the last call on the state

    def _slot_array(self, slots: Optional[Iterable[int]]):
        """``(int32 array, n)`` of the slots ``reset(slots)`` names; ``(None, 0)`` for all of them."""
        if slots is None:
            return None, 0
        idx = [int(s) for s in slots]
        if any(s < 0 or s >= self.batch_size for s in idx):
            raise IndexError(f"slots {idx} out of range for batch_size={self.batch_size}")
        return (C.c_int32 * max(1, len(idx)))(*idx), len(idx)

    def _out(self, out: Optional[torch.Tensor], shape: tuple) -> torch.Tensor:
        """``out``, checked to be a contiguous fp32 tensor of ``shape`` on the stream's device, or a new one."""
        if out is None:
            return torch.empty(shape, dtype=torch.float32, device=self.device)
        if tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != self.device \
                or not out.is_contiguous():
            raise RuntimeError(f"out must be a contiguous fp32 tensor {list(shape)} on {self.device}")
        return out

    @contextlib.contextmanager
    def _ordered(self, *buffers):
        """The body runs on the stream's device after the previous call, and ``buffers`` are recorded on the current
        stream.  Only a body that returns counts as the last call: a refused one leaves the order as it was."""
        with torch.cuda.device(self.device):
            cur = _engine._enter_stream(self._order, self.device, buffers)
            yield
            _engine._leave_stream(self._order, cur)


def _granule(cfg: N.SdrConfig) -> int:
    """The chunk granule of a ``CausalSuDORMRF`` configuration; the other models are refused."""
    if cfg.variant != 2:
        raise RuntimeError("only CausalSuDORMRF can be streamed: the other models normalise over the whole clip")
    granule = N.lib().sdr_stream_granule(C.byref(cfg))
    if granule < 0:
        N.check(int(granule), "sdr_stream_granule")
    return int(granule)


class CausalStream(SlotStream):
    """``batch_size`` independent streams (slots) of ``chunk_samples`` samples per step.

    Owns its state and step workspace, apart from the model's forward workspace, so ``model(x)`` and open streams
    can interleave.  Every step reads the model's weights through the same packed-weight cache as ``forward``, so
    changed weights are picked up on the next step.  Steps run on the current CUDA stream, never synchronise and can
    be captured in a CUDA graph (``step(chunk, out=...)`` with fixed buffers).  A step, reset or flush on another
    CUDA stream than the previous one waits for it on the device, so consecutive calls may switch streams."""

    def __init__(self, model, batch_size: int, chunk_samples: int, mixture_consistency: bool = False):
        lib = N.lib()
        cfg = _engine.make_config(model)
        granule = _granule(cfg)
        # the arguments are checked before the device, so that each refusal names the limit it hit
        B, Cs = int(batch_size), int(chunk_samples)
        if B <= 0 or B > MAX_SLOTS:
            raise ValueError(f"batch_size={batch_size} is outside the slots a step takes (1 .. {MAX_SLOTS})")
        if Cs <= 0 or Cs % granule:
            raise ValueError(f"chunk_samples must be a positive multiple of the granule ({granule} samples); "
                             f"got chunk_samples={chunk_samples}")
        max_chunk = MAX_CHUNK_FRAMES * (cfg.enc_kernel_size // 2)
        if Cs > max_chunk:
            raise ValueError(f"chunk_samples={Cs} is longer than a step takes (at most {max_chunk} samples: "
                             f"{MAX_CHUNK_FRAMES} frames of hop {cfg.enc_kernel_size // 2})")
        if mixture_consistency and cfg.in_audio_channels != 1:
            raise RuntimeError("mixture consistency (mixture_consistency.py:14-36) is defined for mono mixtures only; "
                               f"this model has in_audio_channels={cfg.in_audio_channels}")
        ws_bytes = lib.sdr_stream_workspace_bytes(C.byref(cfg), B, Cs)
        if ws_bytes == 0:
            raise ValueError(f"sdr_stream_workspace_bytes refused batch_size={B}, chunk_samples={Cs}")
        super().__init__(_engine._model_device(model, "sudo_rm_rf_b200 streams on CUDA (sm_90a) only and has no CPU "
                                                      "path: move the model to an H100 (`model.cuda()`)"), B)
        self.model = model
        self.chunk_samples = Cs
        self.granule = granule
        self.latency = cfg.enc_kernel_size // 2
        self.mixture_consistency = bool(mixture_consistency)
        self._cfg = cfg
        self._state = torch.empty(lib.sdr_stream_state_bytes(C.byref(cfg), B), dtype=torch.uint8, device=self.device)
        self._ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
        self.reset()

    def reset(self, slots: Optional[Iterable[int]] = None) -> None:
        """Start slots over (all of them when ``slots`` is None): their next step is the start of a new stream."""
        arr, n = self._slot_array(slots)
        with self._ordered(self._state):
            N.check(N.lib().sdr_stream_reset(C.byref(self._cfg), N.ptr(self._state), self.batch_size, arr, n,
                                             N.stream(self.device)), "sdr_stream_reset")

    def _reset_masked(self, mask: torch.Tensor) -> None:
        """Starts over the slots whose byte in ``mask`` (device uint8 [B]) is set, on the current stream, inside the
        caller's ``_ordered`` section right after a step: the mask is read on the device, so a captured graph resets
        whichever slots it names at replay."""
        N.check(N.lib().sdr_stream_reset_masked(C.byref(self._cfg), N.ptr(self._state), self.batch_size, N.ptr(mask),
                                                N.stream(self.device)), "sdr_stream_reset_masked")

    def step(self, chunk: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, A, C] chunk -> [B, S*A, C] estimates of the model's output samples ``c*C - hop .. (c+1)*C - hop - 1``."""
        cfg = self._cfg
        x = _engine._check_input(self.model, cfg, chunk)
        B, Cs = self.batch_size, self.chunk_samples
        if x.shape[0] != B or x.shape[2] != Cs:
            raise RuntimeError(f"expected a chunk of shape [{B}, {cfg.in_audio_channels}, {Cs}], got {list(chunk.shape)}")
        if x.device != self.device:
            raise RuntimeError(f"chunk is on {x.device}, the stream on {self.device}")
        out = self._out(out, (B, cfg.num_sources * cfg.in_audio_channels, Cs))
        with self._ordered(self._state, self._ws):
            packed = _engine.packed_for(self.model, cfg, self.device, torch.cuda.current_stream(self.device))
            N.check(N.lib().sdr_stream_step(C.byref(cfg), N.ptr(packed), N.ptr(self._state), N.ptr(x), N.ptr(out), B,
                                            Cs, 1 if self.mixture_consistency else 0, N.ptr(self._ws),
                                            self._ws.numel(), N.stream(self.device)), "sdr_stream_step")
        return out

    def flush(self) -> torch.Tensor:
        """[B, S*A, hop]: the last ``hop`` output samples, which only the end of the stream completes.  The state is
        left as it is; ``reset()`` starts the slots over."""
        cfg = self._cfg
        tail = torch.empty((self.batch_size, cfg.num_sources * cfg.in_audio_channels, self.latency),
                           dtype=torch.float32, device=self.device)
        with self._ordered(self._state):
            N.check(N.lib().sdr_stream_flush(C.byref(cfg), N.ptr(self._state), N.ptr(tail), self.batch_size,
                                             1 if self.mixture_consistency else 0, N.stream(self.device)),
                    "sdr_stream_flush")
        return tail
