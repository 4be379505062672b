"""Windowed separation taken step by step (DESIGN.md section 7f).

``separate_long`` gives every model, including the ones that normalise over the whole clip, a local semantics: windows
of W samples every H samples (W/2 <= H < W), each separated on its own, its sources put in the order of the window
before it and the overlaps cross-faded.  Everything it outputs below sample n - H depends only on the input below n,
so a stream that keeps the last H input samples, the last window's raw estimate and its order per slot produces it
step by step, one hop late::

    cat(step(x_0), ..., step(x_{j-1}))[..., H:] == separate_long(x[..., :n])[..., :n - H]       (n = j C)
    flush() == separate_long(x[..., :n])[..., n - H:n]

Each step separates q = C / H windows per slot (q - 1 in a slot's first step) through ``separate`` or ``forward`` on
the model's shared workspace, so its cost and memory stay the same however long the stream runs.
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from . import _engine
from . import _native as N
from .streaming import MAX_SLOTS, SlotStream
from .windowed import window_hop


class WindowedStream(SlotStream):
    """``batch_size`` independent streams (slots) of ``chunk_samples`` samples per step, separated in windows of
    ``window`` samples every ``hop``.

    A step's output [B, S*A, C] is the slot's samples ``n - hop .. n + C - hop - 1`` of ``separate_long`` on
    everything the slot has received (zeros below 0), where n counts the samples since its last reset.  The window
    counters live on the device: ``step(chunk, out=...)`` with fixed buffers never synchronises and can be captured in
    a CUDA graph.  Every step reads the model's weights through the packed-weight cache, so changed weights are used
    from the next step on.  A call on another CUDA stream than the previous one waits for it on the device."""

    def __init__(self, model, batch_size: int, chunk_samples: int, window: int, hop: Optional[int] = None,
                 normalize: bool = True, mixture_consistency: bool = False):
        lib = N.lib()
        cfg = _engine.make_config(model)
        W, H = window_hop(window, hop)
        B, Cs = batch_size, chunk_samples
        # the arguments are checked before the device, so that each refusal names the limit it hit
        if isinstance(B, bool) or not isinstance(B, int) or B <= 0 or B > MAX_SLOTS:
            raise ValueError(f"batch_size={batch_size!r} is outside the slots a step takes (1 .. {MAX_SLOTS})")
        if isinstance(Cs, bool) or not isinstance(Cs, int) or Cs <= 0 or Cs % H:
            raise ValueError(f"chunk_samples must be a positive multiple of the hop ({H} samples); "
                             f"got chunk_samples={chunk_samples!r}")
        A, S = cfg.in_audio_channels, cfg.num_sources
        if normalize and A != 1:
            raise RuntimeError("separate() follows the README recipe, which is written for mono mixtures")
        if mixture_consistency and A != 1:
            raise RuntimeError("mixture consistency (mixture_consistency.py:14-36) is defined for mono mixtures only; "
                               f"this model has in_audio_channels={A}")
        state_bytes = lib.sdr_window_stream_state_bytes(B, S, A, W, H)
        scratch_bytes = lib.sdr_window_stream_merge_scratch_bytes(B, S, Cs, H)
        if state_bytes == 0 or scratch_bytes == 0:
            raise N.NativeError(f"windowed streams support 1 to 4 sources and windows of at most 2^24 samples "
                                f"(num_sources={S}, window={W})")
        super().__init__(_engine._model_device(model, "sudo_rm_rf_b200 streams on CUDA (sm_90a) only and has no CPU "
                                                      "path: move the model to an H100 (`model.cuda()`)"), B)
        device = self.device
        self.model = model
        self.chunk_samples = Cs
        self.window, self.hop = W, H
        self.latency = H
        self.normalize = bool(normalize)
        self.mixture_consistency = bool(mixture_consistency)
        self._cfg = cfg
        self._q = Cs // H
        self._state = torch.empty(state_bytes, dtype=torch.uint8, device=device)
        self._batch = torch.empty((B * self._q, A, W), dtype=torch.float32, device=device)
        self._scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=device)
        self.reset()

    def _shape(self):
        cfg = self._cfg
        return self.batch_size, cfg.num_sources, cfg.in_audio_channels, self.window, self.hop

    def _run(self, wav):
        run = _engine.separate if self.normalize else _engine.forward
        return run(self.model, wav, mixture_consistency=self.mixture_consistency)

    def reset(self, slots: Optional[Iterable[int]] = None) -> None:
        """Start slots over (all of them when ``slots`` is None): their next step is the start of a new stream."""
        arr, n = self._slot_array(slots)
        with self._ordered(self._state):
            N.check(N.lib().sdr_window_stream_reset(N.ptr(self._state), *self._shape(), arr, n, N.stream(self.device)),
                    "sdr_window_stream_reset")

    def _reset_masked(self, mask: torch.Tensor) -> None:
        """``CausalStream._reset_masked`` for the window counters and carries."""
        N.check(N.lib().sdr_window_stream_reset_masked(N.ptr(self._state), *self._shape(), N.ptr(mask),
                                                       N.stream(self.device)), "sdr_window_stream_reset_masked")

    def step(self, chunk: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, A, C] chunk -> [B, S*A, C]: the slots' separated samples ``n - hop .. n + C - hop - 1``."""
        lib = N.lib()
        cfg = self._cfg
        if chunk.requires_grad:
            raise RuntimeError("a windowed stream is inference-only: the chunk requires grad (pass chunk.detach())")
        x = _engine._check_input(self.model, cfg, chunk)
        B, S, A, W, H = self._shape()
        Cs = self.chunk_samples
        if x.shape[0] != B or x.shape[2] != Cs:
            raise RuntimeError(f"expected a chunk of shape [{B}, {A}, {Cs}], got {list(chunk.shape)}")
        if x.device != self.device:
            raise RuntimeError(f"chunk is on {x.device}, the stream on {self.device}")
        out = self._out(out, (B, S * A, Cs))
        with self._ordered(self._state, self._batch, self._scratch):
            N.check(lib.sdr_window_stream_gather(N.ptr(self._state), N.ptr(x), N.ptr(self._batch), B, S, A, Cs, W, H,
                                                 N.stream(self.device)), "sdr_window_stream_gather")
            # the model's shared workspace and packed weights, as for any forward of B q windows
            est = self._run(self._batch)
            N.check(lib.sdr_window_stream_merge(N.ptr(est), N.ptr(self._state), N.ptr(out), B, S, A, Cs, W, H,
                                                N.ptr(self._scratch), N.stream(self.device)), "sdr_window_stream_merge")
        return out

    def flush(self) -> torch.Tensor:
        """[B, S*A, hop]: each slot's last ``hop`` samples of ``separate_long`` on everything it has received (zeros
        for a slot without a step since its reset).  The state is left as it is; ``reset()`` starts slots over."""
        lib = N.lib()
        B, S, A, W, H = self._shape()
        with self._ordered(self._state):
            win = torch.empty((B, A, W), dtype=torch.float32, device=self.device)
            N.check(lib.sdr_window_stream_gather(N.ptr(self._state), None, N.ptr(win), B, S, A, 0, W, H,
                                                 N.stream(self.device)), "sdr_window_stream_gather")
            # a slot that has received H samples is one window long: separate_long separates them unpadded
            single = self._run(win[..., :H].contiguous())
            est = self._run(win) if W < 2 * H else None
            scratch = torch.empty(lib.sdr_window_stream_flush_scratch_bytes(B, S), dtype=torch.uint8,
                                  device=self.device)
            tail = torch.empty((B, S * A, H), dtype=torch.float32, device=self.device)
            N.check(lib.sdr_window_stream_flush(N.ptr(single), N.ptr(est), N.ptr(self._state), N.ptr(tail), B, S, A, W,
                                                H, N.ptr(scratch), N.stream(self.device)), "sdr_window_stream_flush")
        return tail
