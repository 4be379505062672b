"""Streaming at any sample rate (DESIGN.md section 7h): ``resample_poly`` chunk by chunk, and the model streams behind
a resampler into and out of the model's rate.

``ResampleStream`` carries per slot a step counter and an input history on the device, so that each step emits
exactly the samples ``resample_poly`` gives on everything the slot has received, ``delay`` samples late, bit for bit::

    cat(step(x_0), ..., step(x_{j-1})) == resample_poly(s)[j C p/q - delay ...]      s = lead zeros + x

``ResampledStream`` wraps a ``CausalStream`` or a ``WindowedStream`` running at the model's rate between two of them,
and so produces ``separate`` / ``separate_long`` with ``sample_rate`` and ``model_rate``, ``latency`` samples late.
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from . import _engine
from . import _native as N
from .resample import _ratio, check_rates
from .streaming import MAX_SLOTS, CausalStream, SlotStream, _granule
from .window_stream import WindowedStream
from .windowed import window_hop


def _int(v, name, low):
    if isinstance(v, bool) or not isinstance(v, int) or v < low:
        raise ValueError(f"{name} must be an integer of at least {low}, got {v!r}")
    return v


def min_delay(up, down, lead=0):
    """The smallest ``delay`` of a ``ResampleStream``: floor((L - lead p) / q), L = 10 max(p, q).  By then every
    output a step emits has its whole filter support received."""
    p, q = _ratio(up, down)
    return (10 * max(p, q) - lead * p) // q


class ResampleStream(SlotStream):
    """``resample_poly`` taken chunk by chunk for ``batch_size`` independent slots of ``rows`` rows each.

    Per slot, let s be ``lead`` zeros followed by everything the slot received since its reset, and r
    ``resample_poly(s, up, down)``.  Step j returns [B, rows, C p / q]: samples ``j C p/q - delay .. (j+1) C p/q -
    delay - 1`` of r (zeros below 0), bitwise what ``resample_poly`` gives on the concatenation.  ``chunk_samples`` C
    is a positive multiple of q (``up / down`` reduced to ``p / q``, p != q, ``max(p, q) <= 4096``); ``delay`` is at
    least, and by default, ``min_delay(up, down, lead)``.  The counters live on the device: ``step(chunk, out=...)``
    with fixed buffers never synchronises and can be captured in a CUDA graph.  Chunks of any float dtype and stride
    are taken as contiguous fp32.  No autograd and no CPU path."""

    def __init__(self, batch_size: int, rows: int, chunk_samples: int, up: int, down: int, *,
                 delay: Optional[int] = None, lead: int = 0, device=None):
        lib = N.lib()
        p, q = _ratio(up, down)
        if p == q:
            raise ValueError(f"up / down = {up} / {down} reduces to 1: there is nothing to resample")
        # the arguments are checked before the device, so that each refusal names the limit it hit
        if isinstance(batch_size, bool) or not isinstance(batch_size, int) or not 1 <= batch_size <= MAX_SLOTS:
            raise ValueError(f"batch_size={batch_size!r} is outside the slots a step takes (1 .. {MAX_SLOTS})")
        _int(rows, "rows", 1)
        if isinstance(chunk_samples, bool) or not isinstance(chunk_samples, int) or chunk_samples <= 0 \
                or chunk_samples % q:
            raise ValueError(f"chunk_samples must be a positive multiple of q = {q} (up / down = {up} / {down} "
                             f"reduced to {p} / {q}); got chunk_samples={chunk_samples!r}")
        _int(lead, "lead", 0)
        least = min_delay(up, down, lead)
        if delay is None:
            delay = least
        elif isinstance(delay, bool) or not isinstance(delay, int) or delay < least:
            raise ValueError(f"delay must be an integer of at least floor((L - lead p) / q) = {least} "
                             f"(L = {10 * max(p, q)}, lead = {lead}); got delay={delay!r}")
        args = (batch_size, rows, chunk_samples, up, down, delay, lead)
        state_bytes = lib.sdr_resample_stream_state_bytes(*args)
        if state_bytes == 0:
            raise N.NativeError(f"sdr_resample_stream_state_bytes refused batch_size={batch_size}, rows={rows}, "
                                f"chunk_samples={chunk_samples}, delay={delay}, lead={lead} (64-bit sizes)")
        super().__init__(_engine._cuda_device(device if device is not None else "cuda",
                                              "sudo_rm_rf_b200 resamples on CUDA (sm_90a) only and has no CPU path"),
                         batch_size)
        self.rows, self.chunk_samples = rows, chunk_samples
        self.up, self.down, self.p, self.q = up, down, p, q
        self.delay, self.lead = delay, lead
        self.latency = delay
        self.out_samples = chunk_samples // q * p
        self._args = args
        self._state = torch.empty(state_bytes, dtype=torch.uint8, device=self.device)
        self.reset()

    def flush_samples(self, tail_samples: int = 0) -> int:
        """The length of ``flush`` with a tail of ``tail_samples``: ceil((lead + t) p / q) + delay."""
        return -(-(self.lead + tail_samples) * self.p // self.q) + self.delay

    def _check(self, x, what, length=None):
        B, R = self.batch_size, self.rows
        if not torch.is_tensor(x) or not x.is_cuda or not x.dtype.is_floating_point:
            raise RuntimeError(f"the {what} must be a floating-point CUDA tensor")
        if x.dim() != 3 or x.shape[0] != B or x.shape[1] != R or (length is not None and x.shape[2] != length):
            want = f"[{B}, {R}, {length if length is not None else 't'}]"
            raise RuntimeError(f"expected a {what} of shape {want}, got {list(x.shape)}")
        if x.device != self.device:
            raise RuntimeError(f"the {what} is on {x.device}, the stream on {self.device}")
        if torch.is_grad_enabled() and x.requires_grad:
            raise RuntimeError("a resampling stream has no autograd: wrap the call in torch.no_grad()")
        return x.detach().to(torch.float32).contiguous()

    def reset(self, slots: Optional[Iterable[int]] = None) -> None:
        """Start slots over (all of them when ``slots`` is None): their next step is the start of a new stream."""
        arr, n = self._slot_array(slots)
        with self._ordered(self._state):
            N.check(N.lib().sdr_resample_stream_reset(N.ptr(self._state), self._state.numel(), *self._args, arr, n,
                                                      N.stream(self.device)), "sdr_resample_stream_reset")

    def step(self, chunk: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, rows, C] chunk -> [B, rows, C p / q]: samples ``j C p/q - delay ..`` of each slot's resampled input."""
        return self._step(chunk, out, None)

    def _step(self, chunk, out, zero):
        """``step``; the chunks of the slots whose ``zero`` byte (device uint8 [B], or None) is set read as zeros."""
        x = self._check(chunk, "chunk", self.chunk_samples)
        out = self._out(out, (self.batch_size, self.rows, self.out_samples))
        with self._ordered(self._state):
            N.check(N.lib().sdr_resample_stream_step(N.ptr(self._state), self._state.numel(), N.ptr(x), N.ptr(zero),
                                                     N.ptr(out), *self._args, N.stream(self.device)),
                    "sdr_resample_stream_step")
        return out

    def flush(self, tail: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, rows, flush_samples(t)]: the rest of each slot's resampled input, with s extended by ``tail``
        [B, rows, t] (any t >= 0), up to ceil(len(s) p / q).  The state is left as it was."""
        return self._flush(tail, None)

    def _flush(self, tail, zero):
        x = self._check(tail, "tail") if tail is not None else None
        t = x.shape[-1] if x is not None else 0
        out = self._out(None, (self.batch_size, self.rows, self.flush_samples(t)))
        with self._ordered(self._state):
            N.check(N.lib().sdr_resample_stream_flush(N.ptr(self._state), self._state.numel(), N.ptr(x if t else None),
                                                      t, N.ptr(zero), N.ptr(out), *self._args, N.stream(self.device)),
                    "sdr_resample_stream_flush")
        return out


class ResampledStream(SlotStream):
    """A model stream (``inner``: a ``CausalStream`` or a ``WindowedStream`` at ``model_rate``) fed and read at
    ``sample_rate``.  ``chunk_samples`` C counts input-rate samples; with ``model_rate / sample_rate = p / q``, the
    inner stream takes Cm = C p / q samples per step.  For a slot that has received n = j C samples,
    ``cat(steps)[..., D:]`` is ``ref[..., :n - D]`` and ``flush()`` is ``ref[..., n - D:n]``, where ref is
    ``separate`` (causal) or ``separate_long`` (windowed) with the same rates, and the latency
    D = C + floor((lat q + L) / p) (lat: the inner stream's latency, L = 10 max(p, q)).

    Each step resamples its chunk into model-rate samples [(j-1) Cm, j Cm) (an input resampler ``delay``ed by Cm),
    steps the inner stream on them and resamples its estimate back (an output resampler whose ``lead`` puts the
    model's first sample on the input's sample grid).  A slot's first step after a reset is the chunk before its
    origin: the inner stream resets that slot after it, and its estimate counts as zeros.  Which slots are in that
    step is a device-side mask, so a step captured in a CUDA graph stays right across later resets."""

    def __init__(self, make_inner, chunk_samples: int, sample_rate: int, model_rate: int, unit: int, unit_name: str):
        p, q = _ratio(model_rate, sample_rate, ("model_rate", "sample_rate"))
        L = 10 * max(p, q)
        Cs = chunk_samples
        if isinstance(Cs, bool) or not isinstance(Cs, int) or Cs <= 0 or Cs % q:
            raise ValueError(f"chunk_samples must be a positive multiple of q = {q} (model_rate / sample_rate = "
                             f"{model_rate} / {sample_rate} reduced to {p} / {q}); got chunk_samples={Cs!r}")
        Cm = Cs // q * p
        if Cm < L // q:
            raise ValueError(f"chunk_samples={Cs} gives {Cm} samples at the model's rate per step, fewer than the "
                             f"input resampler's delay floor(L / q) = {L // q}: take chunks of at least "
                             f"{-(-(L // q) // p) * q} samples")
        if Cm % unit:
            raise ValueError(f"chunk_samples={Cs} gives {Cm} samples at the model's rate per step, which is not a "
                             f"multiple of the inner stream's {unit_name} ({unit} samples)")
        inner = make_inner(Cm)
        super().__init__(inner.device, inner.batch_size)
        B, dev = self.batch_size, self.device
        cfg = inner._cfg
        A, SA = cfg.in_audio_channels, cfg.num_sources * cfg.in_audio_channels
        lat = inner.latency
        m = -(-(Cm + lat) // p)
        self.inner = inner
        self.chunk_samples = Cs
        self.sample_rate, self.model_rate = sample_rate, model_rate
        self._to_model = ResampleStream(B, A, Cs, model_rate, sample_rate, delay=Cm, device=dev)
        self._to_input = ResampleStream(B, SA, Cm, sample_rate, model_rate, lead=m * p - (Cm + lat), device=dev)
        self.latency = Cs + (lat * q + L) // p
        assert self.latency == self._to_input.delay + m * q
        self._mid = torch.empty((B, A, Cm), dtype=torch.float32, device=dev)
        self._est = torch.empty((B, SA, Cm), dtype=torch.float32, device=dev)
        self._fresh = torch.empty(B, dtype=torch.uint8, device=dev)
        self.reset()

    def reset(self, slots: Optional[Iterable[int]] = None) -> None:
        """Start slots over (all of them when ``slots`` is None): their next step is the start of a new stream."""
        arr, n = self._slot_array(slots)
        idx = None if arr is None else arr[:n]
        with self._ordered(self._fresh):
            self._to_model.reset(idx)
            self._to_input.reset(idx)
            if idx is None:
                self._fresh.fill_(1)
            elif idx:
                self._fresh.index_fill_(0, torch.tensor(idx, dtype=torch.long).to(self.device, non_blocking=True), 1)

    def step(self, chunk: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, A, C] chunk at ``sample_rate`` -> [B, S*A, C]: the slots' separated samples ``n - D .. n + C - D - 1``
        at ``sample_rate``."""
        with self._ordered(self._mid, self._est, self._fresh):
            mid = self._to_model.step(chunk, out=self._mid)
            est = self.inner.step(mid, out=self._est)
            self.inner._reset_masked(self._fresh)
            out = self._to_input._step(est, out, self._fresh)
            self._fresh.zero_()
        return out

    def flush(self) -> torch.Tensor:
        """[B, S*A, latency]: each slot's last ``latency`` samples of the separation of everything it received (zeros
        for a slot without a step since its reset).  Every state is left as it was."""
        inner = self.inner
        with self._ordered(self._fresh):
            mid = self._to_model.flush()                # model-rate samples [(j-1) Cm, j Cm): one inner chunk
            saved = inner._state.clone()
            est = inner.step(mid)
            tail = torch.cat([est, inner.flush()], dim=-1)
            inner._state.copy_(saved)
            out = self._to_input._flush(tail, self._fresh)
        return out


def causal_stream(model, batch_size, chunk_samples, mixture_consistency, sample_rate, model_rate):
    """``CausalSuDORMRF.stream``: a ``CausalStream``, or with two different rates a ``ResampledStream`` around one."""
    check_rates(sample_rate, model_rate)
    if sample_rate == model_rate:
        return CausalStream(model, batch_size, chunk_samples, mixture_consistency=mixture_consistency)
    return ResampledStream(lambda Cm: CausalStream(model, batch_size, Cm, mixture_consistency=mixture_consistency),
                           chunk_samples, sample_rate, model_rate, _granule(_engine.make_config(model)), "granule")


def windowed_stream(model, batch_size, chunk_samples, window, hop, normalize, mixture_consistency, sample_rate,
                    model_rate):
    """``stream_windows``: a ``WindowedStream``, or with two different rates a ``ResampledStream`` around one (``window``
    and ``hop`` count model-rate samples)."""
    check_rates(sample_rate, model_rate)
    if sample_rate == model_rate:
        return WindowedStream(model, batch_size, chunk_samples, window, hop, normalize=normalize,
                              mixture_consistency=mixture_consistency)
    W, H = window_hop(window, hop)
    return ResampledStream(lambda Cm: WindowedStream(model, batch_size, Cm, W, H, normalize=normalize,
                                                     mixture_consistency=mixture_consistency),
                           chunk_samples, sample_rate, model_rate, H, "hop")
