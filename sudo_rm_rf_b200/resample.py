"""Polyphase resampling on the GPU (DESIGN.md section 7g): ``scipy.signal.resample_poly`` with its defaults, and the
conversion into and out of a model's rate that ``separate`` / ``separate_long`` do with ``sample_rate`` and
``model_rate``.

The filter is designed on the device and every output is summed in fp64 in a fixed order (``sdr_resample_poly`` in
``libsudormrf_b200.so``), so a call never copies from the host, can be captured in a CUDA graph and repeats bit for
bit, whatever the batch.
"""
import math

import torch

from . import _native as N

MAX_RATIO = 4096             # largest max(p, q) of the reduced ratio: any pair of 8 .. 192 kHz standard rates fits


def _ratio(up, down, what=("up", "down")):
    """(p, q): up / down reduced by their gcd, after the checks."""
    for v, name in zip((up, down), what):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"{name} must be a positive integer, got {v!r}")
    g = math.gcd(up, down)
    p, q = up // g, down // g
    if max(p, q) > MAX_RATIO:
        raise ValueError(f"{what[0]} / {what[1]} = {up} / {down} reduces to {p} / {q}; max(p, q) must be at most "
                         f"{MAX_RATIO}")
    return p, q


def resample_poly(x, up, down):
    """``scipy.signal.resample_poly(x, up, down)`` on the last axis of a CUDA tensor, with scipy's defaults
    (``window=('kaiser', 5.0)``, ``padtype='constant'``).

    ``x`` is ``[..., T]`` of any floating dtype and stride, computed on as contiguous fp32; returns fp32
    ``[..., ceil(T p / q)]`` with ``up / down`` reduced to ``p / q`` (``p == q``: a copy).  ``up`` and ``down`` are
    positive integers whose reduced ratio has ``max(p, q) <= 4096``.  Each output is summed in fp64 and rounded once:
    it agrees with scipy on the fp64 input to about one fp32 rounding.  A NaN or infinity makes non-finite exactly the
    outputs whose filter support holds it.  No CPU path and no autograd."""
    p, q = _ratio(up, down)
    if not torch.is_tensor(x) or not x.is_cuda:
        raise RuntimeError("sudo_rm_rf_b200.resample_poly runs on CUDA tensors only (no CPU path)")
    if not x.dtype.is_floating_point:
        raise RuntimeError(f"expected a floating-point tensor, got {x.dtype}")
    if x.dim() < 1 or x.shape[-1] == 0 or x.numel() == 0:
        raise RuntimeError("expected a non-empty tensor [..., T] with T >= 1")
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError("sudo_rm_rf_b200.resample_poly has no autograd: wrap the call in torch.no_grad()")
    lead, T = tuple(x.shape[:-1]), x.shape[-1]
    rows = x.numel() // T
    dev = x.device
    lib = N.lib()
    nbytes = lib.sdr_resample_poly_scratch_bytes(up, down)
    src = x.detach().to(torch.float32).contiguous()
    with torch.cuda.device(dev):
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(lead + (-(-T * p // q),), dtype=torch.float32, device=dev)
        # The scratch and the output are allocated here on the current stream and released to it: the caching
        # allocator orders their reuse, and no state outlives the call.
        N.check(lib.sdr_resample_poly(N.ptr(src), N.ptr(out), rows, T, up, down, N.ptr(scratch), nbytes,
                                      N.stream(dev)), "sdr_resample_poly")
    return out


def check_rates(sample_rate, model_rate):
    """Refuses anything but both rates or neither, as positive integers whose ratio ``resample_poly`` takes."""
    if (sample_rate is None) != (model_rate is None):
        raise ValueError("give both sample_rate and model_rate, or neither")
    if sample_rate is not None:
        _ratio(model_rate, sample_rate, ("model_rate", "sample_rate"))


def at_model_rate(run, wav, sample_rate, model_rate):
    """``run(wav)`` for a mixture ``wav [..., T]`` recorded at ``sample_rate`` by a model trained at ``model_rate``:
    the mixture resampled to ``model_rate``, ``run`` there, every source resampled back to ``sample_rate`` and cropped
    to ``T`` (a view).  Without rates, or with equal ones, exactly ``run(wav)``."""
    check_rates(sample_rate, model_rate)
    if sample_rate == model_rate:
        return run(wav)
    est = run(resample_poly(wav, model_rate, sample_rate))
    return resample_poly(est, sample_rate, model_rate)[..., :wav.shape[-1]]
