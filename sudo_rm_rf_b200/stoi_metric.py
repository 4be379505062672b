"""Short-time objective intelligibility on the GPU: pystoi's ``stoi(x, y, fs_sig, extended=False)``.

The ``stoi`` that asteroid's ``get_metrics(..., metrics_list='all')`` reports, and that the reference's evaluation
scripts (``utils/simple_whamr_evaluation.py`` and the two notebooks) score separations with (``input_stoi`` for the
mixture).  Per (clean x, processed y): both are resampled to 10 kHz as Octave's ``resample`` does, the frames of x more
than 40 dB below its loudest are dropped from both, and the 30-frame segment correlations of the 15 third-octave band
magnitudes of x and of y (scaled to x and clipped 15 dB above it) are averaged.

The whole computation runs in fp64 from the fp32 inputs in ``libsudormrf_b200.so`` (``sdr_stoi``) without
synchronising with the host, so a call can be captured in a CUDA graph, and repeats bit for bit.
"""
import torch

from . import _native as N


def stoi(x, y, fs_sig, extended=False, mixture=None, lengths=None):
    """pystoi's ``stoi`` on CUDA tensors, for every row at once.

    ``x`` (clean) and ``y`` (processed) are ``[T]``, ``[S, T]`` or ``[B, S, T]`` of one shape; row j of ``y`` is scored
    against row j of ``x``.  ``fs_sig`` is an integer sampling rate >= 1000 Hz whose ratio to 10 kHz reduces to
    p / q with max(p, q) <= 441 (8, 16, 22.05, 44.1 and 48 kHz among them).  Returns fp64 of the leading shape
    (``[]``, ``[S]`` or ``[B, S]``).  Fewer than 30 analysed frames give 1e-5, as pystoi (which also warns then).

    ``mixture`` (``[T]`` for ``[T]`` or ``[S, T]`` inputs; ``[B, T]`` or ``[B, 1, T]``) is scored against every row of
    ``x`` too, and the call returns ``(stoi, input_stoi)``.  ``lengths`` (``[B]`` integers, a tensor or a sequence)
    scores item b over its first ``lengths[b]`` samples only: unlike BSS-eval, zero padding changes STOI, so a ragged
    corpus needs it.  A length outside [1, T] gives NaN for its item.  A NaN or infinity in ``x[j]`` or ``y[j]`` makes
    score j NaN; one in the mixture makes the mixture's scores NaN.

    Inputs of any floating dtype and stride are computed on as contiguous fp32.  ``extended=True`` (ESTOI) is not
    implemented.  Metric only: no autograd."""
    if extended:
        raise NotImplementedError("sudo_rm_rf_b200.stoi computes STOI only: extended=True (ESTOI) is not implemented")
    if x.dim() not in (1, 2, 3) or y.shape != x.shape:
        raise RuntimeError("expected x and y of one shape, [T], [S, T] or [B, S, T]")
    if not (x.is_cuda and y.is_cuda) or (mixture is not None and not mixture.is_cuda):
        raise RuntimeError("sudo_rm_rf_b200.stoi runs on CUDA tensors only (no CPU path)")
    if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad
                                    or (mixture is not None and mixture.requires_grad)):
        raise RuntimeError("sudo_rm_rf_b200.stoi is the evaluation metric only (no autograd): "
                           "wrap the call in torch.no_grad()")
    lead = x.shape[:-1]
    ref = x.reshape((-1,) + tuple(x.shape[-2:]) if x.dim() == 3 else (1, -1, x.shape[-1]))
    est = y.reshape(ref.shape)
    B, S, T = ref.shape
    if B == 0 or S == 0 or T == 0:
        raise RuntimeError("empty batch or zero-length signals")
    fs = int(fs_sig)
    if fs != fs_sig:
        raise RuntimeError("fs_sig must be an integer sampling rate")
    dev = x.device
    lib = N.lib()
    nbytes = lib.sdr_stoi_scratch_bytes(B, S, T, fs)
    if nbytes == 0:
        raise N.NativeError("sdr_stoi supports integer sampling rates >= 1000 Hz whose ratio to 10 kHz reduces to "
                            "p / q with max(p, q) <= 441")
    ref = ref.detach().to(torch.float32).contiguous()
    est = est.detach().to(device=dev, dtype=torch.float32).contiguous()
    mix = None
    if mixture is not None:
        mix = mixture.detach()
        if mix.numel() != B * T or mix.shape[-1] != T:
            raise RuntimeError(f"expected a mixture of {B} x {T} samples ([T], [B, T] or [B, 1, T])")
        mix = mix.reshape(B, T).to(device=dev, dtype=torch.float32).contiguous()
    lens = None
    if lengths is not None:
        lens = torch.as_tensor(lengths).reshape(-1)
        if lens.numel() != B or lens.dtype.is_floating_point or lens.dtype.is_complex:
            raise RuntimeError(f"expected {B} integer lengths")
        lens = lens.to(device=dev, dtype=torch.int64).contiguous()
    with torch.cuda.device(dev):
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty((1 if mix is None else 2, B, S), dtype=torch.float64, device=dev)
        # Every buffer of the call is allocated here on the current stream and released to it: the caching allocator
        # orders their reuse, and no state outlives the call (tests/test_gpu_stoi.py runs it across streams and threads).
        N.check(lib.sdr_stoi(N.ptr(ref), N.ptr(est), N.ptr(mix), N.ptr(lens), N.ptr(out[0]),
                             N.ptr(out[1] if mix is not None else None), B, S, T, fs, N.ptr(scratch), N.stream(dev)),
                "sdr_stoi")
    out = out.reshape((out.shape[0],) + tuple(lead))
    return out[0] if mix is None else (out[0], out[1])
