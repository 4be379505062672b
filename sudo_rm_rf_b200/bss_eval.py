"""BSS-eval v3 source criteria on the GPU: ``mir_eval.separation.bss_eval_sources``.

The ``sdr``, ``sir`` and ``sar`` that asteroid's ``get_metrics(..., metrics_list='all')`` reports, and that the
reference's evaluation scripts (``utils/simple_whamr_evaluation.py`` and the two notebooks) score separations with.
Per item, with F-tap distortion filters (512, as mir_eval) and the projections ``P_j e`` of an estimate onto the
delays of reference j and ``P_all e`` onto the delays of every reference::

    SDR = 10 log10(|P_j e|^2 / |e - P_j e|^2)
    SIR = 10 log10(|P_j e|^2 / |P_all e - P_j e|^2)
    SAR = 10 log10(|P_all e|^2 / |e - P_all e|^2)

The whole computation (fp64 lagged correlations, a block-Levinson solve per item, the projections as FIR filters and
the permutation search) runs in ``libsudormrf_b200.so`` (``sdr_bss_eval``) without synchronising with the host, so a
call can be captured in a CUDA graph.  Zero-padding an item to a longer length changes none of its values, so a
ragged corpus can be scored in zero-padded batches.
"""
import torch

from . import _native as N


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True, filter_length=512,
                     mixture=None):
    """mir_eval's ``bss_eval_sources`` on CUDA tensors.

    ``reference_sources`` and ``estimated_sources`` are ``[S, T]`` (mir_eval's shape) or ``[B, S, T]``, 1 <= S <= 4,
    1 <= filter_length <= 512 and T >= (S - 1) * filter_length + 1 (no more delayed references than dimensions).
    Returns ``(sdr, sir, sar, perm)`` on the device: fp64 ``[..., S]`` in dB and int64 ``[..., S]`` where ``perm[j]``
    is the estimate scored against reference j.  With ``compute_permutation`` that is the assignment with the largest
    mean SIR (the first in ``itertools.permutations`` order), otherwise estimate j.  Where mir_eval raises on an
    all-zero reference or estimate row, and where such a row holds a NaN or an infinity, that item gets NaN in every
    output and ``perm = -1``.  So does an item whose references are too close to dependent for the normal equations
    (several band-limited references with deep stop bands), where the solve would give no projection.

    With ``mixture`` (``[T]``, ``[1, T]``, ``[B, T]`` or ``[B, 1, T]``) the call also returns the mixture scored as the
    estimate of every reference and the improvements, as a dict ``{"sdr", "sir", "sar"}`` of the mixture's scores and
    ``{"sdri", "siri", "sari"}`` = score - mixture score, each ``[..., S]``:
    ``(sdr, sir, sar, perm, extra)``.

    Inputs of any floating dtype and stride are computed on as contiguous fp32.  Metric only: no autograd."""
    ref, est = reference_sources, estimated_sources
    if ref.dim() not in (2, 3) or est.shape != ref.shape:
        raise RuntimeError("expected reference_sources and estimated_sources of one shape, [S, T] or [B, S, T]")
    if not (ref.is_cuda and est.is_cuda) or (mixture is not None and not mixture.is_cuda):
        raise RuntimeError("sudo_rm_rf_b200.bss_eval runs on CUDA tensors only (no CPU path)")
    if torch.is_grad_enabled() and (ref.requires_grad or est.requires_grad
                                    or (mixture is not None and mixture.requires_grad)):
        raise RuntimeError("sudo_rm_rf_b200.bss_eval is the evaluation metric only (no autograd): "
                           "wrap the call in torch.no_grad()")
    single = ref.dim() == 2
    if single:
        ref, est = ref.unsqueeze(0), est.unsqueeze(0)
    B, S, T = ref.shape
    F = int(filter_length)
    dev = ref.device
    if B == 0 or T == 0:
        raise RuntimeError("empty batch or zero-length signals")
    lib = N.lib()
    nbytes = lib.sdr_bss_eval_scratch_bytes(B, S, T, F)
    if nbytes == 0:
        raise N.NativeError("sdr_bss_eval supports 1..4 sources, filter lengths 1..512 and items of at least "
                            "(S - 1) * filter_length + 1 samples")
    ref = ref.detach().to(torch.float32).contiguous()
    est = est.detach().to(device=dev, dtype=torch.float32).contiguous()
    mix = None
    if mixture is not None:
        mix = mixture.detach()
        if mix.numel() != B * T or mix.shape[-1] != T:
            raise RuntimeError(f"expected a mixture of {B} x {T} samples ([T], [1, T], [B, T] or [B, 1, T])")
        mix = mix.reshape(B, T).to(device=dev, dtype=torch.float32).contiguous()
    with torch.cuda.device(dev):
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty((3 if mix is None else 6, B, S), dtype=torch.float64, device=dev)
        perm = torch.empty((B, S), dtype=torch.int32, device=dev)
        if mix is None:
            N.check(lib.sdr_bss_eval(N.ptr(ref), N.ptr(est), N.ptr(out[0]), N.ptr(out[1]), N.ptr(out[2]), N.ptr(perm),
                                     B, S, T, F, 1 if compute_permutation else 0, N.ptr(scratch), N.stream(dev)),
                    "sdr_bss_eval")
        else:
            N.check(lib.sdr_bss_eval_mixture(
                N.ptr(ref), N.ptr(est), N.ptr(mix), N.ptr(out[0]), N.ptr(out[1]), N.ptr(out[2]), N.ptr(perm),
                N.ptr(out[3]), N.ptr(out[4]), N.ptr(out[5]), B, S, T, F, 1 if compute_permutation else 0,
                N.ptr(scratch), N.stream(dev)), "sdr_bss_eval_mixture")
    if single:
        out, perm = out[:, 0], perm[0]
    sdr, sir, sar = out[0], out[1], out[2]
    perm = perm.long()
    if mix is None:
        return sdr, sir, sar, perm
    extra = {"sdr": out[3], "sir": out[4], "sar": out[5],
             "sdri": sdr - out[3], "siri": sir - out[4], "sari": sar - out[5]}
    return sdr, sir, sar, perm, extra
