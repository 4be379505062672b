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

``bss_eval_sources_framewise`` is mir_eval's framewise form for long recordings: the same criteria in fixed windows at
a fixed hop (``sdr_bss_eval_framewise``), each window read in place from the recording.

``bss_eval_images`` and ``bss_eval_images_framewise`` are mir_eval's source-image criteria for multichannel
separations (SDR, ISR, SIR and SAR; ``sdr_bss_eval_images``), the same kernels with each source's C channel rows
projected together.

``bss_eval_v4`` is museval's BSS-eval v4 (``sdr_bss_eval_v4``), the SiSEC 2018 / MUSDB18 criteria: the image criteria
per window, with distortion filters solved once from the whole recording.
"""
import torch

from . import _native as N


def _checked(ref, est, mixture):
    """The shape, device and autograd checks of every entry -> (ref, est as [B, S, T], whether they were [S, T])."""
    if ref.dim() not in (2, 3) or est.shape != ref.shape:
        raise RuntimeError("expected reference_sources and estimated_sources of one shape, [S, T] or [B, S, T]")
    _usable(ref, est, mixture)
    single = ref.dim() == 2
    if single:
        ref, est = ref.unsqueeze(0), est.unsqueeze(0)
    if ref.shape[0] == 0 or ref.shape[2] == 0:
        raise RuntimeError("empty batch or zero-length signals")
    return ref, est, single


def _usable(ref, est, mixture):
    """The device and autograd checks of every entry."""
    if not (ref.is_cuda and est.is_cuda) or (mixture is not None and not mixture.is_cuda):
        raise RuntimeError("sudo_rm_rf_b200.bss_eval runs on CUDA tensors only (no CPU path)")
    if torch.is_grad_enabled() and (ref.requires_grad or est.requires_grad
                                    or (mixture is not None and mixture.requires_grad)):
        raise RuntimeError("sudo_rm_rf_b200.bss_eval is the evaluation metric only (no autograd): "
                           "wrap the call in torch.no_grad()")


def _fp32(ref, est, mixture):
    """Contiguous fp32 copies on ref's device (none when the inputs already are) -> (ref, est, mixture [B, T] or
    None)."""
    B, _, T = ref.shape
    dev = ref.device
    ref = ref.detach().to(torch.float32).contiguous()
    est = est.detach().to(device=dev, dtype=torch.float32).contiguous()
    mix = None
    if mixture is not None:
        mix = mixture.detach()
        if mix.numel() != B * T or mix.shape[-1] != T:
            raise RuntimeError(f"expected a mixture of {B} x {T} samples ([T], [1, T], [B, T] or [B, 1, T])")
        mix = mix.reshape(B, T).to(device=dev, dtype=torch.float32).contiguous()
    return ref, est, mix


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True, filter_length=512,
                     mixture=None, *, _windows=None, _images=False, _v4=False):
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

    Inputs of any floating dtype and stride are computed on as contiguous fp32.  Metric only: no autograd.

    ``_windows`` = ``(window, hop, lengths)`` is ``bss_eval_sources_framewise``'s call (see ``_framewise``): the
    outputs gain a last dimension of windows.  ``_images`` is ``bss_eval_images``' call (see ``_images_call``):
    inputs ``[..., S, T, C]`` and outputs ``(sdr, isr, sir, sar, perm)``; with ``_v4`` as well, ``bss_eval_v4``'s.
    Every BSS-eval entry allocates and enqueues here, on the caller's stream, so the stream and thread tests of this
    entry cover them all."""
    if _images:
        ref, est, single = _images_checked(reference_sources, estimated_sources)
        B, S, T, C = ref.shape
        F = int(filter_length)
        dev = ref.device
        nbytes, shape, enqueue = (_v4_call if _v4 else _images_call)(B, S, C, T, F, _windows, dev)
        ref, est, mix = _rows(ref, dev), _rows(est, dev), None
    else:
        ref, est, single = _checked(reference_sources, estimated_sources, mixture)
        B, S, T = ref.shape
        F = int(filter_length)
        dev = ref.device
        nbytes, shape, enqueue = _whole(B, S, T, F) if _windows is None else _framewise(B, S, T, F, *_windows, dev)
        ref, est, mix = _fp32(ref, est, mixture)
    with torch.cuda.device(dev):
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty((4 if _images else 3 if mix is None else 6,) + shape, dtype=torch.float64, device=dev)
        perm = torch.empty(shape, dtype=torch.int32, device=dev)
        code, what = enqueue(ref, est, mix, out, perm, 1 if compute_permutation else 0, scratch, N.stream(dev))
        N.check(code, what)
    if len(shape) == 3:                                     # [B, nwin, S] -> [B, S, nwin]
        out, perm = out.transpose(-1, -2).contiguous(), perm.transpose(-1, -2).contiguous()
    if single:
        out, perm = out[:, 0], perm[0]
    if _images:
        return out[0], out[1], out[2], out[3], perm.long()
    sdr, sir, sar = out[0], out[1], out[2]
    perm = perm.long()
    if mix is None:
        return sdr, sir, sar, perm
    extra = {"sdr": out[3], "sir": out[4], "sar": out[5],
             "sdri": sdr - out[3], "siri": sir - out[4], "sari": sar - out[5]}
    return sdr, sir, sar, perm, extra


def _whole(B, S, T, F):
    """sdr_bss_eval's scratch size, outputs [B, S] and call, refused before anything is allocated."""
    lib = N.lib()
    nbytes = lib.sdr_bss_eval_scratch_bytes(B, S, T, F)
    if nbytes == 0:
        raise N.NativeError("sdr_bss_eval supports 1..4 sources, filter lengths 1..512 and items of at least "
                            "(S - 1) * filter_length + 1 samples")

    def enqueue(ref, est, mix, out, perm, cp, scratch, stream):
        if mix is None:
            return lib.sdr_bss_eval(N.ptr(ref), N.ptr(est), N.ptr(out[0]), N.ptr(out[1]), N.ptr(out[2]), N.ptr(perm),
                                    B, S, T, F, cp, N.ptr(scratch), stream), "sdr_bss_eval"
        return lib.sdr_bss_eval_mixture(
            N.ptr(ref), N.ptr(est), N.ptr(mix), N.ptr(out[0]), N.ptr(out[1]), N.ptr(out[2]), N.ptr(perm),
            N.ptr(out[3]), N.ptr(out[4]), N.ptr(out[5]), B, S, T, F, cp, N.ptr(scratch), stream), "sdr_bss_eval_mixture"
    return nbytes, (B, S), enqueue


def _framewise(B, S, T, F, W, H, lengths, dev):
    """sdr_bss_eval_framewise's scratch size, outputs [B, nwin, S] and call, refused before anything is allocated."""
    lib = N.lib()
    nbytes = lib.sdr_bss_eval_framewise_scratch_bytes(B, S, T, W, H, F)
    if nbytes == 0:
        raise N.NativeError("sdr_bss_eval_framewise supports 1..4 sources, filter lengths 1..512 and windows (or, "
                            "when the whole item is scored, items) of at least (S - 1) * filter_length + 1 samples")
    lens = _lengths(lengths, B, dev)

    def enqueue(ref, est, mix, out, perm, cp, scratch, stream):
        m = [None] * 3 if mix is None else [out[3], out[4], out[5]]
        return lib.sdr_bss_eval_framewise(
            N.ptr(ref), N.ptr(est), N.ptr(mix), N.ptr(lens), N.ptr(out[0]), N.ptr(out[1]), N.ptr(out[2]), N.ptr(perm),
            N.ptr(m[0]), N.ptr(m[1]), N.ptr(m[2]), B, S, T, W, H, F, cp, N.ptr(scratch), stream), \
            "sdr_bss_eval_framewise"
    return nbytes, (B, window_count(T, W, H), S), enqueue


def _lengths(lengths, B, dev):
    """Per-recording lengths as a contiguous int64 CUDA tensor (None without them)."""
    if lengths is None:
        return None
    lens = torch.as_tensor(lengths).reshape(-1)
    if lens.numel() != B or lens.dtype.is_floating_point or lens.dtype.is_complex:
        raise RuntimeError(f"expected {B} integer lengths")
    if not lens.is_cuda and torch.cuda.is_current_stream_capturing():
        raise RuntimeError("lengths on the host are copied to the device with a host synchronisation, which a "
                           "CUDA graph cannot capture: pass them as a CUDA tensor")
    return lens.to(device=dev, dtype=torch.int64).contiguous()


def window_count(T, window, hop):
    """mir_eval's framewise window count, ``floor((T - window + hop) / hop)``, and 1 (the whole item) when that is
    below 2, that is when ``T < window + hop``."""
    return 1 if T - window < hop else (T - window) // hop + 1


def bss_eval_sources_framewise(reference_sources, estimated_sources, window=1323000, hop=661500,
                               compute_permutation=False, filter_length=512, mixture=None, lengths=None):
    """mir_eval's ``bss_eval_sources_framewise`` on CUDA tensors: the criteria of ``bss_eval_sources`` in windows of
    ``window`` samples every ``hop`` samples (the defaults are mir_eval's, 30 s and 15 s at 44.1 kHz).

    ``reference_sources`` and ``estimated_sources`` are ``[S, T]`` or ``[B, S, T]``; the outputs ``(sdr, sir, sar,
    perm)`` are ``[S, nwin]`` or ``[B, S, nwin]``, fp64 in dB and int64, with ``nwin = window_count(T, window, hop)``.
    Column k scores the slice ``[k hop, k hop + window)`` exactly as ``bss_eval_sources`` scores it (bit for bit), its
    permutation searched in that window alone when ``compute_permutation``.  When fewer than two windows fit
    (``T < window + hop``) the one column is ``bss_eval_sources`` of the whole item, as mir_eval does.  The windows
    are read in place: nothing is copied, and the scratch holds at most 128 windows, however long the recordings.

    A window in which a reference or estimate row is all zeros gets NaN in every output and ``perm = -1`` (mir_eval
    writes NaN there too); so does a window holding a NaN or an infinity, and windows that do not contain it keep their
    values.  mir_eval raises when a whole row is silent; here every window of such an item is NaN.

    ``lengths`` (``[B]`` integers) gives each recording its own length: item b has ``window_count(lengths[b],
    window, hop)`` columns, with the same whole-item fallback, and its columns past that are NaN with ``perm = -1``.
    The lengths are read on the device, so the output width follows from T and a length outside [1, T], or a fallback
    item shorter than ``(S - 1) * filter_length + 1``, gives NaN columns instead of an error.  As a CUDA tensor they
    cost no host synchronisation and the call can be captured in a CUDA graph; a sequence or a CPU tensor is copied to
    the device first, which synchronises with the host and is refused during graph capture.  ``mixture`` is as in
    ``bss_eval_sources`` and adds the same dict, per window.

    Limits are those of ``bss_eval_sources`` applied to the window: 1 <= S <= 4, 1 <= filter_length <= 512, and
    ``window >= (S - 1) * filter_length + 1`` (T, when the fallback applies).  Metric only: no autograd."""
    W, H = int(window), int(hop)
    if W < 1 or H < 1:
        raise RuntimeError("window and hop must be positive")
    return bss_eval_sources(reference_sources, estimated_sources, compute_permutation, filter_length, mixture,
                            _windows=(W, H, lengths))


def bss_eval_images(reference_sources, estimated_sources, compute_permutation=True, filter_length=512):
    """mir_eval's ``bss_eval_images`` on CUDA tensors: the BSS-eval criteria of multichannel source images.

    ``reference_sources`` and ``estimated_sources`` are in mir_eval's layout, ``[S, T, C]`` (S images of C channels,
    time before channels), or ``[B, S, T, C]`` for a batch; ``[S, T]`` is read as C = 1, as mir_eval does.  (A
    three-dimensional input is mir_eval's ``[S, T, C]``, so a batch of mono items is passed as ``[B, S, T, 1]``.)
    Per item, with F-tap distortion filters, ``P_j e_i`` projects each channel of estimate image i onto the F delays
    of all C channels of reference image j, ``P_all e_i`` onto the delays of every reference channel, and the
    energies sum over channels::

        SDR = 10 log10(|s_j|^2 / |e_i - s_j|^2)           ISR = 10 log10(|s_j|^2 / |P_j e_i - s_j|^2)
        SIR = 10 log10(|P_j e_i|^2 / |P_all e_i - P_j e_i|^2)
        SAR = 10 log10(|P_all e_i|^2 / |e_i - P_all e_i|^2)

    Returns ``(sdr, isr, sir, sar, perm)``, each ``[..., S]`` on the device: fp64 in dB, and int64 ``perm`` where
    ``perm[j]`` is the estimate scored against reference j (the assignment with the largest mean SIR with
    ``compute_permutation``, the first in ``itertools.permutations`` order; else estimate j).  For C = 1, SIR and SAR
    are ``bss_eval_sources``'s; SDR is measured against ``s_j`` itself rather than ``P_j e``.

    An all-zero channel of a non-silent image is dropped from its projections (the projection onto its other
    channels, as mir_eval's least-squares fallback gives).  An item in which a reference or estimate image is all
    zeros, or holds a NaN or an infinity, gets NaN in every output and ``perm = -1``; so does one whose references are
    too close to dependent for the normal equations (see ``bss_eval_sources``).

    Limits: 1 <= S * C <= 4, 1 <= filter_length <= 512 and T >= (S * C - 1) * filter_length + 1; two stereo sources
    fit, MUSDB's four stereo stems do not.  Inputs of any floating dtype and stride are copied once into a contiguous
    fp32 ``[B, S, C, T]`` tensor (not at all when they already are that, transposed).  Metric only: no autograd.

    A stereo model's ``[B, S*C, T]`` output (channel rows of each source together), scored against targets laid out
    the same way::

        sdr, isr, sir, sar, perm = bss_eval_images(tgt.view(B, S, C, T).transpose(-1, -2),
                                                   out.view(B, S, C, T).transpose(-1, -2))
    """
    return bss_eval_sources(reference_sources, estimated_sources, compute_permutation, filter_length, _images=True)


def bss_eval_images_framewise(reference_sources, estimated_sources, window=1323000, hop=661500,
                              compute_permutation=False, filter_length=512, lengths=None):
    """mir_eval's ``bss_eval_images_framewise`` on CUDA tensors: the criteria of ``bss_eval_images`` in windows of
    ``window`` samples every ``hop`` samples, with the layout of ``bss_eval_images``.

    Returns ``(sdr, isr, sir, sar, perm)``, each ``[..., S, nwin]`` with ``nwin = window_count(T, window, hop)``.
    Column k is ``bss_eval_images`` of the slice ``[k hop, k hop + window)``, bit for bit; when fewer than two windows
    fit (``T < window + hop``) the one column is the whole item.  Windows are read in place and the scratch holds at
    most 128 windows.  A window with a silent image, a NaN or an infinity is NaN with ``perm = -1``, alone.
    ``lengths`` is as in ``bss_eval_sources_framewise``: as a CUDA tensor it costs no host synchronisation, host
    lengths are refused during graph capture, and columns past a recording's windows are NaN with ``perm = -1``.

    Limits: 1 <= S * C <= 4, 1 <= filter_length <= 512, ``window >= (S * C - 1) * filter_length + 1`` (T when the
    fallback applies).  Metric only: no autograd."""
    W, H = int(window), int(hop)
    if W < 1 or H < 1:
        raise RuntimeError("window and hop must be positive")
    return bss_eval_sources(reference_sources, estimated_sources, compute_permutation, filter_length,
                            _windows=(W, H, lengths), _images=True)


def _images_checked(ref, est):
    """The checks of the image entries -> (ref, est as [B, S, T, C] views, whether they had no batch dimension)."""
    if ref.dim() not in (2, 3, 4) or est.shape != ref.shape:
        raise RuntimeError("expected reference_sources and estimated_sources of one shape, [S, T], [S, T, C] or "
                           "[B, S, T, C]")
    _usable(ref, est, None)
    single = ref.dim() < 4
    if ref.dim() == 2:
        ref, est = ref.unsqueeze(-1), est.unsqueeze(-1)
    if single:
        ref, est = ref.unsqueeze(0), est.unsqueeze(0)
    if ref.shape[0] == 0 or ref.shape[2] == 0 or ref.shape[3] == 0:
        raise RuntimeError("empty batch, zero-length signals or no channels")
    return ref, est, single


def _images_call(B, S, C, T, F, windows, dev):
    """sdr_bss_eval_images' (windows None) or sdr_bss_eval_images_framewise's scratch size, outputs [B, S] or
    [B, nwin, S] and call, refused before anything is allocated."""
    lib = N.lib()
    if windows is None:
        nbytes, shape, what = lib.sdr_bss_eval_images_scratch_bytes(B, S, C, T, F), (B, S), "sdr_bss_eval_images"
    else:
        W, H, lengths = windows
        nbytes = lib.sdr_bss_eval_images_framewise_scratch_bytes(B, S, C, T, W, H, F)
        shape, what = (B, window_count(T, W, H), S), "sdr_bss_eval_images_framewise"
    if nbytes == 0:
        raise N.NativeError(f"{what} supports 1 <= sources * channels <= 4, filter lengths 1..512 and "
                            + ("items" if windows is None else "windows (or, when the whole item is scored, items)")
                            + " of at least (sources * channels - 1) * filter_length + 1 samples; got "
                            f"{S} sources x {C} channels, filter_length {F}")
    lens = None if windows is None else _lengths(lengths, B, dev)

    def enqueue(ref, est, mix, out, perm, cp, scratch, stream):
        o = [N.ptr(out[i]) for i in range(4)]
        if windows is None:
            return lib.sdr_bss_eval_images(N.ptr(ref), N.ptr(est), *o, N.ptr(perm), B, S, C, T, F, cp,
                                           N.ptr(scratch), stream), what
        return lib.sdr_bss_eval_images_framewise(N.ptr(ref), N.ptr(est), N.ptr(lens), *o, N.ptr(perm), B, S, C, T,
                                                 W, H, F, cp, N.ptr(scratch), stream), what
    return nbytes, shape, enqueue


def bss_eval_v4(reference_sources, estimated_sources, window=44100, hop=44100, compute_permutation=False,
                filter_length=512, lengths=None):
    """museval's BSS-eval v4 (``museval.evaluate(..., mode='v4')``, the SiSEC 2018 / MUSDB18 metric) on CUDA tensors.

    ``reference_sources`` and ``estimated_sources`` are in ``bss_eval_images``' layout: ``[S, T, C]``, ``[S, T]``
    (C = 1) or ``[B, S, T, C]``.  The distortion filters are solved once per recording, from the correlations of its
    whole length: they are those ``bss_eval_images`` computes on the whole recording.  Window k, ``[k hop, k hop +
    window)``, then filters its own reference slice (zero outside the window) with them, and with ``s_j`` the reference
    slice, ``P_j e_i`` and ``P_all e_i`` the slice filtered by the own and joint filters and ``e_i`` the estimate
    slice, energies summed over channels::

        SDR = 10 log10(|s_j|^2 / |e_i - s_j|^2)           ISR = 10 log10(|s_j|^2 / |P_j e_i - s_j|^2)
        SIR = 10 log10(|P_j e_i|^2 / |P_all e_i - P_j e_i|^2)
        SAR = 10 log10(|P_all e_i|^2 / |e_i - P_all e_i|^2)

    (a zero denominator is +inf).  The defaults are museval's: one-second windows and hops at 44.1 kHz, no permutation
    search.  Returns ``(sdr, isr, sir, sar, perm)``, each ``[..., S, nwin]`` with ``nwin = (T - window) // hop + 1``,
    fp64 in dB and int64; with ``compute_permutation`` each window takes the assignment with the largest mean SIR in
    that window.  There is no whole-recording fallback: T < window is refused.

    A window in which a reference or estimate image is all zeros is NaN with ``perm = -1``.  A NaN or an infinity
    anywhere in a recording poisons its whole-track correlations, so every window of that recording is NaN with
    ``perm = -1`` (unlike ``bss_eval_images_framewise``, where only the windows holding it are); so is every window of
    a recording whose whole-track filters are no projection (see ``bss_eval_sources``).  Other recordings keep their
    values.  ``lengths`` (``[B]`` integers) gives each recording its own length, filters and window count; columns
    past that count are NaN with ``perm = -1``, and so is every column of a recording shorter than ``window`` or than
    ``(S * C - 1) * filter_length + 1``.  As a CUDA tensor they cost no host synchronisation and the call can be
    captured in a CUDA graph; host lengths are refused during capture.  A recording's columns are the same, bit for
    bit, in any batch.

    Limits: 1 <= S * C <= 4 (four mono stems, or stereo vocals and accompaniment; not four stereo stems),
    1 <= filter_length <= 512, T >= window and T >= (S * C - 1) * filter_length + 1.  The scratch stops growing with
    T past a few million samples per recording.  Metric only: no autograd."""
    W, H = int(window), int(hop)
    if W < 1 or H < 1:
        raise RuntimeError("window and hop must be positive")
    return bss_eval_sources(reference_sources, estimated_sources, compute_permutation, filter_length,
                            _windows=(W, H, lengths), _images=True, _v4=True)


def _v4_call(B, S, C, T, F, windows, dev):
    """sdr_bss_eval_v4's scratch size, outputs [B, nwin, S] and call, refused before anything is allocated."""
    lib = N.lib()
    W, H, lengths = windows
    nbytes = lib.sdr_bss_eval_v4_scratch_bytes(B, S, C, T, W, H, F)
    if nbytes == 0:
        raise N.NativeError("sdr_bss_eval_v4 supports 1 <= sources * channels <= 4, filter lengths 1..512 and "
                            "recordings of at least one window and (sources * channels - 1) * filter_length + 1 "
                            f"samples; got {S} sources x {C} channels, {T} samples, window {W}, filter_length {F}")
    lens = _lengths(lengths, B, dev)

    def enqueue(ref, est, mix, out, perm, cp, scratch, stream):
        o = [N.ptr(out[i]) for i in range(4)]
        return lib.sdr_bss_eval_v4(N.ptr(ref), N.ptr(est), N.ptr(lens), *o, N.ptr(perm), B, S, C, T, W, H, F, cp,
                                   N.ptr(scratch), stream), "sdr_bss_eval_v4"
    return nbytes, (B, (T - W) // H + 1, S), enqueue


def _rows(x, dev):
    """[B, S, T, C] -> contiguous fp32 [B, S, C, T] on dev: one copy, none when x already is that, transposed."""
    x = x.detach().transpose(-1, -2)
    if x.dtype == torch.float32 and x.device == dev and x.is_contiguous():
        return x
    return torch.empty(x.shape, dtype=torch.float32, device=dev).copy_(x)
