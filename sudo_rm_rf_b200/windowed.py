"""Separation of recordings of any length in overlapping windows (DESIGN.md section 7e).

A whole-clip forward holds every encoder frame of the clip in its workspace and refuses clips past 2^31 elements per
layer, and its GlobLN / GroupNorm statistics span the whole clip, while the models are trained on a few seconds.
``separate_long`` cuts the recording into windows of ``window`` samples every ``hop`` samples, separates them in
batches of at most ``max_windows`` per recording through ``separate`` (``sdr_separate``) or ``forward``
(``sdr_forward``) on the model's shared workspace, puts each window's sources in the order of the window before it (the permutation that maximises the
centred correlation over their overlap) and cross-fades the overlaps.  Its memory is set by the window batch, not by
the length.  Everything after the input checks runs on the current stream without a host synchronisation.

``separate_long_corpus`` separates a corpus of recordings of different lengths in window batches they share
(DESIGN.md section 7i), each recording's result that of ``separate_long`` on it alone.
"""
import bisect
from typing import List, NamedTuple, Tuple

import torch

from . import _engine
from . import _native as N
from . import corpus


def window_hop(window, hop=None):
    """(W, H) after the checks: integers with W/2 <= H < W; the default hop is ceil(W / 2)."""
    if isinstance(window, bool) or not isinstance(window, int) or window < 2:
        raise ValueError(f"window must be an integer number of samples >= 2, got {window!r}")
    if hop is None:
        hop = (window + 1) // 2
    if isinstance(hop, bool) or not isinstance(hop, int) or not (window <= 2 * hop and hop < window):
        raise ValueError(f"hop must be an integer with window / 2 <= hop < window ({window}), got {hop!r}")
    return window, hop


def window_plan(T, W, H):
    """(K, starts, overlaps): the window count, window k's first sample k H, and O_k = min(W - H, T - k H), the length
    of the overlap of windows k-1 and k below T, for k >= 1."""
    K = 1 if T <= W else 1 + -(-(T - W) // H)
    return K, [k * H for k in range(K)], [min(W - H, T - k * H) for k in range(1, K)]


class CorpusPlan(NamedTuple):
    """How ``separate_long_corpus`` packs a corpus (DESIGN.md section 7i).  ``long`` and ``short``: the indices of the
    recordings longer than the window and of the others, in corpus order.  Per long recording j: ``offsets[j]``, its
    first sample per channel in the flat buffers (the sum of the lengths before it), ``firsts[j]``, its first global
    window (the sum of the window counts before it), and ``counts[j]``, its window count.  ``batches``: (g0, M) of
    every window batch, contiguous and in order.  ``windows`` and ``samples``: the totals over the long recordings."""
    long: List[int]
    short: List[int]
    offsets: List[int]
    firsts: List[int]
    counts: List[int]
    batches: List[Tuple[int, int]]
    windows: int
    samples: int

    def locate(self, g):
        """(j, k): global window g is window k of long recording j."""
        j = bisect.bisect_right(self.firsts, g) - 1
        return j, g - self.firsts[j]


def corpus_plan(lengths, W, H, max_windows):
    """The packing of recordings of ``lengths`` samples into batches of at most ``max_windows`` windows: recording-major
    in corpus order, each batch a contiguous range of global windows, so that a batch boundary splits at most one
    recording.  Pure host logic."""
    lengths = [int(T) for T in lengths]
    if not lengths:
        raise ValueError("separate_long_corpus needs at least one recording")
    if any(T < 1 for T in lengths):
        raise ValueError("every recording needs at least one sample")
    if max_windows < 1:
        raise ValueError(f"max_windows must be a positive integer, got {max_windows!r}")
    long = [i for i, T in enumerate(lengths) if T > W]
    short = [i for i, T in enumerate(lengths) if T <= W]
    counts = [window_plan(lengths[i], W, H)[0] for i in long]
    offsets, firsts, off, g = [], [], 0, 0
    for i, K in zip(long, counts):
        offsets.append(off)
        firsts.append(g)
        off += lengths[i]
        g += K
    M = min(max_windows, g)
    batches = [(g0, min(M, g - g0)) for g0 in range(0, g, M)] if g else []
    return CorpusPlan(long, short, offsets, firsts, counts, batches, g, off)


# The stage calls below run on buffers the caller allocated on the current stream for this one call (see
# separate_long): the caching allocator orders their reuse, and no state outlives the call.
def gather(x, batch, W, H, k0, M, desc=None):
    """Windows k0 .. k0+M-1 of x [B, A, T] into batch [B, M, A, W] (its first B M A W floats), zeros past T.  With a
    corpus's descriptors ``desc`` ([R, 3] int64, see ``separate_long_corpus``): global windows k0 .. k0+M-1 of the
    flat corpus x into batch [M, A, W]."""
    if desc is not None:
        A = batch.shape[-2]
        N.check(N.lib().sdr_window_gather_ragged(N.ptr(x), N.ptr(desc), desc.shape[0], A, W, H, k0, M, N.ptr(batch),
                                                 N.stream(x.device)), "sdr_window_gather_ragged")
        return
    B, A, T = x.shape
    N.check(N.lib().sdr_window_gather(N.ptr(x), N.ptr(batch), B, A, T, W, H, k0, M, N.stream(x.device)),
            "sdr_window_gather")


def merge(est, carry, perm, out, S, A, W, H, k0, M, scratch, desc=None):
    """Aligns and overlap-adds the estimates [B, M, S A, W] of windows k0 .. k0+M-1 into out [B, S A, T]; ``carry``
    holds what the previous batch's merge left, ``perm`` ([B, K, S] int32 or None) receives each window's order.
    With a corpus's descriptors ``desc``: the estimates [M, S A, W] of global windows k0 .. k0+M-1 into the flat
    corpus output, ``perm`` [G, S]."""
    if desc is not None:
        N.check(N.lib().sdr_window_merge_ragged(N.ptr(est), N.ptr(desc), desc.shape[0], N.ptr(carry), N.ptr(perm),
                                                N.ptr(out), S, A, W, H, k0, M, N.ptr(scratch), N.stream(out.device)),
                "sdr_window_merge_ragged")
        return
    B, T = out.shape[0], out.shape[-1]
    N.check(N.lib().sdr_window_merge(N.ptr(est), N.ptr(carry), N.ptr(perm), N.ptr(out), B, S, A, T, W, H, k0, M,
                                     N.ptr(scratch), N.stream(out.device)), "sdr_window_merge")


def separate_long(model, wav, window, hop=None, normalize=True, mixture_consistency=False, max_windows=32,
                  return_permutations=False):
    """``wav`` [B, A, T] (or [B, T] for mono) -> [B, S A, T] fp32.  ``T <= window``: exactly
    ``model.separate(wav, mixture_consistency=..., normalize=...)``.  Otherwise the windows are separated with the
    per-window README recipe (``normalize=True``, mono) or the plain forward (``normalize=False``) and merged as
    ``sdr_window_merge`` states.  ``return_permutations``: also the [B, K, S] int32 order of every window (output
    source s of window k is its raw source perm[b, k, s]; None for a single window)."""
    W, H = window_hop(window, hop)
    if isinstance(max_windows, bool) or not isinstance(max_windows, int) or max_windows < 1:
        raise ValueError(f"max_windows must be a positive integer, got {max_windows!r}")
    cfg = _engine.make_config(model)
    if wav.dim() == 2:
        wav = wav.unsqueeze(1)
    x = _engine._check_input(model, cfg, wav)
    B, A, T = x.shape
    if normalize and A != 1:
        raise RuntimeError("separate() follows the README recipe, which is written for mono mixtures")
    if mixture_consistency and A != 1:
        raise RuntimeError("mixture consistency (mixture_consistency.py:14-36) is defined for mono mixtures only; "
                           f"this model has in_audio_channels={A}")
    run = _engine.separate if normalize else _engine.forward
    if T <= W:
        out = run(model, wav, mixture_consistency=mixture_consistency)
        return (out, None) if return_permutations else out
    lib = N.lib()
    S = cfg.num_sources
    K = lib.sdr_window_count(T, W, H)
    M = min(max_windows, K)
    carry_bytes = lib.sdr_window_carry_bytes(B, S, A, W)
    scratch_bytes = lib.sdr_window_merge_scratch_bytes(B, S, M)
    if K == 0 or carry_bytes == 0 or scratch_bytes == 0:
        raise N.NativeError(f"windowed separation supports 1 to 4 sources and windows of at most 2^24 samples "
                            f"(num_sources={S}, window={W})")
    device = x.device
    with torch.cuda.device(device):
        batch = torch.empty((B * M, A, W), dtype=torch.float32, device=device)
        carry = torch.empty(carry_bytes, dtype=torch.uint8, device=device)
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=device)
        out = torch.empty((B, S * A, T), dtype=torch.float32, device=device)
        perm = torch.empty((B, K, S), dtype=torch.int32, device=device) if return_permutations else None
        for k0 in range(0, K, M):
            m = min(M, K - k0)
            gather(x, batch, W, H, k0, m)
            # the model's shared workspace and packed weights, as for any forward of B m windows
            est = run(model, batch[:B * m], mixture_consistency=mixture_consistency)
            merge(est, carry, perm, out, S, A, W, H, k0, m, scratch)
    return (out, perm) if return_permutations else out


def separate_long_corpus(model, wavs, window, hop=None, normalize=True, mixture_consistency=False, max_windows=32,
                         return_permutations=False):
    """``separate_long`` over a corpus: ``wavs`` is a sequence of CUDA tensors [A, T_r] (or [T_r] for mono) on one
    device, of any lengths.  Returns a list of [S A, T_r] fp32 tensors, and with ``return_permutations`` also a list
    of [K_r, S] int32 window orders (None for a recording of one window).  Recording r's result is
    ``separate_long(model, wavs[r][None], window, hop, normalize, mixture_consistency)[0]``, whatever shares its
    batches and whatever ``max_windows`` is.

    The windows of the recordings longer than ``window`` are laid out recording-major in corpus order and separated in
    shared batches of ``max_windows``; a batch boundary splits at most one recording, whose last window the carry
    holds.  The others are separated whole, grouped by padded length (``corpus.plan_buckets``).  Memory: the corpus's
    input and output, plus what one ``separate_long`` call with the same window batch takes."""
    W, H = window_hop(window, hop)
    if isinstance(max_windows, bool) or not isinstance(max_windows, int) or max_windows < 1:
        raise ValueError(f"max_windows must be a positive integer, got {max_windows!r}")
    wavs = list(wavs)
    if not wavs:
        raise ValueError("separate_long_corpus needs at least one recording")
    cfg = _engine.make_config(model)
    xs = [_engine._check_input(model, cfg, w.reshape(1, 1, -1) if w.dim() == 1 else w.unsqueeze(0))[0] for w in wavs]
    device = xs[0].device
    if any(x.device != device for x in xs):
        raise RuntimeError("separate_long_corpus takes every recording on one device")
    S, A = cfg.num_sources, xs[0].shape[0]
    if normalize and A != 1:
        raise RuntimeError("separate() follows the README recipe, which is written for mono mixtures")
    if mixture_consistency and A != 1:
        raise RuntimeError("mixture consistency (mixture_consistency.py:14-36) is defined for mono mixtures only; "
                           f"this model has in_audio_channels={A}")
    plan = corpus_plan([x.shape[-1] for x in xs], W, H, max_windows)
    outs, perms = [None] * len(xs), [None] * len(xs)
    with torch.cuda.device(device):
        if plan.short:
            _separate_whole(model, cfg, [xs[i] for i in plan.short], plan.short, outs, normalize, mixture_consistency,
                            max_windows)
        if plan.long:
            _separate_windows(model, cfg, xs, plan, outs, perms if return_permutations else None, W, H, S, A,
                              normalize, mixture_consistency)
    return (outs, perms) if return_permutations else outs


def _separate_whole(model, cfg, xs, idx, outs, normalize, mixture_consistency, max_batch):
    """The recordings that fit one window, as ``separate_long`` runs them: ``separate`` (through ``separate_corpus``,
    whose per-recording statistics span the true length) or ``forward`` at their own padded length, in batches of
    recordings that share it.  outs[idx[j]] receives recording j's [S A, T]."""
    if normalize:
        for i, o in zip(idx, corpus.separate_corpus(model, [x[0] for x in xs], max_batch=max_batch,
                                                    mixture_consistency=mixture_consistency)):
            outs[i] = o
        return
    A = xs[0].shape[0]
    for Tp, group in corpus.plan_buckets([x.shape[-1] for x in xs], corpus.model_padding_rule(cfg), max_batch):
        batch = torch.zeros((len(group), A, Tp), dtype=torch.float32, device=xs[0].device)
        for b, j in enumerate(group):
            batch[b, :, :xs[j].shape[-1]] = xs[j]
        est = _engine.forward(model, batch, mixture_consistency=mixture_consistency)
        for b, j in enumerate(group):
            outs[idx[j]] = est[b, :, :xs[j].shape[-1]].clone()


def _separate_windows(model, cfg, xs, plan, outs, perms, W, H, S, A, normalize, mixture_consistency):
    """The recordings longer than one window, in the shared window batches of ``plan``; outs (and perms, unless None)
    receive views of the flat output (and orders)."""
    lib = N.lib()
    M = plan.batches[0][1]
    carry_bytes = lib.sdr_window_ragged_carry_bytes(S, A, W)
    scratch_bytes = lib.sdr_window_ragged_scratch_bytes(S, M)
    if carry_bytes == 0 or scratch_bytes == 0:
        raise N.NativeError(f"windowed separation supports 1 to 4 sources and windows of at most 2^24 samples "
                            f"(num_sources={S}, window={W})")
    device = xs[0].device
    run = _engine.separate if normalize else _engine.forward
    x = torch.cat([xs[i].reshape(-1) for i in plan.long])
    # (off_r, T_r, g_r) per recording: the one upload of the call
    desc = torch.tensor([[o, xs[i].shape[-1], g] for i, o, g in zip(plan.long, plan.offsets, plan.firsts)],
                        dtype=torch.int64).to(device)
    batch = torch.empty((M, A, W), dtype=torch.float32, device=device)
    carry = torch.empty(carry_bytes, dtype=torch.uint8, device=device)
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=device)
    out = torch.empty(S * A * plan.samples, dtype=torch.float32, device=device)
    perm = torch.empty((plan.windows, S), dtype=torch.int32, device=device) if perms is not None else None
    for g0, m in plan.batches:
        gather(x, batch, W, H, g0, m, desc=desc)
        # the model's shared workspace and packed weights, as for any forward of m windows
        est = run(model, batch[:m], mixture_consistency=mixture_consistency)
        merge(est, carry, perm, out, S, A, W, H, g0, m, scratch, desc=desc)
    for j, i in enumerate(plan.long):
        T = xs[i].shape[-1]
        outs[i] = out[S * A * plan.offsets[j]:S * A * (plan.offsets[j] + T)].view(S * A, T)
        if perm is not None:
            perms[i] = perm[plan.firsts[j]:plan.firsts[j] + plan.counts[j]]
