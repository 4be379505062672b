"""Separation of recordings of any length in overlapping windows (DESIGN.md section 7e).

A whole-clip forward holds every encoder frame of the clip in its workspace and refuses clips past 2^31 elements per
layer, and its GlobLN / GroupNorm statistics span the whole clip, while the models are trained on a few seconds.
``separate_long`` cuts the recording into windows of ``window`` samples every ``hop`` samples, separates them in
batches of at most ``max_windows`` per recording through ``separate`` (``sdr_separate``) or ``forward``
(``sdr_forward``) on the model's shared workspace, puts each window's sources in the order of the window before it (the permutation that maximises the
centred correlation over their overlap) and cross-fades the overlaps.  Its memory is set by the window batch, not by
the length.  Everything after the input checks runs on the current stream without a host synchronisation.
"""
import torch

from . import _engine
from . import _native as N


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


# The stage calls below run on buffers the caller allocated on the current stream for this one call (see
# separate_long): the caching allocator orders their reuse, and no state outlives the call.
def gather(x, batch, W, H, k0, M):
    """Windows k0 .. k0+M-1 of x [B, A, T] into batch [B, M, A, W] (its first B M A W floats), zeros past T."""
    B, A, T = x.shape
    N.check(N.lib().sdr_window_gather(N.ptr(x), N.ptr(batch), B, A, T, W, H, k0, M, N.stream(x.device)),
            "sdr_window_gather")


def merge(est, carry, perm, out, S, A, W, H, k0, M, scratch):
    """Aligns and overlap-adds the estimates [B, M, S A, W] of windows k0 .. k0+M-1 into out [B, S A, T]; ``carry``
    holds what the previous batch's merge left, ``perm`` ([B, K, S] int32 or None) receives each window's order."""
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
