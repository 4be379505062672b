"""mir_eval 0.7's bss_eval_images and bss_eval_images_framewise restated in fp64 numpy.

Per item: S reference images s_j and S estimated images e_i of C channels, in mir_eval's layout [S, T, C], and F-tap
distortion filters.  Each channel lives in R^(T+F-1), zero-padded.  P_j e_i projects each channel of e_i onto the span
of the F delays of all C channels of s_j, P_all e_i onto all S C F delayed reference channels, and energies sum over
channels (mir_eval's _bss_decomp_mtifilt_images and _bss_image_crit):
    SDR = |s_j|^2 / |e_i - s_j|^2,          ISR = |s_j|^2 / |P_j e_i - s_j|^2,
    SIR = |P_j e_i|^2 / |P_all e_i - P_j e_i|^2,  SAR = |P_all e_i|^2 / |e_i - P_all e_i|^2    in dB, 0 denominator +inf
The projections are least squares on the explicit matrix of delayed reference channels (QR with column pivoting),
so an all-zero channel, or any other dependent delay, drops out of the span.  With compute_permutation, the
assignment with the largest mean SIR (the first maximum in itertools.permutations order).

Where this restatement (and the GPU) differ from mir_eval, on purpose: an item with an all-zero reference or estimate
image, or one holding a NaN or an infinity, is NaN with perm -1 (mir_eval raises on a silent reference)."""
import itertools

import numpy as np
import scipy.linalg

from bss_framewise_oracle import spans


def _db(num, den):
    with np.errstate(divide="ignore"):
        return np.inf if den == 0 else 10.0 * np.log10(num / den)


def _delays(x, F):
    """x [T] -> [T + F - 1, F], column l = x delayed by l samples."""
    T = len(x)
    A = np.zeros((T + F - 1, F))
    for l in range(F):
        A[l:l + T, l] = x
    return A


def _project(A, Y):
    """Orthogonal projection of the columns of Y onto the column span of A."""
    coef = scipy.linalg.lstsq(A, Y, lapack_driver="gelsy")[0]
    return A @ coef


def _as_images(x):
    x = np.asarray(x, np.float64)
    return x[..., None] if x.ndim == 2 else x


def scorable(refs, ests):
    """Every image has positive, finite energy."""
    refs, ests = _as_images(refs), _as_images(ests)
    energies = np.concatenate([np.sum(refs ** 2, axis=(1, 2)), np.sum(ests ** 2, axis=(1, 2))])
    return bool(np.all(np.isfinite(energies)) and np.all(energies > 0))


def criteria(refs, ests, F=512):
    """All pairs: (sdr, isr, sir, sar) [S_est, S_ref] for refs, ests [S, T, C] (or [S, T], C = 1)."""
    refs, ests = _as_images(refs), _as_images(ests)
    S, T, C = refs.shape
    L = T + F - 1
    pad = np.zeros((S, L, C))
    pad[:, :T] = refs
    Y = np.zeros((L, S * C))                          # every estimate channel, padded: column i C + c
    for i in range(S):
        Y[:T, i * C:(i + 1) * C] = ests[i]
    own = [np.hstack([_delays(refs[j, :, c], F) for c in range(C)]) for j in range(S)]
    p_all = _project(np.hstack(own), Y)
    p_own = [_project(A, Y) for A in own]
    out = np.zeros((4, S, S))
    for i in range(S):
        cols = slice(i * C, (i + 1) * C)
        e, pa = Y[:, cols], p_all[:, cols]
        for j in range(S):
            s, pj = pad[j], p_own[j][:, cols]
            s2 = np.sum(s ** 2)
            out[:, i, j] = (_db(s2, np.sum((e - s) ** 2)), _db(s2, np.sum((pj - s) ** 2)),
                            _db(np.sum(pj ** 2), np.sum((pa - pj) ** 2)), _db(np.sum(pa ** 2), np.sum((e - pa) ** 2)))
    return out


def bss_eval_images(refs, ests, compute_permutation=True, F=512):
    """refs, ests [S, T, C] (or [S, T]) -> (sdr, isr, sir, sar, perm), each [S], perm[j] the estimate given j."""
    refs, ests = _as_images(refs), _as_images(ests)
    S = refs.shape[0]
    if not scorable(refs, ests):
        nan = np.full(S, np.nan)
        return nan, nan.copy(), nan.copy(), nan.copy(), np.full(S, -1)
    crit = criteria(refs, ests, F)
    perm = np.arange(S)
    if compute_permutation:
        best = -np.inf
        for p in itertools.permutations(range(S)):
            m = np.mean([crit[2, p[j], j] for j in range(S)])
            if m > best:
                best, perm = m, np.array(p)
    idx = np.arange(S)
    return crit[0, perm, idx], crit[1, perm, idx], crit[2, perm, idx], crit[3, perm, idx], perm


def bss_eval_images_framewise(refs, ests, W, H, compute_permutation=False, F=512, length=None):
    """refs, ests [S, T, C] -> (sdr, isr, sir, sar, perm) [S, ncol], mir_eval's windows and fallback
    (bss_framewise_oracle.spans with S C rows); ``length`` as in bss_framewise_oracle."""
    refs, ests = _as_images(refs), _as_images(ests)
    S, T, C = refs.shape
    cols = []
    for sp in spans(T, W, H, S * C, F, length):
        if sp is None:
            nan = np.full(S, np.nan)
            cols.append((nan, nan, nan, nan, np.full(S, -1)))
        else:
            cols.append(bss_eval_images(refs[:, sp[0]:sp[1]], ests[:, sp[0]:sp[1]], compute_permutation, F))
    return tuple(np.stack([c[i] for c in cols], 1) for i in range(5))
