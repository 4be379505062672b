"""fp64 numpy/scipy restatements of the BSS-eval v3 source criteria (mir_eval.separation.bss_eval_sources).

``bss_eval`` forms the normal equations from FFT correlations (G block-Toeplitz through ``scipy.linalg.toeplitz``),
solves them with ``np.linalg.solve`` (``lstsq`` when G is singular), builds the projections with ``fftconvolve`` and
picks the assignment with the largest mean SIR.  ``bss_eval_direct`` is an independent formulation for small T: the
delayed references as explicit columns and ``np.linalg.lstsq``.  Both take ``[S, T]`` arrays."""
import itertools

import numpy as np
from scipy.linalg import toeplitz
from scipy.signal import fftconvolve


def _db(num, den):
    if den == 0:
        return np.inf
    with np.errstate(divide="ignore"):
        return 10 * np.log10(num / den)


def _criteria(e, p_target, p_all):
    """(sdr, sir, sar) of estimate e (zero-padded to T + F - 1) from its two projections."""
    return (_db(np.sum(p_target ** 2), np.sum((e - p_target) ** 2)),
            _db(np.sum(p_target ** 2), np.sum((p_all - p_target) ** 2)),
            _db(np.sum(p_all ** 2), np.sum((e - p_all) ** 2)))


def _project_fft(refs, e, F):
    """Projection of e onto the F delays of every row of refs, in R^(T+F-1)."""
    S, T = refs.shape
    n = 1 << int(np.ceil(np.log2(T + F - 1)))
    rf = np.fft.rfft(refs, n=n, axis=1)
    ef = np.fft.rfft(e, n=n)
    G = np.zeros((S * F, S * F))
    D = np.zeros(S * F)
    for i in range(S):
        for j in range(S):
            c = np.fft.irfft(rf[i] * np.conj(rf[j]), n=n)        # c[k] = sum_t s_i[t + k] s_j[t]
            # G[(i,l),(j,m)] = sum_t s_i[t] s_j[t + l - m] = c[m - l]
            G[i * F:(i + 1) * F, j * F:(j + 1) * F] = toeplitz(np.r_[c[0], c[-1:-F:-1]], c[:F])
        d = np.fft.irfft(rf[i] * np.conj(ef), n=n)               # D[(i,l)] = sum_t s_i[t] e[t + l] = d[-l]
        D[i * F:(i + 1) * F] = np.r_[d[0], d[-1:-F:-1]]
    try:
        if S * F > T + F - 1:                    # more delayed references than dimensions: G is singular
            raise np.linalg.LinAlgError
        c = np.linalg.solve(G, D)
    except np.linalg.LinAlgError:
        c = np.linalg.lstsq(G, D, rcond=None)[0]
    return sum(fftconvolve(c[i * F:(i + 1) * F], refs[i]) for i in range(S))


def _project_direct(refs, e, F):
    S, T = refs.shape
    cols = [np.r_[np.zeros(l), r, np.zeros(F - 1 - l)] for r in refs for l in range(F)]
    A = np.stack(cols, 1)
    ep = np.r_[e, np.zeros(F - 1)]
    return A @ np.linalg.lstsq(A, ep, rcond=None)[0]


def _bss_eval(refs, ests, compute_permutation, F, project, margin=False):
    refs = np.asarray(refs, np.float64)
    ests = np.asarray(ests, np.float64)
    S, T = refs.shape
    if not (np.any(refs, axis=1).all() and np.any(ests, axis=1).all()):
        nan = np.full(S, np.nan)
        return (nan, nan.copy(), nan.copy(), np.full(S, -1)) + ((np.inf,) if margin else ())
    pad = lambda x: np.r_[x, np.zeros(F - 1)]      # noqa: E731
    pairs = [(i, j) for i in range(S) for j in range(S)] if compute_permutation else [(j, j) for j in range(S)]
    crit = np.full((3, S, S), np.nan)
    p_all = {}
    for i, j in pairs:
        if i not in p_all:
            p_all[i] = project(refs, ests[i], F)
        crit[:, i, j] = _criteria(pad(ests[i]), project(refs[j:j + 1], ests[i], F), p_all[i])
    idx = np.arange(S)
    if compute_permutation:
        perms = list(itertools.permutations(range(S)))
        mean_sir = [np.mean(crit[1][list(p), idx]) for p in perms]
        perm = np.array(perms[int(np.argmax(mean_sir))])
        top = np.sort(np.asarray(mean_sir))[::-1]
        gap = top[0] - top[1] if len(top) > 1 else np.inf
    else:
        perm, gap = idx, np.inf
    return (crit[0][perm, idx], crit[1][perm, idx], crit[2][perm, idx], perm) + ((gap,) if margin else ())


def bss_eval(refs, ests, compute_permutation=True, F=512, margin=False):
    """-> (sdr, sir, sar, perm) of one item, [S] each; NaN and perm -1 when a row is all zeros.  With margin, also the
    best mean SIR minus the runner-up's (the permutation is only determined up to that)."""
    return _bss_eval(refs, ests, compute_permutation, F, _project_fft, margin)


def bss_eval_direct(refs, ests, compute_permutation=True, F=512):
    """The same through explicit delayed-reference matrices and np.linalg.lstsq (small T only)."""
    return _bss_eval(refs, ests, compute_permutation, F, _project_direct)


def bss_eval_mixture(refs, mix, F=512):
    """(sdr, sir, sar) [S] of the mixture scored as the estimate of every reference."""
    S = refs.shape[0]
    out = [bss_eval(refs, np.stack([mix] * S), False, F)[k] for k in range(3)]
    return tuple(out)
