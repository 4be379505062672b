"""fp64 numpy/scipy restatements of the BSS-eval v3 source criteria (mir_eval.separation.bss_eval_sources).

``bss_eval`` forms the normal equations from FFT correlations (G block-Toeplitz through ``scipy.linalg.toeplitz``),
solves them with ``np.linalg.solve`` (``lstsq`` when G is singular), builds the projections with ``fftconvolve`` and
picks the assignment with the largest mean SIR.  ``bss_eval_direct`` is an independent formulation for small T: the
delayed references as explicit columns and ``np.linalg.lstsq``.  ``bss_eval_span`` projects by Householder QR onto
the delayed references the GPU's recursion keeps (see its docstring); it is the oracle for near-degenerate references,
where the normal equations are too ill-conditioned for ``np.linalg.solve``.  All take ``[S, T]`` arrays."""
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


def _defect(e, p):
    """| |p|^2 + |e - p|^2 - |e|^2 | / |e|^2: zero up to rounding for an orthogonal projection p of e."""
    return abs(np.sum(p ** 2) + np.sum((e - p) ** 2) - np.sum(e ** 2)) / np.sum(e ** 2)


def _bss_eval(refs, ests, compute_permutation, F, project, margin=False, defect_limit=None):
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
        p_target = project(refs[j:j + 1], ests[i], F)
        if defect_limit is not None and max(_defect(pad(ests[i]), p) for p in (p_target, p_all[i])) > defect_limit:
            nan = np.full(S, np.nan)
            return (nan, nan.copy(), nan.copy(), np.full(S, -1)) + ((np.inf,) if margin else ())
        crit[:, i, j] = _criteria(pad(ests[i]), p_target, p_all[i])
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


def bss_eval_mixture(refs, mix, F=512, oracle=bss_eval):
    """(sdr, sir, sar) [S] of the mixture scored as the estimate of every reference."""
    S = refs.shape[0]
    out = oracle(refs, np.stack([mix] * S), False, F)
    return tuple(out[:3])


# ---------------------------------------------------------------------------------------------------------------------
# span oracle: QR onto the delayed references that bsseval.cu's block-Levinson recursion keeps
# ---------------------------------------------------------------------------------------------------------------------
PIVOT_TOL = 1e-10           # bsseval.cu's kBssPivotTol, on unit-energy references


def _ginv(P):
    """The sweep operator of bss_ginv: pivots in channel order, one at or below PIVOT_TOL is skipped.  -> (the
    generalised inverse, which pivots were kept)."""
    M = P.shape[0]
    W = np.array(P, np.float64)
    kept = np.zeros(M, bool)
    for p in range(M):
        d = W[p, p]
        kept[p] = d > PIVOT_TOL
        if not kept[p]:
            continue
        o = np.arange(M) != p
        W[np.ix_(o, o)] -= np.outer(W[o, p], W[p, o]) / d
        W[o, p] /= d
        W[p, o] /= d
        W[p, p] = -1.0 / d
    return np.where(np.outer(kept, kept), -W, 0.0), kept


def _lag_correlations(refs, F):
    """R[k][r][q] = sum_t s_r[t] s_q[t + k] / sqrt(E_r E_q), k < F: the block-Toeplitz matrix in unit energy."""
    M, T = refs.shape
    n = 1 << int(np.ceil(np.log2(T + F)))
    rf = np.fft.rfft(refs, n=n, axis=1)
    c = np.fft.irfft(np.conj(rf)[:, None, :] * rf[None, :, :], n=n, axis=2)[:, :, :F]
    inv = 1.0 / np.sqrt(np.sum(refs * refs, axis=1))
    return np.transpose(c, (2, 0, 1)) * inv[None, :, None] * inv[None, None, :]


def _levinson(refs, F, e=None):
    """bsseval.cu's block-Levinson recursion restated in fp64 on unit-energy references.  Forward and backward
    predictors A, B and prediction-error matrices Pf, Pb grow by one lag per step, each inverted by _ginv; with an
    estimate e, the solution grows as x[k] += B_{n+1}[k] g, g = Pb^- (D[n+1] - eps).  -> (kept [F, M]: whether the
    sweep of the order-l backward error Pb kept pivot r, the filters [F, M] or None)."""
    refs = np.asarray(refs, np.float64)
    M, T = refs.shape
    R = _lag_correlations(refs, F)
    A = np.zeros((F, M, M))
    Br = np.zeros((F, M, M))
    A[0] = Br[0] = np.eye(M)
    Pf, Pb = R[0].copy(), R[0].copy()
    kept = np.zeros((F, M), bool)
    Pbi, kept[0] = _ginv(Pb)
    if e is not None:
        inv = 1.0 / np.sqrt(np.sum(refs * refs, axis=1))
        n2 = 1 << int(np.ceil(np.log2(T + F)))
        d = np.fft.irfft(np.conj(np.fft.rfft(refs, n=n2, axis=1)) * np.fft.rfft(e, n=n2)[None], n=n2, axis=1)
        rhs = (d[:, :F] * inv[:, None]).T                              # [F, M]: sum_t s_r[t] e[t + k] / sqrt(E_r)
        x = np.zeros((F, M))
        x[0] = Pbi @ rhs[0]
    for n in range(F - 1):
        D = np.einsum("kij,kjc->ic", R[n + 1:0:-1], A[:n + 1])          # sum_k R_{n+1-k} A[k]
        Pfi = _ginv(Pf)[0]
        Kf, Kb = Pbi @ D, Pfi @ D.T
        nPf, nPb = Pf - D.T @ Kf, Pb - D @ Kb
        Pf, Pb = 0.5 * (nPf + nPf.T), 0.5 * (nPb + nPb.T)
        Pbi, kept[n + 1] = _ginv(Pb)
        a, b = A[:n + 2].copy(), Br[n + 1::-1].copy()                  # A[k] and Brev[n + 1 - k]
        A[:n + 2] = a - b @ Kf
        Br[n + 1::-1] = b - a @ Kb
        if e is not None:
            g = Pbi @ (rhs[n + 1] - np.einsum("kij,kj->i", R[n + 1:0:-1], x[:n + 1]))
            x[:n + 2] += Br[n + 1::-1] @ g
    return kept, (x * inv[None, :] if e is not None else None)


def kept_delays(refs, F):
    """[F, M] bools: which delayed references (lag l, row r) the recursion keeps.  Pivot r of the order-l backward
    error is the energy of s_r delayed by l left after projecting out every shorter delay of every row and rows < r
    at delay l; the solve gives a dropped pivot's direction no weight."""
    return _levinson(refs, F)[0]


def _span_basis(refs, F):
    """An orthonormal basis (Householder QR) of the kept delays of refs' unit-energy rows, in R^(T+F-1)."""
    M, T = refs.shape
    kept = kept_delays(refs, F)
    unit = refs / np.sqrt(np.sum(refs * refs, axis=1, keepdims=True))
    A = np.zeros((T + F - 1, int(kept.sum())))
    for c, (l, r) in enumerate(zip(*np.nonzero(kept))):
        A[l:l + T, c] = unit[r]
    return np.linalg.qr(A)[0]


def bss_eval_span(refs, ests, compute_permutation=True, F=512, margin=False):
    """bss_eval with the projections onto the span of the delays that bsseval.cu keeps, by Householder QR of the
    explicit [T + F - 1, K] matrix of those delays: no normal equations, so no squared condition number.

    Why this is the GPU's answer, as long as the recursion keeps its prediction-error matrices positive
    semi-definite: the normal equations' matrix G is the Gram matrix of the delays in the order (lag, row).
    kept_delays restates the recursion's drop rule; every pivot it keeps is the energy of a delay orthogonal to the
    earlier ones, so the kept delays are linearly independent, and every dropped one lies within sqrt(PIVOT_TOL)
    (relative) of the span of the earlier ones.  Where nothing is dropped (white or AR references), this is the full
    projection, and it agrees with bss_eval and bss_eval_direct.  A row's prediction error never grows with the
    order, so once delay (r, l) is dropped the longer delays of r are dropped too: each row keeps a prefix of lags.
    None of this holds once the recursion loses definiteness (several band-limited references with deep stop bands,
    G's condition number near 1 / eps): its pivots then go non-positive where the true ones are ~1e-8, it drops
    delays that are not in the span, the kept lags need not be a prefix, and its solution is no projection; the GPU
    reports such an item NaN (PROJECTION_DEFECT), and this oracle says nothing about it.  Where something is dropped
    (a windowed tone's delays span a few dimensions to 1e-15), the full projection also collects whatever noise the
    dropped delays' residual directions happen to hold, which np.linalg.solve on the 1e15-conditioned G reports as
    several dB of error and QR of all delays as a little extra |P e|; this oracle projects onto the kept delays
    only.  The recursion itself is not exactly that projection: its generalised inverses still let a little of the
    dropped directions into the predictors, which moves a value by up to a few hundredths of a dB
    (bss_eval_recursion restates it exactly)."""
    cache = {}

    def project(r, e, F):
        key = r.tobytes()
        if key not in cache:
            cache[key] = _span_basis(r, F)
        Q = cache[key]
        ep = np.r_[e, np.zeros(F - 1)]
        return Q @ (Q.T @ ep)

    return _bss_eval(refs, ests, compute_permutation, F, project, margin)


def _project_recursion(refs, e, F):
    """Projection of e by the filters the restated recursion solves for."""
    c = _levinson(refs, F, e)[1]
    return sum(fftconvolve(c[:, r], refs[r]) for r in range(refs.shape[0]))


PROJECTION_DEFECT = 1e-2    # bsseval.cu's kBssProjectionDefect


def bss_eval_recursion(refs, ests, compute_permutation=True, F=512, margin=False):
    """bss_eval through the restated recursion (_project_recursion): the GPU's algorithm in fp64 on the host.  Where
    the recursion drops delays it differs from bss_eval_span by up to a few hundredths of a dB (see
    tests/test_gpu_bss_eval_space.py), because the generalised inverses still let the dropped delays' directions
    into the predictors; this restatement tells such a difference from a kernel error.  Like the GPU, it reports an
    item NaN and perm -1 when a projection it forms is not one: |p|^2 + |e - p|^2 off |e|^2 by more than
    PROJECTION_DEFECT |e|^2, which happens when the recursion loses definiteness."""
    return _bss_eval(refs, ests, compute_permutation, F, _project_recursion, margin, PROJECTION_DEFECT)


def recursion_defect(refs, e, F):
    """The Pythagoras defect (_defect) of the restated recursion's projection of e onto every delay of refs."""
    return _defect(np.r_[e, np.zeros(F - 1)], _project_recursion(np.asarray(refs, np.float64), e, F))


def span_defect(refs, e, F):
    """The same for QR onto the kept delays."""
    Q = _span_basis(np.asarray(refs, np.float64), F)
    ep = np.r_[e, np.zeros(F - 1)]
    return _defect(ep, Q @ (Q.T @ ep))
