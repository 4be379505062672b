"""museval's BSS-eval v4 (``museval.evaluate(..., mode='v4')``, the SiSEC 2018 / MUSDB18 metric) restated in fp64
numpy from its definition; museval's source was not at hand, so this is a restatement, not a copy.

Per recording: S reference images s_j and S estimated images e_i of C channels, in mir_eval's layout [S, n, C], R = S C
rows, F-tap distortion filters.
- Filters once per recording, from the whole length n: the joint filters project each estimate channel onto all R F
  delayed reference channels, source j's own filters onto its C F delays.  The normal equations G c = D are formed
  from lagged correlations (by FFT) and solved with np.linalg.solve: the filters bss_eval_images computes on the whole
  recording.
- Windows: nwin = (n - W) // H + 1 for n >= W, none otherwise (no whole-recording fallback); window k covers
  [k H, k H + W).  Its reference and estimate slices are signals of their own, zero outside the window; in
  R^(W + F - 1), with P_j and P_all the slice filtered by the own and joint filters and energies summed over channels:
      SDR = |s|^2 / |e - s|^2,  ISR = |s|^2 / |P_j - s|^2,  SIR = |P_j|^2 / |P_all - P_j|^2,  SAR = |P_all|^2 / |e - P_all|^2
  in dB, a zero denominator +inf.  (s_true = s, e_spat = P_j - s, e_interf = P_all - P_j, e_artif = e - P_all.)
- A window in which any reference or estimate image is all zeros is NaN with perm -1.  A NaN or an infinity anywhere
  in the recording makes every window NaN with perm -1; so does a recording shorter than W or than (R - 1) F + 1.
- With compute_permutation, each window takes the assignment with the largest mean SIR in that window (the first
  maximum in itertools.permutations order); otherwise estimate j for reference j.
Recalled, not checked against museval: that it has no whole-recording fallback, and its silence test on estimates."""
import itertools

import numpy as np

from bss_images_oracle import _as_images, _db


def _xcorr(a, b, F):
    """X[k] = sum_t a[t] b[t + k], k < F, for rows a [n], b [n]."""
    n = len(a)
    N = 1 << int(np.ceil(np.log2(n + F)))
    return np.fft.irfft(np.conj(np.fft.rfft(a, N)) * np.fft.rfft(b, N), N)[:F]


def _normal_equations(rows, ests, F):
    """rows [M, n] reference rows, ests [E, n] -> G [M F, M F], D [M F, E], G[(r,l),(q,m)] = X_rq[l - m]."""
    M = len(rows)
    X = {(r, q): _xcorr(rows[r], rows[q], F) for r in range(M) for q in range(M)}
    G = np.zeros((M * F, M * F))
    lag = np.arange(F)[:, None] - np.arange(F)[None, :]                 # l - m
    for r in range(M):
        for q in range(M):
            G[r * F:(r + 1) * F, q * F:(q + 1) * F] = np.where(lag >= 0, X[(r, q)][np.abs(lag)],
                                                               X[(q, r)][np.abs(lag)])
    D = np.stack([np.concatenate([_xcorr(rows[r], e, F) for r in range(M)]) for e in ests], 1)
    return G, D


def track_filters(refs, ests, F):
    """Whole-recording filters of refs, ests [S, n, C]: (cj, ct), each [R, R, F]: estimate row e's joint filters on
    reference row r, and its own-source filters (row r of source r // C, from that source's own system)."""
    refs, ests = _as_images(refs), _as_images(ests)
    S, n, C = refs.shape
    R = S * C
    rows = refs.transpose(0, 2, 1).reshape(R, n)
    erows = ests.transpose(0, 2, 1).reshape(R, n)
    G, D = _normal_equations(rows, erows, F)
    cj = np.linalg.solve(G, D).T.reshape(R, R, F)
    ct = np.zeros((R, R, F))
    for j in range(S):
        Gj, Dj = _normal_equations(rows[j * C:(j + 1) * C], erows, F)
        ct[:, j * C:(j + 1) * C] = np.linalg.solve(Gj, Dj).T.reshape(R, C, F)
    return cj, ct


def window_criteria(refs, ests, cj, ct, start, W):
    """All pairs' (sdr, isr, sir, sar) [4, S_est, S_ref] of the window [start, start + W) under fixed filters."""
    refs, ests = _as_images(refs), _as_images(ests)
    S, _, C = refs.shape
    R = S * C
    F = cj.shape[-1]
    s = refs[:, start:start + W].transpose(0, 2, 1).reshape(R, W)
    e = ests[:, start:start + W].transpose(0, 2, 1).reshape(R, W)
    L = W + F - 1
    spad = np.zeros((R, L))
    spad[:, :W] = s
    epad = np.zeros((R, L))
    epad[:, :W] = e
    pa = np.stack([sum(np.convolve(cj[x, r], s[r]) for r in range(R)) for x in range(R)])           # [R est rows, L]
    pj = np.stack([[sum(np.convolve(ct[x, j * C + c], s[j * C + c]) for c in range(C)) for j in range(S)]
                   for x in range(R)])                                                               # [R, S, L]
    out = np.zeros((4, S, S))
    for i in range(S):
        xs = range(i * C, (i + 1) * C)
        for j in range(S):
            sj = np.stack([spad[j * C + x % C] for x in xs])
            ej = epad[list(xs)]
            pjj = np.stack([pj[x, j] for x in xs])
            paj = pa[list(xs)]
            s2 = np.sum(sj ** 2)
            out[:, i, j] = (_db(s2, np.sum((ej - sj) ** 2)), _db(s2, np.sum((pjj - sj) ** 2)),
                            _db(np.sum(pjj ** 2), np.sum((paj - pjj) ** 2)),
                            _db(np.sum(paj ** 2), np.sum((ej - paj) ** 2)))
    return out


def window_count(T, W, H):
    return (T - W) // H + 1


def bss_eval_v4(refs, ests, W, H, compute_permutation=False, F=512, length=None):
    """refs, ests [S, T, C] (or [S, T]) -> (sdr, isr, sir, sar, perm), each [S, nwin] with nwin = window_count(T, W,
    H); ``length`` scores the recording as its first ``length`` samples (its own filters and windows, NaN past them)."""
    refs, ests = _as_images(refs), _as_images(ests)
    S, T, C = refs.shape
    ncol = window_count(T, W, H)
    out = [np.full((S, ncol), np.nan) for _ in range(4)] + [np.full((S, ncol), -1)]
    n = T if length is None else int(length)
    if n < W or n < (S * C - 1) * F + 1 or n > T:
        return tuple(out)
    refs, ests = refs[:, :n], ests[:, :n]
    if not (np.isfinite(refs).all() and np.isfinite(ests).all()):
        return tuple(out)
    if any(not np.any(x[j]) for x in (refs, ests) for j in range(S)):        # silent over the whole recording
        return tuple(out)
    cj, ct = track_filters(refs, ests, F)
    for k in range(window_count(n, W, H)):
        a = k * H
        if any(not np.any(x[j, a:a + W]) for x in (refs, ests) for j in range(S)):
            continue
        crit = window_criteria(refs, ests, cj, ct, a, W)
        perm = np.arange(S)
        if compute_permutation:
            best = -np.inf
            for p in itertools.permutations(range(S)):
                m = np.mean([crit[2, p[j], j] for j in range(S)])
                if m > best:
                    best, perm = m, np.array(p)
        idx = np.arange(S)
        for q in range(4):
            out[q][:, k] = crit[q, perm, idx]
        out[4][:, k] = perm
    return tuple(out)
