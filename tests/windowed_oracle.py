"""fp64 numpy restatement of windowed separation (DESIGN.md section 7e): the window plan, the alignment of each
window's sources with the window before it, and the fp32 cross-fade."""
import itertools

import numpy as np


def plan(T, W, H):
    """(K, starts, overlaps): K windows, window k starting at k H, overlap k (k >= 1) of O_k samples below T."""
    if T <= W:
        return 1, [0], []
    K = 1 + int(np.ceil((T - W) / H))
    starts = [k * H for k in range(K)]
    overlaps = [len(range(k * H, min((k - 1) * H + W, T))) for k in range(1, K)]
    return K, starts, overlaps


def windows(x, W, H):
    """x [B, A, T] -> [B, K, A, W], zeros past T."""
    B, A, T = x.shape
    K, starts, _ = plan(T, W, H)
    out = np.zeros((B, K, A, W), dtype=x.dtype)
    for k, s in enumerate(starts):
        n = min(W, T - s)
        out[:, k, :, :n] = x[:, :, s:s + n]
    return out


def correlation(prev, cur, H, O):
    """C[i][j] = sum_a sum_t (p_ia - mean p_ia)(c_ja - mean c_ja) over the overlap; prev, cur [S, A, W]."""
    p = prev[:, :, H:H + O].astype(np.float64)
    c = cur[:, :, :O].astype(np.float64)
    p = p - p.mean(axis=-1, keepdims=True)
    c = c - c.mean(axis=-1, keepdims=True)
    return np.einsum("iat,jat->ij", p, c)


def best(C):
    """(rho, margin): the first maximum of sum_i C[i][rho(i)] over itertools.permutations (the identity when C is not
    finite) and the relative gap between the best score and the runner-up (inf when there is none)."""
    S = C.shape[0]
    if S == 1 or not np.all(np.isfinite(C)):
        return tuple(range(S)), np.inf
    scores = []
    for p in itertools.permutations(range(S)):
        s = 0.0
        for i in range(S):
            s = s + C[i][p[i]]
        scores.append((s, p))
    top = max(s for s, _ in scores)
    rho = next(p for s, p in scores if s == top)
    rest = sorted((s for s, _ in scores), reverse=True)[1]
    scale = max(abs(top), abs(rest), 1e-300)
    return rho, (top - rest) / scale


def align(est, T, W, H):
    """est [B, K, S, A, W] -> (pi [B, K, S], margin [B, K]): pi_0 = id, pi_k(s) = rho_k(pi_{k-1}(s))."""
    B, K, S = est.shape[:3]
    _, _, overlaps = plan(T, W, H)
    pi = np.zeros((B, K, S), dtype=np.int64)
    margin = np.full((B, K), np.inf)
    for b in range(B):
        cur = list(range(S))
        pi[b, 0] = cur
        for k in range(1, K):
            rho, margin[b, k] = best(correlation(est[b, k - 1], est[b, k], H, overlaps[k - 1]))
            cur = [rho[s] for s in cur]
            pi[b, k] = cur
    return pi, margin


def fade(prev, cur, j, overlap):
    """The fp32 cross-fade of overlap samples j (an array; prev and cur have j's shape in front), operation for
    operation as the kernel's window_fade: r = (j + 1) / (overlap + 1), (1 - r) prev + r cur."""
    f = np.float32
    r = np.asarray(j + 1).astype(f) / f(overlap + 1)
    r = r.reshape(r.shape + (1,) * (prev.ndim - r.ndim))
    return (f(1) - r) * prev.astype(f) + r * cur.astype(f)


def overlap_add(est, pi, T, W, H):
    """est [B, K, S, A, W] fp32 and pi [B, K, S] -> [B, S A, T] fp32."""
    B, K, S, A, _ = est.shape
    out = np.zeros((B, S, A, T), dtype=np.float32)
    t = np.arange(T)
    k = np.minimum(t // H, K - 1)
    j = t - k * H
    two = (k > 0) & (j < W - H)
    kp = np.maximum(k - 1, 0)
    for b in range(B):
        for s in range(S):
            cur = est[b, k, pi[b, k, s], :, j]                   # [T, A]
            prev = est[b, kp, pi[b, kp, s], :, np.minimum(j + H, W - 1)]
            out[b, s] = np.where(two[:, None], fade(prev, cur, j, W - H), cur).T
    return out.reshape(B, S * A, T)
