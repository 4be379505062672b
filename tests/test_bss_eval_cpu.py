"""BSS-eval without a GPU: the fp64 oracle formulations agree (the span oracle with the others where the recursion
drops nothing; on windowed tones the normal equations fail), the C-ABI symbols bind, the scratch query refuses
unsupported arguments, and the Python entry refuses CPU tensors and inputs that require grad."""
import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from bss_oracle import _criteria, bss_eval, bss_eval_direct, bss_eval_recursion, bss_eval_span, kept_delays

SYMBOLS = ("sdr_bss_eval_scratch_bytes", "sdr_bss_eval", "sdr_bss_eval_mixture")


def agree(a, b, tol):
    """Equal where infinite or NaN, within tol elsewhere."""
    a, b = np.asarray(a), np.asarray(b)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    return bool(np.all(same | (np.abs(a - b) <= tol)))


@pytest.mark.parametrize("S,T,F,seed", [(1, 60, 8, 0), (2, 200, 16, 1), (3, 150, 24, 2), (4, 120, 12, 3),
                                        (2, 90, 30, 4)])
def test_oracle_formulations_agree(S, T, F, seed):
    rng = np.random.default_rng(seed)
    refs = rng.standard_normal((S, T))
    refs[-1] = np.convolve(refs[-1], [1.0, 0.9, 0.5])[:T]                    # one coloured reference
    ests = rng.standard_normal((S, S)) @ refs + 0.05 * rng.standard_normal((S, T))
    ests[0] = np.convolve(ests[0], [0.7, -0.2, 0.1])[:T]
    for perm in (True, False):
        a, b = bss_eval(refs, ests, perm, F), bss_eval_direct(refs, ests, perm, F)
        for x, y in zip(a[:3], b[:3]):
            assert agree(x, y, 1e-9), (x, y)
        assert np.array_equal(a[3], b[3])


def test_oracle_silent_rows():
    refs = np.ones((2, 50))
    ests = np.ones((2, 50))
    ests[1] = 0
    sdr, sir, sar, perm = bss_eval(refs, ests, True, 4)
    assert np.isnan(sdr).all() and np.isnan(sir).all() and np.isnan(sar).all() and (perm == -1).all()


def test_symbols_bind_and_scratch_limits():
    lib = N.lib()
    for name in SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 32000, 512) > 0
    assert lib.sdr_bss_eval_scratch_bytes(1, 4, 4, 1) > 0 and lib.sdr_bss_eval_scratch_bytes(1, 4, 3, 1) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 5, 1000, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 0, 1000, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 1000, 0) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 1000, 513) == 0
    assert lib.sdr_bss_eval_scratch_bytes(0, 2, 1000, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 0, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 1, 1, 512) > 0                    # one reference: any length
    assert lib.sdr_bss_eval_scratch_bytes(4, 3, 1025, 512) > 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 3, 1024, 512) == 0                # 3 x 512 delays in R^1535
    # null buffers are refused before anything is enqueued
    assert lib.sdr_bss_eval(None, None, None, None, None, None, 1, 2, 100, 16, 1, None, None) == -2


def test_refusals():
    x = torch.zeros(2, 100)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.bss_eval_sources(x, x)
    with pytest.raises(RuntimeError, match="shape"):
        P.bss_eval_sources(x, torch.zeros(3, 100))
    g = torch.zeros(2, 100, requires_grad=True)
    with pytest.raises(RuntimeError, match="CUDA|no autograd"):
        P.bss_eval_sources(g, x)
    assert P.bss_eval_sources is P.bss_eval.bss_eval_sources


@pytest.mark.parametrize("S,T,F,seed", [(1, 60, 8, 0), (2, 200, 16, 1), (3, 150, 24, 2), (4, 120, 12, 3),
                                        (2, 90, 30, 4)])
def test_span_oracle_equals_full_projection_when_nothing_is_dropped(S, T, F, seed):
    """On the well-conditioned cases above the recursion keeps every delay, and QR onto them and the restated
    recursion give the normal equations' and lstsq's values within 1e-9 dB."""
    rng = np.random.default_rng(seed)
    refs = rng.standard_normal((S, T))
    refs[-1] = np.convolve(refs[-1], [1.0, 0.9, 0.5])[:T]
    ests = rng.standard_normal((S, S)) @ refs + 0.05 * rng.standard_normal((S, T))
    ests[0] = np.convolve(ests[0], [0.7, -0.2, 0.1])[:T]
    assert kept_delays(refs, F).all()
    for perm in (True, False):
        a, b = bss_eval(refs, ests, perm, F), bss_eval_direct(refs, ests, perm, F)
        c, d = bss_eval_span(refs, ests, perm, F), bss_eval_recursion(refs, ests, perm, F)
        for x, y, z, w in zip(a[:3], b[:3], c[:3], d[:3]):
            assert agree(x, z, 1e-9) and agree(y, z, 1e-9) and agree(w, z, 1e-9), (x, y, z, w)
        assert np.array_equal(a[3], c[3]) and np.array_equal(a[3], d[3])


@pytest.mark.parametrize("S,pole", [(1, 0.0), (2, 0.9), (4, 0.95), (2, 0.999)])
def test_nothing_dropped_on_white_and_ar_references(S, pole):
    rng = np.random.default_rng(20 + S)
    refs = lfilter([1.0], [1.0, -pole], rng.standard_normal((S, 4000)), axis=1).astype(np.float32)
    assert kept_delays(refs.astype(np.float64), 512).all()


def windowed_tones(T=32000):
    t = np.arange(T)
    return (sum(np.sin(2 * np.pi * f / 16000 * t + i) for i, f in enumerate((100, 200, 300)))
            * np.hanning(T)).astype(np.float32).astype(np.float64)


def test_windowed_tones_defeat_the_normal_equations():
    """A Hann-windowed sum of three tones (fp32) with an estimate at 20 dB SNR, T = 32000, F = 512.  Its 512 delays
    span a handful of dimensions to 1e-15, so G's condition number is ~1e15: np.linalg.solve (mir_eval's method)
    reports an SDR many dB off (1.1 dB with one LAPACK build; the figure depends on the build), QR onto every delay
    20.06 dB, QR onto the kept delays 20.00 dB, the noise level.  The recursion keeps a prefix of 5 lags, then
    nothing."""
    rng = np.random.default_rng(0)
    T, F = 32000, 512
    ref = windowed_tones(T)[None]
    noise = rng.standard_normal(T)
    est = (ref[0] + noise * np.sqrt(np.sum(ref[0] ** 2) / np.sum(noise ** 2) / 100)).astype(np.float32)
    est = est.astype(np.float64)[None]
    kept = kept_delays(ref, F)[:, 0]
    n = int(kept.sum())
    assert 3 <= n <= 12 and kept[:n].all(), n
    span = bss_eval_span(ref, est, False, F)[0][0]
    solve = bss_eval(ref, est, False, F)[0][0]
    cols = np.stack([np.r_[np.zeros(l), ref[0], np.zeros(F - 1 - l)] for l in range(F)], 1)
    Q = np.linalg.qr(cols)[0]
    e = np.r_[est[0], np.zeros(F - 1)]
    full = _criteria(e, Q @ (Q.T @ e), Q @ (Q.T @ e))[0]
    assert abs(span - 20.0) < 0.05, span
    assert 0.0 <= full - span < 0.2, (full, span)
    assert abs(solve - full) > 3.0, (solve, full)
