"""BSS-eval v4 without a GPU: the fp64 numpy restatement of museval's v4 (bss_v4_oracle.py) checked against itself
(its whole-track filters against explicit-matrix least squares, one whole-recording window against bss_eval_images,
silent windows); the bindings, scratch query and refusals of sdr_bss_eval_v4; the Python entry's refusals, which come
before any allocation, and its shapes."""
import contextlib
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from bss_images_oracle import _delays, bss_eval_images
from bss_v4_oracle import bss_eval_v4, track_filters, window_count
from test_bss_eval_images_cpu import close, images

BAD_ARGUMENT, UNSUPPORTED = -2, -5
HEADER = Path(__file__).resolve().parents[1] / "include" / "sudormrf_b200.h"
ENTRIES = ("sdr_bss_eval_v4_scratch_bytes", "sdr_bss_eval_v4")
TRACK_CHUNK, TRACK_BLOCKS = 8192, 512       # bsseval.cu's kBssTrackChunk and kBssTrackBlocks


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against itself
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,C,n,F", [(1, 1, 300, 8), (2, 1, 400, 16), (4, 1, 300, 12), (1, 2, 300, 8),
                                     (2, 2, 500, 10), (1, 4, 260, 6)])
def test_filters_are_least_squares(S, C, n, F):
    rng = np.random.default_rng(10 * S + C)
    refs, ests = images(rng, S, n, C)
    cj, ct = track_filters(refs, ests, F)
    R = S * C
    rows = [refs[j, :, c] for j in range(S) for c in range(C)]
    Y = np.zeros((n + F - 1, R))
    for x in range(R):
        Y[:n, x] = ests[x // C, :, x % C]
    A = np.hstack([_delays(r, F) for r in rows])
    want = np.linalg.lstsq(A, Y, rcond=None)[0].T.reshape(R, R, F)
    assert np.max(np.abs(cj - want)) <= 1e-9 * max(1.0, np.max(np.abs(want)))
    for j in range(S):
        Aj = np.hstack([_delays(r, F) for r in rows[j * C:(j + 1) * C]])
        wj = np.linalg.lstsq(Aj, Y, rcond=None)[0].T.reshape(R, C, F)
        assert np.max(np.abs(ct[:, j * C:(j + 1) * C] - wj)) <= 1e-9 * max(1.0, np.max(np.abs(wj)))


@pytest.mark.parametrize("S,C,n,F,perm", [(1, 1, 200, 8, False), (2, 1, 300, 16, True), (3, 1, 200, 12, True),
                                          (1, 2, 200, 8, False), (2, 2, 240, 8, True), (1, 3, 150, 6, False)])
def test_one_whole_window_is_bss_eval_images(S, C, n, F, perm):
    rng = np.random.default_rng(100 * S + C)
    refs, ests = images(rng, S, n, C)
    got = bss_eval_v4(refs, ests, n, n, perm, F)
    want = bss_eval_images(refs, ests, perm, F)
    assert got[0].shape == (S, 1)
    assert np.array_equal(got[4][:, 0], want[4])
    for g, w in zip(got[:4], want[:4]):
        assert close(g[:, 0], w, 1e-9), (g[:, 0], w)


def test_silent_stem_windows_are_nan_exactly_there():
    rng = np.random.default_rng(5)
    S, C, W, H, F = 2, 1, 100, 100, 8
    n = 6 * W + 37
    refs, ests = images(rng, S, n, C)
    refs[1, 2 * W:3 * W] = 0.0                          # a silent reference stem in window 2
    ests[0, 4 * W:5 * W] = 0.0                          # a silent estimate in window 4
    got = bss_eval_v4(refs, ests, W, H, True, F)
    assert got[0].shape == (S, 6)
    for k in range(6):
        nan = k in (2, 4)
        assert all(np.isnan(x[:, k]).all() == nan and np.isnan(x[:, k]).any() == nan for x in got[:4]), k
        assert (got[4][:, k] == -1).all() == nan, k
    # a NaN anywhere poisons every window; a recording shorter than the window or the filters has none
    bad = refs.copy()
    bad[0, 5] = np.nan
    assert np.isnan(bss_eval_v4(bad, ests, W, H, True, F)[0]).all()
    assert np.isnan(bss_eval_v4(refs, ests, W, H, True, F, length=W - 1)[0]).all()
    short = bss_eval_v4(refs, ests, W, H, True, F, length=2 * W + 5)
    assert np.isfinite(short[0][:, :2]).all() and np.isnan(short[0][:, 2:]).all() and (short[4][:, 2:] == -1).all()


def test_window_count():
    assert window_count(44100 * 3, 44100, 44100) == 3 and window_count(44100 * 3 - 1, 44100, 44100) == 2
    assert window_count(1000, 300, 200) == 4 and window_count(300, 300, 200) == 1


# ---------------------------------------------------------------------------------------------------------------------
# the C-ABI entries
# ---------------------------------------------------------------------------------------------------------------------
def test_symbols_bind_and_are_declared():
    lib = N.lib()
    text = HEADER.read_text()
    for name in ENTRIES:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\b" + name + r"\(", text), name
    assert lib.sdr_abi_version() == 2
    assert "bss_eval_v4" in P.__all__ and P.bss_eval_v4 is P.bss_eval.bss_eval_v4


@pytest.mark.parametrize("S,C", [(1, 1), (2, 1), (3, 1), (4, 1), (1, 2), (2, 2), (1, 3), (1, 4)])
@pytest.mark.parametrize("F", [1, 16, 512])
def test_scratch_grid(S, C, F):
    q = N.lib().sdr_bss_eval_v4_scratch_bytes
    R = S * C
    T = max((R - 1) * F + 1, 64)
    assert q(1, S, C, T, T, T, F) > 0 and q(4, S, C, 44100 * 10, 44100, 44100, F) > 0
    if R > 1:
        shortest = (R - 1) * F + 1                                   # too short for the joint system below this
        assert q(1, S, C, shortest, 1, 1, F) > 0 and q(1, S, C, shortest - 1, 1, 1, F) == 0
    assert q(1, S, C, T, T + 1, 1, F) == 0                           # T < W: no window
    # constant in T once one launch's chunks (512 per batch) no longer cover it
    for B in (1, 8):
        span = TRACK_CHUNK * max(1, TRACK_BLOCKS // B)
        sizes = [q(B, S, C, T, 44100, 44100, F) for T in (span + 44100 * 128, 3 * span + 44100 * 128, 1 << 36)]
        assert sizes[0] == sizes[1] == sizes[2] > 0, (B, sizes)
    for args in ((0, S, C, T, T, T, F), (1, S, C, 0, T, T, F), (1, S, C, T, 0, T, F), (1, S, C, T, T, 0, F),
                 (1, S, C, T, T, T, 0), (1, S, C, T, T, T, 513), (1, S, 0, T, T, T, F), (1, 0, C, T, T, T, F)):
        assert q(*args) == 0, args


@pytest.mark.parametrize("S,C", [(5, 1), (1, 5), (3, 2), (2, 3), (4, 2), (2, 4)])
def test_scratch_refuses_more_than_four_rows(S, C):
    assert N.lib().sdr_bss_eval_v4_scratch_bytes(1, S, C, 1 << 22, 44100, 44100, 16) == 0


X = 1 << 20                 # fake device addresses: every refused call returns before any CUDA call
M4 = X + 4
NAMES = "ref est lengths sdr isr sir sar perm B S C T W H F cp scratch stream".split()
BASE = dict(ref=X, est=X, lengths=None, sdr=X, isr=X, sir=X, sar=X, perm=None, B=2, S=2, C=2, T=441000, W=44100,
            H=44100, F=512, cp=0, scratch=X, stream=None)


@pytest.mark.parametrize("kw,want", [
    (dict(ref=None), BAD_ARGUMENT), (dict(est=None), BAD_ARGUMENT), (dict(sdr=None), BAD_ARGUMENT),
    (dict(isr=None), BAD_ARGUMENT), (dict(sir=None), BAD_ARGUMENT), (dict(sar=None), BAD_ARGUMENT),
    (dict(scratch=None), BAD_ARGUMENT), (dict(scratch=M4), BAD_ARGUMENT), (dict(lengths=M4), BAD_ARGUMENT),
    (dict(B=0), BAD_ARGUMENT), (dict(T=0), BAD_ARGUMENT), (dict(W=0), BAD_ARGUMENT), (dict(H=0), BAD_ARGUMENT),
    (dict(W=-1), BAD_ARGUMENT), (dict(H=-5), BAD_ARGUMENT),
    (dict(S=5, C=1), UNSUPPORTED), (dict(S=4, C=2), UNSUPPORTED), (dict(C=3), UNSUPPORTED), (dict(C=0), UNSUPPORTED),
    (dict(S=0), UNSUPPORTED), (dict(F=0), UNSUPPORTED), (dict(F=513), UNSUPPORTED), (dict(T=44099), UNSUPPORTED),
    (dict(T=3 * 512, W=1000), UNSUPPORTED), (dict(B=1 << 30), UNSUPPORTED),
    (dict(scratch=M4, C=3), BAD_ARGUMENT), (dict(isr=None, F=513), BAD_ARGUMENT), (dict(lengths=M4, T=0), BAD_ARGUMENT),
], ids=lambda v: str(v))
def test_entry_refusals(kw, want):
    a = dict(BASE, **kw)
    assert N.lib().sdr_bss_eval_v4(*[a[n] for n in NAMES]) == want


# ---------------------------------------------------------------------------------------------------------------------
# the Python entry
# ---------------------------------------------------------------------------------------------------------------------
def test_python_checks():
    x = torch.zeros(2, 1000, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.bss_eval_v4(x, x, 100, 100)
    with pytest.raises(RuntimeError, match="shape"):
        P.bss_eval_v4(x, torch.zeros(2, 1000, 3), 100, 100)
    with pytest.raises(RuntimeError, match="shape"):
        P.bss_eval_v4(torch.zeros(1, 1, 2, 1000, 2), torch.zeros(1, 1, 2, 1000, 2))
    for w, h in ((0, 10), (10, 0), (-1, 10)):
        with pytest.raises(RuntimeError, match="positive"):
            P.bss_eval_v4(x, x, w, h)


@pytest.mark.parametrize("shape,W,F,what", [((3, 2000, 2), 500, 16, "sources \\* channels <= 4"),
                                            ((2, 2, 2000, 3), 500, 16, "sources \\* channels <= 4"),
                                            ((2, 1000, 2), 500, 513, "filter lengths 1..512"),
                                            ((2, 1000, 2), 500, 512, "\\(sources \\* channels - 1\\)"),
                                            ((2, 1000, 1), 1001, 16, "at least one window")])
def test_python_refuses_before_allocating(monkeypatch, shape, W, F, what):
    """The limits are refused from the library's scratch query, before any tensor is allocated or copied."""
    monkeypatch.setattr(P.bss_eval, "_usable", lambda *a: None)        # CPU tensors stand in for CUDA ones

    def boom(*a, **k):
        raise AssertionError("allocated before the refusal")
    monkeypatch.setattr(torch, "empty", boom)
    x = torch.zeros(shape)
    with pytest.raises(N.NativeError, match=what):
        P.bss_eval_v4(x, x, window=W, hop=W, filter_length=F)


@pytest.mark.parametrize("shape,single", [((2, 1000), True), ((2, 1000, 2), True), ((3, 2, 1000, 2), False)])
def test_python_shapes(monkeypatch, shape, single):
    """[S, T] is C = 1, [S, T, C] one recording, [B, S, T, C] a batch; outputs [..., S, nwin] with museval's count."""
    monkeypatch.setattr(P.bss_eval, "_usable", lambda *a: None)
    seen = {}

    def fake_call(B, S, C, T, F, windows, dev):
        seen.update(B=B, S=S, C=C, T=T, windows=windows[:2])
        nwin = (T - windows[0]) // windows[1] + 1

        def enqueue(ref, est, mix, out, perm, cp, scratch, stream):
            assert ref.shape == (B, S, C, T) and ref.is_contiguous() and mix is None
            out.zero_()
            perm.zero_()
            return 0, "fake"
        return 8, (B, nwin, S), enqueue
    monkeypatch.setattr(P.bss_eval, "_v4_call", fake_call)
    monkeypatch.setattr(N, "stream", lambda dev: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    x = torch.zeros(shape)
    out = P.bss_eval_v4(x, x, window=300, hop=200)
    S = shape[-3] if len(shape) == 4 else shape[0]
    lead = () if single else (shape[0],)
    assert len(out) == 5 and all(o.shape == lead + (S, 4) for o in out) and out[4].dtype == torch.int64
    assert seen["C"] == (1 if len(shape) == 2 else shape[-1]) and seen["windows"] == (300, 200)


def test_defaults_are_museval():
    import inspect
    sig = inspect.signature(P.bss_eval_v4)
    assert list(sig.parameters) == ["reference_sources", "estimated_sources", "window", "hop", "compute_permutation",
                                    "filter_length", "lengths"]
    d = {k: v.default for k, v in sig.parameters.items()}
    assert d["window"] == 44100 and d["hop"] == 44100 and d["compute_permutation"] is False
    assert d["filter_length"] == 512 and d["lengths"] is None
