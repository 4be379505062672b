"""BSS-eval of source images without a GPU: the fp64 numpy restatement of mir_eval's bss_eval_images
(bss_images_oracle.py) checked against itself (the sources' criteria at C = 1, invariance under an orthogonal channel
mix, a silent channel, the framewise windows); the bindings, scratch queries and refusals of the four C-ABI entries;
the Python entries' refusals, which come before any allocation, and their layout handling."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.bss_eval import _rows
from bss_images_oracle import _delays, _project, bss_eval_images, bss_eval_images_framewise, criteria
from bss_oracle import bss_eval

BAD_ARGUMENT, UNSUPPORTED = -2, -5
HEADER = Path(__file__).resolve().parents[1] / "include" / "sudormrf_b200.h"
ENTRIES = ("sdr_bss_eval_images_scratch_bytes", "sdr_bss_eval_images", "sdr_bss_eval_images_framewise_scratch_bytes",
           "sdr_bss_eval_images_framewise")


def close(a, b, tol):
    """Equal within tol dB, infinities equal to themselves."""
    a, b = np.asarray(a), np.asarray(b)
    with np.errstate(invalid="ignore"):
        return bool(np.all((a == b) | (np.abs(a - b) <= tol)))


def images(rng, S, T, C, noise=0.1):
    """References [S, T, C] and estimates mixed across sources and channels, noised and shuffled."""
    refs = rng.standard_normal((S, T, C))
    mixm = np.eye(S * C) + 0.3 * rng.standard_normal((S * C, S * C))
    flat = refs.transpose(0, 2, 1).reshape(S * C, T)
    ests = (mixm @ flat + noise * rng.standard_normal((S * C, T))).reshape(S, C, T).transpose(0, 2, 1)
    return refs, ests[rng.permutation(S)]


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against itself
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,T,F,perm", [(1, 200, 8, True), (2, 300, 16, True), (3, 200, 12, False),
                                        (4, 160, 10, True), (2, 33, 16, True)])
def test_mono_sir_sar_are_the_sources(S, T, F, perm):
    rng = np.random.default_rng(S * 100 + F)
    refs, ests = images(rng, S, T, 1)
    sdr, isr, sir, sar, p = bss_eval_images(refs, ests, perm, F)
    want = bss_eval(refs[..., 0], ests[..., 0], perm, F)
    assert np.array_equal(p, want[3])
    assert close(sir, want[1], 1e-9) and close(sar, want[2], 1e-9)
    assert np.all(np.isfinite(sdr)) and np.all(np.isfinite(isr))


@pytest.mark.parametrize("S,C,T,F", [(1, 2, 200, 8), (2, 2, 240, 8), (1, 3, 150, 6), (1, 4, 120, 5)])
def test_orthogonal_channel_mix_changes_nothing(S, C, T, F):
    rng = np.random.default_rng(7 * C + S)
    refs, ests = images(rng, S, T, C)
    q, _ = np.linalg.qr(rng.standard_normal((C, C)))
    a = bss_eval_images(refs, ests, True, F)
    b = bss_eval_images(refs @ q.T, ests @ q.T, True, F)
    assert np.array_equal(a[4], b[4])
    for x, y in zip(a[:4], b[:4]):
        assert close(x, y, 1e-8)


def test_silent_channel_is_the_projection_onto_the_others():
    rng = np.random.default_rng(3)
    S, C, T, F = 2, 2, 200, 8
    refs, ests = images(rng, S, T, C)
    refs[1, :, 0] = 0.0                                  # source 1's first channel is silent, the image is not
    crit = criteria(refs, ests, F)
    L = T + F - 1
    pad = lambda x: np.concatenate([x, np.zeros(F - 1)])
    own = [np.hstack([_delays(refs[0, :, c], F) for c in range(C)]), _delays(refs[1, :, 1], F)]
    both = np.hstack(own)
    for i in range(S):
        e = np.stack([pad(ests[i, :, c]) for c in range(C)], 1)
        pa = _project(both, e)
        for j in range(S):
            s = np.stack([pad(refs[j, :, c]) for c in range(C)], 1)
            pj = _project(own[j], e)
            sir = 10 * np.log10(np.sum(pj ** 2) / np.sum((pa - pj) ** 2))
            isr = 10 * np.log10(np.sum(s ** 2) / np.sum((pj - s) ** 2))
            sar = 10 * np.log10(np.sum(pa ** 2) / np.sum((e - pa) ** 2))
            assert abs(crit[2, i, j] - sir) < 1e-8 and abs(crit[1, i, j] - isr) < 1e-8
            assert abs(crit[3, i, j] - sar) < 1e-8 and e.shape[0] == L


def test_silent_or_nonfinite_image_is_nan():
    rng = np.random.default_rng(4)
    refs, ests = images(rng, 2, 100, 2)
    for r, e in ((np.where(np.arange(2)[:, None, None] == 1, 0.0, refs), ests),
                 (refs, np.where(np.arange(2)[:, None, None] == 0, 0.0, ests)),
                 (np.where(np.arange(100)[None, :, None] == 5, np.nan, refs), ests),
                 (refs, np.where(np.arange(100)[None, :, None] == 9, np.inf, ests))):
        out = bss_eval_images(r, e, True, 4)
        assert all(np.isnan(x).all() for x in out[:4]) and (out[4] == -1).all()


def test_framewise_windows_and_fallback():
    rng = np.random.default_rng(6)
    S, C, T, W, H, F = 1, 2, 400, 150, 100, 8
    refs, ests = images(rng, S, T, C)
    got = bss_eval_images_framewise(refs, ests, W, H, False, F)
    assert got[0].shape == (S, 3)
    for k in range(3):
        want = bss_eval_images(refs[:, k * H:k * H + W], ests[:, k * H:k * H + W], False, F)
        for x, y in zip(got, want):
            assert np.array_equal(x[:, k], y)
    fb = bss_eval_images_framewise(refs, ests, W, H, False, F, length=200)       # 200 < W + H: the whole item
    want = bss_eval_images(refs[:, :200], ests[:, :200], False, F)
    assert all(np.array_equal(x[:, 0], y) for x, y in zip(fb, want)) and np.isnan(fb[0][:, 1:]).all()
    assert (fb[4][:, 1:] == -1).all()
    assert np.isnan(bss_eval_images_framewise(refs, ests, W, H, False, F, length=F)[0]).all()  # < (S C - 1) F + 1


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


@pytest.mark.parametrize("S,C", [(1, 1), (2, 1), (3, 1), (4, 1), (1, 2), (2, 2), (1, 3), (1, 4)])
def test_scratch_limits(S, C):
    lib = N.lib()
    q, fq = lib.sdr_bss_eval_images_scratch_bytes, lib.sdr_bss_eval_images_framewise_scratch_bytes
    R = S * C
    T = (R - 1) * 512 + 1
    assert q(1, S, C, T, 512) > 0 and q(3, S, C, 48000, 16) > 0
    assert q(1, S, C, T, 513) == 0
    if R > 1:
        assert q(1, S, C, T - 1, 512) == 0 and fq(1, S, C, 10 * T, T - 1, 100, 512) == 0
    assert fq(1, S, C, 10 * T, T, 100, 512) > 0
    for args in ((0, S, C, T, 512), (1, S, C, 0, 512), (1, S, C, T, 0), (1, S, 0, T, 512), (1, 0, C, T, 512)):
        assert q(*args) == 0, args


@pytest.mark.parametrize("S,C", [(5, 1), (1, 5), (3, 2), (2, 3), (4, 2), (2, 4)])
def test_scratch_refuses_more_than_four_rows(S, C):
    lib = N.lib()
    assert lib.sdr_bss_eval_images_scratch_bytes(1, S, C, 1 << 20, 16) == 0
    assert lib.sdr_bss_eval_images_framewise_scratch_bytes(1, S, C, 1 << 20, 1 << 16, 1 << 15, 16) == 0


def test_framewise_scratch_is_bounded():
    lib = N.lib()
    fq = lib.sdr_bss_eval_images_framewise_scratch_bytes
    sizes = [fq(1, 2, 2, T, 240000, 120000, 512) for T in (240000, 8000 * 3600, 1 << 40)]
    assert sizes[0] > 0 and sizes[1] == sizes[2] <= 128 * sizes[0]
    # one window's scratch is the whole-item scratch of W samples
    assert fq(1, 2, 2, 8000, 8000, 4000, 512) == lib.sdr_bss_eval_images_scratch_bytes(1, 2, 2, 8000, 512)


X = 1 << 20                 # fake device addresses: every refused call returns before any CUDA call
M4 = X + 4
NAMES = "ref est sdr isr sir sar perm B S C T F cp scratch stream".split()
BASE = dict(ref=X, est=X, sdr=X, isr=X, sir=X, sar=X, perm=None, B=2, S=2, C=2, T=48000, F=512, cp=1, scratch=X,
            stream=None)
FW_NAMES = "ref est lengths sdr isr sir sar perm B S C T W H F cp scratch stream".split()
FW_BASE = dict(BASE, lengths=None, T=100000, W=8000, H=4000)


@pytest.mark.parametrize("kw,want", [
    (dict(ref=None), BAD_ARGUMENT), (dict(est=None), BAD_ARGUMENT), (dict(isr=None), BAD_ARGUMENT),
    (dict(sar=None), BAD_ARGUMENT), (dict(scratch=None), BAD_ARGUMENT), (dict(scratch=M4), BAD_ARGUMENT),
    (dict(B=0), BAD_ARGUMENT), (dict(T=0), BAD_ARGUMENT), (dict(S=5, C=1), UNSUPPORTED), (dict(C=3), UNSUPPORTED),
    (dict(C=0), UNSUPPORTED), (dict(S=0), UNSUPPORTED), (dict(F=0), UNSUPPORTED), (dict(F=513), UNSUPPORTED),
    (dict(T=3 * 512), UNSUPPORTED), (dict(B=1 << 30), UNSUPPORTED), (dict(scratch=M4, C=3), BAD_ARGUMENT),
    (dict(isr=None, F=513), BAD_ARGUMENT),
], ids=lambda v: str(v))
def test_entry_refusals(kw, want):
    a = dict(BASE, **kw)
    assert N.lib().sdr_bss_eval_images(*[a[n] for n in NAMES]) == want


@pytest.mark.parametrize("kw,want", [
    (dict(ref=None), BAD_ARGUMENT), (dict(isr=None), BAD_ARGUMENT), (dict(scratch=M4), BAD_ARGUMENT),
    (dict(lengths=M4), BAD_ARGUMENT), (dict(B=0), BAD_ARGUMENT), (dict(W=0), BAD_ARGUMENT),
    (dict(H=-1), BAD_ARGUMENT), (dict(C=3), UNSUPPORTED), (dict(F=513), UNSUPPORTED), (dict(W=3 * 512), UNSUPPORTED),
    (dict(W=200000, T=3 * 512), UNSUPPORTED), (dict(lengths=M4, C=3), BAD_ARGUMENT),
], ids=lambda v: str(v))
def test_framewise_entry_refusals(kw, want):
    a = dict(FW_BASE, **kw)
    assert N.lib().sdr_bss_eval_images_framewise(*[a[n] for n in FW_NAMES]) == want


# ---------------------------------------------------------------------------------------------------------------------
# the Python entries
# ---------------------------------------------------------------------------------------------------------------------
def test_python_checks():
    x = torch.zeros(2, 1000, 2)
    for f in (P.bss_eval_images, P.bss_eval_images_framewise):
        with pytest.raises(RuntimeError, match="CUDA"):
            f(x, x)
        with pytest.raises(RuntimeError, match="shape"):
            f(x, torch.zeros(2, 1000, 3))
        with pytest.raises(RuntimeError, match="shape"):
            f(torch.zeros(1, 1, 2, 1000, 2), torch.zeros(1, 1, 2, 1000, 2))
    with pytest.raises(RuntimeError, match="positive"):
        P.bss_eval_images_framewise(x, x, 0, 10)
    for name in ("bss_eval_images", "bss_eval_images_framewise"):
        assert name in P.__all__ and getattr(P, name) is getattr(P.bss_eval, name)


@pytest.mark.parametrize("shape,F,what", [((3, 2000, 2), 16, "sources \\* channels <= 4"),
                                          ((2, 2, 2000, 3), 16, "sources \\* channels <= 4"),
                                          ((2, 1000, 2), 513, "filter lengths 1..512"),
                                          ((2, 1000, 2), 512, "\\(sources \\* channels - 1\\) \\* filter_length")])
@pytest.mark.parametrize("framewise", [False, True])
def test_python_refuses_before_allocating(monkeypatch, shape, F, what, framewise):
    """The limits are refused from the library's scratch query, before any tensor is allocated or copied."""
    monkeypatch.setattr(P.bss_eval, "_usable", lambda *a: None)        # CPU tensors stand in for CUDA ones

    def boom(*a, **k):
        raise AssertionError("allocated before the refusal")
    monkeypatch.setattr(torch, "empty", boom)
    x = torch.zeros(shape)
    with pytest.raises(N.NativeError, match=what):
        if framewise:
            P.bss_eval_images_framewise(x, x, window=shape[-2], hop=shape[-2], filter_length=F)
        else:
            P.bss_eval_images(x, x, filter_length=F)


def test_rows_layout():
    """mir_eval's [B, S, T, C] becomes contiguous fp32 [B, S, C, T], copied once, and not at all when it already is."""
    dev = torch.device("cpu")
    x = torch.randn(2, 3, 50, 2, dtype=torch.float64)
    r = _rows(x, dev)
    assert r.shape == (2, 3, 2, 50) and r.dtype == torch.float32 and r.is_contiguous()
    assert torch.equal(r, x.transpose(-1, -2).float())
    model_out = torch.randn(2, 3 * 2, 50)                               # a stereo model's [B, S*C, T]
    view = model_out.view(2, 3, 2, 50).transpose(-1, -2)               # the documented [B, S, T, C] view
    r = _rows(view, dev)
    assert r.data_ptr() == model_out.data_ptr() and torch.equal(r, model_out.view(2, 3, 2, 50))
    for s in range(3):                                                 # source s, channel c is row s C + c
        for c in range(2):
            assert torch.equal(r[:, s, c], model_out[:, s * 2 + c])


def test_defaults_are_mir_eval_signature():
    import inspect
    sig = inspect.signature(P.bss_eval_images)
    assert list(sig.parameters) == ["reference_sources", "estimated_sources", "compute_permutation", "filter_length"]
    assert sig.parameters["compute_permutation"].default is True and sig.parameters["filter_length"].default == 512
    sig = inspect.signature(P.bss_eval_images_framewise)
    assert list(sig.parameters)[:5] == ["reference_sources", "estimated_sources", "window", "hop",
                                        "compute_permutation"]
    assert sig.parameters["window"].default == 30 * 44100 and sig.parameters["hop"].default == 15 * 44100
    assert sig.parameters["compute_permutation"].default is False
