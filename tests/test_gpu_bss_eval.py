"""BSS-eval on the GPU (sdr_bss_eval) against the fp64 restatement in bss_oracle.py: parity over source counts,
lengths, filter lengths and batches; invariances (zero padding, estimate order, reproducibility, CUDA graphs);
degenerate and rank-deficient reference sets; the mixture improvements; batches past 65535; input dtypes and strides."""
import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import sudo_rm_rf_b200 as P
from bss_oracle import _criteria, _project_fft, bss_eval

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def make_item(rng, S, T, F, coloured):
    """References (white or AR-coloured), estimates = mixing matrix x references + noise at -10..40 dB, then a short
    FIR filter shorter or longer than F; estimates in a random order."""
    refs = rng.standard_normal((S, T))
    if coloured:
        for i in range(S):
            refs[i] = lfilter([1.0], [1.0, -rng.uniform(0.5, 0.95)], refs[i])
    mixing = np.eye(S) + rng.uniform(0.05, 0.4) * rng.standard_normal((S, S))
    ests = mixing @ refs
    for i in range(S):
        snr = rng.uniform(-10, 40)
        noise = rng.standard_normal(T)
        ests[i] += noise * np.sqrt(np.sum(ests[i] ** 2) / np.sum(noise ** 2) / 10 ** (snr / 10))
        taps = int(rng.choice([max(1, F // 2), F + 7]))
        fir = rng.standard_normal(taps) * np.exp(-np.arange(taps) / 4.0)
        fir[0] = 1.0
        ests[i] = lfilter(fir, [1.0], ests[i])
    ests = ests[rng.permutation(S)]
    return refs.astype(np.float32), ests.astype(np.float32)


def run(refs, ests, perm=True, F=512, **kw):
    with torch.no_grad():
        out = P.bss_eval_sources(torch.from_numpy(np.ascontiguousarray(refs)).to(DEV),
                                 torch.from_numpy(np.ascontiguousarray(ests)).to(DEV), perm, F, **kw)
    return [o.cpu().numpy() if torch.is_tensor(o) else {k: v.cpu().numpy() for k, v in o.items()} for o in out]


def low_tolerance(amp_db):
    """The tolerance below -20 dB.  The solve's error in a projection is absolute and relative to the estimate:
    |P e - P~ e| ~ eps |e|.  A criterion with |P e|^2 in its numerator then moves by about 8.7 eps |e| / |P e| dB.
    For |P_j e| (SDR and SIR), |e|^2 / |P_j e|^2 = 1 + 10^(-SDR/10); for |P_all e| (SAR) the same with SAR.  So the
    tolerance is the [-20, 60] band's 1e-3 dB scaled by sqrt(1 + 10^(-a/10)) / sqrt(1 + 10^2), a the pair's SDR
    (for SDR and SIR) or SAR: 1e-3 dB at -20 dB, 1e-2 at -40, 0.1 at -60."""
    return 1e-3 * np.maximum(1.0, np.sqrt((1 + 10 ** (-np.asarray(amp_db, np.float64) / 10)) / 101))


def check_values(got, ref, label, amp_db=None):
    """|d| <= 1e-3 dB where the oracle lies in [-20, 60] dB; below -20 dB within low_tolerance(amp_db), amp_db the
    oracle's SDR of the same pairs for an SIR and the value itself otherwise; within 0.05 dB for finite values in (60,
    120]; both above 100 dB past 120 dB, where |e - P e|^2 is rounding noise in either computation; inf and NaN where
    the oracle has them."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (label, got, ref)
    mid = (ref >= -20) & (ref <= 60)
    assert np.all(np.abs(got - ref)[mid] <= 1e-3), (label, got[mid], ref[mid])
    low = np.isfinite(ref) & (ref < -20)
    tol = low_tolerance(ref if amp_db is None else np.broadcast_to(amp_db, ref.shape))
    assert np.all(np.abs(got - ref)[low] <= tol[low]), (label, got[low], ref[low], tol[low])
    high = np.isfinite(ref) & (ref > 60) & (ref <= 120)
    assert np.all(np.abs(got - ref)[high] <= 0.05), (label, got[high], ref[high])
    top = (ref > 120)
    assert np.all(got[top] > 100), (label, got[top], ref[top])


def check_item(got, refs, ests, perm=True, F=512, label=""):
    """The permutation where the oracle's best mean SIR beats the runner-up by more than 1e-3 dB and lies below 120 dB
    (past that both computations rank rounding noise, e.g. T + F - 1 <= S F, where every estimate is in the span);
    the values wherever the permutations agree."""
    sdr, sir, sar, p, gap = bss_eval(refs.astype(np.float64), ests.astype(np.float64), perm, F, margin=True)
    if gap > 1e-3 and np.mean(sir) <= 120:
        assert np.array_equal(got[3], p), (label, got[3], p)
    if np.array_equal(got[3], p):
        for g, r, name in zip(got[:3], (sdr, sir, sar), ("sdr", "sir", "sar")):
            check_values(g, r, f"{label} {name}", sdr if name == "sir" else None)


CASES = [(1, 1, 1, 3), (1, 1, 512, 2), (1, 511, 512, 2), (1, 512, 512, 2), (2, 100, 16, 8), (3, 2000, 512, 2),
         (2, 513, 512, 2), (4, 513, 16, 4),
         (4, 100, 1, 64), (2, 8000, 512, 6), (3, 8000, 16, 8), (4, 8000, 512, 2), (1, 32000, 512, 2),
         (2, 32000, 512, 3), (3, 32000, 16, 2), (2, 56000, 512, 2), (4, 56000, 16, 2)]


@pytest.mark.parametrize("S,T,F,B", CASES)
def test_parity(S, T, F, B):
    rng = np.random.default_rng(1000 * S + T + F)
    items = [make_item(rng, S, T, F, coloured=(b % 2 == 1)) for b in range(B)]
    refs = np.stack([i[0] for i in items])
    ests = np.stack([i[1] for i in items])
    got = run(refs, ests, True, F)
    for b in range(B):
        check_item([g[b] for g in got], refs[b], ests[b], True, F, f"S{S} T{T} F{F} item {b}")
    if B <= 4:                                          # the fixed assignment
        got = run(refs, ests, False, F)
        assert np.array_equal(got[3], np.tile(np.arange(S), (B, 1)))
        for b in range(B):
            check_item([g[b] for g in got], refs[b], ests[b], False, F, f"fixed S{S} T{T} F{F} item {b}")


def test_zero_padding_and_estimate_order():
    rng = np.random.default_rng(5)
    S, T, F = 3, 6000, 512
    refs, ests = make_item(rng, S, T, F, True)
    alone = run(refs, ests)
    pad = lambda x: np.concatenate([x, np.zeros((S, 2345), np.float32)], 1)      # noqa: E731
    refs2 = np.stack([pad(refs), rng.standard_normal((S, T + 2345)).astype(np.float32)])
    ests2 = np.stack([pad(ests), rng.standard_normal((S, T + 2345)).astype(np.float32)])
    padded = run(refs2, ests2)
    for a, p in zip(alone[:3], padded[:3]):
        assert np.all(np.abs(a - p[0]) <= 1e-6), (a, p[0])
    assert np.array_equal(alone[3], padded[3][0])
    order = rng.permutation(S)
    shuffled = run(refs, ests[order])
    for a, s in zip(alone[:3], shuffled[:3]):
        assert np.all(np.abs(a - s) <= 1e-9)
    assert np.array_equal(order[shuffled[3]], alone[3])


def test_bitwise_reproducible_and_graph_capture():
    rng = np.random.default_rng(6)
    items = [make_item(rng, 2, 8000, 512, b % 2 == 0) for b in range(4)]
    r = torch.from_numpy(np.stack([i[0] for i in items])).to(DEV)
    e = torch.from_numpy(np.stack([i[1] for i in items])).to(DEV)
    with torch.no_grad():
        a = P.bss_eval_sources(r, e)
        b = P.bss_eval_sources(r, e)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            P.bss_eval_sources(r, e)                    # warm-up: sets the kernels' shared-memory limits
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c = P.bss_eval_sources(r, e)
        g.replay()
        torch.cuda.synchronize()
    for x, y in zip(a, c):
        assert torch.equal(x, y)


def test_silent_rows_stay_in_their_item():
    rng = np.random.default_rng(7)
    items = [make_item(rng, 2, 3000, 256, False) for _ in range(3)]
    refs = np.stack([i[0] for i in items])
    ests = np.stack([i[1] for i in items])
    refs[0, 1] = 0
    ests[2, 0] = 0
    got = run(refs, ests, F=256)
    for b in (0, 2):
        assert all(np.isnan(g[b]).all() for g in got[:3]) and (got[3][b] == -1).all()
    check_item([g[1] for g in got], refs[1], ests[1], True, 256, "neighbour")


@pytest.mark.parametrize("kind", ["identical", "scaled", "delayed"])
def test_dependent_references(kind):
    """Two references that span the same delays (equal, a scaled copy) or a copy delayed by 37 < F samples: the joint
    span is that of the first reference with F (+ 37) taps, which the oracle solves without the rank deficiency."""
    rng = np.random.default_rng(8)
    T, F, d = 4000, 512, 37
    base = np.r_[lfilter([1.0], [1.0, -0.8], rng.standard_normal(T - d)), np.zeros(d)]
    dup = {"identical": base, "scaled": -2.0 * base, "delayed": np.r_[np.zeros(d), base[:-d]]}[kind]
    refs = np.stack([base, dup]).astype(np.float32)
    ests = (refs + 0.05 * rng.standard_normal((2, T))).astype(np.float32)
    sdr, sir, sar, perm = run(refs, ests, False, F)
    if kind != "delayed":
        assert np.all((sir >= 150) | np.isinf(sir)), sir
    r64 = refs.astype(np.float64)
    for j in range(2):
        e = ests[j].astype(np.float64)
        p_all = _project_fft(r64[:1], e, F + (d if kind == "delayed" else 0))[:T + F - 1]
        want = _criteria(np.r_[e, np.zeros(F - 1)], _project_fft(r64[j:j + 1], e, F), p_all)
        for g, w, name in zip((sdr, sir, sar), want, ("sdr", "sir", "sar")):
            check_values(g[j:j + 1], np.array([w]), f"{kind} {name} {j}")


def test_filtered_reference_and_short_signals():
    rng = np.random.default_rng(9)
    T, F = 8000, 512
    refs = rng.standard_normal((2, T)).astype(np.float32)
    refs[:, T - F:] = 0                                 # the filtered estimates end within T
    fir = rng.standard_normal(F) * np.exp(-np.arange(F) / 50.0)
    ests = np.stack([np.convolve(refs[1], fir)[:T], np.convolve(refs[0], fir[:40])[:T]]).astype(np.float32)
    sdr, sir, sar, perm = run(refs, ests, True, F)
    assert np.array_equal(perm, [1, 0]) and np.all(sdr >= 100), (sdr, perm)
    for T in (1, 7, 300):                               # T < F: one source; more would outnumber the dimensions
        refs, ests = make_item(rng, 1, T, F, False)
        got = run(refs, ests, True, F)
        assert all(np.all(~np.isnan(g)) for g in got[:3])
        check_item(got, refs, ests, True, F, f"T{T}")
    refs, ests = make_item(rng, 2, F, F, False)
    with pytest.raises(P._native.NativeError, match="samples"):
        run(refs, ests, True, F)


def test_mixture_improvements():
    rng = np.random.default_rng(10)
    S, T, F, B = 2, 8000, 512, 3
    items = [make_item(rng, S, T, F, True) for _ in range(B)]
    refs = np.stack([i[0] for i in items])
    ests = np.stack([i[1] for i in items])
    mix = refs.sum(1) + 0.01 * rng.standard_normal((B, T)).astype(np.float32)
    sdr, sir, sar, perm, extra = run(refs, ests, True, F, mixture=torch.from_numpy(mix).to(DEV).unsqueeze(1))
    plain = run(refs, ests, True, F)
    for a, b in zip((sdr, sir, sar, perm), plain):
        assert np.array_equal(a, b)
    for b in range(B):
        o = bss_eval(refs[b].astype(np.float64), ests[b].astype(np.float64), True, F)
        m = bss_eval(refs[b].astype(np.float64), np.stack([mix[b]] * S).astype(np.float64), False, F)
        for k, name in enumerate(("sdr", "sir", "sar")):
            check_values(extra[name][b], m[k], f"mixture {name}")
            d = o[k] - m[k]
            ok = np.isfinite(d)
            assert np.all(np.abs(extra[name + "i"][b] - d)[ok] <= 2e-3), (name, extra[name + "i"][b], d)


def test_batch_past_grid_limit():
    rng = np.random.default_rng(11)
    B, S, T, F = 65537, 2, 6, 4
    refs = torch.from_numpy(rng.standard_normal((B, S, T)).astype(np.float32)).to(DEV)
    ests = torch.from_numpy(rng.standard_normal((B, S, T)).astype(np.float32)).to(DEV)
    with torch.no_grad():
        full = P.bss_eval_sources(refs, ests, True, F)
        h = B // 2
        lo = P.bss_eval_sources(refs[:h], ests[:h], True, F)
        hi = P.bss_eval_sources(refs[h:], ests[h:], True, F)
    for f, a, b in zip(full, lo, hi):
        assert torch.equal(f, torch.cat([a, b]))


def test_dtypes_and_strides():
    rng = np.random.default_rng(12)
    refs, ests = make_item(rng, 3, 5000, 128, True)
    r = torch.from_numpy(refs).to(DEV)
    e = torch.from_numpy(ests).to(DEV)
    with torch.no_grad():
        for dt in (torch.float16, torch.bfloat16, torch.float64):
            rc, ec = r.to(dt), e.to(dt)
            a = P.bss_eval_sources(rc, ec, True, 128)
            b = P.bss_eval_sources(rc.float(), ec.float(), True, 128)
            for x, y in zip(a, b):
                assert torch.equal(x, y), dt
        wide = torch.zeros(3, 2 * 5000, device=DEV)
        wide[:, ::2] = e
        a = P.bss_eval_sources(r.t().contiguous().t(), wide[:, ::2], True, 128)
        b = P.bss_eval_sources(r, e, True, 128)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
