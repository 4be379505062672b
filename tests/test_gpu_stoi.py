"""STOI on the GPU (sdr_stoi) against the fp64 restatement in stoi_oracle.py, within 1e-9: sampling rates, the 30-frame
and frame-grid length edges, lengths up to a 10-minute item, source counts and batches, speech-like signals whose
silent-frame mask keeps and drops frames with a 1 dB margin, degenerate rows, per-item lengths, non-finite
containment, poisoned scratch, reproducibility across calls, graphs, streams and threads, input dtypes and strides."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
import stoi_oracle as O
from guards import POISON_HUGE, POISON_NAN, Guards, check_bands, poisoned

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-9


def clean(rng, n, fs, kind):
    """white, AR-coloured, or amplitude-modulated noise with silent gaps and stretches 39 and 41 dB below the loud
    parts (the mask keeps the first and drops the second, with a 1 dB margin)."""
    x = rng.standard_normal(n)
    if kind == "ar":
        x = lfilter([1.0], [1.0, -0.9], x)
    elif kind == "speechlike":
        t = np.arange(n) / fs
        x = lfilter([1.0], [1.0, -0.7], x) * (1.0 + 0.8 * np.sin(2 * np.pi * 3.0 * t))
        seg = max(n // 10, 1)
        x[seg:2 * seg] = 0.0                                              # silent gap
        x[3 * seg:4 * seg] *= 10 ** (-39 / 20)
        x[5 * seg:6 * seg] *= 10 ** (-41 / 20)
        x[7 * seg:7 * seg + seg // 3] = 0.0
    return x


def processed(rng, x, how):
    n = len(x)
    if how == "noisy":
        snr = rng.uniform(-10, 30)
        e = rng.standard_normal(n)
        return x + e * np.sqrt(np.sum(x ** 2) / max(np.sum(e ** 2), 1e-30) / 10 ** (snr / 10))
    if how == "filtered":
        return lfilter([0.6, 0.3, -0.2], [1.0, -0.3], x) + 0.05 * np.std(x) * rng.standard_normal(n)
    return x + 20 * np.std(x) * rng.standard_normal(n)                   # "clipped": the clip binds everywhere


def batch(rng, B, S, n, fs, kinds=("white", "ar", "speechlike"), hows=("noisy", "filtered", "clipped")):
    x = np.stack([[clean(rng, n, fs, kinds[(b * S + j) % len(kinds)]) for j in range(S)] for b in range(B)])
    y = np.stack([[processed(rng, x[b, j], hows[(b + j) % len(hows)]) for j in range(S)] for b in range(B)])
    mix = x.sum(1) + 0.1 * rng.standard_normal((B, n))
    return x.astype(np.float32), y.astype(np.float32), mix.astype(np.float32)


def gpu(x, y, fs, mix=None, lengths=None):
    with torch.no_grad():
        out = P.stoi(torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV), fs,
                     mixture=None if mix is None else torch.from_numpy(mix).to(DEV),
                     lengths=None if lengths is None else torch.tensor(lengths, device=DEV))
    return out.cpu().numpy() if mix is None else (out[0].cpu().numpy(), out[1].cpu().numpy())


def oracle(x, y, fs, mix=None, lengths=None):
    B, S, T = x.shape
    d = np.zeros((B, S))
    m = np.zeros((B, S))
    for b in range(B):
        n = T if lengths is None else lengths[b]
        for j in range(S):
            xr = x[b, j, :n].astype(np.float64)
            d[b, j] = O.stoi(xr, y[b, j, :n].astype(np.float64), fs)
            if mix is not None:
                m[b, j] = O.stoi(xr, mix[b, :n].astype(np.float64), fs)
    return d if mix is None else (d, m)


def close(got, want, label):
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (label, got, want)
    ok = ~np.isnan(want)
    assert np.all(np.abs(got - want)[ok] <= TOL), (label, np.max(np.abs(got - want)[ok]), got, want)


def check(x, y, fs, mix, label, lengths=None):
    g = gpu(x, y, fs, mix, lengths)
    w = oracle(x, y, fs, mix, lengths)
    if mix is None:
        close(g, w, label)
    else:
        close(g[0], w[0], label + " estimate")
        close(g[1], w[1], label + " mixture")
        close(gpu(x, y, fs, None, lengths), w[0], label + " without mixture")


@pytest.mark.parametrize("fs", [8000, 10000, 16000, 22050, 44100, 48000])
def test_sampling_rates(fs):
    rng = np.random.default_rng(fs)
    x, y, mix = batch(rng, 2, 2, 4 * fs, fs)
    check(x, y, fs, mix, f"fs {fs}")


def boundary_lengths():
    """(fs, n): 30 spectral frames +-1 for white noise (3277 samples at 8 kHz is the first real value), and resampled
    lengths where len - 256 is a multiple of 128 +-1 (the last frame dropped or not)."""
    out = [(8000, n) for n in (3276, 3277, 3278)]
    out += [(10000, 256 + 128 * 40 + d) for d in (-1, 0, 1)]
    for fs in (8000, 16000):
        for k in (40, 300):
            want = 256 + 128 * k
            n = next(n for n in range(1, 10 * want) if O.resampled_length(n, fs) >= want)
            out += [(fs, m) for m in (n - 1, n, n + 1)]
    return out


@pytest.mark.parametrize("fs,n", boundary_lengths())
def test_length_edges(fs, n):
    rng = np.random.default_rng(n)
    x, y, mix = batch(rng, 1, 2, n, fs, kinds=("white",), hows=("noisy",))
    check(x, y, fs, mix, f"fs {fs} n {n}")


@pytest.mark.parametrize("seconds", [4, 10])
def test_long_items(seconds):
    rng = np.random.default_rng(seconds)
    x, y, mix = batch(rng, 2, 2, seconds * 16000, 16000)
    check(x, y, 16000, mix, f"{seconds} s")


def test_ten_minute_item():
    rng = np.random.default_rng(600)
    x, y, mix = batch(rng, 1, 1, 600 * 16000, 16000, kinds=("speechlike",), hows=("noisy",))
    check(x, y, 16000, mix, "10 min")


@pytest.mark.parametrize("S", [1, 2, 3, 4, 16])
def test_source_counts(S):
    rng = np.random.default_rng(100 + S)
    x, y, mix = batch(rng, 2, S, 20000, 8000)
    check(x, y, 8000, mix, f"S {S}")


@pytest.mark.parametrize("B", [1, 3, 257])
def test_batches(B):
    rng = np.random.default_rng(200 + B)
    x, y, mix = batch(rng, B, 2, 6000, 8000)
    check(x, y, 8000, mix, f"B {B}")


def test_degenerate_rows():
    """Silent clean rows and silent estimates give exactly 0.0 and rows too short for 30 frames exactly 1e-5, as the
    oracle.  A constant row is within tolerance of nothing: its segment magnitudes are constant, so what remains after
    the mean is removed is rounding residue, which the normalisation scales up.  It must be finite, bounded and
    reproducible."""
    rng = np.random.default_rng(7)
    n, fs = 24000, 8000
    x, y, mix = batch(rng, 2, 4, n, fs)
    x[0, 0] = 0.0                                   # silent clean row
    y[0, 1] = 0.0                                   # silent estimate
    x[1, 0] = 0.0
    y[1, 0] = 0.0                                   # both silent
    x[1, 2] = 0.25                                  # constant clean row
    y[1, 3] = -1.0                                  # constant estimate
    d, m = gpu(x, y, fs, mix)
    assert d[0, 0] == 0.0 and d[0, 1] == 0.0 and d[1, 0] == 0.0 and m[0, 0] == 0.0 and m[1, 0] == 0.0
    w = oracle(x, y, fs, mix)
    for b, j in ((0, 2), (0, 3), (1, 1)):
        assert abs(d[b, j] - w[0][b, j]) <= TOL and abs(m[b, j] - w[1][b, j]) <= TOL, (b, j)
    assert np.all(np.isfinite(d[1, 2:])) and np.all(np.abs(d[1, 2:]) <= 1.0 + 1e-9)
    d2, m2 = gpu(x, y, fs, mix)
    assert np.array_equal(d, d2) and np.array_equal(m, m2)
    sx, sy, smix = batch(rng, 1, 2, 3000, fs)
    got = gpu(sx, sy, fs, smix)
    assert np.all(got[0] == 1e-5) and np.all(got[1] == 1e-5)
    tx, ty, _ = batch(rng, 1, 1, 150, fs)           # no frame at all after resampling
    assert np.all(gpu(tx, ty, fs) == 1e-5)


def test_lengths_equal_items_scored_alone():
    """Item b scored over lengths[b] equals the same item alone at that length, bit for bit; NaN in the padding
    changes nothing; a length outside [1, T] gives NaN for its item only."""
    rng = np.random.default_rng(8)
    fs, T = 16000, 40000
    lens = [40000, 31234, 9000, 5000]
    x, y, mix = batch(rng, 4, 2, T, fs)
    for b, n in enumerate(lens):
        x[b, :, n:] = 0.0
        y[b, :, n:] = 0.0
        mix[b, n:] = 0.0
    d, m = gpu(x, y, fs, mix, lens)
    for b, n in enumerate(lens):
        a = gpu(np.ascontiguousarray(x[b:b + 1, :, :n]), np.ascontiguousarray(y[b:b + 1, :, :n]), fs,
                np.ascontiguousarray(mix[b:b + 1, :n]))
        assert np.array_equal(a[0][0], d[b]) and np.array_equal(a[1][0], m[b]), b
    close(d, oracle(x, y, fs, None, lens), "lengths")
    xn, yn, mn = x.copy(), y.copy(), mix.copy()
    for b, n in enumerate(lens):
        xn[b, :, n:] = np.nan
        yn[b, :, n:] = np.inf
        mn[b, n:] = np.nan
    dn, mn_ = gpu(xn, yn, fs, mn, lens)
    assert np.array_equal(dn.view(np.int64), d.view(np.int64)) and np.array_equal(mn_.view(np.int64), m.view(np.int64))
    bad = [40000, 0, 40001, 5000]
    db, mb = gpu(x, y, fs, mix, bad)
    assert np.isnan(db[1:3]).all() and np.isnan(mb[1:3]).all()
    assert np.array_equal(db[[0, 3]], d[[0, 3]]) and np.array_equal(mb[[0, 3]], m[[0, 3]])


@pytest.mark.parametrize("where", ["estimate", "reference", "mixture"])
@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
def test_nonfinite_containment(where, value):
    rng = np.random.default_rng(9)
    fs = 8000
    x, y, mix = batch(rng, 3, 2, 12000, fs)
    d0, m0 = gpu(x, y, fs, mix)
    {"estimate": y, "reference": x, "mixture": mix[:, None]}[where][1, 1 if where != "mixture" else 0, 5000] = value
    d, m = gpu(x, y, fs, mix)
    nan_d = np.zeros_like(d0, bool)
    nan_m = np.zeros_like(m0, bool)
    if where == "estimate":
        nan_d[1, 1] = True
    elif where == "reference":
        nan_d[1, 1] = nan_m[1, 1] = True
    else:
        nan_m[1, :] = True
    assert np.array_equal(np.isnan(d), nan_d) and np.array_equal(np.isnan(m), nan_m), (where, d, m)
    assert np.array_equal(d[~nan_d], d0[~nan_d]) and np.array_equal(m[~nan_m], m0[~nan_m])


def abi_call(x, y, mix, lens, fs, pattern):
    """One sdr_stoi call with every buffer guarded and a scratch of exactly the queried size filled with `pattern`
    (0: clean).  -> (stoi, mix_stoi), after checking the bands and that no input changed."""
    B, S, T = x.shape
    lib = N.lib()
    scratch = poisoned(lib.sdr_stoi_scratch_bytes(B, S, T, fs), pattern)
    g = Guards()
    r, e, m, ln = g.input("reference", x), g.input("estimate", y), g.input("mixture", mix), g.input("lengths", lens)
    nan = torch.full((B, S), float("nan"), dtype=torch.float64, device=DEV)
    out, mout = g.output("stoi", nan), g.output("mix_stoi", nan)
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    rc = lib.sdr_stoi(p(r), p(e), p(m), p(ln), p(out), p(mout), B, S, T, fs, p(scratch),
                      C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    assert rc == 0, rc
    g.check()
    check_bands(scratch, "scratch")
    return out.clone(), mout.clone()


@pytest.mark.parametrize("fs", [8000, 44100])
def test_poisoned_scratch_and_guards(fs):
    rng = np.random.default_rng(10)
    T = 3 * fs
    x, y, mix = batch(rng, 3, 2, T, fs)
    t = lambda a: torch.from_numpy(a).to(DEV)   # noqa: E731
    lens = torch.tensor([T, T - 777, T // 2], dtype=torch.int64, device=DEV)
    clean_ = abi_call(t(x), t(y), t(mix), lens, fs, 0)
    assert not any(torch.isnan(o).any() for o in clean_)
    for pattern in (POISON_NAN, POISON_HUGE):
        got = abi_call(t(x), t(y), t(mix), lens, fs, pattern)
        for a, b in zip(got, clean_):
            assert torch.equal(a.view(torch.int64), b.view(torch.int64)), hex(pattern)


def test_reproducible_graph_side_stream_and_threads():
    rng = np.random.default_rng(11)
    fs = 16000
    x, y, mix = batch(rng, 4, 2, 3 * fs, fs)
    r, e, m = (torch.from_numpy(a).to(DEV) for a in (x, y, mix))
    lens = torch.tensor([3 * fs, 40000, 30000, 20000], device=DEV)
    with torch.no_grad():
        a = P.stoi(r, e, fs, mixture=m, lengths=lens)
        b = P.stoi(r, e, fs, mixture=m, lengths=lens)
        for u, v in zip(a, b):
            assert torch.equal(u, v)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            c = P.stoi(r, e, fs, mixture=m, lengths=lens)
        torch.cuda.current_stream().wait_stream(s)
        for u, v in zip(a, c):
            assert torch.equal(u, v)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            gr = P.stoi(r, e, fs, mixture=m, lengths=lens)
        g.replay()
        torch.cuda.synchronize()
    for u, v in zip(a, gr):
        assert torch.equal(u, v)
    results, errors = [None] * 4, []

    def worker(i):
        try:
            st = torch.cuda.Stream()
            with torch.no_grad(), torch.cuda.stream(st):
                out = P.stoi(r, e, fs, mixture=m, lengths=lens)
            st.synchronize()
            results[i] = out
        except Exception as ex:                 # noqa: BLE001
            errors.append(ex)
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for out in results:
        for u, v in zip(a, out):
            assert torch.equal(u, v)


def test_dtypes_strides_and_shapes():
    rng = np.random.default_rng(12)
    fs = 8000
    x, y, mix = batch(rng, 1, 3, 16000, fs)
    r, e = torch.from_numpy(x[0]).to(DEV), torch.from_numpy(y[0]).to(DEV)
    with torch.no_grad():
        for dt in (torch.float16, torch.bfloat16, torch.float64):
            rc, ec = r.to(dt), e.to(dt)
            assert torch.equal(P.stoi(rc, ec, fs), P.stoi(rc.float(), ec.float(), fs)), dt
        wide = torch.zeros(3, 2 * 16000, device=DEV)
        wide[:, ::2] = e
        assert torch.equal(P.stoi(r.t().contiguous().t(), wide[:, ::2], fs), P.stoi(r, e, fs))
        full = P.stoi(r, e, fs)
        assert full.shape == (3,) and full.dtype == torch.float64 and full.device == r.device
        one = P.stoi(r[1], e[1], fs)
        assert one.shape == () and torch.equal(one, full[1])
        d, mi = P.stoi(r, e, fs, mixture=torch.from_numpy(mix[0]).to(DEV))
        assert torch.equal(d, full) and mi.shape == (3,)
