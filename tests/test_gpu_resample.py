"""Polyphase resampling on the GPU (DESIGN.md section 7g) against scipy.signal.resample_poly on the fp64 input.

The bar per sample is |got - ref| <= 2^-23 |ref| + 1e-9 max|x|: one fp32 rounding of an fp64 sum, plus the fp64
design of the filter.  Cases: every ordered pair of twelve standard rates, the length edges of the filter support,
batch shapes up to 4096 rows held bitwise to each row alone, strides and dtypes, the non-finite rule, past 2^31 output
elements, poisoned and guarded scratch, CUDA graphs, streams and threads, STOI unchanged, and the model methods'
``sample_rate`` / ``model_rate`` against the composition of the public pieces and the fp64 chain."""
import ctypes as C
import itertools
import math
import threading

import numpy as np
import pytest
import scipy.signal as ss
import torch

import sudo_rm_rf_b200 as P
from guards import POISON_HUGE, POISON_NAN, check_bands, guarded_copy, poisoned, poisoned_like
from oracle import sudormrf_oracle as O
from sudo_rm_rf_b200 import _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000)
SPREAD = 1e-5      # run-to-run spread of the non-causal forwards, whose fp64 statistics are summed by atomics
worst = {}         # largest error seen over the bar's scale, per test


@pytest.fixture(autouse=True, scope="module")
def release_device_memory():
    """Leaves the device as the module found it: the cached models and the allocator's cached blocks (the 2^31 case
    alone caches about 13 GB) are released when the module ends."""
    yield
    _cache.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def ratio(up, down):
    g = math.gcd(up, down)
    return up // g, down // g


def signal(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape)


def gpu(x64):
    return torch.from_numpy(np.ascontiguousarray(x64)).float().to(DEV)


def check(got, x32, up, down, what):
    """got (device) against scipy on the fp64 values of x32 (device fp32); returns the largest |err| / bar."""
    x = x32.double().cpu().numpy()
    ref = ss.resample_poly(x, up, down, axis=-1)
    got = got.double().cpu().numpy()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bar = 2.0 ** -23 * np.abs(ref) + 1e-9 * max(np.abs(x).max(), 1e-300)
    err = np.abs(got - ref)
    r = float((err / bar).max())
    worst[what] = max(worst.get(what, 0.0), r)
    assert r <= 1.0, (what, up, down, r, float(err.max()))
    return r


def bits(t):
    return t.contiguous().view(torch.int32)


def direct(x, up, down, idx):
    """Outputs idx of resample_poly(x) by its definition: sum_t h[i q + L - t p] x[t] over the taps in [0, 2L], with
    scipy's filter; x fp64 numpy [T]."""
    p, q = ratio(up, down)
    L = 10 * max(p, q)
    h = ss.firwin(2 * L + 1, 1.0 / max(p, q), window=("kaiser", 5.0)) * p
    out = []
    for i in idx:
        c = i * q + L
        t = np.arange(max(0, -(-(c - 2 * L) // p)), min(c // p, len(x) - 1) + 1)
        out.append(np.dot(h[c - t * p], x[t]))
    return np.array(out)


def test_direct_definition_is_scipy():
    x = signal(5000, 1)
    for up, down in ((1, 6), (6, 1), (80, 441), (147, 160)):
        ref = ss.resample_poly(x, up, down)
        idx = [0, 1, len(ref) // 2, len(ref) - 1]
        assert np.abs(direct(x, up, down, idx) - ref[idx]).max() <= 1e-12 * np.abs(x).max()


@pytest.mark.parametrize("a", RATES)
def test_every_rate_pair(a):
    for b in RATES:
        if a == b:
            continue
        x = gpu(signal((2, a // 4 + 17), a + b))            # a quarter of a second and a bit
        check(P.resample_poly(x, b, a), x, b, a, "rate pairs")
    print(f"\nrate pairs from {a}: largest error / bar {worst['rate pairs']:.3f}")


@pytest.mark.parametrize("up,down", [(1, 6), (6, 1), (80, 441), (441, 80), (160, 441), (147, 2560), (2560, 147),
                                     (1, 2), (3, 2), (1, 4096)])
def test_length_edges(up, down):
    p, q = ratio(up, down)
    L = 10 * max(p, q)
    lengths = {1, 2, max(q - 1, 1), q, q + 1, L - 1, L, L + 1, 2 * L - 1, 2 * L + 1, 3 * 44100 * q // max(p, q) + 7}
    for T in sorted(lengths):
        x = gpu(signal((3, T), T))
        got = P.resample_poly(x, up, down)
        assert got.shape == (3, -(-T * p // q))
        check(got, x, up, down, "length edges")
    print(f"\nlength edges {up}/{down}: largest error / bar {worst['length edges']:.3f}")


def test_copy_when_the_ratio_is_one():
    x = gpu(signal((3, 1001), 3))
    for up in (1, 7):
        got = P.resample_poly(x, up, up)
        assert torch.equal(bits(got), bits(x)) and got.data_ptr() != x.data_ptr()


@pytest.mark.parametrize("up,down", [(80, 441), (6, 1), (147, 2560)])
def test_shapes_rows_are_independent(up, down):
    gen = signal((4096, 3000), 7)
    x = gpu(gen)
    whole = P.resample_poly(x, up, down)
    parts = torch.cat([P.resample_poly(x[i:i + 1000], up, down) for i in range(0, 4096, 1000)])
    assert torch.equal(bits(whole), bits(parts))
    for r in (0, 1, 2047, 4095):
        assert torch.equal(bits(whole[r]), bits(P.resample_poly(x[r], up, down))), r
    three = P.resample_poly(x.reshape(64, 64, 3000), up, down)
    assert three.shape == (64, 64, whole.shape[-1]) and torch.equal(bits(three.reshape(4096, -1)), bits(whole))
    check(whole[:8], x[:8], up, down, "shapes")


def test_strides_and_dtypes():
    x = gpu(signal((6, 4000), 9))
    want = P.resample_poly(x[::2, ::3].contiguous(), 80, 441)
    assert torch.equal(bits(P.resample_poly(x[::2, ::3], 80, 441)), bits(want))
    xt = x.t().contiguous().t()                                   # column-major view of the same values
    assert torch.equal(bits(P.resample_poly(xt, 6, 1)), bits(P.resample_poly(x, 6, 1)))
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        xd = x.to(dt)
        got = P.resample_poly(xd, 80, 441)
        assert got.dtype == torch.float32
        assert torch.equal(bits(got), bits(P.resample_poly(xd.float(), 80, 441))), dt
    x64 = torch.from_numpy(signal((2, 3000), 10)).to(DEV)
    check(P.resample_poly(x64, 441, 80), x64.float(), 441, 80, "dtypes")


@pytest.mark.parametrize("up,down", [(1, 6), (6, 1), (80, 441), (441, 80)])
def test_nonfinite_reaches_exactly_its_support(up, down):
    p, q = ratio(up, down)
    L = 10 * max(p, q)
    T = 4 * L + 3 * q + 11
    clean = signal((1, T), 11)
    n = -(-T * p // q)
    base = P.resample_poly(gpu(clean), up, down)
    for t, v in itertools.product((0, 1, T // 2, T - 1), (np.nan, np.inf, -np.inf)):
        x = clean.copy()
        x[0, t] = v
        got = P.resample_poly(gpu(x), up, down)[0].cpu().numpy()
        i = np.arange(n)
        c = i * q + L
        inside = (c - t * p >= 0) & (c - t * p <= 2 * L)
        assert (~np.isfinite(got[inside])).all(), (t, v)
        assert np.array_equal(got[~inside], base[0].cpu().numpy()[~inside]), (t, v)


def test_past_2_31_output_elements():
    rows, T = 3, 120_000_000                   # 8 -> 48 kHz: 3 x 720 M outputs
    g = torch.Generator(device=DEV).manual_seed(12)
    x = torch.randn(rows, T, device=DEV, generator=g)
    torch.cuda.reset_peak_memory_stats()
    out = P.resample_poly(x, 6, 1)
    torch.cuda.synchronize()
    print(f"\npast 2^31: {out.numel()} outputs, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert out.numel() > 2 ** 31
    alone = P.resample_poly(x[-1:].clone(), 6, 1)
    assert torch.equal(bits(out[-1]), bits(alone[0]))
    last = x[-1].double().cpu().numpy()
    n = out.shape[-1]
    idx = list(range(n - 300, n)) + list(range(n // 2, n // 2 + 50))
    ref = direct(last, 6, 1, idx)
    got = out[-1, idx].double().cpu().numpy()
    bar = 2.0 ** -23 * np.abs(ref) + 1e-9 * np.abs(last).max()
    assert (np.abs(got - ref) <= bar).all()
    del out, alone, x


def raw(x, out, up, down, scratch):
    """The C-ABI entry on caller-made buffers, on the current stream."""
    rows, T = x.shape
    return N.lib().sdr_resample_poly(x.data_ptr(), out.data_ptr(), rows, T, up, down, scratch.data_ptr(),
                                     scratch.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream))


@pytest.mark.parametrize("up,down", [(80, 441), (441, 80), (6, 1), (147, 2560)])
def test_poisoned_and_guarded_buffers(up, down):
    x = gpu(signal((5, 7001), 13))
    want = P.resample_poly(x, up, down)
    nbytes = N.lib().sdr_resample_poly_scratch_bytes(up, down)
    for pattern in (0, POISON_NAN, POISON_HUGE):
        xs = guarded_copy(x)
        before = xs.clone()
        out = poisoned_like(want, pattern)
        scratch = poisoned(nbytes, pattern, align=8)
        assert raw(xs, out, up, down, scratch) == 0
        torch.cuda.synchronize()
        for t, what in ((xs, "x"), (out, "out"), (scratch, "scratch")):
            check_bands(t, what)
        assert torch.equal(xs, before)
        assert torch.equal(bits(out), bits(want)), pattern


def test_graph_capture_and_replay():
    x = gpu(signal((4, 20000), 14))
    want = P.resample_poly(x, 160, 441)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        P.resample_poly(x, 160, 441)                     # warm the allocator on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = P.resample_poly(x, 160, 441)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(out), bits(want))
    x.copy_(gpu(signal((4, 20000), 15)))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(out), bits(P.resample_poly(x, 160, 441)))


def test_side_stream_and_threads():
    xs = [gpu(signal((8, 30000), 16 + i)) for i in range(2)]
    want = [P.resample_poly(x, 80, 441) for x in xs]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = P.resample_poly(xs[0], 80, 441)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(bits(got), bits(want[0]))
    results, errs = {}, []

    def worker(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(5):
                    r = P.resample_poly(xs[i], 80, 441)
                st.synchronize()
            results[i] = r
        except Exception as e:          # noqa: BLE001  (reported below)
            errs.append(e)
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(120)
    assert not errs, errs
    for i in range(2):
        assert torch.equal(bits(results[i]), bits(want[i])), i


# STOI of the commit before its resampling filter and support bounds moved into resample.cuh, on an H100, in hex
STOI_BEFORE = {
    44100: (["0x1.98e4e8e0dc659p-1", "0x1.8fc02974f56bdp-1", "0x1.91e44ee171760p-1", "0x1.942b7beacb681p-1"],
            ["0x1.ea25758887603p-2", "0x1.e7e8a5bffa4f4p-2", "0x1.0181bccb61d75p-1", "0x1.e459b7ffd8ebap-2"]),
    16000: (["0x1.8fa7a5060dbd0p-1", "0x1.9266e494230edp-1", "0x1.96118cd52c764p-1", "0x1.98ce3a8ca73d0p-1"],
            ["0x1.0e1b1139ffeecp-1", "0x1.f4c158dec5b7bp-2", "0x1.fe2cf427d0c70p-2", "0x1.00a42184411ffp-1"]),
    8000: (["0x1.937f2035afc56p-1", "0x1.95e3cd01cc635p-1", "0x1.9124761d1a57ap-1", "0x1.8eaae94d90717p-1"],
           ["0x1.f199cd3ae92e2p-2", "0x1.01904b5cb411ep-1", "0x1.e460e0b9db174p-2", "0x1.0042b6c466389p-1"]),
}


@pytest.mark.parametrize("fs", list(STOI_BEFORE))
def test_stoi_is_unchanged(fs):
    rng = np.random.default_rng(fs)
    T = 3 * fs + 7
    x = rng.standard_normal((2, 2, T))
    x[:, :, fs // 2:fs] *= 1e-3
    y = x + 0.5 * rng.standard_normal((2, 2, T))
    m = x.sum(1) + 0.1 * rng.standard_normal((2, T))
    s, ms = P.stoi(gpu(x), gpu(y), fs, mixture=gpu(m))
    assert [float(v).hex() for v in s.flatten().tolist()] == STOI_BEFORE[fs][0]
    assert [float(v).hex() for v in ms.flatten().tolist()] == STOI_BEFORE[fs][1]


# ---------------------------------------------------------------------------------------------------------------------
# the models at another rate
# ---------------------------------------------------------------------------------------------------------------------
MODELS = {
    "improved": (P.SuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                  enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    "groupcomm": (P.GroupCommSudoRmRf, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                            enc_kernel_size=21, enc_num_basis=64, num_sources=2, group_size=4)),
    "causal": (P.CausalSuDORMRF, dict(in_audio_channels=1, out_channels=64, in_channels=128, num_blocks=2,
                                      upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    "original": (P.OriginalSuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                          enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
}
PAIRS = ((44100, 8000), (48000, 16000), (16000, 8000), (8000, 16000))
_cache = {}


def model(name):
    if name not in _cache:
        cls, kw = MODELS[name]
        sd = O.make_state_dict(O.Config(variant=name, **kw), seed=21)
        m = cls(**kw)
        m.load_state_dict(sd)
        _cache[name] = (m.to(DEV).eval(), O.Config(variant=name, **kw), sd)
    return _cache[name]


def mixture(B, T, fs, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64) / fs
    tone = torch.sin(2 * np.pi * 220.0 * t) * torch.sin(2 * np.pi * 0.3 * t)
    return (0.3 * torch.randn(B, 1, T, generator=g, dtype=torch.float64) + tone + 0.1).float().to(DEV)


def same(got, want, exact):
    assert got.shape == want.shape
    if exact:
        assert torch.equal(bits(got), bits(want))
    else:
        assert float((got - want).abs().max() / want.abs().max()) <= SPREAD


def cases():
    for name, (sr, mr), normalize, mc in itertools.product(MODELS, PAIRS, (True, False), (True, False)):
        yield pytest.param(name, sr, mr, normalize, mc, id=f"{name}-{sr}-{mr}-norm{int(normalize)}-mc{int(mc)}")


@pytest.mark.parametrize("name,sr,mr,normalize,mc", list(cases()))
def test_separate_at_another_rate(name, sr, mr, normalize, mc):
    m, cfg, sd = model(name)
    exact = name == "causal"
    T = sr // 2 + 123
    x = mixture(2, T, sr, sr + mr)
    with torch.no_grad():
        got = m.separate(x, mixture_consistency=mc, normalize=normalize, sample_rate=sr, model_rate=mr)
        down = P.resample_poly(x, mr, sr)
        est = m.separate(down, mixture_consistency=mc, normalize=normalize)
        want = P.resample_poly(est, sr, mr)[..., :T]
        same(got, want, exact)
        assert got.shape == (2, m.num_sources, T)
        # the fp64 chain: scipy around the oracle
        d64 = torch.from_numpy(ss.resample_poly(x.double().cpu().numpy(), mr, sr, axis=-1))
        if normalize:
            e64 = O.separate(cfg, sd, d64[:, 0], apply_mixture_consistency=mc, dtype=torch.float64)
        else:
            e64 = O.forward(cfg, sd, d64, dtype=torch.float64)
            if mc:
                e64 = O.mixture_consistency(e64, d64)
        r64 = torch.from_numpy(ss.resample_poly(e64.numpy(), sr, mr, axis=-1))[..., :T]
        e = O.parity_errors(got, r64)
        assert max(e) < 1e-3, e
        # equal rates: the existing call
        plain = m.separate(x, mixture_consistency=mc, normalize=normalize)
        same(m.separate(x, mixture_consistency=mc, normalize=normalize, sample_rate=sr, model_rate=sr), plain, exact)


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("normalize", [True, False])
def test_separate_long_at_another_rate(name, normalize):
    m, _, _ = model(name)
    exact = name == "causal"
    sr, mr, W, H = 44100, 8000, 4000, 2500
    T = 5 * sr + 17
    x = mixture(2, T, sr, 31)
    with torch.no_grad():
        got = m.separate_long(x, W, H, normalize=normalize, max_windows=4, sample_rate=sr, model_rate=mr)
        est = m.separate_long(P.resample_poly(x, mr, sr), W, H, normalize=normalize, max_windows=4)
        want = P.resample_poly(est, sr, mr)[..., :T]
        same(got, want, exact)
        plain = m.separate_long(x, W, H, normalize=normalize, max_windows=4)
        same(m.separate_long(x, W, H, normalize=normalize, max_windows=4, sample_rate=sr, model_rate=sr), plain,
             exact)


def test_ten_minutes_at_44k1_through_u16_at_8k():
    kw = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
              enc_num_basis=512, num_sources=2)
    sd = O.make_state_dict(O.Config(variant="improved", **kw), seed=3)
    m = P.SuDORMRF(**kw)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    sr, mr = 44100, 8000
    T = 600 * sr
    x = mixture(1, T, sr, 41)
    with torch.no_grad():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        got = m.separate_long(x, 4 * mr, 2 * mr, sample_rate=sr, model_rate=mr)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        est = m.separate_long(P.resample_poly(x, mr, sr), 4 * mr, 2 * mr)
        want = P.resample_poly(est, sr, mr)[..., :T]
    print(f"\n10 min at 44.1 kHz through U16/512 at 8 kHz: peak {peak / 2**30:.2f} GiB")
    assert got.shape == (1, 2, T) and torch.isfinite(got).all()
    same(got, want, False)
