"""Streaming at any sample rate on the GPU (DESIGN.md section 7h).

``ResampleStream`` against ``resample_poly`` on the concatenation, bitwise: every ordered pair of twelve standard rates,
chunk sizes, rows, delays, leads, slot counts up to 65535 and past 2^31 output elements; resets, flush, graph replay,
dtypes and strides, non-finite inputs, poisoned and guarded buffers, CUDA streams and host threads.  The model streams
at another rate against ``separate`` / ``separate_long`` with ``sample_rate`` and ``model_rate``: bitwise for the
causal model, within the windowed stream's rule for the others, and ten minutes at 44.1 kHz with constant memory."""
import itertools
import math
import threading

import ctypes as C
import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
import windowed_oracle as WO
from guards import POISON_HUGE, POISON_NAN, check_bands, guarded_copy, poisoned, poisoned_like
from oracle import sudormrf_oracle as O
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.resample_stream import ResampleStream, ResampledStream, min_delay
from sudo_rm_rf_b200.streaming import CausalStream
from sudo_rm_rf_b200.window_stream import WindowedStream

pytestmark = pytest.mark.gpu
DEV = "cuda"
RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000)
SPREAD = 1e-5      # run-to-run spread of the non-causal forwards, whose fp64 statistics are summed by atomics
MARGIN = 1e-6


@pytest.fixture(autouse=True, scope="module")
def release_device_memory():
    """The cached models and the allocator's cached blocks (the 2^31 case alone caches about 12 GB) are released
    when the module ends."""
    yield
    _cache.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def ratio(up, down):
    g = math.gcd(up, down)
    return up // g, down // g


def bits(t):
    return t.contiguous().view(torch.int32)


def signal(shape, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal(shape)).float().to(DEV)


def expected(x, up, down, delay, lead, start, n):
    """Samples [start - delay, start - delay + n) of resample_poly(lead zeros + x), zeros below 0."""
    B, R, _ = x.shape
    s = torch.cat([torch.zeros(B, R, lead, device=DEV), x], dim=-1)
    r = P.resample_poly(s, up, down)
    a = start - delay
    out = torch.zeros(B, R, n, device=DEV)
    lo, hi = max(a, 0), min(a + n, r.shape[-1])
    if hi > lo:
        out[..., lo - a:hi - a] = r[..., lo:hi]
    return out


def run(st, x, tail=None):
    """(cat of the steps over x, flush with tail)."""
    C_ = st.chunk_samples
    steps = [st.step(x[..., j:j + C_]) for j in range(0, x.shape[-1], C_)]
    return torch.cat(steps, dim=-1), st.flush(tail)


def check_stream(up, down, B, rows, C_, steps, delay=None, lead=0, tail=5, seed=0):
    p, q = ratio(up, down)
    st = ResampleStream(B, rows, C_, up, down, delay=delay, lead=lead)
    x = signal((B, rows, steps * C_), seed)
    t = signal((B, rows, tail), seed + 1)
    got, fl = run(st, x, t)
    P_ = C_ // q * p
    assert got.shape == (B, rows, steps * P_)
    want = expected(x, up, down, st.delay, lead, 0, steps * P_)
    assert torch.equal(bits(got), bits(want)), (up, down, C_, rows, delay, lead)
    full = torch.cat([x, t], dim=-1)
    n_end = -(-(lead + full.shape[-1]) * p // q)
    want_f = expected(full, up, down, st.delay, lead, steps * P_, n_end - (steps * P_ - st.delay))
    assert fl.shape == want_f.shape == (B, rows, st.flush_samples(tail))
    assert torch.equal(bits(fl), bits(want_f)), (up, down, "flush")
    return got


# ---------------------------------------------------------------------------------------------------------------------
# 1. the resampler against resample_poly
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("up,down", list(itertools.permutations(RATES, 2)))
def test_every_rate_pair_is_resample_poly_bitwise(up, down):
    p, q = ratio(up, down)
    least = min_delay(up, down)
    # chunks of q and 3q, rows 1 and 2, the smallest delay and one above it, a lead
    a = check_stream(up, down, 3, 1, q, 7, seed=up + down)
    check_stream(up, down, 2, 2, 3 * q, 3, delay=least + 7, seed=up)
    check_stream(up, down, 2, 1, q, 5, lead=3, seed=down)
    check_stream(up, down, 2, 1, 3 * q, 3, lead=q + 1, delay=min_delay(up, down, q + 1) + 2, seed=7)
    # two chunk sizes give the same bits
    st = ResampleStream(3, 1, 7 * q, up, down)
    x = signal((3, 1, 7 * q), up + down)
    assert torch.equal(bits(st.step(x)), bits(a))


@pytest.mark.parametrize("B", [1, 3, 300, 65535])
def test_slot_counts(B):
    up, down = 8000, 44100
    p, q = ratio(up, down)
    C_ = q
    st = ResampleStream(B, 1, C_, up, down)
    x = signal((B, 1, 4 * C_), B)
    got, fl = run(st, x)
    want = expected(x, up, down, st.delay, 0, 0, 4 * p)
    assert torch.equal(bits(got), bits(want))
    assert torch.equal(bits(fl), bits(expected(x, up, down, st.delay, 0, 4 * p, st.delay)))


# ---------------------------------------------------------------------------------------------------------------------
# 2. lifecycle
# ---------------------------------------------------------------------------------------------------------------------
def test_reset_starts_a_slot_over_and_leaves_the_others():
    up, down, B, C_ = 8000, 44100, 4, 441
    x = signal((B, 2, 12 * C_), 5)
    ref = ResampleStream(B, 2, C_, up, down)
    whole = torch.cat([ref.step(x[..., j * C_:(j + 1) * C_]) for j in range(12)], dim=-1)
    st = ResampleStream(B, 2, C_, up, down)
    a = [st.step(x[..., j * C_:(j + 1) * C_]) for j in range(5)]
    st.reset([2])
    b = [st.step(x[..., j * C_:(j + 1) * C_]) for j in range(5, 12)]
    got = torch.cat(a + b, dim=-1)
    keep = [0, 1, 3]
    assert torch.equal(bits(got[keep]), bits(whole[keep]))
    fresh = ResampleStream(1, 2, C_, up, down)
    want = torch.cat([fresh.step(x[2:3, :, j * C_:(j + 1) * C_]) for j in range(5, 12)], dim=-1)
    assert torch.equal(bits(torch.cat(b, dim=-1)[2:3]), bits(want))


def test_flush_keeps_the_state():
    up, down, C_ = 8000, 48000, 6
    x = signal((2, 1, 10 * C_), 6)
    a = ResampleStream(2, 1, C_, up, down)
    b = ResampleStream(2, 1, C_, up, down)
    for j in range(10):
        ch = x[..., j * C_:(j + 1) * C_]
        b.flush(signal((2, 1, 3), j))
        b.flush()
        assert torch.equal(bits(a.step(ch)), bits(b.step(ch))), j
    assert torch.equal(bits(a.flush()), bits(b.flush()))


def test_captured_step_with_resets_is_the_eager_step():
    up, down, B, C_ = 16000, 44100, 3, 441
    steps = 21
    x = signal((B, 1, steps * C_), 8)
    eager_st = ResampleStream(B, 1, C_, up, down)
    st = ResampleStream(B, 1, C_, up, down)
    chunk = torch.empty(B, 1, C_, device=DEV)
    out = torch.empty(B, 1, st.out_samples, device=DEV)
    chunk.copy_(x[..., :C_])
    st.step(chunk, out=out)
    eager = [eager_st.step(x[..., :C_])]
    got = [out.clone()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st.step(chunk, out=out)
    st.reset()
    eager_st.reset()
    for j in range(steps):                       # 21 replays, with resets of one slot and of all slots between them
        if j == 7:
            st.reset([1])
            eager_st.reset([1])
        if j == 14:
            st.reset()
            eager_st.reset()
        chunk.copy_(x[..., j * C_:(j + 1) * C_])
        g.replay()
        got.append(out.clone())
        eager.append(eager_st.step(x[..., j * C_:(j + 1) * C_]))
    torch.cuda.synchronize()
    assert torch.equal(bits(torch.cat(got, -1)), bits(torch.cat(eager, -1)))


def test_dtypes_and_strides_give_the_fp32_bits():
    up, down, C_ = 48000, 8000, 6
    x = signal((2, 3, 8 * C_), 9)
    want, wf = run(ResampleStream(2, 3, C_, up, down), x)
    got, gf = run(ResampleStream(2, 3, C_, up, down), x.double())          # fp64 of fp32 values: the same input
    assert torch.equal(bits(got), bits(want)) and torch.equal(bits(gf), bits(wf))
    h = x.half()
    got, gf = run(ResampleStream(2, 3, C_, up, down), h)
    ref, rf = run(ResampleStream(2, 3, C_, up, down), h.float())
    assert torch.equal(bits(got), bits(ref)) and torch.equal(bits(gf), bits(rf))
    wide = torch.zeros(3, 2, 8 * C_ * 2, device=DEV)
    strided = wide.transpose(0, 1)[..., ::2]
    strided.copy_(x)
    st = ResampleStream(2, 3, C_, up, down)
    got = torch.cat([st.step(strided[..., j * C_:(j + 1) * C_]) for j in range(8)], dim=-1)
    assert torch.equal(bits(got), bits(want))


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
@pytest.mark.parametrize("up,down", [(8000, 44100), (44100, 8000)])
def test_a_bad_value_reaches_exactly_its_support(bad, up, down):
    p, q = ratio(up, down)
    C_ = q
    steps = 12
    B = 3
    x = signal((B, 1, steps * C_), 10)
    # inside a chunk, at a chunk's first sample (read from the history by the next steps) and its last
    for pos in (5 * C_ + C_ // 2, 6 * C_, 7 * C_ - 1):
        y = x.clone()
        y[1, 0, pos] = bad
        st = ResampleStream(B, 1, C_, up, down)
        got, fl = run(st, y)
        want = expected(y, up, down, st.delay, 0, 0, steps * p)
        assert torch.equal(torch.isfinite(got), torch.isfinite(want)), pos
        assert not torch.isfinite(got[1]).all()
        assert torch.equal(bits(got[[0, 2]]), bits(want[[0, 2]]))
        ok = torch.isfinite(want)
        assert torch.equal(bits(got[ok]), bits(want[ok]))
        st.reset([1])                          # slot 1 starts over; a reset clears the bad value from its history
        again, _ = run(st, x)
        assert torch.isfinite(again[1]).all()
        assert torch.equal(bits(again[1:2]), bits(expected(x[1:2], up, down, st.delay, 0, 0, steps * p)))


def raw_stream(state, x, outs, zero, B, rows, C_, up, down, delay, lead):
    lib = N.lib()
    cur = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (B, rows, C_, up, down, delay, lead)
    N.check(lib.sdr_resample_stream_reset(C.c_void_p(state.data_ptr()), state.numel(), *args, None, 0, cur), "reset")
    for j, out in enumerate(outs):
        chunk = guarded_copy(x[..., j * C_:(j + 1) * C_].contiguous())
        N.check(lib.sdr_resample_stream_step(C.c_void_p(state.data_ptr()), state.numel(), C.c_void_p(chunk.data_ptr()),
                                             zero, C.c_void_p(out.data_ptr()), *args, cur), "step")
        check_bands(chunk, "chunk")


@pytest.mark.parametrize("pattern", [POISON_NAN, POISON_HUGE])
@pytest.mark.parametrize("up,down", [(44100, 8000), (8000, 44100), (11025, 192000)])
def test_poisoned_and_guarded_state_and_outputs(pattern, up, down):
    p, q = ratio(up, down)
    B, rows, C_, steps = 3, 2, q, 6
    delay, lead = min_delay(up, down, 2) + 3, 2
    lib = N.lib()
    nbytes = lib.sdr_resample_stream_state_bytes(B, rows, C_, up, down, delay, lead)
    x = signal((B, rows, steps * C_), 11)
    results = []
    for pat in (0, pattern):
        state = poisoned(nbytes, pat)
        outs = [poisoned_like(torch.empty(B, rows, C_ // q * p, device=DEV), pat) for _ in range(steps)]
        raw_stream(state, x, outs, None, B, rows, C_, up, down, delay, lead)
        n = (lead + 0) * p
        tail = poisoned_like(torch.empty(B, rows, -(-n // q) + delay, device=DEV), pat)
        N.check(lib.sdr_resample_stream_flush(C.c_void_p(state.data_ptr()), nbytes, None, 0, None,
                                              C.c_void_p(tail.data_ptr()), B, rows, C_, up, down, delay, lead,
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream)), "flush")
        for t, what in [(state, "state"), (tail, "flush")] + [(o, f"out {i}") for i, o in enumerate(outs)]:
            check_bands(t, what)
        results.append(torch.cat(outs + [tail], dim=-1).clone())
    assert torch.equal(bits(results[0]), bits(results[1]))
    want = expected(x, up, down, delay, lead, 0, results[0].shape[-1])
    assert torch.equal(bits(results[0]), bits(want))
    # a state one byte short, or misaligned, is refused before anything is enqueued
    state = poisoned(nbytes, 0)
    cur = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (B, rows, C_, up, down, delay, lead)
    assert lib.sdr_resample_stream_reset(C.c_void_p(state.data_ptr()), nbytes - 1, *args, None, 0, cur) == -3
    assert lib.sdr_resample_stream_reset(C.c_void_p(state.data_ptr() + 16), nbytes, *args, None, 0, cur) == -2


def test_alternating_cuda_streams_and_host_threads():
    up, down, B, C_ = 8000, 44100, 4, 441
    x = signal((B, 1, 16 * C_), 12)
    want, wf = run(ResampleStream(B, 1, C_, up, down), x)
    st = ResampleStream(B, 1, C_, up, down)
    sides = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    for j in range(16):
        with torch.cuda.stream(sides[j % 2]):
            outs.append(st.step(x[..., j * C_:(j + 1) * C_]))
            if j == 15:
                fl = st.flush()
    torch.cuda.synchronize()
    assert torch.equal(bits(torch.cat(outs, -1)), bits(want)) and torch.equal(bits(fl), bits(wf))

    results, errors = {}, []

    def worker(i):
        try:
            s = ResampleStream(B, 1, C_, up, down)
            with torch.cuda.stream(torch.cuda.Stream()):
                got, f = run(s, x)
                torch.cuda.current_stream().synchronize()
            results[i] = (got, f)
        except Exception as e:          # noqa: BLE001 - reported below
            errors.append(e)
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for got, f in results.values():
        assert torch.equal(bits(got), bits(want)) and torch.equal(bits(f), bits(wf))


def test_one_step_past_2_31_outputs():
    up, down = 48000, 8000                   # p / q = 6 / 1
    B, C_ = 1024, 350000                      # 1024 x 2.1 M = 2.15 G outputs in one step
    st = ResampleStream(B, 1, C_, up, down)
    x = torch.empty(B, 1, C_, device=DEV)
    x[-1].copy_(signal((1, C_), 13))
    x[:-1].fill_(0.25)
    out = st.step(x)
    assert out.numel() > 2 ** 31
    last = out[-1:].clone()
    del out
    torch.cuda.synchronize()
    alone = ResampleStream(1, 1, C_, up, down).step(x[-1:])
    assert torch.equal(bits(last), bits(alone))
    assert torch.equal(bits(last), bits(expected(x[-1:], up, down, st.delay, 0, 0, 6 * C_)))


# ---------------------------------------------------------------------------------------------------------------------
# 3. the causal model at another rate
# ---------------------------------------------------------------------------------------------------------------------
SMALL = dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64,
             num_sources=2)
MODELS = {
    "improved": (P.SuDORMRF, "improved", SMALL),
    "groupcomm": (P.GroupCommSudoRmRf, "groupcomm", dict(SMALL, group_size=4)),
    "causal": (P.CausalSuDORMRF, "causal", dict(SMALL, in_audio_channels=1)),
    "causal_stereo": (P.CausalSuDORMRF, "causal", dict(SMALL, in_audio_channels=2)),
    "original": (P.OriginalSuDORMRF, "original", SMALL),
}
_cache = {}


def model(name, seed=11):
    if (name, seed) not in _cache:
        cls, variant, kw = MODELS[name]
        sd = O.make_state_dict(O.Config(variant=variant, **kw), seed=seed)
        m = cls(**kw)
        m.load_state_dict(sd)
        _cache[name, seed] = m.to(DEV).eval()
    return _cache[name, seed]


def mixture(B, A, T, fs, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64) / fs
    tone = torch.sin(2 * np.pi * 220.0 * t) * torch.sin(2 * np.pi * 0.3 * t)
    return (0.3 * torch.randn(B, A, T, generator=g, dtype=torch.float64) + tone + 0.1).float().to(DEV)


def stream_all(st, x):
    C_ = st.chunk_samples
    return torch.cat([st.step(x[..., j:j + C_]) for j in range(0, x.shape[-1], C_)], dim=-1)


# chunk sizes of 80 model-rate samples (one granule of the small causal model) per step
CAUSAL_PAIRS = [(44100, 8000, 441), (48000, 8000, 480), (16000, 8000, 160), (8000, 16000, 40)]


@pytest.mark.parametrize("sr,mr,C_", CAUSAL_PAIRS)
@pytest.mark.parametrize("name,mc", [("causal", False), ("causal", True), ("causal_stereo", False)])
def test_causal_stream_is_separate_at_another_rate(name, mc, sr, mr, C_):
    m = model(name)
    A = MODELS[name][2]["in_audio_channels"]
    p, q = ratio(mr, sr)
    L = 10 * max(p, q)
    steps = 24                                     # n p / q = 24 x 80: a multiple of hop 2^depth = 160
    x = mixture(2, A, steps * C_, sr, sr + mr)
    n = x.shape[-1]
    with torch.no_grad():
        st = m.stream(2, C_, mixture_consistency=mc, sample_rate=sr, model_rate=mr)
        assert isinstance(st, ResampledStream) and isinstance(st.inner, CausalStream)
        D = st.latency
        assert D == C_ + (st.inner.latency * q + L) // p
        assert not st.flush().any()                                       # no step since the reset: zeros
        got = torch.cat([stream_all(st, x), st.flush()], dim=-1)[..., D:]
        want = m.separate(x, mixture_consistency=mc, sample_rate=sr, model_rate=mr)
        assert got.shape == want.shape
        assert torch.equal(bits(got), bits(want))
        # a prefix: the steps so far and the flush
        half = steps // 2 * C_
        st.reset()
        got = torch.cat([stream_all(st, x[..., :half]), st.flush()], dim=-1)[..., D:]
        assert torch.equal(bits(got), bits(m.separate(x[..., :half], mixture_consistency=mc, sample_rate=sr,
                                                      model_rate=mr)))
    if sr == 44100 and name == "causal" and not mc:
        assert D == 551 and n > D


def test_default_causal_model_latency():
    m = P.CausalSuDORMRF().to(DEV).eval()
    st = m.stream(1, 441, sample_rate=44100, model_rate=8000)
    assert st.latency == 551 and st.chunk_samples == 441 and st.batch_size == 1


def test_causal_slot_reset_mid_stream_and_graph_replay_across_it():
    m = model("causal")
    sr, mr, C_ = 44100, 8000, 441
    B, steps, cut = 3, 20, 8
    x = mixture(B, 1, steps * C_, sr, 17)
    with torch.no_grad():
        st = m.stream(B, C_, sample_rate=sr, model_rate=mr)
        D = st.latency
        a = stream_all(st, x[..., :cut * C_])
        st.reset([1])
        b = stream_all(st, x[..., cut * C_:])
        fl = st.flush()
        whole = m.separate(x, sample_rate=sr, model_rate=mr)
        got = torch.cat([a, b, fl], dim=-1)[..., D:]
        assert torch.equal(bits(got[[0, 2]]), bits(whole[[0, 2]]))
        fresh = m.separate(x[1:2, :, cut * C_:], sample_rate=sr, model_rate=mr)
        assert torch.equal(bits(torch.cat([b, fl], dim=-1)[1:2, :, D:]), bits(fresh))
        # a captured step, replayed across a reset of slot 1 and one of every slot, is the eager step
        eager = m.stream(B, C_, sample_rate=sr, model_rate=mr)
        cap = m.stream(B, C_, sample_rate=sr, model_rate=mr)
        chunk = torch.empty(B, 1, C_, device=DEV)
        out = torch.empty(B, 2, C_, device=DEV)
        chunk.copy_(x[..., :C_])
        cap.step(chunk, out=out)
        want = [eager.step(x[..., :C_])]
        got = [out.clone()]
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cap.step(chunk, out=out)
        for j in range(1, steps):
            if j == cut:
                cap.reset([1])
                eager.reset([1])
            if j == steps - 4:
                cap.reset()
                eager.reset()
            chunk.copy_(x[..., j * C_:(j + 1) * C_])
            g.replay()
            got.append(out.clone())
            want.append(eager.step(x[..., j * C_:(j + 1) * C_]))
        torch.cuda.synchronize()
        assert torch.equal(bits(torch.cat(got, -1)), bits(torch.cat(want, -1)))
        assert torch.equal(bits(cap.flush()), bits(eager.flush()))


# ---------------------------------------------------------------------------------------------------------------------
# 4. the windowed models at another rate
# ---------------------------------------------------------------------------------------------------------------------
def clear_end(m, xm, W, H, normalize, mc):
    """The first model-rate sample of xm's windowed separation that a near-tie of the alignment may change."""
    B, A, T = xm.shape
    if T <= W:
        return T
    K = WO.plan(T, W, H)[0]
    batch = torch.from_numpy(WO.windows(xm.cpu().numpy(), W, H)).to(DEV).reshape(B * K, A, W)
    est = m.separate(batch, mixture_consistency=mc, normalize=normalize).cpu().numpy()
    _, margin = WO.align(est.reshape(B, K, -1, A, W), T, W, H)
    close = np.nonzero((margin[:, 1:] <= MARGIN).any(axis=0))[0]
    return T if close.size == 0 else (1 + int(close[0])) * H


@pytest.mark.parametrize("normalize,mc", [(True, False), (False, True)])
@pytest.mark.parametrize("name", ["causal", "improved", "groupcomm", "original"])
def test_windowed_stream_is_separate_long_at_another_rate(name, normalize, mc):
    m = model(name)
    sr, mr, W, H = 44100, 8000, 4000, 2000
    C_ = 11025                                     # 2000 model-rate samples: one hop per step
    p, q = ratio(mr, sr)
    L = 10 * max(p, q)
    steps = 10
    x = mixture(2, 1, steps * C_, sr, 23)
    n = x.shape[-1]
    with torch.no_grad():
        st = m.stream_windows(2, C_, W, H, normalize=normalize, mixture_consistency=mc, sample_rate=sr, model_rate=mr)
        assert isinstance(st.inner, WindowedStream) and st.latency == C_ + (H * q + L) // p
        got = torch.cat([stream_all(st, x), st.flush()], dim=-1)[..., st.latency:]
        want = m.separate_long(x, W, H, normalize=normalize, mixture_consistency=mc, sample_rate=sr, model_rate=mr)
        assert got.shape == want.shape
        if name == "causal":
            assert torch.equal(bits(got), bits(want))
        else:
            end_m = clear_end(m, P.resample_poly(x, mr, sr), W, H, normalize, mc)
            end = n if end_m >= n * p // q else max(0, (end_m * q - L) // p)
            g, w = got[..., :end], want[..., :end]
            assert float((g - w).abs().max()) <= (MARGIN + SPREAD) * float(want.abs().max())


def test_windowed_latency_of_4s_windows_every_2s():
    m = model("improved")
    st = m.stream_windows(1, 88200, 32000, 16000, sample_rate=44100, model_rate=8000)
    assert st.latency == 176455 and st.chunk_samples == 88200


def test_ten_minutes_at_44k1_through_u16_512_at_8k():
    kw = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
              enc_num_basis=512, num_sources=2)
    sd = O.make_state_dict(O.Config(variant="improved", **kw), seed=3)
    m = P.SuDORMRF(**kw)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    sr, mr, C_ = 44100, 8000, 88200
    steps = 300                                   # ten minutes
    g = torch.Generator(device=DEV).manual_seed(5)
    peaks = []
    with torch.no_grad():
        st = m.stream_windows(1, C_, 4 * mr, 2 * mr, sample_rate=sr, model_rate=mr)
        chunk = torch.empty(1, 1, C_, device=DEV)
        out = torch.empty(1, 2, C_, device=DEV)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        for j in range(steps):
            chunk.normal_(generator=g)
            st.step(chunk, out=out)
            if j in (9, steps - 1):
                torch.cuda.synchronize()
                peaks.append(torch.cuda.max_memory_allocated())
        assert torch.isfinite(out).all() and out.abs().max() > 0
    print(f"\n10 min at 44.1 kHz through U16/512 at 8 kHz, streamed: peak {peaks[-1] / 2**30:.3f} GiB")
    assert peaks[-1] == peaks[0]
