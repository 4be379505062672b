"""Streaming at any sample rate without a GPU (DESIGN.md section 7h): an fp64 numpy restatement of ``ResampleStream``
(history, counter, delay, lead, flush tail) against ``scipy.signal.resample_poly`` on the concatenation, the same for
``ResampledStream`` around an identity and a causal FIR model, the bindings, the state size and the refusals."""
import ctypes
import itertools
import math
import os
import re

import numpy as np
import pytest
import scipy.signal as ss

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.resample_stream import ResampleStream, min_delay
from sudo_rm_rf_b200.streaming import CausalStream
from sudo_rm_rf_b200.window_stream import WindowedStream

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000)
ENTRIES = ("sdr_resample_stream_state_bytes", "sdr_resample_stream_reset", "sdr_resample_stream_step",
           "sdr_resample_stream_flush", "sdr_stream_reset_masked", "sdr_window_stream_reset_masked")
ERR_BAD_ARGUMENT, ERR_WORKSPACE, ERR_UNSUPPORTED = -2, -3, -5


def ratio(up, down):
    g = math.gcd(up, down)
    return up // g, down // g


class Restated:
    """One slot of ResampleStream in fp64: the counter j, the history of Hs samples, and V = [history | chunk] with
    V[k] = s[lead + j C - Hs + k]; output o sums h[c - t p] s[t] over resample_poly's support, c = o q + L."""

    def __init__(self, up, down, C, delay=None, lead=0):
        self.p, self.q = ratio(up, down)
        p, q = self.p, self.q
        self.L = L = 10 * max(p, q)
        self.h = ss.firwin(2 * L + 1, 1.0 / max(p, q), window=("kaiser", 5.0)) * p
        self.C, self.lead = C, lead
        self.delay = min_delay(up, down, lead) if delay is None else delay
        self.Hs = lead + (self.delay * q + L) // p + 1
        self.hist = np.zeros(self.Hs)
        self.j = 0

    def _outputs(self, V, o0, n, length):
        p, q, L = self.p, self.q, self.L
        base = self.lead + self.j * self.C - self.Hs
        out = np.zeros(n)
        for i in range(n):
            o = o0 + i
            if o < 0:
                continue
            c = o * q + L
            cp, r = divmod(c, p)
            t0, t1 = max(cp - (2 * L - r) // p, 0), min(cp, length - 1)
            if t1 < t0:
                continue
            assert t0 >= base, "the history does not reach the support"
            t = np.arange(t0, t1 + 1)
            out[i] = np.dot(self.h[r + (cp - t) * p], V[t - base])
        return out

    def step(self, chunk):
        V = np.concatenate([self.hist, chunk])
        P_ = self.C // self.q * self.p
        out = self._outputs(V, self.j * P_ - self.delay, P_, self.lead + (self.j + 1) * self.C)
        self.hist = V[self.C:]
        self.j += 1
        return out

    def flush(self, tail=np.zeros(0)):
        V = np.concatenate([self.hist, tail])
        P_ = self.C // self.q * self.p
        n = -(-(self.lead + len(tail)) * self.p // self.q) + self.delay
        return self._outputs(V, self.j * P_ - self.delay, n, self.lead + self.j * self.C + len(tail))


def reference(s, up, down, start, n):
    r = ss.resample_poly(s, up, down)
    out = np.zeros(n)
    lo, hi = max(start, 0), min(start + n, len(r))
    if hi > lo:
        out[lo - start:hi - start] = r[lo:hi]
    return out


@pytest.mark.parametrize("up,down", list(itertools.permutations(RATES, 2)))
def test_restatement_is_resample_poly(up, down):
    p, q = ratio(up, down)
    g = np.random.default_rng(up * 7 + down)
    for steps, lead, extra, C in ((1, 0, 0, q), (4, 0, 3, q), (3, 2, 0, 2 * q), (2, q + 3, 5, q)):
        st = Restated(up, down, C, None if extra == 0 else min_delay(up, down, lead) + extra, lead)
        x = g.standard_normal(steps * C)
        tail = g.standard_normal(3)
        got = np.concatenate([st.step(x[j * C:(j + 1) * C]) for j in range(steps)])
        s = np.concatenate([np.zeros(lead), x, tail])
        P_ = steps * C // q * p
        want = reference(s, up, down, -st.delay, P_)
        assert np.allclose(got, want, rtol=0, atol=1e-12), (steps, lead, extra)
        fl = st.flush(tail)
        n_end = -(-len(s) * p // q)
        assert len(fl) == n_end - (P_ - st.delay)
        assert np.allclose(fl, reference(s, up, down, P_ - st.delay, len(fl)), rtol=0, atol=1e-12)


def test_smallest_delays_of_the_issue_examples():
    assert min_delay(8000, 44100) == 10 and min_delay(44100, 8000) == 55        # 44.1 -> 8 kHz and 8 -> 44.1 kHz


class Composite:
    """ResampledStream in fp64 around a causal model f that streams with latency lat (identity: f = x)."""

    def __init__(self, sr, mr, C, f, lat):
        self.p, self.q = p, q = ratio(mr, sr)
        self.L = 10 * max(p, q)
        self.C, self.Cm = C, C // q * p
        self.f, self.lat = f, lat
        self.inp = Restated(mr, sr, C, self.Cm)
        m = -(-(self.Cm + lat) // p)
        self.out = Restated(sr, mr, self.Cm, None, m * p - (self.Cm + lat))
        self.latency = C + (lat * q + self.L) // p
        assert self.latency == self.out.delay + m * q
        self.xm = np.zeros(0)                  # what the inner stream received since its (deferred) reset
        self.fresh = True

    def _inner(self, xm):
        """The inner stream's step: f's output samples [n - lat, n + Cm - lat) of everything received."""
        n = len(self.xm)
        self.xm = np.concatenate([self.xm, xm])
        y = self.f(self.xm)
        return np.concatenate([np.zeros(max(0, self.lat - n)), y[max(0, n - self.lat):n + self.Cm - self.lat]])

    def step(self, chunk):
        est = self._inner(self.inp.step(chunk))
        if self.fresh:
            est[:] = 0
            self.xm = np.zeros(0)
            self.fresh = False
        return self.out.step(est)

    def flush(self):
        keep = self.xm
        est = self._inner(self.inp.flush())
        y = self.f(self.xm)
        tail = np.concatenate([est, y[len(self.xm) - self.lat:]])
        self.xm = keep
        if self.fresh:
            tail[:] = 0
        return self.out.flush(tail)


@pytest.mark.parametrize("sr,mr,C", [(44100, 8000, 441), (48000, 8000, 480), (8000, 16000, 40), (16000, 8000, 160),
                                     (11025, 16000, 441)])
@pytest.mark.parametrize("model,lat", [("identity", 0), ("identity", 10), ("fir", 10), ("fir", 37)])
def test_composite_restatement_is_separate_at_another_rate(sr, mr, C, model, lat):
    g = np.random.default_rng(sr + mr + lat)
    taps = g.standard_normal(9)
    f = (lambda v: v.copy()) if model == "identity" else (lambda v: np.convolve(v, taps)[:len(v)] + 0.25)
    for steps in (1, 2, 5):
        st = Composite(sr, mr, C, f, lat)
        x = g.standard_normal(steps * C)
        got = np.concatenate([st.step(x[j * C:(j + 1) * C]) for j in range(steps)] + [st.flush()])
        want = ss.resample_poly(f(ss.resample_poly(x, mr, sr)), sr, mr)[:len(x)]
        D = st.latency
        assert len(got) == len(x) + D
        assert np.allclose(got[D:], want, rtol=0, atol=1e-10), (steps, D)
    p, q = ratio(mr, sr)
    assert st.latency == C + (lat * q + 10 * max(p, q)) // p


def test_composite_latencies_of_the_issue_examples():
    assert Composite(44100, 8000, 441, None, 10).latency == 551
    assert Composite(44100, 8000, 88200, None, 16000).latency == 176455


# ---------------------------------------------------------------------------------------------------------------------
# bindings, state size, refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_entries_bind_and_match_the_header():
    lib = N.lib()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(REPO, "include", "sudormrf_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(sdr_[a-z_0-9]+)\s*\(", hdr))
    for name in ENTRIES:
        assert name in declared and name in N.EXPORTED_SYMBOLS and hasattr(lib, name), name
    assert lib.sdr_abi_version() == 2
    assert P.ResampleStream is ResampleStream


@pytest.mark.parametrize("B,rows,C,up,down,delay,lead", [(1, 1, 441, 8000, 44100, 10, 0), (3, 2, 441, 8000, 44100, 20, 7),
                                                         (65535, 1, 80, 44100, 8000, 55, 0),
                                                         (2, 3, 2560, 11025, 192000, 10, 0),
                                                         (5, 1, 147, 192000, 11025, 174, 0)])
def test_state_size(B, rows, C, up, down, delay, lead):
    p, q = ratio(up, down)
    L = 10 * max(p, q)
    r = lambda v: (v + 255) // 256 * 256             # noqa: E731
    Hs = lead + (delay * q + L) // p + 1
    want = r(8 * (2 * L + 1)) + r(8 * B) + 2 * B * rows * Hs * 4
    assert N.lib().sdr_resample_stream_state_bytes(B, rows, C, up, down, delay, lead) == want


def test_abi_refusals_before_any_launch():
    lib = N.lib()
    x = 256                     # any non-null, aligned address: these calls return before reading a buffer
    args = (2, 1, 441, 8000, 44100, 10, 0)
    need = lib.sdr_resample_stream_state_bytes(*args)
    assert lib.sdr_resample_stream_state_bytes(2, 1, 440, 8000, 44100, 10, 0) == 0          # C not a multiple of q
    assert lib.sdr_resample_stream_state_bytes(2, 1, 441, 8000, 44100, 9, 0) == 0           # delay below its least
    assert lib.sdr_resample_stream_state_bytes(0, 1, 441, 8000, 44100, 10, 0) == 0
    assert lib.sdr_resample_stream_state_bytes(65536, 1, 441, 8000, 44100, 10, 0) == 0
    assert lib.sdr_resample_stream_state_bytes(2, 0, 441, 8000, 44100, 10, 0) == 0
    assert lib.sdr_resample_stream_state_bytes(2, 1, 4097, 1, 4097, 10, 0) == 0             # ratio past 4096
    assert lib.sdr_resample_stream_state_bytes(2, 1, 3, 3, 3, 10, 0) == 0                   # nothing to resample
    assert lib.sdr_resample_stream_state_bytes(2, 1, 441, 8000, 44100, 10, -1) == 0

    def reset(st, nb, a=args):
        return lib.sdr_resample_stream_reset(st, nb, *a, None, 0, None)
    assert reset(None, need) == ERR_BAD_ARGUMENT
    assert reset(x, need - 1) == ERR_WORKSPACE
    assert reset(x + 16, need) == ERR_BAD_ARGUMENT
    assert reset(x, need, (2, 1, 441, 1, 4097, 10, 0)) == ERR_UNSUPPORTED
    assert reset(x, need, (2, 1, 441, 8000, 44100, 9, 0)) == ERR_BAD_ARGUMENT
    assert lib.sdr_resample_stream_reset(x, need, *args, (ctypes.c_int32 * 1)(2), 1, None) == ERR_BAD_ARGUMENT

    def step(st, nb, chunk, out):
        return lib.sdr_resample_stream_step(st, nb, chunk, None, out, *args, None)
    assert step(None, need, x, x) == ERR_BAD_ARGUMENT
    assert step(x, need, None, x) == ERR_BAD_ARGUMENT
    assert step(x, need, x, None) == ERR_BAD_ARGUMENT
    assert step(x, need - 1, x, x) == ERR_WORKSPACE
    assert step(x + 8, need, x, x) == ERR_BAD_ARGUMENT

    def flush(st, nb, tail, t, out):
        return lib.sdr_resample_stream_flush(st, nb, tail, t, None, out, *args, None)
    assert flush(None, need, None, 0, x) == ERR_BAD_ARGUMENT
    assert flush(x, need, None, 0, None) == ERR_BAD_ARGUMENT
    assert flush(x, need, None, 3, x) == ERR_BAD_ARGUMENT                                  # a tail without data
    assert flush(x, need, x, -1, x) == ERR_BAD_ARGUMENT
    assert flush(x, need - 1, None, 0, x) == ERR_WORKSPACE
    assert flush(x + 8, need, None, 0, x) == ERR_BAD_ARGUMENT
    assert lib.sdr_window_stream_reset_masked(None, 1, 2, 1, 10, 5, x, None) == ERR_BAD_ARGUMENT
    assert lib.sdr_window_stream_reset_masked(x, 1, 2, 1, 10, 5, None, None) == ERR_BAD_ARGUMENT
    assert lib.sdr_window_stream_reset_masked(x, 1, 5, 1, 10, 5, x, None) == ERR_UNSUPPORTED


@pytest.mark.parametrize("kw,msg", [
    (dict(chunk_samples=440), "multiple of q = 441"),
    (dict(chunk_samples=0), "multiple of q = 441"),
    (dict(delay=9), "at least floor\\(\\(L - lead p\\) / q\\) = 10"),
    (dict(lead=-1), "lead"),
    (dict(batch_size=0), "1 .. 65535"),
    (dict(batch_size=65536), "1 .. 65535"),
    (dict(rows=0), "rows"),
    (dict(up=1, down=4097, chunk_samples=4097), "at most 4096"),
    (dict(up=3, down=3, chunk_samples=3), "nothing to resample"),
])
def test_resample_stream_refusals(kw, msg):
    args = dict(batch_size=2, rows=1, chunk_samples=441, up=8000, down=44100)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        ResampleStream(args.pop("batch_size"), args.pop("rows"), args.pop("chunk_samples"), args.pop("up"),
                       args.pop("down"), **args)


KW = dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=2, enc_kernel_size=21, enc_num_basis=16,
          num_sources=2)
CLASSES = ((P.SuDORMRF, {}), (P.GroupCommSudoRmRf, dict(group_size=4)), (P.CausalSuDORMRF, {}),
           (P.OriginalSuDORMRF, {}))


def test_model_stream_refusals():
    causal = P.CausalSuDORMRF(**KW).eval()          # granule 10 x max(4, 2) = 40 samples
    cases = [
        (dict(chunk_samples=440), "multiple of q = 441"),
        (dict(chunk_samples=6 * 41, sample_rate=48000, model_rate=8000),
         "not a multiple of the inner stream's granule \\(40 samples\\)"),
        (dict(chunk_samples=12, sample_rate=48000, model_rate=8000), "fewer than the input resampler's delay"),
    ]
    for kw, msg in cases:
        args = dict(sample_rate=44100, model_rate=8000)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            causal.stream(2, args.pop("chunk_samples"), **args)
    # Cm = 80 at 16 -> 8 kHz: the least is floor(20 / 2) = 10, and 80 is a multiple of the granule
    with pytest.raises(RuntimeError, match="CUDA"):
        causal.stream(2, 160, sample_rate=16000, model_rate=8000)
    for cls, extra in CLASSES:
        m = cls(**KW, **extra).eval()
        with pytest.raises(ValueError, match="not a multiple of the inner stream's hop \\(2000 samples\\)"):
            m.stream_windows(1, 441 * 26, 4000, 2000, sample_rate=44100, model_rate=8000)
        with pytest.raises(RuntimeError, match="CUDA"):
            m.stream_windows(1, 441 * 25, 4000, 2000, sample_rate=44100, model_rate=8000)


@pytest.mark.parametrize("rates", [dict(sample_rate=44100), dict(model_rate=8000), dict(sample_rate=0, model_rate=8000),
                                   dict(sample_rate=44100, model_rate=-8000), dict(sample_rate=44100.0, model_rate=8000),
                                   dict(sample_rate=True, model_rate=8000), dict(sample_rate=8000, model_rate=8000 * 4097)])
def test_bad_rates_are_separates_refusals(rates):
    x = np.zeros(1)
    for cls, extra in CLASSES:
        m = cls(**KW, **extra).eval()
        with pytest.raises(ValueError) as want:
            m.separate(x, **rates)
        with pytest.raises(ValueError) as got:
            m.stream_windows(1, 4000, 4000, 2000, **rates)
        assert str(got.value) == str(want.value)
        if cls is P.CausalSuDORMRF:
            with pytest.raises(ValueError) as got:
                m.stream(1, 80, **rates)
            assert str(got.value) == str(want.value)


def test_equal_rates_or_none_are_the_existing_streams():
    import inspect
    for cls, extra in CLASSES:
        sw = inspect.signature(cls.stream_windows).parameters
        assert list(sw)[-2:] == ["sample_rate", "model_rate"]
        m = cls(**KW, **extra).eval()
        for rates in (dict(), dict(sample_rate=16000, model_rate=16000)):
            with pytest.raises(RuntimeError) as plain:
                WindowedStream(m, 1, 2000, 4000, 2000)
            with pytest.raises(RuntimeError) as same:
                m.stream_windows(1, 2000, 4000, 2000, **rates)
            assert str(plain.value) == str(same.value)
    causal = P.CausalSuDORMRF(**KW).eval()
    with pytest.raises(RuntimeError) as plain:
        CausalStream(causal, 1, 80)
    for rates in (dict(), dict(sample_rate=8000, model_rate=8000)):
        with pytest.raises(RuntimeError) as same:
            causal.stream(1, 80, **rates)
        assert str(plain.value) == str(same.value)
