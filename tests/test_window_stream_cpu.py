"""Windowed streams without a GPU (DESIGN.md section 7f): the bindings, the state size, the refusals, and an fp64 numpy
restatement of the stream that, fed the same window estimates, gives ``separate_long``'s output on every prefix."""
import os
import re

import numpy as np
import pytest

import sudo_rm_rf_b200 as P
import windowed_oracle as WO
from sudo_rm_rf_b200 import _native

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("sdr_window_stream_state_bytes", "sdr_window_stream_reset", "sdr_window_stream_gather",
           "sdr_window_stream_merge_scratch_bytes", "sdr_window_stream_merge", "sdr_window_stream_flush_scratch_bytes",
           "sdr_window_stream_flush", "sdr_window_stream_launch_count")


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
def estimator(S, A, W, seed):
    """A deterministic stand-in for a separator: window k's samples [A, L] -> [S, A, L] fp32, its sources in an order
    that changes with k.  It is not sample-wise (every source depends on the window's mean), so a window of L < W
    samples is not the first L samples of its zero-padded estimate, as with the normalising models."""
    g = np.random.default_rng(seed)
    gains = g.uniform(0.2, 2.0, (S, A, W)).astype(np.float32)

    def f(win, k):
        L = win.shape[-1]
        mean = win.mean(axis=-1, keepdims=True, dtype=np.float64).astype(np.float32)
        src = np.stack([gains[s, :, :L] * win + np.float32(s + 1) * mean for s in range(S)])
        order = np.random.default_rng(seed * 7919 + k + 2).permutation(S)
        return src[order].astype(np.float32)
    return f


def separate_long(x, W, H, f):
    """x [B, A, T] -> [B, S A, T]: windowed separation (windowed.separate_long) with window estimates f."""
    B, A, T = x.shape
    if T <= W:
        return np.stack([f(x[b], 0) for b in range(B)]).reshape(B, -1, T)
    wins = WO.windows(x, W, H)
    est = np.stack([np.stack([f(wins[b, k], k) for k in range(wins.shape[1])]) for b in range(B)])
    pi, _ = WO.align(est, T, W, H)
    return WO.overlap_add(est, pi, T, W, H)


class StreamOracle:
    """The stream's state and stages as DESIGN.md section 7f states them, one slot at a time: history, carry (raw
    estimate and order of the last window) and window counter c; a step completes windows c-1 .. c+q-2."""

    def __init__(self, B, S, A, C, W, H, f):
        self.B, self.S, self.A, self.C, self.W, self.H, self.f = B, S, A, C, W, H, f
        self.hist = np.zeros((B, A, H), np.float32)
        self.carry = np.zeros((B, S, A, W), np.float32)
        self.pi = np.tile(np.arange(S), (B, 1))
        self.count = np.zeros(B, np.int64)

    def reset(self, slots):
        for b in slots:
            self.hist[b], self.carry[b], self.pi[b], self.count[b] = 0, 0, np.arange(self.S), 0

    def _out(self, prev, prev_pi, cur, cur_pi, k, js):
        """[S, A, len(js)] of window k at offsets js, cross-faded with window k-1 (prev) in the overlap."""
        S, W, H = self.S, self.W, self.H
        o = np.zeros((S, self.A, len(js)), np.float32)
        for s in range(S):
            c = cur[cur_pi[s]][:, js].T                       # [len, A]
            if k > 0:
                p = prev[prev_pi[s]][:, np.minimum(js + H, W - 1)].T
                c = np.where((js < W - H)[:, None], WO.fade(p, c, js, W - H), c)
            o[s] = c.T
        return o

    def step(self, chunk):
        B, S, A, C, W, H = self.B, self.S, self.A, self.C, self.W, self.H
        q = C // H
        out = np.zeros((B, S, A, C), np.float32)
        for b in range(B):
            ext = np.concatenate([self.hist[b], chunk[b]], axis=-1)
            c0 = int(self.count[b])
            prev, pi = self.carry[b], list(self.pi[b]) if c0 > 1 else list(range(S))
            for m in range(q):
                k = c0 - 1 + m
                win = ext[:, m * H:m * H + W] if k >= 0 else np.zeros((A, W), np.float32)
                cur = self.f(win, k)
                rho = WO.best(WO.correlation(prev, cur, H, W - H))[0] if k > 0 else tuple(range(S))
                new = [rho[s] for s in pi]
                if k >= 0:
                    out[b, :, :, m * H:(m + 1) * H] = self._out(prev, pi, cur, new, k, np.arange(H))
                prev, pi = cur, new
            self.carry[b], self.pi[b], self.count[b] = prev, pi, c0 + q
            self.hist[b] = chunk[b][:, C - H:]
        return out.reshape(B, S * A, C)

    def flush(self):
        B, S, A, W, H = self.B, self.S, self.A, self.W, self.H
        out = np.zeros((B, S, A, H), np.float32)
        for b in range(B):
            c = int(self.count[b])
            if c == 1:                                        # one window long: separated unpadded
                out[b] = self.f(self.hist[b], 0)
            elif c > 1 and W == 2 * H:                        # the carry's window ends at n
                out[b] = self._out(None, None, self.carry[b], self.pi[b], 0, np.arange(H, 2 * H))
            elif c > 1:                                       # one more window, zero-padded past n
                win = np.concatenate([self.hist[b], np.zeros((A, W - H), np.float32)], axis=-1)
                cur = self.f(win, c - 1)
                rho = WO.best(WO.correlation(self.carry[b], cur, H, W - H))[0]
                new = [rho[s] for s in self.pi[b]]
                out[b] = self._out(self.carry[b], self.pi[b], cur, new, c - 1, np.arange(H))
        return out.reshape(B, S * A, H)


def prefix_output(x, n, C, W, H, f):
    """Samples [n - H, n + C - H) of separate_long(x[..., :n + C]), zeros below 0."""
    full = separate_long(x[..., :n + C], W, H, f)
    want = np.zeros(full.shape[:2] + (C,), np.float32)
    lo = max(n - H, 0)
    want[..., lo - (n - H):] = full[..., lo:n + C - H]
    return want


SHAPES = [(12, 6), (9, 6), (11, 6), (7, 4), (10, 5)]       # W = 2H even, W < 2H even and odd


@pytest.mark.parametrize("W,H", SHAPES)
@pytest.mark.parametrize("q", [1, 2, 5])
@pytest.mark.parametrize("S,A", [(1, 1), (2, 2), (3, 1), (4, 2)])
def test_restatement_is_separate_long_on_every_prefix(W, H, q, S, A):
    B, C = 2, q * H
    f = estimator(S, A, W, seed=W * 100 + H * 10 + S + A)
    steps = max(2, -(-14 * H // C))                           # past 12 windows
    x = np.random.default_rng(q * 31 + S * 7 + A).standard_normal((B, A, steps * C)).astype(np.float32)
    st = StreamOracle(B, S, A, C, W, H, f)
    for j in range(steps):
        n = j * C
        # the flush before this step: the last H samples of separate_long on what has arrived
        tail = st.flush()
        if n == 0:
            assert not tail.any()
        else:
            assert np.array_equal(tail, separate_long(x[..., :n], W, H, f)[..., n - H:n]), (j, "flush")
        got = st.step(x[..., n:n + C])
        assert np.array_equal(got, prefix_output(x, n, C, W, H, f)), j
    outs = []
    st2 = StreamOracle(B, S, A, C, W, H, f)
    for j in range(steps):
        outs.append(st2.step(x[..., j * C:(j + 1) * C]))
    whole = separate_long(x, W, H, f)
    assert np.array_equal(np.concatenate(outs + [st2.flush()], axis=-1)[..., H:], whole)


def test_restatement_reset_slot_equals_a_fresh_stream():
    S, A, W, H, C = 2, 1, 9, 6, 12
    f = estimator(S, A, W, seed=4)
    x = np.random.default_rng(0).standard_normal((3, A, 6 * C)).astype(np.float32)
    st = StreamOracle(3, S, A, C, W, H, f)
    for j in range(3):
        st.step(x[..., j * C:(j + 1) * C])
    st.reset([1])
    fresh = StreamOracle(1, S, A, C, W, H, f)
    for j in range(3, 6):
        got = st.step(x[..., j * C:(j + 1) * C])
        assert np.array_equal(got[1:2], fresh.step(x[1:2, :, j * C:(j + 1) * C])), j


# ---------------------------------------------------------------------------------------------------------------------
# bindings, state size, refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_entries_bind_and_match_the_header():
    lib = _native.lib()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(REPO, "include", "sudormrf_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(sdr_[a-z_0-9]+)\s*\(", hdr))
    for name in ENTRIES:
        assert name in declared and name in _native.EXPORTED_SYMBOLS and hasattr(lib, name), name
    assert lib.sdr_abi_version() == 2
    # refused before anything is enqueued (no device needed)
    assert lib.sdr_window_stream_reset(None, 1, 2, 1, 10, 5, None, 0, None) == -2
    assert lib.sdr_window_stream_gather(None, None, None, 1, 2, 1, 10, 10, 5, None) == -2
    assert lib.sdr_window_stream_merge(None, None, None, 1, 2, 1, 10, 10, 5, None, None) == -2
    assert lib.sdr_window_stream_flush(None, None, None, None, 1, 2, 1, 10, 5, None, None) == -2
    assert lib.sdr_window_stream_launch_count(1, 2, 1, 10, 10, 5) == 6
    assert lib.sdr_window_stream_launch_count(1, 5, 1, 10, 10, 5) == -5
    assert lib.sdr_window_stream_launch_count(1, 2, 1, 7, 10, 5) == -2


@pytest.mark.parametrize("B,S,A,W,H", [(1, 1, 1, 10, 5), (3, 2, 2, 9, 6), (3, 1, 1, 101, 51), (7, 4, 1, 32000, 16000),
                                       (65535, 3, 2, 2 ** 24, 2 ** 23)])
def test_state_size(B, S, A, W, H):
    lib = _native.lib()
    r = lambda v: (v + 255) // 256 * 256             # noqa: E731
    carry = lib.sdr_window_carry_bytes(B, S, A, W)
    assert carry == r(B * S * 4) + B * S * A * W * 4
    assert lib.sdr_window_stream_state_bytes(B, S, A, W, H) == r(carry) + r(B * A * H * 4) + 8 * B
    assert lib.sdr_window_stream_merge_scratch_bytes(B, S, 3 * H, H) == (B * 3 * S + B * 4 * S) * 4
    assert lib.sdr_window_stream_flush_scratch_bytes(B, S) == (B * S + 2 * B * S) * 4


def test_state_size_refusals():
    lib = _native.lib()
    assert lib.sdr_window_stream_state_bytes(1, 5, 1, 10, 5) == 0             # S > 4
    assert lib.sdr_window_stream_state_bytes(1, 0, 1, 10, 5) == 0
    assert lib.sdr_window_stream_state_bytes(0, 2, 1, 10, 5) == 0
    assert lib.sdr_window_stream_state_bytes(1, 2, 1, 10, 4) == 0             # H < W / 2
    assert lib.sdr_window_stream_state_bytes(1, 2, 1, 10, 10) == 0            # H = W
    assert lib.sdr_window_stream_state_bytes(1, 2, 1, 2 ** 24 + 2, 2 ** 23 + 1) == 0
    assert lib.sdr_window_stream_merge_scratch_bytes(1, 2, 7, 5) == 0         # C not a multiple of H
    assert lib.sdr_window_stream_merge_scratch_bytes(1, 2, 0, 5) == 0


KW = dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=2, enc_kernel_size=5, enc_num_basis=16,
          num_sources=2)


@pytest.mark.parametrize("kw,msg", [
    (dict(batch_size=1, chunk_samples=3000, window=4000, hop=2000), "multiple of the hop"),
    (dict(batch_size=1, chunk_samples=0, window=4000, hop=2000), "multiple of the hop"),
    (dict(batch_size=1, chunk_samples=2000, window=4000, hop=1999), "hop must be"),
    (dict(batch_size=1, chunk_samples=4000, window=4000, hop=4000), "hop must be"),
    (dict(batch_size=1, chunk_samples=2, window=1), "window must be"),
    (dict(batch_size=0, chunk_samples=2000, window=4000), "batch_size"),
    (dict(batch_size=65536, chunk_samples=2000, window=4000), "batch_size"),
    (dict(batch_size=True, chunk_samples=2000, window=4000), "batch_size"),
])
def test_argument_refusals(kw, msg):
    m = P.SuDORMRF(**KW).eval()
    with pytest.raises(ValueError, match=msg):
        m.stream_windows(**kw)


def test_other_refusals():
    with pytest.raises(RuntimeError, match="mono"):
        P.GroupCommSudoRmRf(**KW, group_size=4, in_audio_channels=2).stream_windows(1, 2000, 4000, normalize=False)
    with pytest.raises(RuntimeError, match="README recipe"):
        P.GroupCommSudoRmRf(**KW, group_size=4, in_audio_channels=2).stream_windows(1, 2000, 4000,
                                                                                     mixture_consistency=False)
    with pytest.raises(_native.NativeError, match="1 to 4 sources"):
        P.SuDORMRF(**dict(KW, num_sources=5)).stream_windows(1, 2000, 4000)
    with pytest.raises(_native.NativeError, match="2\\^24"):
        P.SuDORMRF(**KW).stream_windows(1, 2 ** 24 + 2, 2 ** 24 + 2)
    for cls, extra in ((P.SuDORMRF, {}), (P.GroupCommSudoRmRf, dict(group_size=4)), (P.CausalSuDORMRF, {}),
                       (P.OriginalSuDORMRF, {})):
        with pytest.raises(RuntimeError, match="CUDA"):               # a CPU model
            cls(**KW, **extra).eval().stream_windows(2, 4000, 4000, 2000)


def test_defaults_follow_separate():
    """The public signatures of the methods the four classes share, defaults included: GroupComm applies mixture
    consistency by default everywhere but in ``forward_host``."""
    import inspect
    want = {
        "separate": "(self, input_wav, mixture_consistency={mc}, normalize=False, sample_rate=None, model_rate=None)",
        "separate_long": "(self, input_wav, window, hop=None, normalize=True, mixture_consistency={mc}, "
                         "max_windows=32, sample_rate=None, model_rate=None)",
        "stream_windows": "(self, batch_size, chunk_samples, window, hop=None, normalize=True, "
                          "mixture_consistency={mc}, sample_rate=None, model_rate=None)",
        "forward_host": "(self, host_wav, host_out=None, mixture_consistency=False)",
        "pad_to_appropriate_length": "(self, x)",
        "remove_trailing_zeros": "(padded_x, initial_x)",
    }
    for cls in (P.SuDORMRF, P.GroupCommSudoRmRf, P.CausalSuDORMRF, P.OriginalSuDORMRF):
        for name, sig in want.items():
            got = str(inspect.signature(getattr(cls, name)))
            assert got == sig.format(mc=cls is P.GroupCommSudoRmRf), (cls, name, got)
        sep = inspect.signature(cls.separate).parameters["mixture_consistency"].default
        sw = inspect.signature(cls.stream_windows).parameters
        assert sw["mixture_consistency"].default == sep and sw["normalize"].default is True, cls
    assert str(inspect.signature(P.CausalSuDORMRF.stream)) == \
        "(self, batch_size, chunk_samples, mixture_consistency=False, sample_rate=None, model_rate=None)"
    assert P.WindowedStream is P.window_stream.WindowedStream
