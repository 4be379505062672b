"""BSS-eval of source images on the GPU (sdr_bss_eval_images, sdr_bss_eval_images_framewise): SDR, ISR, SIR and SAR
against the fp64 least-squares restatement of mir_eval's bss_eval_images (bss_images_oracle.py) within section 7c's
bar, over every (S, C) with S C <= 4, F 1, 16 and 512, the shortest accepted length and one past a correlation chunk,
white and AR references mixed, filtered and noised at -10..40 dB, with and without the permutation; SIR and SAR at
C = 1 against bss_eval_sources; a zero channel in a non-silent image; silent and non-finite images confined to their
item or window; repeat calls and CUDA-graph replay bit for bit; framewise columns bit for bit the sliced windows,
ragged lengths, the fallback, NaN columns, and an hour of stereo within twice its inputs' memory."""
import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import sudo_rm_rf_b200 as P
from bss_images_oracle import bss_eval_images as oracle, bss_eval_images_framewise as oracle_framewise, criteria
from test_gpu_bss_eval import low_tolerance

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PAIRS = [(1, 1), (2, 1), (3, 1), (4, 1), (1, 2), (1, 3), (1, 4), (2, 2)]
CHUNK = 128                 # bsseval.cu's kBssFramewiseItems: windows per launch


def make_images(rng, S, C, T, F, coloured):
    """References [S, T, C] (white or AR-coloured rows) and estimates: every row mixed from all S C reference rows,
    noised at -10..40 dB and filtered by a short FIR shorter or longer than F, the images in a random order."""
    R = S * C
    refs = rng.standard_normal((R, T))
    if coloured:
        for r in range(R):
            refs[r] = lfilter([1.0], [1.0, -rng.uniform(0.5, 0.95)], refs[r])
    ests = (np.eye(R) + rng.uniform(0.05, 0.4) * rng.standard_normal((R, R))) @ refs
    for r in range(R):
        snr = rng.uniform(-10, 40)
        noise = rng.standard_normal(T)
        ests[r] += noise * np.sqrt(np.sum(ests[r] ** 2) / np.sum(noise ** 2) / 10 ** (snr / 10))
        taps = int(rng.choice([max(1, F // 2), F + 7]))
        fir = rng.standard_normal(taps) * np.exp(-np.arange(taps) / 4.0)
        fir[0] = 1.0
        ests[r] = lfilter(fir, [1.0], ests[r])
    refs = refs.reshape(S, C, T).transpose(0, 2, 1)
    ests = ests.reshape(S, C, T).transpose(0, 2, 1)[rng.permutation(S)]
    return refs.astype(np.float32), ests.astype(np.float32)


def gpu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def images(refs, ests, perm=True, F=512):
    with torch.no_grad():
        return P.bss_eval_images(refs, ests, perm, F)


def framewise(refs, ests, W, H, perm=False, F=512, **kw):
    with torch.no_grad():
        return P.bss_eval_images_framewise(refs, ests, W, H, perm, F, **kw)


def host(out):
    return [o.cpu().numpy() for o in out]


def assert_equal(got, want, label=""):
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == w.dtype, label
        assert torch.equal(g, w) or bool(((g == w) | (torch.isnan(g) & torch.isnan(w))).all()), label


def check_values(got, ref, label, amp_db=None):
    """|d| <= 1e-3 dB where the oracle lies in [-20, 60] dB; below -20 dB within low_tolerance (amp_db the oracle's
    SDR of the same pairs for an SIR); above 60 dB, where |e - P e|^2 approaches the solve's rounding (the delays
    filling the space at T = (S C - 1) F + 1, or a noiseless estimate), above 40 dB; NaN where the oracle has it."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (label, got, ref)
    mid = (ref >= -20) & (ref <= 60)
    assert np.all(np.abs(got - ref)[mid] <= 1e-3), (label, got[mid], ref[mid])
    low = np.isfinite(ref) & (ref < -20)
    tol = low_tolerance(ref if amp_db is None else np.broadcast_to(amp_db, ref.shape))
    assert np.all(np.abs(got - ref)[low] <= tol[low]), (label, got[low], ref[low], tol[low])
    high = ref > 60
    assert np.all(got[high] > 40), (label, got[high], ref[high])


def check_against_oracle(got, refs, ests, perm, F, label):
    """The values wherever the permutations agree; where they do not, the oracle scores the GPU's assignment within
    1e-3 dB of its best mean SIR, or its best lies above 60 dB, where both rank rounding noise."""
    r, e = refs.astype(np.float64), ests.astype(np.float64)
    want = oracle(r, e, perm, F)
    if np.array_equal(got[4], want[4]):
        for g, w, name in zip(got[:4], want[:4], ("sdr", "isr", "sir", "sar")):
            check_values(g, w, f"{label} {name}", want[0] if name == "sir" else None)
    else:
        p = np.asarray(got[4])
        assert (p >= 0).all(), (label, got[4], want[4])
        theirs = np.mean(criteria(r, e, F)[2, p, np.arange(len(p))])
        assert np.mean(want[2]) - theirs <= 1e-3 or np.mean(want[2]) > 60, (label, got[4], want[4])


# =====================================================================================================================
# 1. accuracy
# =====================================================================================================================
@pytest.mark.parametrize("F", [1, 16, 512])
@pytest.mark.parametrize("S,C", PAIRS)
@pytest.mark.parametrize("long", [False, True])
def test_against_oracle(S, C, F, long):
    """Two items per call (white, AR), T the shortest accepted length or past the first correlation chunk."""
    rng = np.random.default_rng(1000 * S + 100 * C + F + long)
    T = 4096 + 331 if long else max((S * C - 1) * F + 1, 64)      # past a chunk, or the shortest (64 at least)
    items = [make_images(rng, S, C, T, F, coloured=bool(b)) for b in range(2)]
    refs, ests = np.stack([i[0] for i in items]), np.stack([i[1] for i in items])
    for perm in (True, False):
        got = host(images(gpu(refs), gpu(ests), perm, F))
        assert got[0].shape == (2, S) and got[4].dtype == np.int64
        for b in range(2):
            check_against_oracle([g[b] for g in got], refs[b], ests[b], perm, F, f"S={S} C={C} F={F} T={T} b={b}")


@pytest.mark.parametrize("S", [1, 2, 3, 4])
def test_mono_sir_sar_are_bss_eval_sources(S):
    rng = np.random.default_rng(S)
    F, T = 64, 3000
    items = [make_images(rng, S, 1, T, F, coloured=bool(b % 2)) for b in range(4)]
    refs, ests = gpu(np.stack([i[0] for i in items])), gpu(np.stack([i[1] for i in items]))
    sdr, isr, sir, sar, perm = images(refs, ests, True, F)
    with torch.no_grad():
        s = P.bss_eval_sources(refs[..., 0], ests[..., 0], True, F)
    assert torch.equal(perm, s[3])
    for got, want in ((sir, s[1]), (sar, s[2])):
        assert ((got == want) | ((got - want).abs() <= 1e-9)).all(), (got, want)
    # mono input ([S, T]) is read as C = 1
    one = images(refs[0, ..., 0], ests[0, ..., 0], True, F)
    assert_equal(one, [x[0] for x in (sdr, isr, sir, sar, perm)])


# =====================================================================================================================
# 2. edge items
# =====================================================================================================================
def test_zero_channel_is_scored():
    """A source image with one all-zero channel: the projection onto its other channel, as the oracle's lstsq."""
    rng = np.random.default_rng(21)
    S, C, T, F = 2, 2, 3000, 32
    refs, ests = make_images(rng, S, C, T, F, coloured=False)
    refs[1, :, 0] = 0.0
    got = host(images(gpu(refs[None]), gpu(ests[None]), True, F))
    assert all(np.isfinite(g).all() for g in got[:4]) and (got[4] >= 0).all()
    check_against_oracle([g[0] for g in got], refs, ests, True, F, "zero channel")
    # and in the estimate: a zero estimate channel is an ordinary (poor) estimate
    ests[0, :, 1] = 0.0
    got = host(images(gpu(refs[None]), gpu(ests[None]), True, F))
    check_against_oracle([g[0] for g in got], refs, ests, True, F, "zero estimate channel")


def test_silent_and_nonfinite_items_stay_in_place():
    rng = np.random.default_rng(22)
    S, C, T, F, B = 2, 2, 2000, 16, 5
    items = [make_images(rng, S, C, T, F, coloured=False) for _ in range(B)]
    refs, ests = np.stack([i[0] for i in items]), np.stack([i[1] for i in items])
    clean = images(gpu(refs), gpu(ests), True, F)
    refs[1, 0] = 0.0                        # a silent reference image
    ests[2, 1] = 0.0                        # a silent estimate image
    refs[3, 1, 77, 1] = np.nan
    ests[4, 0, 5, 0] = np.inf
    got = images(gpu(refs), gpu(ests), True, F)
    for b in range(1, B):
        assert all(torch.isnan(g[b]).all() for g in got[:4]) and (got[4][b] == -1).all(), b
    assert_equal([g[0] for g in got], [g[0] for g in clean])


# =====================================================================================================================
# 3. repeatability and graphs
# =====================================================================================================================
def test_repeat_and_graph_replay_are_bitwise():
    rng = np.random.default_rng(31)
    S, C, T, F = 2, 2, 8000, 512
    items = [make_images(rng, S, C, T, F, coloured=bool(b % 2)) for b in range(3)]
    refs, ests = gpu(np.stack([i[0] for i in items])), gpu(np.stack([i[1] for i in items]))
    eager = images(refs, ests, True, F)
    assert_equal(images(refs, ests, True, F), eager)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            P.bss_eval_images(refs, ests, True, F)                                      # warm-up
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cap = P.bss_eval_images(refs, ests, True, F)
        g.replay()
        torch.cuda.synchronize()
    assert_equal(cap, eager)


def test_framewise_graph_replay_with_device_lengths():
    rng = np.random.default_rng(32)
    S, C, W, H, F = 1, 2, 1000, 500, 64
    T = W + 149 * H
    items = [make_images(rng, S, C, T, F, coloured=bool(b)) for b in range(2)]
    refs, ests = gpu(np.stack([i[0] for i in items])), gpu(np.stack([i[1] for i in items]))
    lens = torch.tensor([T, T - 7000], device=DEV)
    eager = framewise(refs, ests, W, H, True, F, lengths=lens)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            P.bss_eval_images_framewise(refs, ests, W, H, True, F, lengths=lens)          # warm-up
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cap = P.bss_eval_images_framewise(refs, ests, W, H, True, F, lengths=lens)
        g.replay()
        torch.cuda.synchronize()
    assert_equal(cap, eager)
    assert torch.isnan(eager[0][1, :, -14:]).all() and torch.isfinite(eager[0][1, :, :-14]).all()
    assert (eager[4][1, :, -14:] == -1).all()


# =====================================================================================================================
# 4. framewise
# =====================================================================================================================
@pytest.mark.parametrize("S,C", PAIRS)
def test_framewise_columns_are_their_slices(S, C):
    """Every column bitwise bss_eval_images of its window, made contiguous; 300 windows cross two launch boundaries
    at S C = 1, fewer elsewhere."""
    rng = np.random.default_rng(40 + 10 * S + C)
    F = 32
    W = max(600, (S * C - 1) * F + 1)
    H = W // 2
    n = 300 if S * C == 1 else 7
    T = W + (n - 1) * H + 13
    refs, ests = make_images(rng, S, C, T, F, coloured=True)
    refs, ests = gpu(refs[None]), gpu(ests[None])
    for perm in (False, True):
        got = framewise(refs, ests, W, H, perm, F)
        assert got[0].shape == (1, S, n)
        cols = [0, n - 1] + ([CHUNK - 1, CHUNK, 2 * CHUNK] if n > 2 * CHUNK else list(range(1, n - 1)))
        for k in cols:
            want = images(refs[:, :, k * H:k * H + W].contiguous(), ests[:, :, k * H:k * H + W].contiguous(), perm, F)
            assert_equal([x[..., k] for x in got], want, f"window {k}")


def test_framewise_against_oracle_ragged_and_fallback():
    """Ragged lengths: a recording with its own window count (NaN columns past it), one that falls back to the whole
    item (shorter than W + H), one too short to score, against the oracle's framewise restatement."""
    rng = np.random.default_rng(50)
    S, C, W, H, F = 2, 2, 1600, 800, 16
    T = W + 4 * H
    items = [make_images(rng, S, C, T, F, coloured=bool(b % 2)) for b in range(4)]
    refs, ests = np.stack([i[0] for i in items]), np.stack([i[1] for i in items])
    lengths = [T, W + 2 * H + 5, W + H - 1, 3 * F]
    got = host(framewise(gpu(refs), gpu(ests), W, H, True, F, lengths=torch.tensor(lengths, device=DEV)))
    for b, n in enumerate(lengths):
        want = oracle_framewise(refs[b].astype(np.float64), ests[b].astype(np.float64), W, H, True, F, length=n)
        assert np.array_equal(got[4][b], want[4]), (b, got[4][b], want[4])
        for g, w, name in zip(got[:4], want[:4], ("sdr", "isr", "sir", "sar")):
            check_values(g[b], w, f"item {b} {name}", want[0] if name == "sir" else None)
    assert np.isnan(got[0][3]).all() and np.isnan(got[0][1][:, 3:]).all() and np.isfinite(got[0][2][:, 0]).all()
    # the whole-item fallback without lengths: one column, bss_eval_images of the item
    short = gpu(refs[:, :, :W + H - 1]), gpu(ests[:, :, :W + H - 1])
    assert_equal([x[..., 0] for x in framewise(*short, W, H, True, F)], images(*short, True, F))


def test_framewise_silent_and_nonfinite_windows():
    rng = np.random.default_rng(51)
    S, C, W, H, F = 1, 2, 1000, 1000, 16
    T = 6 * W
    refs, ests = make_images(rng, S, C, T, F, coloured=False)
    refs[0, 1 * W:2 * W] = 0.0
    ests[0, 3 * W + 10, 1] = np.nan
    refs[0, 5 * W + 3, 0] = -np.inf
    got = framewise(gpu(refs[None]), gpu(ests[None]), W, H, True, F)
    bad = [1, 3, 5]
    for k in range(6):
        col = [x[0, :, k] for x in got]
        if k in bad:
            assert all(torch.isnan(c).all() for c in col[:4]) and (col[4] == -1).all(), k
        else:                               # one source: no interference, SIR = +inf
            assert not any(torch.isnan(c).any() for c in col[:4]) and (col[4] == 0).all(), k


def test_hour_of_stereo_within_twice_its_inputs():
    """One hour of two stereo sources at 8 kHz, W = 30 s, H = 15 s, F = 512: 239 windows in two launches.  The
    signals are held as a stereo model returns them, [B, S, C, T], and passed as the [B, S, T, C] views the docstring
    gives, which are scored without a copy."""
    torch.cuda.empty_cache()
    S, C, T, W, H, F = 2, 2, 8000 * 3600, 240000, 120000, 512
    g = torch.Generator(DEV).manual_seed(12)
    rows = torch.randn(1, S, C, T, device=DEV, generator=g)
    est_rows = torch.randn(1, S, C, T, device=DEV, generator=g).mul_(0.3).add_(rows.flip(1))
    inputs = sum(x.numel() * x.element_size() for x in (rows, est_rows))
    refs, ests = rows.transpose(-1, -2), est_rows.transpose(-1, -2)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    got = framewise(refs, ests, W, H, True, F)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print(f"\npeak {peak / 2**20:.0f} MiB for {inputs / 2**20:.0f} MiB of inputs")
    assert peak < 2 * inputs, (peak, inputs)
    assert got[0].shape == (1, S, 239) and torch.isfinite(got[0]).all()
    assert (got[4] == 1 - torch.arange(S, device=DEV)[:, None]).all()          # estimate 1 - j is reference j's
    for k in (0, CHUNK - 1, CHUNK, 238):
        want = images(refs[:, :, k * H:k * H + W], ests[:, :, k * H:k * H + W], True, F)
        assert_equal([x[..., k] for x in got], want, f"window {k}")


def test_refusal_allocates_nothing():
    x = torch.zeros(3, 2000, 2, device=DEV)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(RuntimeError, match="sources \\* channels <= 4"):
        P.bss_eval_images(x, x, filter_length=16)
    with pytest.raises(RuntimeError, match="sources \\* channels <= 4"):
        P.bss_eval_images_framewise(x, x, 500, 250, filter_length=16)
    assert torch.cuda.memory_allocated() == before


def test_stereo_model_output_layout():
    """A stereo model's [B, S*C, T] output viewed as the docstring says equals scoring the images it holds."""
    rng = np.random.default_rng(60)
    S, C, T, F = 2, 2, 4000, 64
    refs, ests = make_images(rng, S, C, T, F, coloured=False)
    out = gpu(ests.transpose(0, 2, 1).reshape(1, S * C, T))                  # [B, S*C, T], channel rows per source
    tgt = gpu(refs.transpose(0, 2, 1).reshape(1, S * C, T))
    got = images(tgt.view(1, S, C, T).transpose(-1, -2), out.view(1, S, C, T).transpose(-1, -2), True, F)
    assert_equal(got, images(gpu(refs[None]), gpu(ests[None]), True, F))
