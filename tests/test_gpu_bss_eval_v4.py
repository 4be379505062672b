"""BSS-eval v4 on the GPU (sdr_bss_eval_v4): SDR, ISR, SIR and SAR per window against the fp64 restatement of
museval's v4 (bss_v4_oracle.py) within section 7c's bar, over every (S, C) with S C <= 4, F 1, 16 and 512, hops
shorter than, equal to and longer than the window, a length that is no multiple of the hop, with and without the
permutation; one whole-recording window against bss_eval_images; per-window SIR that is not framewise v3's when the
mix changes halfway; a recording's columns bitwise the same alone and in a ragged batch, across correlation launches,
and on a second call; silent windows and non-finite recordings confined; ten minutes of four stems within 1.5 times
their inputs' memory; CUDA-graph replay with device lengths."""
import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
from bss_v4_oracle import bss_eval_v4 as oracle, track_filters, window_criteria
from test_gpu_bss_eval_images import PAIRS, assert_equal, check_values, gpu, host, make_images

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def v4(refs, ests, W, H, perm=False, F=512, **kw):
    with torch.no_grad():
        return P.bss_eval_v4(refs, ests, W, H, perm, F, **kw)


def check_against_oracle(got, refs, ests, W, H, perm, F, label):
    """Every column within check_values of the oracle's where the permutations agree; where they do not, the oracle
    scores the GPU's assignment within 1e-3 dB of its best mean SIR (or its best lies above 60 dB)."""
    r, e = refs.astype(np.float64), ests.astype(np.float64)
    want = oracle(r, e, W, H, perm, F)
    assert got[0].shape == want[0].shape, (label, got[0].shape, want[0].shape)
    cj = ct = None
    for k in range(want[0].shape[1]):
        g, w = [x[:, k] for x in got], [x[:, k] for x in want]
        if np.array_equal(g[4], w[4]):
            for gi, wi, name in zip(g[:4], w[:4], ("sdr", "isr", "sir", "sar")):
                check_values(gi, wi, f"{label} window {k} {name}", w[0] if name == "sir" else None)
            continue
        assert perm and (g[4] >= 0).all(), (label, k, g[4], w[4])
        if cj is None:
            cj, ct = track_filters(r, e, F)
        crit = window_criteria(r, e, cj, ct, k * H, W)
        theirs = np.mean(crit[2, g[4], np.arange(len(g[4]))])
        assert np.mean(w[2]) - theirs <= 1e-3 or np.mean(w[2]) > 60, (label, k, g[4], w[4])


# =====================================================================================================================
# 1. accuracy
# =====================================================================================================================
@pytest.mark.parametrize("F", [1, 16, 512])
@pytest.mark.parametrize("S,C", PAIRS)
def test_against_oracle(S, C, F):
    """One recording past the first 8192-sample correlation chunk, its length no multiple of any hop; H < W (with and
    without the permutation), H = W and H > W."""
    rng = np.random.default_rng(2000 * S + 100 * C + F)
    n = 8192 + 3001
    refs, ests = make_images(rng, S, C, n, F, coloured=bool(F % 2))
    for W, H, perm in ((2000, 1500, False), (2000, 1500, True), (2000, 2000, False), (1500, 2500, True)):
        got = host(v4(gpu(refs), gpu(ests), W, H, perm, F))
        assert got[4].dtype == np.int64 and got[0].shape == (S, (n - W) // H + 1)
        check_against_oracle(got, refs, ests, W, H, perm, F, f"S={S} C={C} F={F} W={W} H={H} perm={perm}")


@pytest.mark.parametrize("S,C", PAIRS)
def test_one_window_is_bss_eval_images(S, C):
    """W = T: one window, the whole recording, whose filters are the window's projection: bss_eval_images."""
    rng = np.random.default_rng(70 + 10 * S + C)
    F, T = 64, 20000
    items = [make_images(rng, S, C, T, F, coloured=bool(b)) for b in range(2)]
    refs, ests = gpu(np.stack([i[0] for i in items])), gpu(np.stack([i[1] for i in items]))
    got = v4(refs, ests, T, T, True, F)
    with torch.no_grad():
        want = P.bss_eval_images(refs, ests, True, F)
    assert torch.equal(got[4][..., 0], want[4])
    for g, w in zip(got[:4], want[:4]):
        assert ((g[..., 0] == w) | ((g[..., 0] - w).abs() <= 1e-6)).all(), (g[..., 0], w)


def test_whole_track_filters_are_not_framewise_v3():
    """The interference gain changes halfway through: framewise v3 solves it per window, v4 applies the whole track's
    filters, so their per-window SIR differs by more than 1 dB in every window."""
    rng = np.random.default_rng(80)
    S, T, W, F = 2, 8 * 8000, 8000, 64
    refs = rng.standard_normal((S, T))
    gain = np.where(np.arange(T) < T // 2, 0.05, 0.5)
    ests = np.stack([refs[0] + gain * refs[1], refs[1] + gain * refs[0]]) + 0.01 * rng.standard_normal((S, T))
    r, e = gpu(refs[..., None].astype(np.float32)), gpu(ests[..., None].astype(np.float32))
    got = v4(r, e, W, W, False, F)
    with torch.no_grad():
        v3 = P.bss_eval_images_framewise(r, e, W, W, False, F)
    assert got[2].shape == v3[2].shape == (S, 8)
    assert ((got[2] - v3[2]).abs() > 1.0).all(), (got[2], v3[2])


# =====================================================================================================================
# 2. batches, reproducibility and isolation
# =====================================================================================================================
def test_ragged_batch_is_bitwise_each_recording_alone():
    """Three recordings of two mono sources over 1.6 M samples: the batch folds its correlations over two launches,
    each recording alone over one; the columns are the same bits, a second call too, and NaN past each count."""
    g = torch.Generator(DEV).manual_seed(3)
    S, T, W, H, F = 2, 1_600_000, 44100, 33075, 64
    refs = torch.randn(3, S, T, 1, device=DEV, generator=g)
    ests = 0.3 * torch.randn(3, S, T, 1, device=DEV, generator=g) + refs.flip(1) * 0.2 + refs
    lens = torch.tensor([T, T - 5000, T - 412345], device=DEV)
    batch = v4(refs, ests, W, H, True, F, lengths=lens)
    assert_equal(v4(refs, ests, W, H, True, F, lengths=lens), batch)
    for b, n in enumerate(lens.tolist()):
        alone = v4(refs[b, :, :n].contiguous(), ests[b, :, :n].contiguous(), W, H, True, F)
        k = (n - W) // H + 1
        assert_equal([x[b][..., :k] for x in batch], alone, f"recording {b}")
        assert torch.isnan(batch[0][b][..., k:]).all() and (batch[4][b][..., k:] == -1).all()
        assert torch.isfinite(alone[0]).all()


def test_silent_windows_and_nonfinite_recordings_are_confined():
    rng = np.random.default_rng(90)
    S, C, W, H, F = 2, 2, 4000, 4000, 32
    T = 6 * W + 123
    items = [make_images(rng, S, C, T, F, coloured=False) for _ in range(4)]
    refs, ests = np.stack([i[0] for i in items]), np.stack([i[1] for i in items])
    clean = host(v4(gpu(refs), gpu(ests), W, H, True, F))
    refs[1, 1, 2 * W:3 * W] = 0.0                       # recording 1: a silent reference image in window 2
    ests[2, 0, 4 * W:5 * W] = 0.0                       # recording 2: a silent estimate image in window 4
    refs[3, 0, T - 3, 1] = np.nan                       # recording 3: a NaN past its last window
    got = host(v4(gpu(refs), gpu(ests), W, H, True, F))
    for x, y in zip(got, clean):
        assert np.array_equal(x[0], y[0], equal_nan=True)
    assert all(np.isnan(x[3]).all() for x in got[:4]) and (got[4][3] == -1).all()
    for b, bad in ((1, 2), (2, 4)):
        assert all(np.isnan(x[b][:, bad]).all() for x in got[:4]) and (got[4][b][:, bad] == -1).all()
        keep = [k for k in range(6) if k != bad]
        assert all(np.isfinite(x[b][:, keep]).all() for x in got[:4]) and (got[4][b][:, keep] >= 0).all()
    # the edited recording's own filters and windows, against the oracle
    check_against_oracle([x[1] for x in got], refs[1], ests[1], W, H, True, F, "silent window")
    ests[0, 1, 7, 0] = np.inf                           # an infinity: every window of that recording only
    got = host(v4(gpu(refs), gpu(ests), W, H, True, F))
    assert np.isnan(got[0][0]).all() and (got[4][0] == -1).all() and np.isfinite(got[0][2][:, :4]).all()


# =====================================================================================================================
# 3. scale and graphs
# =====================================================================================================================
def test_ten_minutes_of_four_stems_within_one_and_a_half_inputs():
    torch.cuda.empty_cache()
    S, T, F = 4, 44100 * 600, 512
    g = torch.Generator(DEV).manual_seed(12)
    refs = torch.randn(S, T, device=DEV, generator=g)
    ests = torch.randn(S, T, device=DEV, generator=g).mul_(0.3).add_(refs)
    inputs = sum(x.numel() * x.element_size() for x in (refs, ests))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    got = v4(refs, ests, 44100, 44100, False, F)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print(f"\npeak {peak / 2**20:.0f} MiB for {inputs / 2**20:.0f} MiB of inputs")
    assert peak < 1.5 * inputs, (peak, inputs)
    assert got[0].shape == (S, 600) and all(torch.isfinite(x).all() for x in got[:4])
    # estimate = reference + 0.3 noise: SDR near 10.5 dB in every window
    assert ((got[0] - 10.46).abs() < 0.5).all(), got[0].min()


def test_graph_replay_with_device_lengths():
    rng = np.random.default_rng(95)
    S, C, W, H, F = 1, 2, 3000, 2000, 64
    T = 40000
    items = [make_images(rng, S, C, T, F, coloured=bool(b)) for b in range(2)]
    refs, ests = gpu(np.stack([i[0] for i in items])), gpu(np.stack([i[1] for i in items]))
    lens = torch.tensor([T, T - 9000], device=DEV)
    eager = v4(refs, ests, W, H, True, F, lengths=lens)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            P.bss_eval_v4(refs, ests, W, H, True, F, lengths=lens)                       # warm-up
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap = P.bss_eval_v4(refs, ests, W, H, True, F, lengths=lens)
        graph.replay()
        torch.cuda.synchronize()
    assert_equal(cap, eager)
    k = (T - 9000 - W) // H + 1
    assert torch.isfinite(eager[0][1, :, :k]).all() and torch.isnan(eager[0][1, :, k:]).all()
