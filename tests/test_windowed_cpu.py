"""Windowed separation without a GPU: the window plan against the oracle, the window / hop checks, the native
plan query and the C-ABI bindings."""
import os
import re

import numpy as np
import pytest

import windowed_oracle as WO
from sudo_rm_rf_b200 import _native, windowed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = [(32000, 16000), (32000, 16001), (32000, 31999), (4, 2), (5, 3), (2, 1)]


def _lengths(W, H):
    return [1, W - 1, W, W + 1, W + H - 1, W + H, W + H + 1, W + 7 * H, W + 7 * H + 1, 3600 * 8000, 10 * 60 * 16000]


@pytest.mark.parametrize("W,H", SHAPES)
def test_window_plan_matches_oracle(W, H):
    for T in _lengths(W, H):
        K, starts, overlaps = windowed.window_plan(T, W, H)
        assert (K, starts, overlaps) == WO.plan(T, W, H), T
        assert _native.lib().sdr_window_count(T, W, H) == K, T
        if K > 1:
            # every sample is covered, the last window starts below T, no sample lies in three windows
            assert starts[-1] < T <= starts[-1] + W
            assert all(1 <= o <= W - H for o in overlaps)
            assert starts[2] >= W if K > 2 else True


def test_window_plan_edges():
    W, H = 10, 6
    assert WO.plan(W, W, H) == (1, [0], [])
    assert WO.plan(W + 1, W, H) == (2, [0, 6], [4])
    assert WO.plan(W + H - 1, W, H) == (2, [0, 6], [4])
    assert WO.plan(W + H, W, H) == (2, [0, 6], [4])
    assert WO.plan(W + H + 1, W, H) == (3, [0, 6, 12], [4, 4])
    # the last window starts as late as it can while the one before it ends below T: every overlap is W - H long


@pytest.mark.parametrize("window,hop", [(100, 49), (100, 100), (100, 101), (100, 0), (100, -60), (101, 50),
                                        (1, None), (0, None), (100, 50.0), (100.0, 50), (True, None), (100, True)])
def test_window_hop_refused(window, hop):
    with pytest.raises(ValueError):
        windowed.window_hop(window, hop)


@pytest.mark.parametrize("window,hop,expect", [(100, None, 50), (101, None, 51), (2, None, 1), (100, 50, 50),
                                               (100, 99, 99), (101, 51, 51)])
def test_window_hop_accepted(window, hop, expect):
    assert windowed.window_hop(window, hop) == (window, expect)


def test_native_queries_refuse_what_the_merge_cannot_run():
    lib = _native.lib()
    assert lib.sdr_window_count(100, 10, 4) == 0          # H < W/2
    assert lib.sdr_window_count(100, 10, 10) == 0         # H = W
    assert lib.sdr_window_count(0, 10, 5) == 0
    assert lib.sdr_window_count(2 ** 40, 2 ** 24 + 2, 2 ** 23 + 1) == 0
    assert lib.sdr_window_count(2 ** 40, 2 ** 24, 2 ** 23) == 1 + (2 ** 40 - 2 ** 24 + 2 ** 23 - 1) // 2 ** 23
    assert lib.sdr_window_carry_bytes(1, 5, 1, 100) == 0
    assert lib.sdr_window_merge_scratch_bytes(1, 5, 4) == 0
    assert lib.sdr_window_merge_scratch_bytes(2, 3, 4) == (2 * 4 * 3 + 2 * 5 * 3) * 4
    assert lib.sdr_window_carry_bytes(2, 3, 2, 100) == 256 + 2 * 3 * 2 * 100 * 4


def test_window_entries_bind_and_refuse_null_buffers():
    lib = _native.lib()
    for name in ("sdr_window_count", "sdr_window_carry_bytes", "sdr_window_merge_scratch_bytes", "sdr_window_gather",
                 "sdr_window_merge"):
        assert name in _native.EXPORTED_SYMBOLS and hasattr(lib, name)
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(REPO, "include", "sudormrf_b200.h")).read(), flags=re.S)
    assert set(re.findall(r"\b(sdr_[a-z_0-9]+)\s*\(", hdr)) == set(_native.EXPORTED_SYMBOLS)
    # refused before anything is enqueued (no device needed)
    assert lib.sdr_window_gather(None, None, 1, 1, 100, 10, 5, 0, 1, None) == -2
    assert lib.sdr_window_merge(None, None, None, None, 1, 2, 1, 100, 10, 5, 0, 1, None, None) == -2


def test_oracle_fade_sums_to_one_and_matches_endpoints():
    W, H = 9, 5
    j = np.arange(W - H)
    ones = WO.fade(np.ones(W - H, np.float32), np.ones(W - H, np.float32), j, W - H)
    assert np.allclose(ones, 1.0, rtol=0, atol=1e-7)
    prev = WO.fade(np.ones(W - H, np.float32), np.zeros(W - H, np.float32), j, W - H)
    assert np.all(np.diff(prev) < 0) and prev[0] < 1 and prev[-1] > 0


def test_oracle_aligns_permuted_windows():
    rng = np.random.default_rng(0)
    B, S, A, T, W, H = 2, 3, 2, 103, 20, 12
    src = rng.standard_normal((B, S, A, T)).astype(np.float32)
    K, _, _ = WO.plan(T, W, H)
    win = WO.windows(src.reshape(B, S * A, T), W, H).reshape(B, K, S, A, W)
    perms = np.array([[rng.permutation(S) for _ in range(K)] for _ in range(B)])
    est = np.stack([np.stack([win[b, k][np.argsort(perms[b, k])] for k in range(K)]) for b in range(B)])
    pi, _ = WO.align(est, T, W, H)
    out = WO.overlap_add(est, pi, T, W, H).reshape(B, S, A, T)
    first = np.argsort(perms[:, 0], axis=-1)        # output s of window 0 is true source first[b][s]
    for b in range(B):
        assert np.allclose(out[b], src[b][first[b]], rtol=0, atol=1e-6)
