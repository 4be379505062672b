"""STOI without a GPU: properties of the fp64 restatement in stoi_oracle.py (and, where pystoi is installed, agreement
with it), the C-ABI symbols and the scratch query's refusals, and the Python entry's refusals."""
import math

import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
import stoi_oracle as O
import stoi_rates

SYMBOLS = ("sdr_stoi_scratch_bytes", "sdr_stoi")


def noise(n, seed=0):
    return np.random.default_rng(seed).standard_normal(n)


@pytest.mark.parametrize("fs", [8000, 10000, 16000])
def test_identity_is_one(fs):
    x = noise(4 * fs, fs)
    assert abs(O.stoi(x, x, fs) - 1.0) <= 1e-12


def test_positive_scaling_changes_nothing():
    rng = np.random.default_rng(1)
    x = rng.standard_normal(32000)
    y = x + 0.7 * rng.standard_normal(32000)
    d = O.stoi(x, y, 8000)
    assert 0.2 < d < 0.99
    for a, b in ((3.0, 1.0), (1.0, 0.01), (1e-3, 250.0)):
        assert abs(O.stoi(a * x, b * y, 8000) - d) <= 1e-12, (a, b)


def test_band_table():
    assert O.band_edges() == [(7, 9), (9, 11), (11, 14), (14, 17), (17, 22), (22, 27), (27, 34), (34, 43), (43, 55),
                              (55, 69), (69, 87), (87, 109), (109, 138), (138, 174), (174, 219)]


@pytest.mark.parametrize("fs,taps", [(8000, 365), (16000, 581), (48000, 1741), (44100, 31947), (22050, 31947)])
def test_filter_lengths_and_output_length(fs, taps):
    g = math.gcd(O.FS, fs)
    p, q = O.FS // g, fs // g
    h = O.resample_window_oct(p, q)
    assert len(h) == taps
    for n in (1, 255, 1000, 4 * fs + 3):
        assert len(O.resample_oct(noise(n), p, q)) == -(-n * p // q) == O.resampled_length(n, fs)


def test_thirty_frame_boundary():
    """White noise at 8 kHz: 3276 samples give 29 spectral frames and 1e-5, 3277 give 30 and a real value; a 4 s item
    has 311 analysis frames."""
    x = noise(3277, 2)
    assert O.spectral_frames(x[:3276], 8000) == 29 and O.stoi(x[:3276], x[:3276], 8000) == 1e-5
    assert O.spectral_frames(x, 8000) == 30 and abs(O.stoi(x, x, 8000) - 1.0) <= 1e-12
    assert O.spectral_frames(noise(32000, 3), 8000) == 310          # 311 analysis frames, all kept


def test_silent_rows_give_zero():
    x = noise(16000, 4)
    assert O.stoi(np.zeros(16000), x, 8000) == 0.0
    assert O.stoi(x, np.zeros(16000), 8000) == 0.0
    assert O.stoi(x[:200], x[:200], 8000) == 1e-5                      # no frame at all (pystoi raises)


def test_against_pystoi():
    pystoi = pytest.importorskip("pystoi")
    rng = np.random.default_rng(5)
    for fs in (8000, 10000, 16000, 44100):
        x = rng.standard_normal(3 * fs)
        x[fs // 2:fs] *= 1e-3
        y = x + 0.5 * rng.standard_normal(3 * fs)
        assert abs(O.stoi(x, y, fs) - pystoi.stoi(x, y, fs, extended=False)) <= 1e-9, fs


def test_symbols_bind_and_scratch_limits():
    lib = N.lib()
    for name in SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
    assert lib.sdr_stoi_scratch_bytes(4, 2, 32000, 8000) > 0
    for B, S, T in ((0, 2, 100), (2, 0, 100), (2, 2, 0), (-1, 2, 100), (2, -1, 100), (2, 2, -5)):
        assert lib.sdr_stoi_scratch_bytes(B, S, T, 8000) == 0, (B, S, T)
    assert lib.sdr_stoi_scratch_bytes(1, 1, 100, 999) == 0 and lib.sdr_stoi_scratch_bytes(1, 1, 100, 1000) > 0
    assert lib.sdr_stoi_scratch_bytes(1, 1, 100, 0) == 0 and lib.sdr_stoi_scratch_bytes(1, 1, 100, -8000) == 0
    # the ratio cap: 44.1 kHz reduces to 100 / 441, 35.36 kHz to 125 / 442, 44.101 kHz to 10000 / 44101
    assert lib.sdr_stoi_scratch_bytes(1, 1, 1000, 44100) > 0 and lib.sdr_stoi_scratch_bytes(1, 1, 1000, 22050) > 0
    assert lib.sdr_stoi_scratch_bytes(1, 1, 1000, 35360) == 0
    assert lib.sdr_stoi_scratch_bytes(1, 1, 1000, 44101) == 0 and lib.sdr_stoi_scratch_bytes(1, 1, 1000, 9999) == 0
    # null buffers are refused before anything is enqueued
    assert lib.sdr_stoi(None, None, None, None, None, None, 1, 2, 100, 8000, None, None) == -2
    x = 8                  # any non-null, 8-byte aligned address: these calls return before reading a buffer
    assert lib.sdr_stoi(x, x, x, None, x, None, 1, 2, 100, 8000, x, None) == -2             # mixture, no mix_stoi
    assert lib.sdr_stoi(x, x, None, None, x, None, 1, 2, 100, 8000, 12, None) == -2           # misaligned scratch
    assert lib.sdr_stoi(x, x, None, None, x, None, 1, 2, 100, 35360, x, None) == -5           # past the cap


def test_scratch_query_accepts_exactly_the_supported_rates():
    """For every integer fs in [1, 4.5 MHz]: the scratch query is non-zero exactly where fs >= 1000 and 10000 / fs
    reduces to p / q with max(p, q) <= 441 (3918 rates, from 1000 Hz to 4.41 MHz)."""
    lib = N.lib()
    want = set(stoi_rates.accepted(1, 4_500_000).tolist())
    assert len(want) == 3918
    got = {fs for fs in range(1, 4_500_001) if lib.sdr_stoi_scratch_bytes(1, 1, 1000, fs) > 0}
    assert got == want, (sorted(got - want)[:10], sorted(want - got)[:10])


def test_scratch_query_size_limits():
    """B S up to 715,827,882 = (2^31 - 1) / 3 (the 3 B S tob rows), T up to 2^40."""
    lib = N.lib()
    top = (2 ** 31 - 1) // 3
    for B, S in ((top, 1), (1, top), (top // 2, 2)):
        assert lib.sdr_stoi_scratch_bytes(B, S, 1000, 8000) > 0, (B, S)
    for B, S in ((top + 1, 1), (1, top + 1), (top // 2 + 1, 2)):
        assert lib.sdr_stoi_scratch_bytes(B, S, 1000, 8000) == 0, (B, S)
    for fs in (1000, 8000, 10000, 44100):
        assert lib.sdr_stoi_scratch_bytes(1, 1, 2 ** 40, fs) > 0, fs
        assert lib.sdr_stoi_scratch_bytes(1, 1, 2 ** 40 + 1, fs) == 0, fs


def test_refusals():
    x = torch.zeros(2, 1000)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.stoi(x, x, 8000)
    with pytest.raises(RuntimeError, match="shape"):
        P.stoi(x, torch.zeros(3, 1000), 8000)
    g = torch.zeros(2, 1000, requires_grad=True)
    with pytest.raises(RuntimeError, match="CUDA|no autograd"):
        P.stoi(g, x, 8000)
    with pytest.raises(NotImplementedError, match="ESTOI"):
        P.stoi(x, x, 8000, extended=True)
    assert P.stoi is P.stoi_metric.stoi
