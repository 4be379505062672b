"""Every sampling rate sdr_stoi accepts, one seeded item per rate, and that item's scores by the fp64 restatement.

test_gpu_stoi_space.py scores the rates' oracle values in spawned worker processes; this module imports numpy, scipy
and stoi_oracle only, so that those workers start quickly and regenerate the same items from their seeds."""
import math

import numpy as np
from scipy.signal import lfilter

import stoi_oracle as O

MAX_RATIO = 441                 # largest reduced max(p, q) of 10000 / fs


def ratio(fs):
    """(p, q): 10000 / fs reduced."""
    g = math.gcd(O.FS, fs)
    return O.FS // g, fs // g


def accepted(lo=1, hi=4_500_000):
    """Every integer fs in [lo, hi] that the entry accepts: fs >= 1000 and max(p, q) <= 441."""
    fs = np.arange(max(lo, 1), hi + 1, dtype=np.int64)
    g = np.gcd(O.FS, fs)
    ok = (fs >= 1000) & (np.maximum(O.FS // g, fs // g) <= MAX_RATIO)
    return fs[ok]


def item(i, fs):
    """Item i of the sweep at fs: (clean, estimate, mixture, n), fp32 rows of T samples, about 6000 samples after
    resampling.  White references at even i, AR(0.9) at odd i; a noisy estimate (SNR -5..20 dB) and a mixture (the
    reference plus noise at 0..10 dB).  In one case in ten the item is scored over n < T samples (a random length in
    [0.85 T, T)), so that its resampled tail ends at a random phase of the filter; else n = T."""
    rng = np.random.default_rng([i, fs])
    p, q = ratio(fs)
    T = -(-int(rng.integers(5500, 6500)) * q // p)
    x = rng.standard_normal(T)
    if i % 2:
        x = lfilter([1.0], [1.0, -0.9], x)
    s = np.std(x)
    y = x + s * 10 ** (-rng.uniform(-5, 20) / 20) * rng.standard_normal(T)
    mix = x + s * 10 ** (-rng.uniform(0, 10) / 20) * rng.standard_normal(T)
    n = int(rng.integers(T * 85 // 100, T)) if i % 10 == 0 else T
    return x.astype(np.float32), y.astype(np.float32), mix.astype(np.float32), n


def scores(i, fs):
    """(stoi of the estimate, stoi of the mixture, kept frames, mask margin in dB) of item(i, fs) by the restatement."""
    x, y, mix, n = item(i, fs)
    (d, m), kept, margin = O.score(x[:n], [y[:n], mix[:n]], fs)
    return d, m, len(kept), margin
