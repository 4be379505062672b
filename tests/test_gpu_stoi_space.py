"""STOI on the GPU across its whole input space, against the fp64 restatement in stoi_oracle.py within 1e-9: every
sampling rate the entry accepts, the resampler's tail at every phase of the long filters, the silent-frame mask at the
kept-frame counts that decide between 1e-5 and a value, the mask compaction's 512-frame tiles, references with very
different masks under one mixture, the grid-stride loops of the resampling and spectra kernels past their grid
limits, amplitudes from fp32 denormals to 3e38, and non-finite samples at the first, the last and the first unscored
sample.

Every row compared with the oracle has its silent-frame mask at least MIN_MARGIN dB from the 40 dB threshold (asserted
with stoi_oracle.mask_margin): a frame energy the GPU rounds differently then cannot flip a frame, so a difference
above 1e-9 is a kernel error and not a legitimate rounding flip at the threshold."""
import multiprocessing as mp
import os
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
import stoi_oracle as O
import stoi_rates
from test_gpu_stoi import DEV, TOL, batch, gpu

pytestmark = pytest.mark.gpu
MIN_MARGIN = 1e-6           # dB
HOP = O.N_FRAME // 2
WORST = {}                  # case group -> (largest |GPU - oracle|, where)

# sdr_stoi's grid limits (stoi.cu): resampling chunks of 256 samples in grid.x and rows in grid.y, at most 65535
# each; spectra work items (a warp group of 4 spectral frames of one tob row) in at most 2^20 CTAs
GRID_X = GRID_Y = 65535
SPECTRA_CTAS = 1 << 20


@pytest.fixture(autouse=True)
def device_memory(request):
    """Frees the cached blocks around each test (the batch past the grid limits takes about 10 GB) and prints its
    peak."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    print(f"\n{request.node.name}: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()


def plan(B, S, T, fs, mix):
    """sdr_stoi's geometry: (Tn, M, resampling chunks, resampling rows, spectra work items)."""
    p, q = stoi_rates.ratio(fs)
    Tn = -(-T * p // q)
    F0 = -(-(Tn - O.N_FRAME) // HOP) if Tn > O.N_FRAME else 0
    M = max(F0 - 1, 0)
    R = B * S
    return Tn, M, -(-Tn // 256), 2 * R + (B if mix else 0), (3 if mix else 2) * R * ((M + 3) // 4)


def compare(group, got, want, label):
    """got within TOL of want, NaN where want is NaN; the worst error recorded under `group`."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (label, got, want)
    ok = ~np.isnan(want)
    if ok.any():
        err = float(np.max(np.abs(got - want)[ok]))
        assert err <= TOL, (label, err, got, want)
        if err > WORST.get(group, (-1.0, ""))[0]:
            WORST[group] = (err, label)


def margin_ok(x, fs, label, K=None):
    """The oracle's kept frames of clean row x; asserts the margin and, when given, the kept count K."""
    kept, margin = O.mask_margin(np.asarray(x, np.float64), fs)
    assert margin >= MIN_MARGIN, (label, margin)
    if K is not None:
        assert len(kept) == K, (label, len(kept), K)
    return kept


def score_all(group, x, y, fs, mix=None, lengths=None, label=""):
    """GPU scores of [B, S, T] x and y (and the mixture) against the oracle, every reference's margin asserted."""
    B, S, T = x.shape
    got = gpu(x, y, fs, mix, lengths)
    d = np.zeros((B, S))
    m = np.zeros((B, S))
    for b in range(B):
        n = T if lengths is None else lengths[b]
        for j in range(S):
            ys = [y[b, j, :n]] + ([] if mix is None else [mix[b, :n]])
            w, kept, margin = O.score(x[b, j, :n], ys, fs)
            assert margin >= MIN_MARGIN, (label, b, j, margin)
            d[b, j] = w[0]
            if mix is not None:
                m[b, j] = w[1]
    if mix is None:
        compare(group, got, d, label)
        return got
    compare(group, got[0], d, label + " estimate")
    compare(group, got[1], m, label + " mixture")
    return got


def noise_blocks(rng, levels, tail=1):
    """A 10 kHz row of 128-sample blocks of white noise at levels[i] dB (None: silence), then `tail` silent samples.
    Frame f (samples 128 f .. 128 f + 255) covers blocks f and f + 1, so with tail = 1 the row has len(levels) - 1
    frames: block 0 is read by frame 0 only and the last block by the last frame only.  A frame that covers a 0 dB block
    lies within about 3 dB of a frame of two; one that covers only blocks at -60 dB or silence lies more than 50 dB
    below, and silence alone is at 20 log10(eps)."""
    x = np.zeros(len(levels) * HOP + tail)
    for i, lv in enumerate(levels):
        if lv is not None:
            x[i * HOP:(i + 1) * HOP] = 10 ** (lv / 20) * rng.standard_normal(HOP)
    return x


def kept_run(nb, first, K):
    """Levels of nb blocks (tail 1) that keep exactly frames first .. first + K - 1: blocks first + 1 .. first + K - 1
    at 0 dB (block first too when first = 0, so that frame 0 has two loud blocks)."""
    lv = [None] * nb
    for i in range(first + (first > 0), first + K):
        lv[i] = 0.0
    return lv


def burst(rng, nb, f):
    """A 10 kHz row of nb blocks that is silent but for 4 samples at the centre of frame f (window 0.9999): the two
    neighbouring frames read them at window values below 6e-4, more than 60 dB down, so exactly frame f is kept."""
    x = np.zeros(nb * HOP + 1)
    x[f * HOP + 126:f * HOP + 130] = rng.standard_normal(4) + 3.0
    return x


def random_levels(rng, nb, count=None, fixed=None):
    """nb random block levels in {0 dB, -60 dB, silence}; `fixed` {block: loud?} pinned.  With count, loud and quiet
    blocks are toggled until exactly `count` frames are kept (frame f kept iff block f or f + 1 is loud)."""
    fixed = fixed or {}
    loud = rng.random(nb) < 0.4
    for i, v in fixed.items():
        loud[i] = v
    kept = lambda: int(np.sum(loud[:-1] | loud[1:]))   # noqa: E731
    free = [i for i in range(nb) if i not in fixed]
    while count is not None and kept() != count:
        i = free[int(rng.integers(len(free)))]
        if (kept() < count) != loud[i]:
            loud[i] = not loud[i]
    quiet = rng.random(nb) < 0.5
    return [0.0 if loud[i] else (-60.0 if quiet[i] else None) for i in range(nb)]


def estimates(rng, x):
    """Noisy estimates of every row of x (the noise also where x is silent) and a mixture of each item's rows."""
    s = np.maximum(np.std(x, axis=-1, keepdims=True), 1e-3)
    y = x + s * rng.uniform(0.1, 1.0, x.shape[:-1] + (1,)) * rng.standard_normal(x.shape)
    mix = x.sum(1) + 0.3 * np.std(x.sum(1), axis=-1, keepdims=True) * rng.standard_normal((x.shape[0], x.shape[-1]))
    return y.astype(np.float32), mix.astype(np.float32)


# =====================================================================================================================
# 1. every accepted rate
# =====================================================================================================================
def test_every_accepted_rate():
    """All 3918 accepted rates, one item each (stoi_rates.item: about 6000 samples after resampling, a random scored
    length in one case in ten), its estimate and its mixture against the oracle, which runs in spawned worker
    processes while the GPU scores the items."""
    rates = stoi_rates.accepted()
    assert len(rates) == 3918 and rates[0] == 1000 and rates[-1] == 4_410_000
    t0 = time.time()
    workers = max(1, min(32, len(os.sched_getaffinity(0)) - 1))
    with ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as pool:
        want = pool.map(stoi_rates.scores, range(len(rates)), [int(f) for f in rates], chunksize=16)
        got = []
        t = lambda a: torch.from_numpy(a).to(DEV).view(1, 1, -1)   # noqa: E731
        with torch.no_grad():
            for i, fs in enumerate(rates):
                x, y, mix, n = stoi_rates.item(i, int(fs))
                d, m = P.stoi(t(x), t(y), int(fs), mixture=t(mix), lengths=None if n == len(x) else [n])
                got.append(torch.stack([d.view(()), m.view(())]))
        got = torch.stack(got).cpu().numpy()
        want = list(want)
    print(f"\n{len(rates)} rates in {time.time() - t0:.1f} s with {workers} oracle workers")
    w = np.array([(d, m) for d, m, _, _ in want])
    K = np.array([k for _, _, k, _ in want])
    margins = np.array([mg for _, _, _, mg in want])
    assert np.all(K > 31), rates[K <= 31]                                 # M = K - 1 > 30: every item gets a value
    assert np.all(margins >= MIN_MARGIN), rates[margins < MIN_MARGIN]
    bad = np.flatnonzero(np.any(np.abs(got - w) > TOL, axis=1) | np.any(np.isnan(got), axis=1))
    assert bad.size == 0, [(int(rates[i]), got[i], w[i]) for i in bad[:10]]
    compare("every rate", got, w, "every rate")


# =====================================================================================================================
# 2. the resampler's tail
# =====================================================================================================================
@pytest.mark.parametrize("fs", [11025, 22050, 44100, 1000])
def test_resampling_tails(fs):
    """Per-item lengths at residues 0, 1, q / 2 and q - 1 mod q (for 1000 Hz, q = 1: residues 0, 1, 5, 9 mod p = 10),
    so that the last output sample meets the filter at each phase: against the oracle, and bitwise against each item
    scored alone at its length."""
    rng = np.random.default_rng(fs + 2)
    p, q = stoi_rates.ratio(fs)
    m = q if q > 1 else p
    base = (-(-5000 * q // p) // m + 1) * m
    lens = [base + r for r in (0, 1, m // 2, m - 1)]
    T = max(lens) + 3
    x, y, mix = batch(rng, 4, 2, T, fs, kinds=("white", "ar"), hows=("noisy", "filtered"))
    got = score_all("resampling tails", x, y, fs, mix, lens, f"fs {fs}")
    for b, n in enumerate(lens):
        a = gpu(np.ascontiguousarray(x[b:b + 1, :, :n]), np.ascontiguousarray(y[b:b + 1, :, :n]), fs,
                np.ascontiguousarray(mix[b:b + 1, :n]))
        assert np.array_equal(a[0][0], got[0][b]) and np.array_equal(a[1][0], got[1][b]), (fs, n)


# =====================================================================================================================
# 3. the kept-frame count
# =====================================================================================================================
def test_mask_count_edges():
    """At 10 kHz, noise blocks in silence so that each frame is kept or dropped by tens of dB: kept counts K = 1, 2,
    30 (M = 29: exactly 1e-5), 31 and 32 (M = 30, 31: values), and the loudest frame first or last.  Every K is the
    oracle's, asserted."""
    rng = np.random.default_rng(31)
    nb = 64
    rows = [(burst(rng, nb, 20), 1), (noise_blocks(rng, kept_run(nb, 10, 2)), 2)]
    rows += [(noise_blocks(rng, kept_run(nb, 7, k)), k) for k in (30, 31, 32)]
    first = kept_run(nb, 0, 31)
    first[0] = 6.0                                          # block 0: only frame 0 reads it
    last = kept_run(nb, nb - 32, 31)
    last[-1] = 6.0                                          # the last block: only the last frame (nb - 2) reads it
    rows += [(noise_blocks(rng, first), 31), (noise_blocks(rng, last), 31)]
    x = np.stack([r[0] for r in rows])[:, None].astype(np.float32)
    for i, (_, k) in enumerate(rows):
        margin_ok(x[i, 0], 10000, f"row {i}", k)
    assert np.argmax(O.frame_energies(x[5, 0])) == 0 and np.argmax(O.frame_energies(x[6, 0])) == nb - 2
    y, mix = estimates(rng, x)
    d, m = score_all("mask counts", x, y, 10000, mix, label="10 kHz")
    assert np.all(d[:3] == 1e-5) and np.all(m[:3] == 1e-5) and np.all(d[3:] != 1e-5)
    assert np.all(np.isfinite(d)) and np.all(np.isfinite(m))


def loud_run(rng, T, start, length):
    x = np.zeros(T)
    x[start:start + length] = rng.standard_normal(length)
    return x


@pytest.mark.parametrize("K", [30, 31])
def test_mask_count_edges_resampled(K):
    """K = 30 / 31 at 44.1 kHz, through the resampler: a loud run in silence, its length searched until the oracle
    keeps K frames with a margin of at least 0.01 dB (the filter's ringing puts frames near the run's ends at any
    level)."""
    fs, T = 44100, 44100
    rng = np.random.default_rng(K)
    seed = int(rng.integers(1 << 30))
    for length in range(int((K - 2) * HOP * 4.41), int((K + 2) * HOP * 4.41), 7):
        x = loud_run(np.random.default_rng(seed), T, 9000, length)
        kept, margin = O.mask_margin(x, fs)
        if len(kept) == K and margin >= 0.01:
            break
    else:
        pytest.fail(f"no run length keeps {K} frames")
    x = x.astype(np.float32)[None, None]
    margin_ok(x[0, 0], fs, f"K {K}", K)
    y, mix = estimates(rng, x)
    d, m = score_all("mask counts", x, y, fs, mix, label=f"44.1 kHz K {K}")
    assert (d[0, 0] == 1e-5) == (K == 30)


# =====================================================================================================================
# 4. the compaction's tiles
# =====================================================================================================================
def test_compaction_tile_edges():
    """Items of 1040 blocks at 10 kHz (13.3 s, F0 = 1039 frames: three 512-frame tiles of the mask kernel's scan),
    random block levels in {0 dB, -60 dB, silence}.  Item 0: frame 511 kept and 512 dropped, 1023 dropped and 1024
    kept.  Items 1 and 2: exactly 512 and 513 frames kept."""
    rng = np.random.default_rng(512)
    nb = 1040
    lv0 = random_levels(rng, nb, fixed={511: True, 512: False, 513: False, 1023: False, 1024: False, 1025: True})
    x = np.stack([noise_blocks(rng, lv) for lv in (lv0, random_levels(rng, nb, 512), random_levels(rng, nb, 513))])
    x = x[:, None].astype(np.float32)
    k0 = set(margin_ok(x[0, 0], 10000, "item 0").tolist())
    assert 511 in k0 and 512 not in k0 and 1023 not in k0 and 1024 in k0
    margin_ok(x[1, 0], 10000, "item 1", 512)
    margin_ok(x[2, 0], 10000, "item 2", 513)
    y, mix = estimates(rng, x)
    score_all("compaction tiles", x, y, 10000, mix, label="tiles")


# =====================================================================================================================
# 5. distinct masks under one mixture
# =====================================================================================================================
def test_distinct_masks_under_one_mixture():
    """S = 4 references in one item keeping K = 1, 31, 513 and all 599 frames, with the mixture of all four: the
    mixture is analysed once per reference, under that reference's mask.  Item 1 holds the same references in reverse
    order, the same estimates and the same mixture (its mixture row is 2R + 1): its scores are item 0's reversed,
    bitwise."""
    rng = np.random.default_rng(4)
    nb = 600
    refs = [burst(rng, nb, 300), noise_blocks(rng, kept_run(nb, 200, 31)),
            noise_blocks(rng, random_levels(rng, nb, 513)), rng.standard_normal(nb * HOP + 1)]
    x = np.stack([np.stack(refs), np.stack(refs[::-1])]).astype(np.float32)
    for j, k in enumerate((1, 31, 513, nb - 1)):
        margin_ok(x[0, j], 10000, f"reference {j}", k)
    y, mix = estimates(rng, x)
    y[1] = y[0, ::-1]
    mix[1] = mix[0]
    d, m = score_all("distinct masks", x, y, 10000, mix, label="S 4")
    assert d[0, 0] == 1e-5 and np.array_equal(d[0], d[1, ::-1]) and np.array_equal(m[0], m[1, ::-1])


# =====================================================================================================================
# 6. the grid-stride loops
# =====================================================================================================================
def test_resample_sample_loop_past_grid_x():
    """One 30-minute item at 8 kHz: 18,000,000 resampled samples, 70,313 chunks of 256 > 65535, so the resampling
    kernel's sample loop wraps; against the oracle."""
    fs, T = 8000, 30 * 60 * 8000
    Tn, _, chunks, _, _ = plan(1, 1, T, fs, True)
    print(f"\nTn = {Tn}, resampling chunks {chunks} > {GRID_X}")
    assert Tn > GRID_X * 256 and chunks > GRID_X
    rng = np.random.default_rng(1800)
    x, y, mix = batch(rng, 1, 1, T, fs, kinds=("speechlike",), hows=("noisy",))
    score_all("grid-stride loops", x, y, fs, mix, label="30 min")


def test_rows_and_spectra_past_grid_limits():
    """B = 16384 items of 2 x 8000 samples at 8 kHz with the mixture: 81,920 resampling rows > 65535 (the row loop
    wraps at the last estimate row and every mixture row) and 1,867,776 spectra work items > 2^20 (the loop wraps from
    the estimate rows of item 11210 on).  Every item bitwise against the same items in sub-batches of 1024; the rows
    past each limit against the oracle."""
    fs, B, S, T = 8000, 16384, 2, 8000
    R = B * S
    Tn, M, _, rows, work = plan(B, S, T, fs, True)
    groups = (M + 3) // 4
    first_wrapped = (SPECTRA_CTAS // groups - R) // S            # the item of the first estimate row past 2^20
    print(f"\nresampling rows {rows} > {GRID_Y}, spectra work items {work} > {SPECTRA_CTAS}, "
          f"estimate rows past it from item {first_wrapped}")
    assert rows > GRID_Y and 2 * R - 1 >= GRID_Y and work > SPECTRA_CTAS and first_wrapped == 11210
    g = torch.Generator(device=DEV).manual_seed(16384)
    x = torch.randn(B, S, T, device=DEV, generator=g)
    x.mul_(torch.rand(B, S, 1, device=DEV, generator=g) + 0.1)
    y = x + torch.randn(B, S, T, device=DEV, generator=g) * torch.logspace(-1.5, 0.5, B, device=DEV).view(B, 1, 1)
    mix = x.sum(1) + 0.3 * torch.randn(B, T, device=DEV, generator=g)
    with torch.no_grad():
        d, m = P.stoi(x, y, fs, mixture=mix)
        parts = [P.stoi(x[a:a + 1024], y[a:a + 1024], fs, mixture=mix[a:a + 1024]) for a in range(0, B, 1024)]
    assert torch.equal(d, torch.cat([u for u, _ in parts])) and torch.equal(m, torch.cat([v for _, v in parts]))
    d, m = d.cpu().numpy(), m.cpu().numpy()
    items = [0, 7000, first_wrapped - 1, first_wrapped, 13001, B - 1]
    for b in items:
        xb, yb, mb = (t[b].cpu().numpy() for t in (x, y, mix))
        for j in range(S):
            w, _, margin = O.score(xb[j], [yb[j], mb], fs)
            assert margin >= MIN_MARGIN, (b, j, margin)
            compare("grid-stride loops", [d[b, j], m[b, j]], w, f"B 16384 item {b} source {j}")


# =====================================================================================================================
# 7. amplitudes
# =====================================================================================================================
@pytest.mark.parametrize("fs", [10000, 16000])
def test_amplitude_extremes(fs):
    """Rows at 1e-30 and 1e30, fp32 denormals (1e-40), a row whose peak is 3e38, and a normal reference against a
    denormal estimate and the other way round: eps then dominates frame energies and segment norms, and the values
    must still be the oracle's."""
    rng = np.random.default_rng(fs + 7)
    T = 3 * fs
    x, y, mix = batch(rng, 1, 1, T, fs, kinds=("ar",), hows=("noisy",))
    x, y = x[0, 0].astype(np.float64), y[0, 0].astype(np.float64)
    peak = max(np.max(np.abs(x)), np.max(np.abs(y)))
    pairs = [(1e-30, 1e-30), (1e30, 1e30), (1e-40, 1e-40), (3e38 / peak, 3e38 / peak), (1.0, 1e-40), (1e-40, 1.0),
             (1.0, 1e30)]
    xs = np.stack([x * a for a, _ in pairs])[None].astype(np.float32)
    ys = np.stack([y * b for _, b in pairs])[None].astype(np.float32)
    assert np.all(np.isfinite(xs)) and np.all(np.isfinite(ys))
    assert max(np.max(np.abs(xs)), np.max(np.abs(ys))) >= 2.9e38
    tiny = np.abs(xs[0, 2]) > 0
    assert np.all(np.abs(xs[0, 2][tiny]) < np.finfo(np.float32).tiny)          # denormals
    mix = (x * 1e-3)[None].astype(np.float32)
    score_all("amplitudes", xs, ys, fs, mix, label=f"fs {fs}")


# =====================================================================================================================
# 8. non-finite samples at the edges
# =====================================================================================================================
@pytest.mark.parametrize("fs", [10000, 44100])
@pytest.mark.parametrize("with_lengths", [False, True], ids=["no_lengths", "lengths"])
@pytest.mark.parametrize("where", ["reference", "estimate", "mixture"])
@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
def test_nonfinite_at_edges(fs, with_lengths, where, value):
    """NaN, inf or -inf at sample 0 or len - 1 of item 1's row: that score (or, in the mixture, that item's mixture
    scores) becomes NaN and nothing else changes, bitwise.  At 10 kHz sample len - 1 is read by no analysed frame, so
    only the documented contract puts NaN there.  With lengths, the same value at sample len changes nothing."""
    rng = np.random.default_rng(88)
    T = int(1.2 * fs)
    x, y, mix = batch(rng, 3, 2, T, fs, kinds=("white", "ar"), hows=("noisy",))
    lens = [T, T - 333, T // 2] if with_lengths else None
    n = lens[1] if with_lengths else T
    d0, m0 = gpu(x, y, fs, mix, lens)
    assert np.all(np.isfinite(d0)) and np.all(np.isfinite(m0))
    nan_d = np.zeros_like(d0, bool)
    nan_m = np.zeros_like(m0, bool)
    if where == "estimate":
        nan_d[1, 1] = True
    elif where == "reference":
        nan_d[1, 1] = nan_m[1, 1] = True
    else:
        nan_m[1, :] = True
    for pos in (0, n - 1) + ((n,) if with_lengths else ()):
        xs, ys, ms = x.copy(), y.copy(), mix.copy()
        row = {"estimate": ys[1, 1], "reference": xs[1, 1], "mixture": ms[1]}[where]
        row[pos] = value
        d, m = gpu(xs, ys, fs, ms, lens)
        wd, wm = (nan_d, nan_m) if pos < n else (np.zeros_like(nan_d), np.zeros_like(nan_m))
        assert np.array_equal(np.isnan(d), wd) and np.array_equal(np.isnan(m), wm), (pos, d, m)
        assert np.array_equal(d[~wd].view(np.int64), d0[~wd].view(np.int64)), pos
        assert np.array_equal(m[~wm].view(np.int64), m0[~wm].view(np.int64)), pos


def test_report_worst_errors():
    """Prints the largest |GPU - oracle| per case group of the module (run with -s to see it)."""
    for group, (err, label) in sorted(WORST.items()):
        print(f"worst {group}: {err:.2e} at {label}")
