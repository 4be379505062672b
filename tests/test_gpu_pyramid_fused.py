"""The fused depthwise stage (sdr_depthwise_pyramid_fused), which the forward runs on every block the pyramid takes.

It runs dw_pyramid_kernel twice over y: a statistics pass that writes no level, the solve, and a merge pass that
rebuilds the same raw convolution chain in registers and writes m (+ its statistics), in place over y in the forward.
So the levels never reach HBM.  Checked here:

- against the level-writing pair (sdr_depthwise_pyramid + sdr_merge_pyramid): the same m, bit for bit up to 1e-6 of
  max |m|, and the same statistics of m to 1e-4;
- against the fp64 level-by-level chain, for every fused instantiation: D = 4 / 5 / 6, the shortest eligible rows
  (L >> (D - 1) == 6), 8 and 9 windows (the 256 -> 1024 thread switch), 17 and 32 windows; shared slopes on both
  sides of 1, per-channel slopes, and no PReLU;
- m in place over y at exactly 4096 samples; the refusals at 4097 samples, at 33 windows and for an m that partly
  overlaps y;
- the statistics of m on ill-conditioned inputs up to r = 100 (the merge's 1e-4 contract);
- (CPU) that the parametrisation reaches every fused instantiation in pyramid.cu.
"""
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
from guards import Guards
from test_gpu_stages import channel_slopes, check_stats, norm_in, p, raw_stats, stream

DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PYR_STEP = {4: 480, 5: 464, 6: 416}       # PyrGeom<D>::kStep: level-0 positions one warp window stores
PYR_MAX_SAMPLES = 4096                    # kPyrMaxSamples
FUSED_LENGTHS = {   # shortest eligible row (1 window), 8 windows, 9 windows, 17 windows, 32 windows
    4: (48, 3840, 3856, 8160, 15360),
    5: (96, 3712, 3728, 7888, 14848),
    6: (192, 3328, 3360, 7072, 13312),
}
PAST_32 = {4: 15376, 5: 14864, 6: 13344}  # the next length the alignment allows: 33 windows
SLOPES = (0.3, 1.7, "pc", None)           # shared slope below 1, above 1, one slope per channel, no PReLU
FUSED_PARAMS = [(D, L, s) for D, Ls in FUSED_LENGTHS.items() for L in Ls for s in SLOPES]


def threads(D, L):
    """Block size the launcher picks: the <= 256-thread instantiation up to 8 windows, else the 1024-thread one."""
    return 256 if 32 * -(-L // PYR_STEP[D]) <= 256 else 1024


def arr(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def stage_inputs(samples, C_, D, L, slope, g):
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.3).to(DEV)
    gy = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    by = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    ws = [torch.randn(C_, 1, 5, generator=g).to(DEV) * 0.6 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    gs = [(1 + 0.3 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    bes = [(0.2 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    sl = None if slope is None else (channel_slopes(C_, g) if slope == "pc" else torch.tensor([slope], device=DEV))
    return y, gy, by, ws, bs, gs, bes, sl


def chain_ref(y, gy, by, ws, bs, gs, bes, sl, slope):
    """fp64 level-by-level chain (improved_sudormrf.py:205-216) -> (z_0, m)."""
    C_ = y.shape[1]
    cur = O.glob_ln(y.double(), gy.double(), by.double())
    if sl is not None:
        cur = O.prelu_c(cur, sl.double()) if slope == "pc" else O.prelu1(cur, sl.double())
    levels, z0 = [], None
    for d in range(len(ws)):
        z = F.conv1d(cur, ws[d].double(), bs[d].double(), stride=1 if d == 0 else 2, padding=2, groups=C_)
        z0 = z if d == 0 else z0
        cur = O.glob_ln(z, gs[d].double(), bes[d].double())
        levels.append(cur)
    for _ in range(len(ws) - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
    return z0, levels[0]


def run_pair(y, nin, ws, bs, gs, bes, samples, C_, D, L):
    """The level-writing pair: z_0 and R_d through HBM."""
    lib = N.lib()
    scratch = torch.zeros(lib.sdr_pyramid_scratch_bytes(samples, C_, D, L), dtype=torch.uint8, device=DEV)
    zs = [torch.empty(samples, C_, L >> d, device=DEV) for d in range(D)]
    st0 = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    stm = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    m = torch.empty(samples, C_, L, device=DEV)
    N.check(lib.sdr_depthwise_pyramid(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(st0),
                                      p(scratch), D, samples, C_, L, stream()))
    N.check(lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(m), p(stm), samples, C_, L, stream()))
    torch.cuda.synchronize()
    return m, st0, stm


def run_fused(y, nin, ws, bs, gs, bes, samples, C_, D, L, in_place=False):
    """sdr_depthwise_pyramid_fused on guarded buffers -> (m, stats0, stats_m)."""
    lib = N.lib()
    gd = Guards()
    scratch = gd.output("scratch", torch.zeros(lib.sdr_pyramid_scratch_bytes(samples, C_, D, L), dtype=torch.uint8,
                                               device=DEV))
    st0 = gd.output("stats0", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    stm = gd.output("stats_m", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    if in_place:
        yg = m = gd.output("y", y)
    else:
        yg = gd.input("y", y)
        m = gd.output("m", torch.full((samples, C_, L), float("nan"), device=DEV))
    N.check(lib.sdr_depthwise_pyramid_fused(p(yg), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), p(m), p(st0),
                                            p(stm), p(scratch), D, samples, C_, L, stream()))
    gd.check()
    return m, st0, stm


def same_as_pair(m, stm, m_pair, stm_pair):
    diff = float((m - m_pair).abs().max())
    assert diff <= 1e-6 * float(m_pair.abs().max()), diff     # (the same instructions: expected bitwise)
    scale = torch.stack([(m[0].numel() * stm_pair[:, 1]).sqrt(), stm_pair[:, 1]], dim=1)
    assert ((stm - stm_pair).abs() / scale).max() < 1e-4, (stm, stm_pair)


@pytest.mark.gpu
@pytest.mark.parametrize("D,L,slope", FUSED_PARAMS, ids=str)
def test_fused_stage(D, L, slope):
    samples, C_ = 2, 12
    g = torch.Generator().manual_seed(131)
    y, gy, by, ws, bs, gs, bes, sl = stage_inputs(samples, C_, D, L, slope, g)
    z0_ref, m_ref = chain_ref(y, gy, by, ws, bs, gs, bes, sl, slope)
    sy = raw_stats(y).to(DEV)                        # (nin holds a raw pointer: keep the statistics alive)
    nin = norm_in(sy, gy, by, sl, C_ * L)
    m, st0, stm = run_fused(y, nin, ws, bs, gs, bes, samples, C_, D, L)
    m_pair, st0_pair, stm_pair = run_pair(y, nin, ws, bs, gs, bes, samples, C_, D, L)
    same_as_pair(m, stm, m_pair, stm_pair)
    check_stats(st0, z0_ref)
    e = O.parity_errors(m, m_ref)
    assert max(e) < 5e-5, e
    check_stats(stm, m_ref, rtol=1e-4)


@pytest.mark.gpu
def test_fused_in_place_at_the_sample_table():
    """m over y itself, as the forward calls it, with all 4096 per-sample (mean, rstd) entries in shared memory."""
    samples, C_, D, L = PYR_MAX_SAMPLES, 4, 4, 448
    g = torch.Generator().manual_seed(137)
    y, gy, by, ws, bs, gs, bes, sl = stage_inputs(samples, C_, D, L, 0.3, g)
    sy = raw_stats(y).to(DEV)
    nin = norm_in(sy, gy, by, sl, C_ * L)
    m_pair, _, stm_pair = run_pair(y, nin, ws, bs, gs, bes, samples, C_, D, L)
    m, _, stm = run_fused(y.clone(), nin, ws, bs, gs, bes, samples, C_, D, L, in_place=True)
    same_as_pair(m, stm, m_pair, stm_pair)
    _, m_ref = chain_ref(y, gy, by, ws, bs, gs, bes, sl, 0.3)
    assert max(O.parity_errors(m, m_ref)) < 5e-5


@pytest.mark.gpu
@pytest.mark.parametrize("samples,D,L,rc", [
    (PYR_MAX_SAMPLES + 1, 4, 448, -5),     # past the per-sample table
    (2, 4, PAST_32[4], -5),                # 33 windows
    (2, 6, PAST_32[6], -5),
    (2, 4, 448, -2),                       # m overlaps y without being y
], ids=str)
def test_fused_refusals(samples, D, L, rc):
    """The entry refuses before launching anything: no output and no statistics are written."""
    lib = N.lib()
    C_ = 4
    y = torch.zeros(samples, C_, L + 16, device=DEV)
    prm = [torch.zeros(C_, 5, device=DEV) for _ in range(D)]
    nb = lib.sdr_pyramid_scratch_bytes(samples, C_, D, L)
    assert (nb == 0) == (rc == -5)
    scratch = torch.zeros(max(nb, lib.sdr_pyramid_scratch_bytes(2, C_, D, 448)), dtype=torch.uint8, device=DEV)
    st0 = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    stm = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    m = torch.zeros(samples, C_, L, device=DEV) if rc == -5 else y.view(-1)[16:]
    nin = norm_in(st0, prm[0][:, 0], prm[0][:, 1], torch.tensor([0.3], device=DEV), C_ * L)
    assert lib.sdr_depthwise_pyramid_fused(p(y), C.byref(nin), arr(prm), arr(prm), arr(prm), arr(prm), p(m), p(st0),
                                           p(stm), p(scratch), D, samples, C_, L, stream()) == rc
    torch.cuda.synchronize()
    assert not y.any() and not m.any() and not st0.any() and not stm.any() and not scratch.any()


COND_R = (0, 1, 10, 30, 100)
COND_SCALES = (1e-3, 1.0, 3e4)


@pytest.mark.gpu
@pytest.mark.parametrize("r,scale", [(r, s) for r in COND_R for s in COND_SCALES], ids=lambda v: f"{v:g}")
def test_fused_merge_statistics_conditioning(r, scale):
    """Level 0's beta offsets m by r of its standard deviations (the sign alternating over r): the (mean, rstd) the
    fused merge's statistics give against the two-pass fp64 values of the m it stored."""
    samples, C_, L, D = 2, 512, 3200, 5               # cfg 2's depthwise stage
    g = torch.Generator().manual_seed(139)
    y, gy, by, ws, bs, gs, bes, sl = stage_inputs(samples, C_, D, L, 0.3, g)
    gs = [x * scale for x in gs]
    bes = [x * scale for x in bes]
    _, m0 = chain_ref(y, gy, by, ws, bs, gs, bes, sl, 0.3)
    bes[0] = bes[0] + (1.0 if COND_R.index(r) % 2 == 0 else -1.0) * r * float(m0.std())
    _, m_ref = chain_ref(y, gy, by, ws, bs, gs, bes, sl, 0.3)
    sy = raw_stats(y).to(DEV)
    nin = norm_in(sy, gy, by, sl, C_ * L)
    m, _, stm = run_fused(y, nin, ws, bs, gs, bes, samples, C_, D, L)
    assert torch.isfinite(m).all() and torch.isfinite(stm).all()
    assert max(O.parity_errors(m, m_ref)) < 5e-5
    s = stm.double().cpu()
    n = C_ * L
    mu, var = s[:, 0] / n, s[:, 1] / n - (s[:, 0] / n) ** 2
    md = m.double().reshape(samples, -1).cpu()
    mu_r = md.mean(1)
    var_r = ((md - mu_r[:, None]) ** 2).mean(1)
    rstd, rstd_r = 1 / (var.clamp_min(0) + 1e-8).sqrt(), 1 / (var_r + 1e-8).sqrt()
    err = max(float(((mu - mu_r).abs() * rstd_r).max()), float((rstd / rstd_r - 1).abs().max()))
    assert var.min() > 0 and err < 1e-4, (r, scale, err)


def test_fused_instantiations_are_all_tested():
    src = open(os.path.join(REPO, "sudo_rm_rf_b200", "csrc", "pyramid.cu")).read()
    fused = {(int(d), int(t), pc == "true")
             for d, t, pc in re.findall(r"dw_pyramid_kernel<(\d),\s*(\d+),\s*\w+,\s*(true|false),\s*M>", src)}
    assert len(fused) == 12, sorted(fused)
    assert set(re.findall(r"launch_fused_pass<(\w+)>\(", src)) == {"kPyrStats", "kPyrMerge"}
    tested = {(D, threads(D, L), slope == "pc") for D, L, slope in FUSED_PARAMS}
    assert fused == tested, (sorted(fused - tested), sorted(tested - fused))
