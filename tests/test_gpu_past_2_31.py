"""Past 2^31 elements: the kernels that test_gpu_scale.py does not reach there.

The one-pass depthwise pyramid (fused and level-writing), the wide merge, the causal pyramid, both TAC kernels, both
encoders, the metrics' Gram kernels, the loss and mixture-consistency backward kernels, the backward stage kernels,
three whole models and STOI.  The method is test_gpu_scale.py's:

1. the rows under test start past element 2^31 (past 2^32 where the tensors fit in about 24 GiB), asserted in Python
   before anything is launched;
2. outputs the test allocates start as NaN inside guard bands (tests/guards.py), so a row nobody writes is non-finite;
3. those rows are held to the same entry on a small tensor that holds only them: bitwise where the kernel sums nothing
   across CTAs, within 1e-6 of max |ref| where per-sample statistics are summed by fp64 atomics;
4. the same rows are held to fp64 at the stage tests' tolerances (parameter gradients, which sum over every sample, to
   an fp64 reference accumulated sample by sample on the GPU);
5. the first rows, where a wrapped index would write, are finite.

A case that does not find the device memory it needs free is skipped with the amount; the fixture prints each case's
peak."""
import ctypes as C
import itertools
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
import stoi_oracle as SO
from guards import GUARD, GUARD_BITS, POISON_NAN, assert_guards_intact, check_bands, guarded, poisoned
from test_gpu_long import CLASSES, normalised_input
from test_gpu_model_space import TOL, build, gc, imp
from test_gpu_pyramid_fused import PYR_MAX_SAMPLES, arr, chain_ref, run_fused, stage_inputs
from test_gpu_scale import (BIG_C, BIG_S, SUB, GiB, assert_rows_close, assert_rows_equal, last_sample_parts, need,
                            norm_parts, ref_glob)
from test_gpu_stages import norm_in, p, raw_stats, stream
from test_gpu_train import grad_errors, ref_norm_act

DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
P_REF = 2048                 # positions held to fp64 where a kernel works position by position


@pytest.fixture(autouse=True)
def device_memory(request):
    """Frees the cached blocks around each GPU test and prints its peak."""
    if "gpu" not in request.keywords:
        yield
        return
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    print(f"\n{request.node.name}: peak device memory {torch.cuda.max_memory_allocated() / GiB:.2f} GiB")
    torch.cuda.empty_cache()


def nan_guarded(*shape):
    """An fp32 tensor of NaN inside guard bands, without a second copy of it (the band pattern is an fp32 NaN)."""
    n = math.prod(shape)
    buf = torch.empty(n + 2 * GUARD, device=DEV)
    buf.view(torch.int32).fill_(GUARD_BITS)
    return buf[GUARD:GUARD + n].view(shape)


def past(offset, bound=2 ** 31):
    assert offset > bound, (offset, bound)


def sample_stats(x, chunk=8):
    """(sum, sumsq) per sample in fp64, a few samples at a time."""
    out = torch.empty(x.shape[0], 2, dtype=torch.float64, device=DEV)
    for i in range(0, x.shape[0], chunk):
        out[i:i + chunk] = raw_stats(x[i:i + chunk])
    return out


def assert_stats_close(got, want, rel=1e-6):
    """fp64 statistics summed in another order: the sum against sqrt(n sumsq) is not needed here, both are large."""
    err = (got - want).abs()
    assert bool((err <= rel * want.abs().max()).all()), (got, want)


def check_grad(got, ref, what, tol=3e-4):
    """rel_max and rel_l2 against fp64 (test_gpu_train.py's measures; its stage bar is 1e-3).  Measured on one H100:
    up to 1e-4 for dgamma / dbeta, which sum 2^31 products of either sign in fp32 partials; a sample lost or read
    twice moves a sum by about 1 / 33."""
    rm, rl = grad_errors(got, ref)
    print(f"{what}: rel_max {rm:.2e} rel_l2 {rl:.2e}")
    assert rm <= tol and rl <= tol, (what, rm, rl)


# =====================================================================================================================
# the one-pass depthwise pyramid
# =====================================================================================================================
FUSED_BIG = [(4, 15360, 0.3), (4, 15360, "pc"), (6, 13312, 0.3), (6, 13312, "pc")]     # 32 windows: 1024 threads


@gpu
@pytest.mark.parametrize("D,L,slope", FUSED_BIG, ids=str)
def test_fused_pyramid_past_2_32_elements(D, L, slope):
    """sdr_depthwise_pyramid_fused over 512 channels at the pyramid's longest rows, m in place over y as the forward
    runs it: the last sample starts past 2^32.  It against the same call on that sample alone (the solve needs its
    statistics), and the fp64 level-by-level chain."""
    lib = N.lib()
    C_ = 512
    samples = 2 ** 32 // (C_ * L) + 2
    past((samples - 1) * C_ * L, 2 ** 32)
    assert samples <= PYR_MAX_SAMPLES and lib.sdr_pyramid_scratch_bytes(samples, C_, D, L) > 0
    need(samples * C_ * L * 4 / GiB + 2)
    y_last, gy, by, ws, bs, gs, bes, sl = stage_inputs(1, C_, D, L, slope, torch.Generator().manual_seed(151))
    y = torch.randn(samples, C_, L, device=DEV, generator=torch.Generator(device=DEV).manual_seed(157))
    y[-1] = y_last[0]
    sy = sample_stats(y)
    nin = norm_in(sy, gy, by, sl, C_ * L)
    scratch = torch.zeros(lib.sdr_pyramid_scratch_bytes(samples, C_, D, L), dtype=torch.uint8, device=DEV)
    st0 = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    stm = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    N.check(lib.sdr_depthwise_pyramid_fused(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), p(y), p(st0),
                                            p(stm), p(scratch), D, samples, C_, L, stream()))
    sy1 = sy[-1:].clone()
    nin1 = norm_in(sy1, gy, by, sl, C_ * L)
    m1, st01, stm1 = run_fused(y_last, nin1, ws, bs, gs, bes, 1, C_, D, L)
    torch.cuda.synchronize()
    assert torch.isfinite(y[0, :SUB]).all()
    assert_rows_close(y[-1:], m1)
    assert_stats_close(st0[-1:], st01)
    assert_stats_close(stm[-1:], stm1)
    del y, scratch
    _, m_ref = chain_ref(y_last, gy, by, ws, bs, gs, bes, sl, slope)
    e = O.parity_errors(m1, m_ref)
    assert max(e) < 5e-5, e


@gpu
def test_level_writing_pyramid_past_2_31_elements():
    """sdr_depthwise_pyramid + sdr_merge_pyramid at D = 4 (z_0..z_3 in HBM, m written over y once the levels exist):
    the last sample starts past 2^31.  z_0..z_3 bitwise, m and both statistics close, against the pair on that sample
    alone; m against the fp64 chain."""
    lib = N.lib()
    C_, D, L = 512, 4, 15360
    samples = 2 ** 31 // (C_ * L) + 2
    past((samples - 1) * C_ * L)
    assert samples <= PYR_MAX_SAMPLES
    nb = lib.sdr_pyramid_scratch_bytes(samples, C_, D, L)
    assert nb > 0
    need(samples * C_ * L * 4 * (1 + 2 - 2 ** (1 - D)) / GiB + 2)
    y_last, gy, by, ws, bs, gs, bes, sl = stage_inputs(1, C_, D, L, 0.3, torch.Generator().manual_seed(163))
    y = torch.randn(samples, C_, L, device=DEV, generator=torch.Generator(device=DEV).manual_seed(167))
    y[-1] = y_last[0]
    sy = sample_stats(y)
    nin = norm_in(sy, gy, by, sl, C_ * L)

    def pair(y, samples, nin, m):
        scratch = torch.zeros(lib.sdr_pyramid_scratch_bytes(samples, C_, D, L), dtype=torch.uint8, device=DEV)
        zs = [nan_guarded(samples, C_, L >> d) for d in range(D)]
        st0 = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        stm = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        N.check(lib.sdr_depthwise_pyramid(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(st0),
                                          p(scratch), D, samples, C_, L, stream()))
        N.check(lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(m), p(stm), samples, C_, L, stream()))
        torch.cuda.synchronize()
        for d, z in enumerate(zs):
            assert_guards_intact(z, f"z_{d}")
        return zs, st0, stm

    zs, st0, stm = pair(y, samples, nin, y)                  # m over y: merge_pyramid reads z and scratch only
    sy1 = sy[-1:].clone()
    nin1 = norm_in(sy1, gy, by, sl, C_ * L)
    m1 = nan_guarded(1, C_, L)
    zs1, st01, stm1 = pair(y_last, 1, nin1, m1)
    assert_guards_intact(m1, "m")
    for d in range(D):
        assert_rows_equal(zs[d][-1:], zs1[d])
        assert torch.isfinite(zs[d][0, :SUB]).all()
    assert torch.isfinite(y[0, :SUB]).all()
    assert_rows_close(y[-1:], m1)
    assert_stats_close(st0[-1:], st01)
    assert_stats_close(stm[-1:], stm1)
    del y, zs
    _, m_ref = chain_ref(y_last, gy, by, ws, bs, gs, bes, sl, 0.3)
    assert max(O.parity_errors(m1, m_ref)) < 5e-5


@gpu
def test_wide_merge_past_2_31_elements():
    """sdr_merge at depth 4 (merge_wide_kernel: L % 16 == 0, 16-byte aligned rows), BIG_S samples of BIG_C channels:
    the last sample starts past 2^31.  Its last SUB channels bitwise against the same call on them alone, fp64."""
    depth, L = 4, 1048592
    past((BIG_S - 1) * BIG_C * L)
    need(sum(BIG_S * BIG_C * (L >> d) * 4 for d in range(depth)) / GiB + BIG_S * BIG_C * L * 4 / GiB + 1.5)
    g = torch.Generator(device=DEV).manual_seed(173)
    zs = [torch.randn(BIG_S, BIG_C, L >> d, device=DEV, generator=g) + 0.3 * d for d in range(depth)]
    parts = [norm_parts(BIG_C, BIG_C * L >> d, g) for d in range(depth)]
    m = nan_guarded(BIG_S, BIG_C, L)
    st = torch.zeros(BIG_S, 2, dtype=torch.float64, device=DEV)
    nins = (N.SdrNormIn * depth)(*[norm_in(s_, g_, b_, None, BIG_C * L >> d) for d, (s_, g_, b_) in enumerate(parts)])
    N.check(N.lib().sdr_merge(arr(zs), nins, depth, p(m), p(st), BIG_S, BIG_C, L, stream()))
    zss = last_sample_parts(*zs)
    sub = [(s_[-1:].contiguous(), g_[-SUB:].contiguous(), b_[-SUB:].contiguous()) for s_, g_, b_ in parts]
    ms = nan_guarded(1, SUB, L)
    sts = torch.zeros(1, 2, dtype=torch.float64, device=DEV)
    nss = (N.SdrNormIn * depth)(*[norm_in(s_, g_, b_, None, BIG_C * L >> d) for d, (s_, g_, b_) in enumerate(sub)])
    N.check(N.lib().sdr_merge(arr(zss), nss, depth, p(ms), p(sts), 1, SUB, L, stream()))
    torch.cuda.synchronize()
    assert_guards_intact(m, "m")
    assert_guards_intact(ms, "m (small)")
    assert_rows_equal(m[-1, -SUB:], ms[0])
    assert torch.isfinite(m[0, :SUB]).all()
    md = m[-1].double()
    want_st = torch.stack([md.sum(), (md * md).sum()])
    assert abs(float(st[-1, 0] - want_st[0])) <= 1e-5 * float((md.numel() * want_st[1]).sqrt())
    assert abs(float(st[-1, 1] - want_st[1])) <= 1e-5 * float(want_st[1])
    del md, m, zs
    want = 0
    for d in reversed(range(depth)):
        lvl = ref_glob(zss[d][0], sub[d][0][0], sub[d][1], sub[d][2], BIG_C * L >> d)
        want = lvl + (F.interpolate(want.unsqueeze(0), scale_factor=2, mode="nearest")[0] if d < depth - 1 else 0)
    assert max(O.parity_errors(ms[0], want)) < 2e-5


# =====================================================================================================================
# the causal pyramid
# =====================================================================================================================
def causal_chain(y, sp, ws, bs, sl):
    """fp64 PReLU -> D x (masked 21-tap depthwise conv + PReLU) -> up-sample / add chain (as test_causal_pyramid)."""
    C_ = y.shape[1]
    cur = O.prelu1(y.double(), sp.double())
    levels = []
    for d in range(len(ws)):
        cur = O.prelu1(F.conv1d(cur, O.causal_weight(ws[d].double()), bs[d].double(), stride=1 if d == 0 else 2,
                                padding=10, groups=C_), sl[d].double())
        levels.append(cur)
    for _ in range(len(ws) - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
    return levels[0]


@gpu
@pytest.mark.parametrize("D", [4, 8])
def test_causal_pyramid_past_2_31_elements(D):
    """sdr_causal_pyramid over BIG_S samples of BIG_C channels x 2^20 + 256 positions (many 4096-position windows per
    row): the last sample starts past 2^31.  Its last SUB channels bitwise against the same call on them alone, and
    against the fp64 chain."""
    L = 2 ** 20 + 256
    past((BIG_S - 1) * BIG_C * L)
    need(2 * BIG_S * BIG_C * L * 4 / GiB + 1.5)
    g = torch.Generator(device=DEV).manual_seed(179 + D)
    y = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    sp = torch.tensor([0.3], device=DEV)
    ws = [torch.randn(BIG_C, 1, 21, device=DEV, generator=g) * 0.4 for _ in range(D)]
    bs = [torch.randn(BIG_C, device=DEV, generator=g) * 0.5 for _ in range(D)]
    sl = [torch.tensor([0.1 + 0.07 * d], device=DEV) for d in range(D)]
    m = nan_guarded(BIG_S, BIG_C, L)
    lib = N.lib()
    N.check(lib.sdr_causal_pyramid(p(y), p(sp), arr(ws), arr(bs), arr(sl), p(m), D, BIG_S, BIG_C, L, stream()))
    ys, = last_sample_parts(y)
    wss = [w[-SUB:].contiguous() for w in ws]
    bss = [b[-SUB:].contiguous() for b in bs]
    ms = nan_guarded(1, SUB, L)
    N.check(lib.sdr_causal_pyramid(p(ys), p(sp), arr(wss), arr(bss), arr(sl), p(ms), D, 1, SUB, L, stream()))
    torch.cuda.synchronize()
    assert_guards_intact(m, "m")
    assert_guards_intact(ms, "m (small)")
    assert_rows_equal(m[-1, -SUB:], ms[0])
    assert torch.isfinite(m[0, :SUB]).all()
    del y, m
    e = O.parity_errors(ms, causal_chain(ys, sp, wss, bss, sl))
    assert max(e) < 2e-5, e


# =====================================================================================================================
# TAC
# =====================================================================================================================
TAC_NAMES = ["TAC_input.0.weight", "TAC_input.0.bias", "TAC_input.1.weight",
             "TAC_mean.0.weight", "TAC_mean.0.bias", "TAC_mean.1.weight",
             "TAC_output.0.weight", "TAC_output.0.bias", "TAC_output.1.weight"]


@gpu
@pytest.mark.parametrize("n", [16, 4, 8, 32])
def test_tac_past_2_31_elements(n):
    """sdr_tac, B = 9 items of G x n x L (tac_mma16_kernel at n = 16, tac_kernel<n> otherwise): the last item starts
    past 2^31.  o of the last item bitwise, its per-group statistics close, against the same call on it alone (its
    groups interact); fp64 O.tac on its last positions (TAC works position by position)."""
    B = 9
    G = 16 if n <= 16 else 8
    L = ((2 ** 31) // ((B - 1) * G * n) + 16) // 16 * 16
    past((B - 1) * G * n * L)
    need(2 * B * G * n * L * 4 / GiB + 1.5)
    cfg = O.Config(variant="groupcomm", out_channels=G * n, in_channels=2 * G * n, num_blocks=1, upsampling_depth=1,
                   group_size=G)
    sd = {k[len("sm.0.TAC."):]: v.to(DEV).contiguous() for k, v in O.make_state_dict(cfg, seed=181).items()
          if k.startswith("sm.0.TAC.")}
    params = (C.c_void_p * 9)(*[sd[k].data_ptr() for k in TAC_NAMES])
    x = torch.randn(B, G, n, L, device=DEV, generator=torch.Generator(device=DEV).manual_seed(191 + n))
    o = nan_guarded(B, G, n, L)
    st = torch.zeros(B * G, 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_tac(p(x), params, p(o), p(st), B, G, n, L, stream()))
    xs = x[-1:]                                              # contiguous: a view, read only
    os_ = nan_guarded(1, G, n, L)
    sts = torch.zeros(G, 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_tac(p(xs), params, p(os_), p(sts), 1, G, n, L, stream()))
    torch.cuda.synchronize()
    assert_guards_intact(o, "o")
    assert_guards_intact(os_, "o (small)")
    assert_rows_equal(o[-1:], os_)
    assert torch.isfinite(o[0, 0, :, :SUB]).all()
    assert_stats_close(st[-G:], sts)
    taps = {}
    O.tac(xs[..., -P_REF:].double(), {k: v.double() for k, v in sd.items()}, "", taps)
    e = O.parity_errors(os_[..., -P_REF:], taps["TAC_output"])
    assert max(e) < (1e-4 if n == 16 else 2e-5), e


# =====================================================================================================================
# encoders
# =====================================================================================================================
ENC_BIG = ["ffma", "mma", "ffma_ex", "mma_ex"]


def enc_window_ref(wav1, w, bias, relu, pad, hop, p0, P):
    """fp64 enc[:, p0:p0+P] of one item: enc[n, q] = act(sum_{a,j} w[n,a,j] wav[a, hop q + j - pad] + bias[n])."""
    A, T = wav1.shape
    K = w.shape[-1]
    start, n = hop * p0 - pad, hop * (P - 1) + K
    seg = torch.zeros(A, n, dtype=torch.float64, device=DEV)
    lo, hi = max(start, 0), min(start + n, T)
    seg[:, lo - start:hi - start] = wav1[:, lo:hi].double()
    out = F.conv1d(seg.unsqueeze(0), w.double(), None if bias is None else bias.double(), stride=hop)[0]
    return torch.relu(out) if relu else out


@gpu
@pytest.mark.parametrize("kind", ENC_BIG)
def test_encoder_past_2_31_elements(kind):
    """sdr_encoder / sdr_encoder_mma, and their _ex forms with bias + ReLU and the causal model's left padding
    (2 hop): B = 3 items of 512 x (2^21 + 64), the last item starts past 2^31.  It bitwise against the same call on
    it alone, its statistics close, and fp64 conv1d on its first and last positions."""
    lib = N.lib()
    B, A, N_, K = 3, 1, 512, 21
    hop = K // 2
    L = 2 ** 21 + 64
    T = hop * L
    past((B - 1) * N_ * L)
    need((B + 1) * N_ * L * 4 / GiB + 1.5)
    mma, ex = kind.startswith("mma"), kind.endswith("_ex")
    g = torch.Generator(device=DEV).manual_seed(193)
    wav = torch.randn(B, A, T, device=DEV, generator=g)
    w = torch.randn(N_, A, K, device=DEV, generator=g)
    bias = torch.randn(N_, device=DEV, generator=g) if ex else None
    pad = 2 * hop if ex else hop
    if mma:
        wpk = torch.empty(lib.sdr_encoder_mma_packed_bytes(N_, A, K), dtype=torch.uint8, device=DEV)
        N.check(lib.sdr_encoder_mma_pack(p(w), N_, A, K, p(wpk), stream()))

    def run(wv, rows):
        enc = nan_guarded(rows, N_, L)
        st = torch.zeros(rows, 2, dtype=torch.float64, device=DEV)
        if ex:
            fn = lib.sdr_encoder_mma_ex if mma else lib.sdr_encoder_ex
            N.check(fn(p(wv), p(wpk if mma else w), p(bias), 1, pad, p(enc), p(st), rows, A, T, N_, K, L, stream()))
        else:
            fn = lib.sdr_encoder_mma if mma else lib.sdr_encoder
            N.check(fn(p(wv), p(wpk if mma else w), p(enc), p(st), rows, A, T, N_, K, L, stream()))
        return enc, st

    enc, st = run(wav, B)
    enc1, st1 = run(wav[-1:], 1)
    torch.cuda.synchronize()
    assert_guards_intact(enc, "enc")
    assert_guards_intact(enc1, "enc (small)")
    assert_rows_equal(enc[-1:], enc1)
    assert torch.isfinite(enc[0, :SUB]).all()
    assert_stats_close(st[-1:], st1)
    del enc
    for p0 in (0, L - P_REF):
        want = enc_window_ref(wav[-1], w, bias, ex, pad, hop, p0, P_REF)
        e = O.parity_errors(enc1[0, :, p0:p0 + P_REF], want)
        assert max(e) < (5e-5 if mma else 2e-5), (p0, e)


# =====================================================================================================================
# metrics and losses: the Gram kernels
# =====================================================================================================================
MB, MS, MT = 5, 2, 270_000_000          # item 4 starts at 8 MT > 2^31; 64 chunks of about 4.2 M samples per item


def metric_batch(seed, with_mix=True):
    """Targets with per-source gain and a DC offset; estimates = 0.8 x the swapped targets plus noise whose level
    grows over the batch; mixture = sum of the targets plus a little noise."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    tgt = torch.randn(MB, MS, MT, device=DEV, generator=g)
    tgt.mul_(0.2 + torch.rand(MB, MS, 1, device=DEV, generator=g)).add_(0.05)
    est = torch.randn(MB, MS, MT, device=DEV, generator=g)
    est.mul_(torch.logspace(-1.5, -0.3, MB, device=DEV).view(MB, 1, 1))
    est.add_(tgt.flip(1), alpha=0.8)
    if not with_mix:
        return est, tgt, None
    mix = torch.randn(MB, 1, MT, device=DEV, generator=g).mul_(0.01)
    mix.add_(tgt.sum(1, keepdim=True))
    return est, tgt, mix


def gram64(rows, chunk=1 << 24):
    """fp64 Gram matrix and row sums of a list of [T] rows, a chunk at a time."""
    R = len(rows)
    G = torch.zeros(R, R, dtype=torch.float64, device=DEV)
    s = torch.zeros(R, dtype=torch.float64, device=DEV)
    for a in range(0, rows[0].shape[-1], chunk):
        X = torch.stack([r[a:a + chunk] for r in rows]).double()
        G += X @ X.T
        s += X.sum(1)
    return G, s


def centred(G, s, T):
    return G - torch.outer(s, s) / T


def sisdr64(Gc, i, j, eps=1e-9):
    """SI-SDR in dB of row i against target row j from a (centred) Gram matrix, as sisdr.py:118-126 forms it."""
    dot, tt, ee = Gc[i, j], Gc[j, j], Gc[i, i]
    a = dot / (tt + eps)
    return float(10 * torch.log10(a * a * tt / (ee - 2 * a * dot + a * a * tt + eps)))


def pairwise64(Gc, i, j, eps=1e-8):
    """-PairwiseNegSDR's SI-SDR in dB (take_log) of estimate row i against target row j, as sisdr.py:425-447 forms
    it: eps in the target energy, in the noise energy and inside the log."""
    dot, tt, ee = Gc[i, j], Gc[j, j], Gc[i, i]
    a = dot / (tt + eps)
    return float(10 * torch.log10(a * a * tt / (ee - 2 * a * dot + a * a * tt + eps) + eps))


def pit64(Gc, S):
    """(best, index) over itertools.permutations(range(S)); rows 0..S-1 estimates, S..2S-1 targets."""
    scores = [sum(sisdr64(Gc, pm[j], S + j) for j in range(S)) / S for pm in itertools.permutations(range(S))]
    best = max(scores)
    return best, scores.index(best)


def scratch_bytes(n):
    return torch.zeros(max(int(n), 8), dtype=torch.uint8, device=DEV)


@gpu
def test_metrics_past_2_31_elements():
    """PIT SI-SDR (atomic Gram mode; with and without the mixture's SI-SDRi baseline), the stabilised metric, the
    pairwise SI-SDR (both Gram modes), the FUSS loss and the utterance statistics on B = 5 items of 2 x 270 M
    samples: the last item starts past 2^31.  The last item against a B = 1 call (bitwise for the ordered Gram mode,
    1e-3 dB and the same permutation for the atomic one, 1e-6 for the statistics), and the fp64 Gram computed slice by
    slice; SI-SDRi against the fp64 batch-mean baseline of the whole batch."""
    lib = N.lib()
    past((MB - 1) * MS * MT)
    need(2.5 * MB * MS * MT * 4 / GiB + 2)
    est, tgt, mix = metric_batch(197)
    e1, t1 = est[-1:], tgt[-1:]                              # views: the last item is contiguous
    sb = lambda B: scratch_bytes(lib.sdr_pit_sisdr_scratch_bytes(B, MS))

    def pit(e, t, m, B, zero_mean, improvement):
        best = torch.full((B,), float("nan"), device=DEV)
        perm = torch.full((B,), -7, dtype=torch.int32, device=DEV)
        N.check(lib.sdr_pit_sisdr(p(e), p(t), p(m), p(best), p(perm), B, MS, MT, zero_mean, improvement, 1e-9,
                                  p(sb(B)), stream()))
        return best, perm

    def stab(e, t, B):
        best = torch.full((B,), float("nan"), device=DEV)
        perm = torch.full((B,), -7, dtype=torch.int32, device=DEV)
        sc = scratch_bytes(lib.sdr_stabilized_sisdr_scratch_bytes(B, MS, MS))
        N.check(lib.sdr_stabilized_sisdr(p(e), p(t), p(best), p(perm), B, MS, MS, MS, MT, 1, 0, 1e-9, p(sc),
                                         stream()))
        return best, perm

    def pairwise(e, t, B):
        out = torch.full((B, MS, MS), float("nan"), device=DEV)
        N.check(lib.sdr_pairwise_neg_sdr(p(e), p(t), p(out), B, MS, MT, 1, 1, 1, p(sb(B)), stream()))
        return out

    def pairwise_train(e, t, B):
        out = torch.full((B, MS, MS), float("nan"), device=DEV)
        coef = scratch_bytes(lib.sdr_pairwise_neg_sdr_coef_bytes(B, MS))
        sc = scratch_bytes(lib.sdr_pairwise_neg_sdr_train_scratch_bytes(B, MS, MT))
        N.check(lib.sdr_pairwise_neg_sdr_train(p(e), p(t), p(out), p(coef), B, MS, MT, 1, 1, 1, p(sc), stream()))
        return out

    def snr(e, t, B):
        val = torch.full((B,), float("nan"), device=DEV)
        perm = torch.full((B,), -7, dtype=torch.int32, device=DEV)
        coef = scratch_bytes(lib.sdr_snr_zero_refs_coef_bytes(B, MS))
        sc = scratch_bytes(lib.sdr_snr_zero_refs_scratch_bytes(B, MS, MT))
        N.check(lib.sdr_snr_zero_refs(p(e), p(t), p(val), p(perm), p(coef), B, MS, MT, 0, -40.0, 1e-8, p(sc),
                                      stream()))
        return val, perm

    def ustats(w, rows):
        ms = torch.full((rows, 2), float("nan"), device=DEV)
        sc = torch.zeros(2 * rows, dtype=torch.float64, device=DEV)
        N.check(lib.sdr_utterance_stats(p(w), p(ms), rows, MT, p(sc), stream()))
        return ms

    big = dict(pit=pit(est, tgt, None, MB, 1, 0), pit_i=pit(est, tgt, mix, MB, 1, 1), stab=stab(est, tgt, MB),
               pw=pairwise(est, tgt, MB), pwt=pairwise_train(est, tgt, MB), snr=snr(est, tgt, MB),
               us=ustats(est, MB * MS))
    one = dict(pit=pit(e1, t1, None, 1, 1, 0), stab=stab(e1, t1, 1), pw=pairwise(e1, t1, 1),
               pwt=pairwise_train(e1, t1, 1), snr=snr(e1, t1, 1), us=ustats(e1, MS))
    torch.cuda.synchronize()
    for k in ("pit", "stab", "snr"):
        assert torch.isfinite(big[k][0]).all(), (k, big[k])
        assert (big[k][1] >= 0).all(), (k, big[k])
    for k in ("pit", "stab"):
        assert abs(float(big[k][0][-1] - one[k][0][0])) < 1e-3, (k, big[k][0], one[k][0])
        assert int(big[k][1][-1]) == int(one[k][1][0]), k
    assert torch.equal(big["snr"][0][-1:], one["snr"][0]) and torch.equal(big["snr"][1][-1:], one["snr"][1])
    assert torch.isfinite(big["pw"]).all() and torch.isfinite(big["pwt"]).all()
    assert float((big["pw"][-1] - one["pw"][0]).abs().max()) < 1e-3
    assert torch.equal(big["pwt"][-1:], one["pwt"])
    assert_rows_close(big["us"][-MS:], one["us"])
    assert torch.isfinite(big["us"]).all()
    # fp64, item by item: the mixture's SI-SDR baseline is a mean over the batch
    base, last = [], None
    for b in range(MB):
        G, s = gram64([est[b, 0], est[b, 1], tgt[b, 0], tgt[b, 1], mix[b, 0]])
        Gc = centred(G, s, MT)
        base.append(sum(sisdr64(Gc, 4, 2 + j) for j in range(MS)) / MS)
        if b == MB - 1:
            last = G, s, Gc
    G, s, Gc = last
    best, idx = pit64(Gc, MS)
    assert abs(float(big["pit"][0][-1]) - best) < 1e-3 and int(big["pit"][1][-1]) == idx, (big["pit"], best, idx)
    want_i = best - sum(base) / MB
    assert abs(float(big["pit_i"][0][-1]) - want_i) < 1e-3 and int(big["pit_i"][1][-1]) == idx, (big["pit_i"], want_i)
    for i in range(MS):
        for j in range(MS):
            assert abs(-float(big["pw"][-1, i, j]) - pairwise64(Gc, i, MS + j)) < 1e-3, (i, j, big["pw"][-1])
    mean = s[:MS] / MT
    std = ((torch.diagonal(G)[:MS] - s[:MS] * mean) / (MT - 1)).sqrt()
    assert torch.allclose(big["us"][-MS:].double(), torch.stack([mean, std], 1), rtol=1e-6, atol=1e-7)


@gpu
def test_loss_backward_past_2_31_elements():
    """sdr_pairwise_neg_sdr_backward and sdr_snr_zero_refs_backward (after their training forwards) write grad_est
    [5, 2, 270 M]: the last item's rows start past 2^31.  They bitwise against the same calls on the last item alone,
    and the first rows finite."""
    lib = N.lib()
    past((MB - 1) * MS * MT)
    need(3.2 * MB * MS * MT * 4 / GiB + 2)
    est, tgt, _ = metric_batch(199, with_mix=False)
    g = torch.Generator(device=DEV).manual_seed(211)
    gpw = torch.randn(MB, MS, MS, device=DEV, generator=g)
    gval = torch.randn(MB, device=DEV, generator=g)

    def pairwise(e, t, gout, B, grad):
        out = torch.full((B, MS, MS), float("nan"), device=DEV)
        coef = scratch_bytes(lib.sdr_pairwise_neg_sdr_coef_bytes(B, MS))
        sc = scratch_bytes(lib.sdr_pairwise_neg_sdr_train_scratch_bytes(B, MS, MT))
        N.check(lib.sdr_pairwise_neg_sdr_train(p(e), p(t), p(out), p(coef), B, MS, MT, 1, 1, 1, p(sc), stream()))
        N.check(lib.sdr_pairwise_neg_sdr_backward(p(e), p(t), p(coef), p(gout), p(grad), B, MS, MT, stream()))

    def snr(e, t, gv, B, grad):
        val = torch.full((B,), float("nan"), device=DEV)
        perm = torch.zeros(B, dtype=torch.int32, device=DEV)
        coef = scratch_bytes(lib.sdr_snr_zero_refs_coef_bytes(B, MS))
        sc = scratch_bytes(lib.sdr_snr_zero_refs_scratch_bytes(B, MS, MT))
        N.check(lib.sdr_snr_zero_refs(p(e), p(t), p(val), p(perm), p(coef), B, MS, MT, 0, -40.0, 1e-8, p(sc),
                                      stream()))
        N.check(lib.sdr_snr_zero_refs_backward(p(e), p(t), p(coef), p(gv), p(grad), B, MS, MT, MT, stream()))

    grad = nan_guarded(MB, MS, MT)
    grad1 = nan_guarded(1, MS, MT)
    for name, fn, gin in (("pairwise", pairwise, gpw), ("snr_zero_refs", snr, gval)):
        grad.fill_(float("nan"))
        grad1.fill_(float("nan"))
        fn(est, tgt, gin, MB, grad)
        fn(est[-1:], tgt[-1:], gin[-1:].contiguous(), 1, grad1)
        torch.cuda.synchronize()
        assert_guards_intact(grad, name)
        assert_guards_intact(grad1, name)
        assert_rows_equal(grad[-1:], grad1)
        assert torch.isfinite(grad[0, :, :SUB]).all(), name


@gpu
@pytest.mark.parametrize("kind", ["uniform", "magsq"])
def test_mixture_consistency_backward_past_2_31_elements(kind):
    """sdr_mixture_consistency_backward (and, for magsq, its per-chunk power pass) on est [5, 2, 270 M]: the last
    item's rows start past 2^31.  grad_est and grad_mix bitwise against the call on the last item alone; for the
    uniform weights, which act position by position, fp64 autograd of the oracle on its last positions."""
    lib = N.lib()
    wt = 0 if kind == "uniform" else 1
    past((MB - 1) * MS * MT)
    need(3.2 * MB * MS * MT * 4 / GiB + 2)
    g = torch.Generator(device=DEV).manual_seed(223)
    est = torch.randn(MB, MS, MT, device=DEV, generator=g)
    mix = torch.randn(MB, 1, MT, device=DEV, generator=g)
    gout = est                                               # any [B, S, T] input does: the same buffer, read only

    def run(e, m, go, B):
        ge, gm = nan_guarded(B, MS, MT), nan_guarded(B, 1, MT)
        sc = scratch_bytes(lib.sdr_mixture_consistency_backward_scratch_bytes(B, MS, MT, wt))
        N.check(lib.sdr_mixture_consistency_backward(p(e), p(m), p(go), p(ge), p(gm), B, MS, MT, wt, p(sc), stream()))
        return ge, gm

    ge, gm = run(est, mix, gout, MB)
    ge1, gm1 = run(est[-1:], mix[-1:], gout[-1:], 1)
    torch.cuda.synchronize()
    for t, what in ((ge, "grad_est"), (gm, "grad_mix"), (ge1, "grad_est (small)"), (gm1, "grad_mix (small)")):
        assert_guards_intact(t, what)
    assert_rows_equal(ge[-1:], ge1)
    assert_rows_equal(gm[-1:], gm1)
    assert torch.isfinite(ge[0, :, :SUB]).all() and torch.isfinite(gm[0, :, :SUB]).all()
    if kind == "uniform":
        e64 = est[-1:, :, -P_REF:].double().requires_grad_(True)
        m64 = mix[-1:, :, -P_REF:].double().requires_grad_(True)
        (O.mixture_consistency(e64, m64) * gout[-1:, :, -P_REF:].double()).sum().backward()
        assert max(O.parity_errors(ge1[..., -P_REF:], e64.grad)) < 1e-6
        assert max(O.parity_errors(gm1[..., -P_REF:], m64.grad)) < 1e-6


# =====================================================================================================================
# backward stage kernels
# =====================================================================================================================
L_BWD = 1048592              # BIG_S x BIG_C x L_BWD: the last sample starts past 2^31


@gpu
def test_norm_act_backward_past_2_31_elements():
    """sdr_norm_act_backward of PReLU(GlobLN(x)) (norm_bwd_reduce_kernel, norm_bwd_apply_kernel): dx of the last
    sample bitwise against the call on that sample alone (its statistics), and fp64 autograd; dgamma, dbeta and
    dslope, which sum over every sample, against fp64 autograd accumulated sample by sample."""
    lib = N.lib()
    L = L_BWD
    past((BIG_S - 1) * BIG_C * L)
    need(3 * BIG_S * BIG_C * L * 4 / GiB + 2)
    g = torch.Generator(device=DEV).manual_seed(227)
    x = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g).mul_(1.5).add_(0.2)
    dp = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    gamma = 1 + 0.3 * torch.randn(BIG_C, device=DEV, generator=g)
    beta = 0.2 * torch.randn(BIG_C, device=DEV, generator=g)
    slope = torch.tensor([0.27], device=DEV)
    st = sample_stats(x)

    def run(xx, dd, stats, samples):
        fin = norm_in(stats, gamma, beta, slope, BIG_C * L)
        dx = nan_guarded(samples, BIG_C, L)
        dg, db, da = (torch.full((n,), float("nan"), device=DEV) for n in (BIG_C, BIG_C, 1))
        sc = scratch_bytes(lib.sdr_norm_act_backward_scratch_bytes(samples, BIG_C))
        N.check(lib.sdr_norm_act_backward(p(xx), C.byref(fin), p(dd), p(dx), 0, p(dg), p(db), p(da), p(sc), samples,
                                          BIG_C, L, stream()))
        return dx, dg, db, da

    dx, dg, db, da = run(x, dp, st, BIG_S)
    st1 = st[-1:].clone()
    dx1, _, _, _ = run(x[-1:], dp[-1:], st1, 1)
    torch.cuda.synchronize()
    assert_guards_intact(dx, "dx")
    assert_guards_intact(dx1, "dx (small)")
    assert_rows_equal(dx[-1:], dx1)
    assert torch.isfinite(dx[0, :SUB]).all()
    del dx
    g64, b64, a64 = (t.double().requires_grad_(True) for t in (gamma, beta, slope))
    for b in range(BIG_S):
        x64 = x[b:b + 1].double().requires_grad_(b == BIG_S - 1)
        (ref_norm_act(x64, g64, b64, a64) * dp[b:b + 1].double()).sum().backward()
    check_grad(dx1, x64.grad, "dx of the last sample", 1e-4)
    check_grad(dg, g64.grad, "dgamma")
    check_grad(db, b64.grad, "dbeta")
    check_grad(da, a64.grad, "dslope")


DW_BWD = [("stride1", 1, 0), ("stride2_pool", 2, 1)]


@gpu
@pytest.mark.parametrize("name,stride,pool", DW_BWD, ids=[c[0] for c in DW_BWD])
def test_depthwise_backward_past_2_31_elements(name, stride, pool):
    """sdr_depthwise_backward (dw_bwd_kernel, dw_finish_kernel) of z = dw5(GlobLN(x)), stride 1, and stride 2 with
    the merge's pooled gradient added: dx of the last SUB channels of the last sample bitwise against the call on
    them alone, and fp64; dw5 and dbias against fp64 autograd accumulated sample by sample."""
    lib = N.lib()
    Lin = L_BWD
    Lout = Lin // stride
    past((BIG_S - 1) * BIG_C * Lin)
    need(BIG_S * BIG_C * (2 * Lin + Lout + pool * Lin) * 4 / GiB + 2)
    g = torch.Generator(device=DEV).manual_seed(229 + stride)
    x = torch.randn(BIG_S, BIG_C, Lin, device=DEV, generator=g).add_(0.1)
    dz = torch.randn(BIG_S, BIG_C, Lout, device=DEV, generator=g)
    dm = torch.randn(BIG_S, BIG_C, Lin * pool, device=DEV, generator=g) if pool else None
    gamma = 1 + 0.3 * torch.randn(BIG_C, device=DEV, generator=g)
    beta = 0.2 * torch.randn(BIG_C, device=DEV, generator=g)
    w5 = 0.4 * torch.randn(BIG_C, 5, device=DEV, generator=g)
    st = sample_stats(x)

    def run(dzz, xx, stats, gm, bt, w, dmm, samples, C_):
        fin = norm_in(stats, gm, bt, None, BIG_C * Lin)
        dx = nan_guarded(samples, C_, Lin)
        dw, db = torch.full((C_, 5), float("nan"), device=DEV), torch.full((C_,), float("nan"), device=DEV)
        sc = scratch_bytes(lib.sdr_depthwise_backward_scratch_bytes(samples, C_))
        N.check(lib.sdr_depthwise_backward(p(dzz), p(xx), C.byref(fin), p(w), p(dmm), pool, p(dx), p(dw), p(db),
                                           p(sc), samples, C_, Lin, stride, stream()))
        return dx, dw, db

    dx, dw, db = run(dz, x, st, gamma, beta, w5, dm, BIG_S, BIG_C)
    parts = last_sample_parts(dz, x) + (last_sample_parts(dm) if pool else [None])
    dzs, xs, dms = parts
    st1 = st[-1:].clone()
    gs, bs_, ws = gamma[-SUB:].contiguous(), beta[-SUB:].contiguous(), w5[-SUB:].contiguous()
    dx1, _, _ = run(dzs, xs, st1, gs, bs_, ws, dms, 1, SUB)
    torch.cuda.synchronize()
    assert_guards_intact(dx, "dx")
    assert_guards_intact(dx1, "dx (small)")
    assert_rows_equal(dx[-1, -SUB:], dx1[0])
    assert torch.isfinite(dx[0, :SUB]).all()
    del dx
    w64 = w5.double().requires_grad_(True)
    b64 = torch.zeros(BIG_C, dtype=torch.float64, device=DEV, requires_grad=True)
    for b in range(BIG_S):
        n = ref_glob(x[b], st[b], gamma, beta, BIG_C * Lin).unsqueeze(0)
        z = F.conv1d(n, w64.unsqueeze(1), b64, stride=stride, padding=2, groups=BIG_C)
        (z * dz[b:b + 1].double()).sum().backward()
    check_grad(dw, w64.grad, f"dw5 {name}")
    check_grad(db, b64.grad, f"dbias {name}")
    want = F.conv_transpose1d(dzs.double(), ws.double().unsqueeze(1), None, stride=stride, padding=2,
                              output_padding=stride - 1, groups=SUB)
    if pool:
        want = want + dms.double().reshape(1, SUB, Lin, pool).sum(-1)
    check_grad(dx1, want, f"dx {name}")


@gpu
def test_mask_backward_past_2_31_elements():
    """sdr_mask_backward (mask_bwd_kernel) of masked = relu(mlog) x enc at B = 33, S = 4, N = 16: dmlog (in place
    over dmasked) and denc of the last item bitwise against the call on it alone, and fp64."""
    B, S, N_, L = BIG_S, 4, 16, L_BWD
    past((B - 1) * S * N_ * L)
    need(B * (2 * S * N_ + 2 * N_) * L * 4 / GiB + 2)
    g = torch.Generator(device=DEV).manual_seed(233)
    mlog = torch.randn(B, S * N_, L, device=DEV, generator=g)
    enc = torch.randn(B, N_, L, device=DEV, generator=g)
    dml = torch.randn(B, S * N_, L, device=DEV, generator=g)
    dmk1 = dml[-1:].clone()
    dml1 = dmk1.clone()
    de = nan_guarded(B, N_, L)
    de1 = nan_guarded(1, N_, L)
    N.check(N.lib().sdr_mask_backward(p(mlog), p(enc), p(dml), p(de), B, S, N_, L, stream()))
    N.check(N.lib().sdr_mask_backward(p(mlog[-1:]), p(enc[-1:]), p(dml1), p(de1), 1, S, N_, L, stream()))
    torch.cuda.synchronize()
    assert_guards_intact(de, "denc")
    assert_guards_intact(de1, "denc (small)")
    assert_rows_equal(dml[-1:], dml1)
    assert_rows_equal(de[-1:], de1)
    assert torch.isfinite(de[0, :SUB]).all() and not torch.equal(dml[0, :SUB], dml[-1, :SUB])
    m64 = mlog[-1:].double().view(1, S, N_, L)
    dk64 = dmk1.double().view(1, S, N_, L)
    e64 = enc[-1:].double().unsqueeze(1)
    assert max(O.parity_errors(dml1, (dk64 * (m64 > 0) * e64).view(1, S * N_, L))) < 1e-6
    assert max(O.parity_errors(de1, (dk64 * torch.relu(m64)).sum(1))) < 1e-6


@gpu
def test_overlap_add_backward_past_2_31_elements():
    """sdr_overlap_add_backward (frame_gather_kernel): grad_frames [33, 2 x 21, L] with the last item past 2^31,
    bitwise against the call on the last item alone, which is held exactly to the gather it states."""
    B, SA, K = BIG_S, 2, 21
    hop = K // 2
    L = 2 ** 31 // ((B - 1) * SA * K) + 16
    T = hop * L - 3
    past((B - 1) * SA * K * L)
    need(B * SA * (K * L + T) * 4 / GiB + 2)
    gout = torch.randn(B, SA, T, device=DEV, generator=torch.Generator(device=DEV).manual_seed(239))
    dF = nan_guarded(B, SA * K, L)
    dF1 = nan_guarded(1, SA * K, L)
    N.check(N.lib().sdr_overlap_add_backward(p(gout), p(dF), B, SA, K, L, T, stream()))
    N.check(N.lib().sdr_overlap_add_backward(p(gout[-1:]), p(dF1), 1, SA, K, L, T, stream()))
    torch.cuda.synchronize()
    assert_guards_intact(dF, "grad_frames")
    assert_guards_intact(dF1, "grad_frames (small)")
    assert_rows_equal(dF[-1:], dF1)
    assert torch.isfinite(dF[0, :SUB]).all()
    del dF
    for s in range(SA):
        for j in range(K):
            idx = hop * torch.arange(L, device=DEV) + j - hop
            ok = (idx >= 0) & (idx < T)
            want = torch.where(ok, gout[-1, s, idx.clamp(0, T - 1)], torch.zeros((), device=DEV))
            assert torch.equal(dF1[0, s * K + j], want), (s, j)


@gpu
def test_encoder_wgrad_past_2_31_elements():
    """sdr_encoder_wgrad (wgrad_partial_kernel, wgrad_reduce_kernel) over denc [33, 64, L] past 2^31: dW against fp64
    autograd accumulated item by item."""
    lib = N.lib()
    B, N_, K, L = BIG_S, BIG_C, 21, L_BWD
    hop = K // 2
    T = hop * L
    past((B - 1) * N_ * L)
    need(B * N_ * L * 4 / GiB + 2)
    g = torch.Generator(device=DEV).manual_seed(241)
    de = torch.randn(B, N_, L, device=DEV, generator=g)
    wav = torch.randn(B, 1, T, device=DEV, generator=g)
    dw = torch.full((N_, K), float("nan"), device=DEV)
    sc = scratch_bytes(lib.sdr_encoder_wgrad_scratch_bytes(B, N_, K, L))
    N.check(lib.sdr_encoder_wgrad(p(de), p(wav), p(dw), p(sc), B, N_, K, L, T, stream()))
    torch.cuda.synchronize()
    W = torch.zeros(N_, 1, K, dtype=torch.float64, device=DEV, requires_grad=True)
    for b in range(B):
        e = F.conv1d(wav[b:b + 1].double(), W, None, stride=hop, padding=hop)
        assert e.shape[-1] == L
        (e * de[b:b + 1].double()).sum().backward()
    check_grad(dw, W.grad.view(N_, K), "encoder dW")


@gpu
def test_pointwise_wgrad_past_2_31_elements():
    """sdr_pointwise_wgrad (wgrad_partial_kernel, wgrad_reduce_kernel) of y = W PReLU(GlobLN(x)) + b over dy and x of
    [33, 64, L] past 2^31: dW and db against fp64 accumulated sample by sample."""
    lib = N.lib()
    M = K = BIG_C
    L = L_BWD
    past((BIG_S - 1) * M * L)
    need(2 * BIG_S * M * L * 4 / GiB + 2)
    g = torch.Generator(device=DEV).manual_seed(251)
    dy = torch.randn(BIG_S, M, L, device=DEV, generator=g)
    x = torch.randn(BIG_S, K, L, device=DEV, generator=g).mul_(2).add_(0.3)
    gamma = 1 + 0.3 * torch.randn(K, device=DEV, generator=g)
    beta = 0.2 * torch.randn(K, device=DEV, generator=g)
    slope = torch.tensor([0.3], device=DEV)
    st = sample_stats(x)
    fin = norm_in(st, gamma, beta, slope, K * L)
    dw = torch.full((M, K), float("nan"), device=DEV)
    db = torch.full((M,), float("nan"), device=DEV)
    sc = scratch_bytes(lib.sdr_pointwise_wgrad_scratch_bytes(BIG_S, M, K, L))
    N.check(lib.sdr_pointwise_wgrad(p(dy), p(x), C.byref(fin), p(dw), p(db), p(sc), BIG_S, M, K, L, stream()))
    torch.cuda.synchronize()
    dw64 = torch.zeros(M, K, dtype=torch.float64, device=DEV)
    db64 = torch.zeros(M, dtype=torch.float64, device=DEV)
    for b in range(BIG_S):
        f = ref_glob(x[b], st[b], gamma, beta, K * L, slope)
        d = dy[b].double()
        dw64 += d @ f.T
        db64 += d.sum(1)
    check_grad(dw, dw64, "pointwise dW")
    check_grad(db, db64, "pointwise db")


# =====================================================================================================================
# whole models
# =====================================================================================================================
BIG_MODELS = [
    # y = B x 512 x 15360 on the fused pyramid (D = 4, the longest rows it takes)
    ("improved_pyramid", "improved", imp(2, 21, 64, Co=128, Ci=512, D=4), 153600),
    # the TAC tensor B x 16 groups x 16 channels x L on tac_mma16_kernel
    ("groupcomm_tac", "groupcomm", gc(2, 1, 21, 16, 16, 16, Ci=256, D=1), 10485800),
    # y = B x 512 x L through the causal pyramid
    ("causal", "causal", dict(in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=1,
                              upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64, num_sources=2), 5243040),
]


@gpu
@pytest.mark.parametrize("name,variant,kw,T", BIG_MODELS, ids=[c[0] for c in BIG_MODELS])
def test_model_past_2_31_elements(name, variant, kw, T):
    """A whole model whose pyramid input y (improved, causal) or TAC tensor (GroupComm) passes 2^31 elements, on the
    path asserted from the library's own queries: its last item against a B = 1 run and the fp64 oracle."""
    lib = N.lib()
    cfg = O.Config(variant=variant, **kw)
    L = O.padded_length(cfg, T) // cfg.hop
    assert O.padded_length(cfg, T) == T
    c = _engine.make_config(CLASSES[variant](**kw))
    D, U = cfg.upsampling_depth, cfg.num_blocks
    width = cfg.out_channels if variant == "groupcomm" else cfg.in_channels
    B = 2 ** 31 // (width * L) + 2
    past((B - 1) * width * L)
    n = lib.sdr_forward_launch_count_for(C.byref(c), B, T)
    if variant == "improved":
        assert B <= PYR_MAX_SAMPLES and lib.sdr_pyramid_scratch_bytes(B, cfg.in_channels, D, L) > 0
        assert n == 2 + U * (2 + 3) + 3, n                   # pyramid + solve, not D level launches
    elif variant == "groupcomm":
        assert cfg.out_channels // cfg.group_size == 16     # 16 channels per group: tac_mma16_kernel
        assert n in (2 + U * (D + 4) + 3, 2 + U * (D + 5) + 3), n
    else:
        assert n == 2 + 3 * U + 3, n                         # the causal pyramid in one launch per block
    ws = lib.sdr_workspace_bytes(C.byref(c), B, T)
    assert ws > 0
    need(ws / GiB + 2 * B * (1 + cfg.num_sources) * T * 4 / GiB + 2)
    cfg, sd, m = build(variant, kw, seed=257)
    x1 = normalised_input(1, 1, T, seed=263).to(DEV)
    ref = O.forward(cfg, sd, x1, dtype=torch.float64)        # first: the oracle's fp64 tensors are freed before the run
    torch.cuda.empty_cache()
    x = torch.randn(B, 1, T, device=DEV, generator=torch.Generator(device=DEV).manual_seed(269))
    x[-1] = x1[0]
    with torch.no_grad():
        one = m(x1)
        big = m(x)
    torch.cuda.synchronize()
    assert torch.isfinite(big[0]).all()
    last = big[-1:].clone()
    del big
    print(f"{name}: B = {B}, L = {L}, workspace {ws / GiB:.1f} GiB, {n} launches")
    assert_rows_close(last, one)
    e = O.parity_errors(last, ref)
    assert max(e) < TOL, e


# =====================================================================================================================
# STOI
# =====================================================================================================================
STOI_BIG = [
    # (name, fs, S, seconds, B, mixture): the rows past 2^31 and where they start
    ("input_rows", 44100, 2, 25, 975, True),     # the last reference and estimate rows start at 2,148,772,500 samples
    ("sig_rows", 8000, 2, 60, 900, False),       # the last estimate row of sig starts at 2,159,400,000 doubles
]
STOI_PERIOD = 7                                  # distinct items, tiled: a row read from the wrong item shows


def stoi_call(ref, est, mix, fs):
    """sdr_stoi on a poisoned scratch of exactly the queried size, outputs NaN inside guard bands."""
    lib = N.lib()
    B, S, T = ref.shape
    sc = poisoned(lib.sdr_stoi_scratch_bytes(B, S, T, fs), POISON_NAN)
    nan = torch.full((B, S), float("nan"), dtype=torch.float64, device=DEV)
    out, mout = guarded(nan), guarded(nan)
    N.check(lib.sdr_stoi(p(ref), p(est), p(mix), None, p(out), p(mout) if mix is not None else None, B, S, T, fs,
                         p(sc), stream()), "sdr_stoi")
    check_bands(sc, "scratch")
    assert_guards_intact(out, "stoi")
    assert_guards_intact(mout, "mix_stoi")
    return out, (mout if mix is not None else None)


@gpu
@pytest.mark.parametrize("name,fs,S,seconds,B,with_mix", STOI_BIG, ids=[c[0] for c in STOI_BIG])
def test_stoi_past_2_31_elements(name, fs, S, seconds, B, with_mix):
    """sdr_stoi with the last item's input rows past 2^31 samples (44.1 kHz) or its resampled estimate rows past 2^31
    doubles of the scratch (8 kHz); both also pass the spectra kernel's 2^20-CTA grid.  The last item bitwise against
    the same call on it alone, and against the fp64 restatement; the first item finite."""
    T = seconds * fs
    R = B * S
    g_ = math.gcd(SO.FS, fs)
    pr, qr = SO.FS // g_, fs // g_
    Tn = -(-T * pr // qr)
    M = -(-(Tn - 256) // 128) - 1
    work = (3 if with_mix else 2) * R * ((M + 3) // 4)
    print(f"\n{name}: last input row at {(R - 1) * T}, last estimate sig row at {(2 * R - 1) * Tn}, "
          f"spectra work items {work}")
    past(work, 1 << 20)
    if name == "input_rows":
        past((R - 1) * T)
    else:
        past((2 * R - 1) * Tn)
    lib = N.lib()
    need((2 * R + B) * T * 4 / GiB + lib.sdr_stoi_scratch_bytes(B, S, T, fs) / GiB + 1)
    g = torch.Generator(device=DEV).manual_seed(231)
    base = torch.randn(STOI_PERIOD, S, T, device=DEV, generator=g)
    base.mul_(torch.rand(STOI_PERIOD, S, 1, device=DEV, generator=g) + 0.1)
    base[:, :, T // 3:T // 2] *= 1e-3                   # a quiet stretch the mask drops
    noise = torch.randn(STOI_PERIOD, S, T, device=DEV, generator=g) * torch.linspace(
        0.1, 2.0, STOI_PERIOD, device=DEV).view(-1, 1, 1)
    idx = torch.arange(B, device=DEV) % STOI_PERIOD
    ref = base[idx]
    est = noise[idx].add_(ref)
    del noise
    mix = (base.sum(1) + 0.3 * torch.randn(STOI_PERIOD, T, device=DEV, generator=g))[idx] if with_mix else None
    del base
    d, m = stoi_call(ref, est, mix, fs)
    one = stoi_call(ref[-1:].contiguous(), est[-1:].contiguous(), None if mix is None else mix[-1:].contiguous(), fs)
    torch.cuda.synchronize()
    assert torch.isfinite(d[0]).all() and torch.isfinite(d[-1]).all(), (d[0], d[-1])
    assert torch.equal(d[-1:], one[0]), (d[-1], one[0])
    if with_mix:
        assert torch.isfinite(m[0]).all() and torch.equal(m[-1:], one[1]), (m[-1], one[1])
    xr, yr = ref[-1].cpu().double().numpy(), est[-1].cpu().double().numpy()
    mr = None if mix is None else mix[-1].cpu().double().numpy()
    for j in range(S):
        w, _, margin = SO.score(xr[j], [yr[j]] + ([] if mr is None else [mr]), fs)
        assert margin >= 1e-6, margin
        err = max(abs(float(d[-1, j]) - w[0]), abs(float(m[-1, j]) - w[1]) if with_mix else 0.0)
        print(f"{name}: source {j} |GPU - oracle| {err:.2e}")
        assert err <= 1e-9, (j, d[-1], m if m is None else m[-1], w)


# =====================================================================================================================
# the list of kernels and the cases that run them past 2^31 (no GPU)
# =====================================================================================================================
COVERED = {
    "dw_pyramid_kernel": ["test_fused_pyramid_past_2_32_elements", "test_level_writing_pyramid_past_2_31_elements"],
    "pyramid_solve_kernel": ["test_fused_pyramid_past_2_32_elements", "test_level_writing_pyramid_past_2_31_elements"],
    "merge_pyramid_kernel": ["test_level_writing_pyramid_past_2_31_elements"],
    "merge_wide_kernel": ["test_wide_merge_past_2_31_elements"],
    "causal_pyramid_kernel": ["test_causal_pyramid_past_2_31_elements", "test_model_past_2_31_elements"],
    "tac_mma16_kernel": ["test_tac_past_2_31_elements", "test_model_past_2_31_elements"],
    "tac_kernel": ["test_tac_past_2_31_elements"],
    "encoder_kernel": ["test_encoder_past_2_31_elements"],
    "pw_mma_kernel": ["test_encoder_past_2_31_elements"],
    "gram_kernel": ["test_metrics_past_2_31_elements", "test_loss_backward_past_2_31_elements"],
    "pit_finalize_kernel": ["test_metrics_past_2_31_elements"],
    "stab_finalize_kernel": ["test_metrics_past_2_31_elements"],
    "pairwise_finalize_kernel": ["test_metrics_past_2_31_elements"],
    "snr_zero_refs_finalize_kernel": ["test_metrics_past_2_31_elements"],
    "row_moments_kernel": ["test_metrics_past_2_31_elements"],
    "pairwise_backward_kernel": ["test_loss_backward_past_2_31_elements"],
    "snr_zero_refs_backward_kernel": ["test_loss_backward_past_2_31_elements"],
    "mc_bwd_partials_kernel": ["test_mixture_consistency_backward_past_2_31_elements"],
    "mc_bwd_coef_kernel": ["test_mixture_consistency_backward_past_2_31_elements"],
    "mc_bwd_apply_kernel": ["test_mixture_consistency_backward_past_2_31_elements"],
    "norm_bwd_reduce_kernel": ["test_norm_act_backward_past_2_31_elements"],
    "norm_bwd_apply_kernel": ["test_norm_act_backward_past_2_31_elements"],
    "dw_bwd_kernel": ["test_depthwise_backward_past_2_31_elements"],
    "dw_finish_kernel": ["test_depthwise_backward_past_2_31_elements"],
    "mask_bwd_kernel": ["test_mask_backward_past_2_31_elements"],
    "frame_gather_kernel": ["test_overlap_add_backward_past_2_31_elements"],
    "wgrad_partial_kernel": ["test_encoder_wgrad_past_2_31_elements", "test_pointwise_wgrad_past_2_31_elements"],
    "wgrad_reduce_kernel": ["test_encoder_wgrad_past_2_31_elements", "test_pointwise_wgrad_past_2_31_elements"],
    "stoi_filter_kernel": ["test_stoi_past_2_31_elements"],
    "stoi_resample_kernel": ["test_stoi_past_2_31_elements"],
    "stoi_mask_kernel": ["test_stoi_past_2_31_elements"],
    "stoi_spectra_kernel": ["test_stoi_past_2_31_elements"],
    "stoi_segment_kernel": ["test_stoi_past_2_31_elements"],
}


def test_past_2_31_kernel_list_is_in_step():
    """Every kernel listed exists in csrc/ and names cases of this module that exist; every kernel of backward.cu is
    listed except the training forward's mask and the weight transpose, which move no activation-sized gradient, and
    every kernel of stoi.cu is listed."""
    csrc = os.path.join(REPO, "sudo_rm_rf_b200", "csrc")
    src = {f: open(os.path.join(csrc, f)).read() for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))}
    defined = {k for s in src.values() for k in re.findall(r"\b(\w+_kernel)\s*\(", s)}
    for k, cases in COVERED.items():
        assert k in defined, k
        assert cases and all(callable(globals().get(c)) for c in cases), (k, cases)
    backward = set(re.findall(r"^(\w+_kernel)\(", src["backward.cu"], re.M)) - {"mask_apply_kernel", "transpose_kernel"}
    assert backward and backward <= set(COVERED), sorted(backward - set(COVERED))
    stoi = set(re.findall(r"__global__[^;{]*?\b(\w+_kernel)\s*\(", src["stoi.cu"]))
    assert len(stoi) == 5 and stoi <= set(COVERED), sorted(stoi - set(COVERED))
