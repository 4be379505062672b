"""Every specialisation the forwards dispatch, at the shapes where kernels go wrong, against fp64 torch references.

- every (ACT, MODE, STATS) instantiation of pw_mma_kernel, and both of its encoder (window) instantiations;
- shared nn.PReLU() slopes on both sides of 0 and of 1 in every kernel that applies one (the kernels pick
  max(y, s*y) or min(y, s*y) from the side of 1 the slope is on);
- the encoder modes of the models (left padding hop or 2*hop, bias + ReLU + statistics) on both encoder kernels;
- GroupComm's proj_1x1 with TAC's residual + norm fused into its operand load, and that residual + norm alone.

Every buffer a kernel is given sits between two guard bands of a fixed bit pattern: a write outside the tensor would
land in the neighbouring workspace segment of the model and show in no output, so the guards are checked after each
call, and the inputs are checked bitwise unchanged.
"""
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn.functional as F

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
from guards import GUARD, Guards, assert_guards_intact, guarded
from test_gpu_stages import channel_slopes, check_stats, close, norm_in, p, raw_stats, stream

DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLOPES = (0.2, -0.4, 0.0, 1.0, 1.7)     # shared PReLU slopes: the usual range, negative, zero, the boundary, above 1


def test_guard_helper_reports_writes_outside():
    for dtype in (torch.float32, torch.float64, torch.uint8):
        t = guarded(torch.ones(3, 8, dtype=dtype))
        t.fill_(7)                                   # the interior is the caller's
        assert_guards_intact(t, "interior writes")
        for where in (GUARD - 1, GUARD + t.numel()):
            t2 = guarded(torch.zeros(3, 8, dtype=dtype))
            t2._base[where] = 1                      # one element just before / just after the tensor
            with pytest.raises(AssertionError, match="written"):
                assert_guards_intact(t2, "stray write")


# ---------------------------------------------------------------------------------------------------------------------
# pw_mma_kernel<WINDOW, ACT, MODE, STATS>: every instantiation
# ---------------------------------------------------------------------------------------------------------------------
# ACT: 0 none, 1 shared slope, 2 per-channel slopes; MODE: 0 bias, 1 + residual, 2 ReLU * gate
MMA_INSTANCES = [(0, 0, False), (0, 0, True), (1, 0, False), (1, 0, True), (0, 1, False), (0, 1, True),
                 (1, 1, False), (1, 1, True), (0, 2, False), (0, 2, True), (1, 2, False), (1, 2, True),
                 (2, 0, False), (2, 0, True)]
MMA_SHAPES = [   # samples, M, K, L, GlobLN on the operand (MODE 1: in place when M fills whole 128-row tiles)
    (2, 128, 64, 200, False),     # a single k-block
    (3, 256, 192, 132, True),     # 3 k-blocks: the 2-stage ring's parity flips between tiles; ragged 2nd position tile
    (3, 42, 128, 36, True),       # 42 rows padded to one 128-row tile (decoder GEMM), L < 128
    (2, 300, 64, 332, True),      # 300 rows padded to 3 tiles, the 3rd position tile ragged
    (40, 512, 64, 332, True),     # 40 x 3 x 4 = 480 tiles: every persistent CTA runs three or four
]
MMA_GATE_SHAPES = [   # samples, M, K, L, GlobLN, gate_channels
    (2, 256, 64, 200, False, 128),
    (3, 768, 192, 132, True, 384),   # two sources
    (2, 768, 64, 36, True, 256),     # three sources
    (2, 768, 128, 332, True, 768),   # one source
    (2, 300, 64, 132, True, 128),    # padded rows, gate rows m % 128
    (40, 512, 64, 332, True, 256),   # many tiles per CTA
]
MMA_PARAMS = [(a, md, st, shape) for (a, md, st) in MMA_INSTANCES
              for shape in (MMA_GATE_SHAPES if md == 2 else MMA_SHAPES)]


def _mma_id(v):
    if isinstance(v, tuple):
        return "x".join(str(int(e)) for e in v)
    return str(int(v)) if isinstance(v, bool) else str(v)


@pytest.mark.gpu
@pytest.mark.parametrize("act,mode,stats,shape", MMA_PARAMS, ids=_mma_id)
def test_pointwise_mma_instantiation(act, mode, stats, shape):
    """pw_mma_kernel<false, act, mode, stats> via sdr_pointwise_mma; ACT 1 runs with every slope in SLOPES."""
    samples, M, K, L, use_norm = shape[:5]
    gate_ch = shape[5] if mode == 2 else 0
    in_place = mode == 1 and M % 128 == 0
    lib = N.lib()
    g = torch.Generator().manual_seed(31)
    x = (torch.randn(samples, K, L, generator=g) + 0.5).to(DEV)
    W = (torch.randn(M, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(M, generator=g).to(DEV)
    gamma = (1 + 0.3 * torch.randn(K, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(K, generator=g)).to(DEV)
    pc_slopes = channel_slopes(K, g)
    residual = torch.randn(samples, M, L, generator=g).to(DEV) if mode == 1 else None
    gate = torch.randn(samples, gate_ch, L, generator=g).to(DEV) if mode == 2 else None
    stats_in = raw_stats(x).to(DEV)
    nbytes = lib.sdr_pointwise_mma_packed_bytes(M, K)
    assert nbytes > 0
    wpk = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_pointwise_mma_pack(p(W), M, K, p(wpk), stream()))

    fx = O.glob_ln(x.double(), gamma.double(), beta.double()) if use_norm else x.double()
    if act == 2:
        fx = O.prelu_c(fx, pc_slopes.double())
    for slope in (SLOPES if act == 1 else (None,)):
        s_t = torch.tensor([slope], device=DEV) if act == 1 else None
        f = O.prelu1(fx, s_t.double()) if act == 1 else fx
        want = torch.einsum("mk,skl->sml", W.double(), f) + bias.double().view(1, -1, 1)
        if mode == 1:
            want = want + residual.double()
        if mode == 2:
            want = torch.relu(want) * gate.double()[:, torch.arange(M, device=DEV) % gate_ch, :]

        gd = Guards()
        xg = gd.input("x", x)
        wg = gd.input("packed weights", wpk)
        bg = gd.input("bias", bias)
        gg = gd.input("gate", gate) if mode == 2 else None
        if in_place:
            y = gd.output("y", residual)
            rg = y
        else:
            y = gd.output("y", torch.full((samples, M, L), float("nan"), device=DEV))
            rg = gd.input("residual", residual) if mode == 1 else None
        st = gd.output("stats", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
        prelu = pc_slopes if act == 2 else s_t
        nin = norm_in(stats_in if use_norm else None, gamma if use_norm else None, beta if use_norm else None,
                      prelu, K * L)
        N.check(lib.sdr_pointwise_mma(p(xg), C.byref(nin), p(wg), p(bg), p(rg), p(gg), gate_ch, p(y),
                                      p(st) if stats else p(None), samples, M, K, L, 1 if mode == 2 else 0, stream()))
        gd.check()
        e = O.parity_errors(y, want)
        assert max(e) < 5e-5, (slope, e)
        if stats:
            check_stats(st, want.float(), rtol=3e-5)
        else:
            assert not st.any()


# ---------------------------------------------------------------------------------------------------------------------
# encoder modes: FFMA (encoder_kernel) and wgmma (pw_mma_kernel<true, 0, 0, STATS>)
# ---------------------------------------------------------------------------------------------------------------------
ENC_CASES = [   # B, A, T, N, K, pad in hops, bias + ReLU, statistics
    (2, 1, 517, 512, 21, 1, True, True),     # the original model's encoder
    (2, 1, 517, 512, 21, 2, False, False),   # the causal model's (left padding 2 * hop)
    (1, 2, 333, 160, 41, 2, False, True),    # A * K = 82 taps straddle two 64-wide k-blocks; T % hop != 0
    (1, 2, 1000, 70, 41, 1, True, True),
    (3, 2, 15, 70, 21, 1, True, True),       # T < K
    (2, 1, 7, 32, 21, 2, True, False),       # T < K, padding 2 * hop
    (2, 1, 3001, 160, 11, 2, True, True),
    (8, 1, 12801, 512, 21, 2, False, True),  # 8 x 11 x 4 = 352 tiles: several per persistent CTA
    (2, 2, 333, 24, 21, 2, True, True),      # N < 32: the FFMA kernel only
    (2, 1, 100, 16, 11, 1, False, True),
]
ENC_PARAMS = [(path,) + c for c in ENC_CASES for path in ("ffma", "mma") if path == "ffma" or c[3] >= 32]


def ref_encoder(wav, w, bias, relu, hop, pad, L):
    """enc[b, n, p] = act(sum_{a,j} w[n, a, j] * wav[b, a, hop*p + j - pad] + bias[n]), wav zero outside [0, T)."""
    K, T = w.shape[-1], wav.shape[-1]
    right = max(0, hop * (L - 1) + K - pad - T)
    frames = F.pad(wav.double(), (pad, right)).unfold(-1, K, hop)[:, :, :L]     # [B, A, L, K]
    out = torch.einsum("bapj,naj->bnp", frames, w.double())
    if bias is not None:
        out = out + bias.double().view(1, -1, 1)
    return torch.relu(out) if relu else out


@pytest.mark.gpu
@pytest.mark.parametrize("path,B,A,T,N_,K,pad_hops,bias_relu,stats", ENC_PARAMS)
def test_encoder_modes(path, B, A, T, N_, K, pad_hops, bias_relu, stats):
    lib = N.lib()
    g = torch.Generator().manual_seed(37)
    hop = K // 2
    pad = pad_hops * hop
    L = (T + hop - 1) // hop + 1              # the last frames read past T
    wav = torch.randn(B, A, T, generator=g).to(DEV)
    w = (torch.randn(N_, A, K, generator=g) / (A * K) ** 0.5).to(DEV)
    bias = (0.3 * torch.randn(N_, generator=g)).to(DEV) if bias_relu else None
    want = ref_encoder(wav, w, bias, bias_relu, hop, pad, L)
    gd = Guards()
    wavg = gd.input("wav", wav)
    bg = gd.input("bias", bias) if bias_relu else None
    enc = gd.output("enc", torch.full((B, N_, L), float("nan"), device=DEV))
    st = gd.output("stats", torch.zeros(B, 2, dtype=torch.float64, device=DEV))
    stp = p(st) if stats else p(None)
    relu = 1 if bias_relu else 0
    if path == "ffma":
        wg = gd.input("weight", w)
        N.check(lib.sdr_encoder_ex(p(wavg), p(wg), p(bg), relu, pad, p(enc), stp, B, A, T, N_, K, L, stream()))
        tol, st_tol = 2e-5, 1e-5
    else:
        nbytes = lib.sdr_encoder_mma_packed_bytes(N_, A, K)
        assert nbytes > 0
        wpk = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        N.check(lib.sdr_encoder_mma_pack(p(w), N_, A, K, p(wpk), stream()))
        wg = gd.input("packed weights", wpk)
        N.check(lib.sdr_encoder_mma_ex(p(wavg), p(wg), p(bg), relu, pad, p(enc), stp, B, A, T, N_, K, L, stream()))
        tol, st_tol = 5e-5, 3e-5
    gd.check()
    close(enc, want, tol=tol)
    if stats:
        check_stats(st, want.float(), rtol=st_tol)
    else:
        assert not st.any()


# ---------------------------------------------------------------------------------------------------------------------
# GroupComm: x + GlobLN(o) fused into proj_1x1 (pw_tile_kernel<true, 16|32>, pw_small_kernel<true>), and on its own
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("samples,M,K,L", [
    (8, 32, 16, 3200),     # proj_1x1 of the published GroupComm models (32 <- 16 channels per group): pw_tile_kernel<true, 32>
    (6, 32, 16, 6400),     # ... at 16 kHz
    (8, 16, 32, 3200),     # 16 <- 32: pw_tile_kernel<true, 16>
    (6, 16, 32, 6400),
    (4, 48, 16, 800),      # M > 32: the tile kernel refuses the shape, pw_small_kernel<true> (three 16-row blocks)
    (3, 16, 48, 132),      # K > 32: pw_small_kernel<true>
])
def test_pointwise_preadd(samples, M, K, L):
    lib = N.lib()
    g = torch.Generator().manual_seed(41)
    x = torch.randn(samples, K, L, generator=g).to(DEV)
    o = (torch.randn(samples, K, L, generator=g) * 1.5 + 0.4).to(DEV)
    gamma = (1 + 0.3 * torch.randn(K, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(K, generator=g)).to(DEV)
    W = (torch.randn(M, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(M, generator=g).to(DEV)
    st_o = raw_stats(o).to(DEV)
    xt_want = x.double() + O.glob_ln(o.double(), gamma.double(), beta.double())
    y_want = torch.einsum("mk,skl->sml", W.double(), xt_want) + bias.double().view(1, -1, 1)
    gd = Guards()
    xg, og, Wg, bg = gd.input("x", x), gd.input("pre_add", o), gd.input("W", W), gd.input("bias", bias)
    xt = gd.output("xt", torch.full_like(x, float("nan")))
    y = gd.output("y", torch.full((samples, M, L), float("nan"), device=DEV))
    st = gd.output("stats", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    pn = norm_in(st_o, gamma, beta, None, K * L)
    N.check(lib.sdr_pointwise_preadd(p(xg), p(og), C.byref(pn), p(xt), p(Wg), p(bg), p(y), p(st),
                                     samples, M, K, L, stream()))
    gd.check()
    close(xt, xt_want)
    close(y, y_want, tol=3e-5)
    check_stats(st, y_want.float(), rtol=3e-5)
    # lengths the streaming kernels cannot load as float4 are refused before any launch
    assert lib.sdr_pointwise_preadd(p(xg), p(og), C.byref(pn), p(xt), p(Wg), p(bg), p(y), p(st),
                                    samples, M, K, L - 2, stream()) == -5


@pytest.mark.gpu
@pytest.mark.parametrize("samples,n,L", [(8, 16, 3200), (6, 8, 517), (3, 32, 36), (2, 4, 6400)])
def test_tac_apply(samples, n, L):
    g = torch.Generator().manual_seed(43)
    x = torch.randn(samples, n, L, generator=g).to(DEV)
    o = (torch.randn(samples, n, L, generator=g) * 0.7 - 0.3).to(DEV)
    gamma = (1 + 0.3 * torch.randn(n, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(n, generator=g)).to(DEV)
    want = x.double() + O.glob_ln(o.double(), gamma.double(), beta.double())
    gd = Guards()
    xg, og = gd.input("x", x), gd.input("o", o)
    out = gd.output("out", torch.full_like(x, float("nan")))
    nrm = norm_in(raw_stats(o).to(DEV), gamma, beta, None, n * L)
    N.check(N.lib().sdr_tac_apply(p(xg), p(og), C.byref(nrm), p(out), samples, n, L, stream()))
    gd.check()
    close(out, want)


# ---------------------------------------------------------------------------------------------------------------------
# shared PReLU slopes on every side, in every other kernel that applies one
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("samples,M,K,L", [
    (2, 130, 33, 100),     # pw_gemm_kernel<128, vec>
    (2, 128, 96, 130),     # pw_gemm_kernel<128, scalar>
    (3, 42, 1024, 200),    # pw_gemm_kernel<64, vec>
    (2, 48, 20, 26),       # pw_gemm_kernel<64, scalar>
    (2, 24, 96, 52),       # pw_gemm_kernel<32, vec>
    (2, 32, 16, 517),      # pw_gemm_kernel<32, scalar>
    (2, 64, 64, 64),       # pw_small_kernel<false>
    (3, 32, 32, 1604),     # pw_tile_kernel<false, 32>
    (4, 16, 32, 96),       # pw_tile_kernel<false, 16>
])
def test_pointwise_ffma_shared_slopes(samples, M, K, L):
    lib = N.lib()
    g = torch.Generator().manual_seed(47)
    x = (torch.randn(samples, K, L, generator=g) + 0.3).to(DEV)
    W = (torch.randn(M, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(M, generator=g).to(DEV)
    gamma = (1 + 0.3 * torch.randn(K, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(K, generator=g)).to(DEV)
    stats_in = raw_stats(x).to(DEV)
    fx = O.glob_ln(x.double(), gamma.double(), beta.double())
    for slope in SLOPES:
        s_t = torch.tensor([slope], device=DEV)
        want = torch.einsum("mk,skl->sml", W.double(), O.prelu1(fx, s_t.double())) + bias.double().view(1, -1, 1)
        gd = Guards()
        xg, Wg = gd.input("x", x), gd.input("W", W)
        y = gd.output("y", torch.full((samples, M, L), float("nan"), device=DEV))
        st = gd.output("stats", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
        nin = norm_in(stats_in, gamma, beta, s_t, K * L)
        N.check(lib.sdr_pointwise(p(xg), C.byref(nin), p(Wg), p(bias), p(None), p(None), 0, p(y), p(st),
                                  samples, M, K, L, 0, stream()))
        gd.check()
        e = O.parity_errors(y, want)
        assert max(e) < 3e-5, (slope, e)
        check_stats(st, want.float(), rtol=3e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,C_,L,stride", [
    (3, 32, 3200, 1), (2, 24, 104, 1), (2, 33, 6400, 2),   # dw5_wide_kernel (Lout % 8 == 0)
    (2, 16, 200, 2),                                       # dw5_vec_kernel
    (5, 7, 26, 1), (5, 7, 26, 2),                          # dw5_scalar_kernel
])
def test_depthwise_shared_slopes(samples, C_, L, stride):
    g = torch.Generator().manual_seed(53)
    x = (torch.randn(samples, C_, L, generator=g) * 2 + 0.7).to(DEV)
    gamma = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    w = torch.randn(C_, 1, 5, generator=g).to(DEV)
    b = torch.randn(C_, generator=g).to(DEV)
    stats_in = raw_stats(x).to(DEV)
    Lout = (L - 1) // stride + 1
    fx = O.glob_ln(x.double(), gamma.double(), beta.double())
    for slope in SLOPES:
        s_t = torch.tensor([slope], device=DEV)
        want = F.conv1d(O.prelu1(fx, s_t.double()), w.double(), b.double(), stride=stride, padding=2, groups=C_)
        gd = Guards()
        xg = gd.input("x", x)
        y = gd.output("y", torch.full((samples, C_, Lout), float("nan"), device=DEV))
        st = gd.output("stats", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
        nin = norm_in(stats_in, gamma, beta, s_t, C_ * L)
        N.check(N.lib().sdr_depthwise(p(xg), C.byref(nin), p(w), p(b), p(y), p(st), samples, C_, L, stride, stream()))
        gd.check()
        e = O.parity_errors(y, want)
        assert max(e) < 2e-5, (slope, e)
        check_stats(st, want)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,C_,L,D", [(3, 7, 48, 4), (2, 6, 1024, 6), (5, 32, 3200, 5)])
def test_depthwise_pyramid_shared_slopes(samples, C_, L, D):
    """Level 0 of sdr_depthwise_pyramid applies proj_1x1's PReLU on load; the merged output carries it through."""
    lib = N.lib()
    g = torch.Generator().manual_seed(59)
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.3).to(DEV)
    gy = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    by = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    ws = [torch.randn(C_, 1, 5, generator=g).to(DEV) * 0.6 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    gs = [(1 + 0.3 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    bes = [(0.2 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    stats_in = raw_stats(y).to(DEV)
    yn = O.glob_ln(y.double(), gy.double(), by.double())
    for slope in SLOPES:
        s_t = torch.tensor([slope], device=DEV)
        cur = O.prelu1(yn, s_t.double())
        levels = []
        for d in range(D):
            z = F.conv1d(cur, ws[d].double(), bs[d].double(), stride=1 if d == 0 else 2, padding=2, groups=C_)
            if d == 0:
                z0 = z
            cur = O.glob_ln(z, gs[d].double(), bes[d].double())
            levels.append(cur)
        for _ in range(D - 1):
            top = levels.pop()
            levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
        gd = Guards()
        yg = gd.input("y", y)
        scratch = gd.output("scratch", torch.zeros(lib.sdr_pyramid_scratch_bytes(samples, C_, D, L),
                                                   dtype=torch.uint8, device=DEV))
        zs = [gd.output(f"z{d}", torch.full((samples, C_, L >> d), float("nan"), device=DEV)) for d in range(D)]
        st0 = gd.output("stats0", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
        stm = gd.output("stats_m", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
        m = gd.output("m", torch.full((samples, C_, L), float("nan"), device=DEV))
        nin = norm_in(stats_in, gy, by, s_t, C_ * L)
        N.check(lib.sdr_depthwise_pyramid(p(yg), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(st0),
                                          p(scratch), D, samples, C_, L, stream()))
        N.check(lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(m), p(stm), samples, C_, L, stream()))
        gd.check()
        e = O.parity_errors(zs[0], z0)
        assert max(e) < 2e-5, (slope, e)
        check_stats(st0, z0)
        e = O.parity_errors(m, levels[0])
        assert max(e) < 5e-5, (slope, e)      # (the affine re-composition reorders fp32 roundings over D levels)
        check_stats(stm, levels[0], rtol=1e-4)


CAUSAL_SLOPES = [   # slope_in, per-level slopes (level d takes entry d): every level crosses to the other side of 1
    (-0.4, (1.7, -0.4, 1.0, 0.0, 1.7, 0.2)),
    (1.7, (0.0, 1.7, -0.4, 1.7, 0.3, 1.7)),
    (0.0, (1.0, 0.2, 1.7, -0.4, 1.7, 0.0)),
    (1.0, (-0.4, 1.7, 0.0, 1.7, -0.4, 1.0)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("samples,C_,L,D", [(2, 32, 3200, 4), (3, 7, 64, 5), (2, 16, 6400, 6)])
def test_causal_pyramid_shared_slopes(samples, C_, L, D):
    lib = N.lib()
    g = torch.Generator().manual_seed(61)
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.1).to(DEV)
    ws = [torch.randn(C_, 1, 21, generator=g).to(DEV) * 0.4 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    for s_in, s_lv in CAUSAL_SLOPES:
        sp = torch.tensor([s_in], device=DEV)
        sl = [torch.tensor([s_lv[d]], device=DEV) for d in range(D)]
        cur = O.prelu1(y.double(), sp.double())
        levels = []
        for d in range(D):
            cur = O.prelu1(F.conv1d(cur, O.causal_weight(ws[d].double()), bs[d].double(), stride=1 if d == 0 else 2,
                                    padding=10, groups=C_), sl[d].double())
            levels.append(cur)
        for _ in range(D - 1):
            top = levels.pop()
            levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
        gd = Guards()
        yg = gd.input("y", y)
        m = gd.output("m", torch.full((samples, C_, L), float("nan"), device=DEV))
        N.check(lib.sdr_causal_pyramid(p(yg), p(sp), arr(ws), arr(bs), arr(sl), p(m), D, samples, C_, L, stream()))
        gd.check()
        e = O.parity_errors(m, levels[0])
        assert max(e) < 2e-5, ((s_in, s_lv[:D]), e)


@pytest.mark.gpu
@pytest.mark.parametrize("B,G,n,L", [(2, 4, 16, 200), (3, 16, 16, 36), (2, 4, 8, 100), (2, 3, 32, 40)])
def test_tac_shared_slopes(B, G, n, L):
    """n = 16 runs on tensor cores (bf16x3), the other group widths on FFMA."""
    cfg = O.Config(variant="groupcomm", out_channels=G * n, in_channels=2 * G * n, num_blocks=1,
                   upsampling_depth=1, group_size=G)
    sd = {k[len("sm.0.TAC."):]: v.to(DEV) for k, v in O.make_state_dict(cfg, seed=9).items()
          if k.startswith("sm.0.TAC.")}
    x = torch.randn(B, G, n, L, generator=torch.Generator().manual_seed(67)).to(DEV)
    names = ["TAC_input.0.weight", "TAC_input.0.bias", "TAC_input.1.weight",
             "TAC_mean.0.weight", "TAC_mean.0.bias", "TAC_mean.1.weight",
             "TAC_output.0.weight", "TAC_output.0.bias", "TAC_output.1.weight"]
    slopes = ["TAC_input.1.weight", "TAC_mean.1.weight", "TAC_output.1.weight"]
    for triple in [(1.7, -0.4, 0.0), (-0.4, 1.0, 1.7), (0.0, 1.7, -0.4)]:
        for k, s in zip(slopes, triple):
            sd[k] = torch.tensor([s], device=DEV)
        taps = {}
        O.tac(x.double(), {k: v.double() for k, v in sd.items()}, "", taps)
        want = taps["TAC_output"]
        gd = Guards()
        xg = gd.input("x", x)
        o = gd.output("o", torch.full((B, G, n, L), float("nan"), device=DEV))
        st = gd.output("stats", torch.zeros(B * G, 2, dtype=torch.float64, device=DEV))
        params = (C.c_void_p * 9)(*[sd[k].data_ptr() for k in names])
        N.check(N.lib().sdr_tac(p(xg), params, p(o), p(st), B, G, n, L, stream()))
        gd.check()
        e = O.parity_errors(o, want)
        assert max(e) < (1e-4 if n == 16 else 2e-5), (triple, e)
        check_stats(st, want.reshape(B * G, n, L), rtol=1e-4 if n == 16 else 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("variant,kw,T", [
    ("improved", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
                      enc_num_basis=256, num_sources=2), 3000),
    ("groupcomm", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
                       enc_num_basis=64, num_sources=2, group_size=4), 3000),
    ("causal", dict(in_audio_channels=1, out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                    enc_kernel_size=21, enc_num_basis=64, num_sources=2), 3000),
])
def test_model_shared_slopes_either_side(variant, kw, T):
    """Every nn.PReLU() slope of the model (shape [1]: proj / final_norm / depthwise levels, TAC's three, mask_net's
    and the causal model's mask_nl_class) set to -0.3 or 1.4, so a slope read from the wrong place or taking the wrong
    branch changes the output."""
    cfg = O.Config(variant=variant, **kw)
    sd = O.make_state_dict(cfg, seed=71)
    shared = [k for k, v in sd.items() if tuple(v.shape) == (1,)]
    assert len(shared) >= 5
    for i, k in enumerate(shared):      # 0, 1, 1, 0, 0, 1, ...: neighbours differ and a role's value changes by block
        sd[k] = torch.tensor([(-0.3, 1.4)[(i + i // 2) % 2]])
    g = torch.Generator().manual_seed(73)
    cls = {"improved": P.SuDORMRF, "groupcomm": P.GroupCommSudoRmRf, "causal": P.CausalSuDORMRF}[variant]
    m = cls(**kw)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    x = torch.randn(2, kw.get("in_audio_channels", 1), T, generator=g)
    with torch.no_grad():
        y = m(x.to(DEV))
    e = O.parity_errors(y, O.forward(cfg, sd, x, dtype=torch.float64))
    assert max(e) < 1e-4, e


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the instantiation matrix above covers exactly what pointwise_mma.cu compiles
# ---------------------------------------------------------------------------------------------------------------------
def test_mma_instantiations_are_all_tested():
    src = open(os.path.join(REPO, "sudo_rm_rf_b200", "csrc", "pointwise_mma.cu")).read()
    b = {"true": True, "false": False}
    compiled = {(False, int(a), int(m), b[s])
                for a, m, s in re.findall(r"SDR_MMA_CASE\((\d+),\s*(\d+),\s*(true|false)\)", src)}
    compiled |= {(b[w], int(a), int(m), b[s])
                 for w, a, m, s in re.findall(r"pw_mma_kernel<(true|false),\s*(\d+),\s*(\d+),\s*(true|false)>", src)}
    assert len(compiled) >= 16
    tested = {(False, a, m, s) for a, m, s, _ in MMA_PARAMS}
    tested |= {(True, 0, 0, stats) for path, *_, stats in ENC_PARAMS if path == "mma"}
    assert compiled == tested, (sorted(compiled - tested), sorted(tested - compiled))
