"""Stage-level parity on the GPU: every per-stage C-ABI entry point against the
same torch ops the oracle uses (fp32).  Tolerances are fp32-reassociation
sized (these kernels are exact fp32 FFMA paths)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def norm_in(stats=None, gamma=None, beta=None, prelu=None, count=1.0):
    """prelu: 1 element = nn.PReLU(); more = one slope per channel (nn.PReLU(C) of the original model)."""
    return N.SdrNormIn(stats.data_ptr() if stats is not None else 0,
                       gamma.data_ptr() if gamma is not None else 0,
                       beta.data_ptr() if beta is not None else 0,
                       prelu.data_ptr() if prelu is not None else 0, float(count),
                       1 if prelu is not None and prelu.numel() > 1 else 0)


def channel_slopes(C_, g):
    """Per-channel PReLU slopes on both sides of 1 and of 0."""
    s = 0.1 + 0.5 * torch.rand(C_, generator=g)
    r = torch.rand(C_, generator=g)
    s = torch.where(r < 0.15, torch.full_like(s, -0.2), torch.where(r > 0.8, torch.full_like(s, 1.3), s))
    return s.to(DEV)


def raw_stats(x):
    """(sum, sumsq) per sample, fp64, as the producers accumulate them."""
    xd = x.double().reshape(x.shape[0], -1)
    return torch.stack([xd.sum(1), (xd * xd).sum(1)], dim=1).contiguous()


def check_stats(got, x, rtol=1e-5):
    want = raw_stats(x)
    n = x[0].numel()
    # the sum may cancel: its error is judged against sqrt(n * sumsq) >= sum|x|
    scale = torch.stack([(n * want[:, 1]).sqrt(), want[:, 1]], dim=1) + 1e-12
    assert ((got - want).abs() / scale).max() < rtol, (got, want)


def close(a, b, tol=2e-5):
    e = O.parity_errors(a, b)
    assert max(e) < tol, e


def ref_norm(x, gamma, beta, prelu=None):
    y = O.glob_ln(x, gamma, beta)
    if prelu is None:
        return y
    return O.prelu_c(y, prelu) if prelu.numel() > 1 else O.prelu1(y, prelu)


@pytest.mark.parametrize("samples,C_,L,stride,prelu", [
    (3, 32, 3200, 1, True), (2, 32, 3200, 2, False), (2, 16, 200, 2, False),
    (2, 24, 104, 1, True), (5, 7, 26, 1, False), (5, 7, 26, 2, False), (1, 3, 2, 2, False),
    (2, 512, 800, 2, False), (4, 5, 4, 1, True),
    (2, 9, 16, 1, False), (2, 9, 16, 2, True), (3, 6, 8, 1, True), (2, 512, 3200, 1, True),
    (2, 33, 6400, 2, False), (1, 4, 40, 1, False),
    (2, 64, 3200, 1, "pc"), (3, 24, 104, 1, "pc"), (2, 7, 26, 1, "pc"), (2, 9, 16, 2, "pc"),   # nn.PReLU(C) (sudormrf.py:33)
])
def test_depthwise(samples, C_, L, stride, prelu):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(samples, C_, L, generator=g) * 2 + 0.7).to(DEV)
    gamma = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    slope = channel_slopes(C_, g) if prelu == "pc" else (torch.tensor([0.3], device=DEV) if prelu else None)
    w = torch.randn(C_, 1, 5, generator=g).to(DEV)
    b = torch.randn(C_, generator=g).to(DEV)
    stats_in = raw_stats(x).to(DEV)
    Lout = (L - 1) // stride + 1
    y = torch.full((samples, C_, Lout), float("nan"), device=DEV)
    stats_out = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    nin = norm_in(stats_in, gamma, beta, slope, C_ * L)
    N.check(N.lib().sdr_depthwise(p(x), C.byref(nin), p(w), p(b), p(y), p(stats_out),
                                  samples, C_, L, stride, stream()))
    want = F.conv1d(ref_norm(x, gamma, beta, slope), w, b, stride=stride, padding=2, groups=C_)
    close(y, want)
    check_stats(stats_out, want)


@pytest.mark.parametrize("samples,C_,L,D,prelu", [
    (3, 512, 3200, 5, True),     # cfg 2 block
    (2, 512, 3200, 6, True),     # cfg 3 block (last level: 100 positions)
    (1, 512, 6400, 6, True),     # cfg 5 block
    (5, 32, 3200, 5, True),      # GroupComm rows
    (3, 7, 48, 4, True),         # shortest eligible rows: L >> (D-1) == 6, every run of the merge is an edge run
    (2, 5, 96, 5, False), (2, 3, 192, 6, True), (4, 9, 112, 4, True), (2, 6, 1024, 6, True), (300, 4, 448, 4, True),
    # one PReLU slope per channel (the original model's UBlock, sudormrf.py:33,171)
    (2, 512, 3200, 4, "pc"), (3, 64, 3200, 5, "pc"), (1, 32, 6400, 6, "pc"), (3, 7, 48, 4, "pc"), (2, 9, 80, 4, "pc"),
])
def test_depthwise_pyramid(samples, C_, L, D, prelu):
    """sdr_depthwise_pyramid + sdr_merge_pyramid == the level-by-level chain in torch (improved_sudormrf.py:205-216)."""
    lib = N.lib()
    g = torch.Generator().manual_seed(11)
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.3).to(DEV)
    gy = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    by = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    slope = channel_slopes(C_, g) if prelu == "pc" else (torch.tensor([0.3], device=DEV) if prelu else None)
    ws = [torch.randn(C_, 1, 5, generator=g).to(DEV) * 0.6 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    gs = [(1 + 0.3 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    bes = [(0.2 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    nbytes = lib.sdr_pyramid_scratch_bytes(samples, C_, D, L)
    assert nbytes > 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    zs = [torch.full((samples, C_, L >> d), float("nan"), device=DEV) for d in range(D)]
    st0 = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    stm = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    m = torch.full((samples, C_, L), float("nan"), device=DEV)
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    nin = norm_in(raw_stats(y).to(DEV), gy, by, slope, C_ * L)
    N.check(lib.sdr_depthwise_pyramid(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(st0),
                                      p(scratch), D, samples, C_, L, stream()))
    N.check(lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(m), p(stm), samples, C_, L, stream()))
    # reference chain
    cur = ref_norm(y, gy, by, slope)
    levels = []
    for d in range(D):
        z = F.conv1d(cur, ws[d], bs[d], stride=1 if d == 0 else 2, padding=2, groups=C_)
        if d == 0:
            close(zs[0], z)
            check_stats(st0, z)
        cur = ref_norm(z, gs[d], bes[d])
        levels.append(cur)
    for _ in range(D - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
    close(m, levels[0], tol=5e-5)            # the affine re-composition reorders fp32 roundings over D levels
    check_stats(stm, levels[0], rtol=1e-4)
    # not eligible: depth 3 or > 6, L not a multiple of 16, rows too short
    assert lib.sdr_pyramid_scratch_bytes(samples, C_, 7, 1024) == 0
    assert lib.sdr_pyramid_scratch_bytes(samples, C_, 3, L) == 0
    assert lib.sdr_pyramid_scratch_bytes(samples, C_, D, L + 8) == 0
    assert lib.sdr_pyramid_scratch_bytes(samples, C_, 6, 96) == 0


@pytest.mark.parametrize("samples,C_,L,D", [
    (2, 32, 3200, 4), (2, 32, 3200, 5), (1, 512, 3200, 4), (3, 7, 64, 5), (2, 5, 32, 5), (2, 9, 16, 2), (2, 4, 8, 1),
    (2, 16, 6400, 6), (1, 8, 4096, 4), (1, 8, 4160, 5), (2, 6, 256, 8), (2, 3, 48, 4),
])
def test_causal_pyramid(samples, C_, L, D):
    """sdr_causal_pyramid == PReLU -> D x (masked 21-tap depthwise conv + PReLU) -> upsample/add chain in torch
    (causal_improved_sudormrf_v3.py:106-116, mask :21-27)."""
    lib = N.lib()
    g = torch.Generator().manual_seed(13)
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.1).to(DEV)
    sp = torch.tensor([0.3], device=DEV)
    ws = [torch.randn(C_, 1, 21, generator=g).to(DEV) * 0.4 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    sl = [torch.tensor([0.1 + 0.07 * d], device=DEV) for d in range(D)]
    m = torch.full((samples, C_, L), float("nan"), device=DEV)
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    N.check(lib.sdr_causal_pyramid(p(y), p(sp), arr(ws), arr(bs), arr(sl), p(m), D, samples, C_, L, stream()))
    cur = O.prelu1(y, sp)
    levels = []
    for d in range(D):
        cur = O.prelu1(F.conv1d(cur, O.causal_weight(ws[d]), bs[d], stride=1 if d == 0 else 2, padding=10, groups=C_),
                       sl[d])
        levels.append(cur)
    for _ in range(D - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
    close(m, levels[0])
    # causality: the first half of the output does not depend on the second half of the input
    y2 = y.clone()
    y2[..., L // 2:] = 7.0
    m2 = torch.empty_like(m)
    N.check(lib.sdr_causal_pyramid(p(y2), p(sp), arr(ws), arr(bs), arr(sl), p(m2), D, samples, C_, L, stream()))
    assert torch.equal(m2[..., :L // 2], m[..., :L // 2])
    # lengths that do not halve D times are refused, not mis-computed
    assert lib.sdr_causal_pyramid(p(y), p(sp), arr(ws), arr(bs), arr(sl), p(m), D, samples, C_, L - 4, stream()) == -5 \
        or (L - 4) % (1 << D) == 0


@pytest.mark.parametrize("samples,C_,L,depth", [
    (2, 32, 3200, 5), (3, 16, 64, 6), (2, 8, 32, 1), (2, 5, 2, 1), (2, 6, 6, 2), (1, 512, 3200, 5),
    (2, 8, 48, 4), (2, 7, 128, 8), (3, 5, 24, 4), (2, 512, 6400, 6),
])
def test_merge(samples, C_, L, depth):
    g = torch.Generator().manual_seed(1)
    zs, gammas, betas, stats = [], [], [], []
    for d in range(depth):
        z = (torch.randn(samples, C_, L >> d, generator=g) + 0.3 * d).to(DEV)
        zs.append(z)
        gammas.append((1 + 0.3 * torch.randn(C_, generator=g)).to(DEV))
        betas.append((0.2 * torch.randn(C_, generator=g)).to(DEV))
        stats.append(raw_stats(z).to(DEV))
    fins = (N.SdrNormIn * depth)(*[norm_in(stats[d], gammas[d], betas[d], None, C_ * (L >> d))
                                  for d in range(depth)])
    zp = (C.c_void_p * depth)(*[z.data_ptr() for z in zs])
    m = torch.full((samples, C_, L), float("nan"), device=DEV)
    st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_merge(zp, fins, depth, p(m), p(st), samples, C_, L, stream()))
    levels = [ref_norm(zs[d], gammas[d], betas[d]) for d in range(depth)]
    for _ in range(depth - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
    close(m, levels[0])
    check_stats(st, levels[0])


@pytest.mark.parametrize("samples,M,K,L,mode", [
    (2, 256, 512, 3200, "norm"),          # bottleneck-like
    (2, 512, 256, 640, "plain_stats"),    # proj_1x1
    (2, 256, 512, 640, "res"),            # res_conv + skip (in place)
    (2, 1024, 256, 384, "mask"),          # mask_net + relu * encoder
    (3, 42, 1024, 200, "plain"),          # decoder GEMM (BM=64 tile)
    (4, 32, 16, 3200, "plain_stats"),     # groupcomm proj (BM=32 tile)
    (4, 16, 32, 96, "res"),               # groupcomm res
    (2, 48, 20, 26, "norm"),              # odd sizes, scalar path (L % 4 != 0)
    (2, 130, 33, 100, "res"),             # M, K not multiples of the tile
    (1, 7, 5, 2, "mask"),
    (32, 32, 16, 3200, "plain_stats"),    # small-channel streaming kernel, two 16-channel output tiles
    (32, 16, 32, 3200, "res"),            # ... with normalised + PReLU input and in-place skip
    (3, 24, 8, 132, "norm"),              # ... M not a multiple of 16, ragged last quad chunk
    (2, 64, 64, 64, "mask"),              # ... largest shape it takes
    (2, 8, 4, 4, "plain_stats"),
    (3, 32, 32, 1604, "norm"), (5, 20, 12, 1604, "res"), (300, 16, 32, 800, "res"),   # tile-staged kernel: ragged last tile, many CTAs
    (2, 32, 16, 517, "pc"), (2, 24, 32, 52, "pc"), (2, 128, 96, 130, "pc"), (2, 16, 64, 3200, "pc"),   # per-channel PReLU slopes
])
def test_pointwise(samples, M, K, L, mode):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(samples, K, L, generator=g) + 0.5).to(DEV)
    W = (torch.randn(M, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(M, generator=g).to(DEV)
    gamma = (1 + 0.3 * torch.randn(K, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(K, generator=g)).to(DEV)
    slope = torch.tensor([0.2], device=DEV)
    stats_in = raw_stats(x).to(DEV)
    y = torch.full((samples, M, L), float("nan"), device=DEV)
    st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    residual = gate = None
    gate_ch = 0
    epi = 0
    if mode == "norm":
        nin = norm_in(stats_in, gamma, beta, None, K * L)
        fx = ref_norm(x, gamma, beta)
    elif mode == "pc":
        slopes = channel_slopes(K, g)
        nin = norm_in(stats_in, gamma, beta, slopes, K * L)
        fx = ref_norm(x, gamma, beta, slopes)
    elif mode == "res":
        nin = norm_in(stats_in, gamma, beta, slope, K * L)
        fx = ref_norm(x, gamma, beta, slope)
        residual = torch.randn(samples, M, L, generator=g).to(DEV)
        y = residual.clone()                  # in-place skip connection
    elif mode == "mask":
        nin = norm_in(None, None, None, slope, 1.0)
        fx = O.prelu1(x, slope)
        gate_ch = max(1, M // 2) if M % 2 == 0 else M
        gate = torch.randn(samples, gate_ch, L, generator=g).to(DEV)
        epi = 1
    else:
        nin = norm_in()
        fx = x
    want = torch.einsum("mk,skl->sml", W.double(), fx.double()) + bias.double().view(1, -1, 1)
    if mode in ("res", "res_out"):
        want = want + residual.double()
        res_ptr = p(y)
    else:
        res_ptr = p(None)
    if mode == "mask":
        idx = torch.arange(M, device=DEV) % gate_ch
        want = torch.relu(want) * gate.double()[:, idx, :]
    want_stats = mode in ("plain_stats", "pc")
    N.check(N.lib().sdr_pointwise(p(x), C.byref(nin), p(W), p(bias), res_ptr, p(gate), gate_ch,
                                  p(y), p(st) if want_stats else p(None),
                                  samples, M, K, L, epi, stream()))
    close(y, want.float(), tol=3e-5)
    if want_stats:
        check_stats(st, want.float(), rtol=3e-5)


@pytest.mark.parametrize("B,A,T,N_,K,D", [
    (2, 1, 32000, 512, 21, 5), (3, 1, 517, 24, 21, 3), (2, 1, 100, 32, 21, 5),
    (2, 2, 333, 16, 11, 3), (1, 1, 7, 70, 21, 1), (1, 1, 3000, 64, 91, 4),
])
def test_encoder(B, A, T, N_, K, D):
    g = torch.Generator().manual_seed(3)
    cfg = O.Config(enc_kernel_size=K, upsampling_depth=D)
    Tp = O.padded_length(cfg, T)
    hop = K // 2
    L = Tp // hop
    wav = torch.randn(B, A, T, generator=g).to(DEV)
    w = torch.randn(N_, A, K, generator=g).to(DEV)
    enc = torch.full((B, N_, L), float("nan"), device=DEV)
    st = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_encoder(p(wav), p(w), p(enc), p(st), B, A, T, N_, K, L, stream()))
    # fp64 reference: an fp32 cuDNN convolution may run in TF32 (~1e-3 relative), far above the kernel's error
    xp = torch.zeros(B, A, Tp, device=DEV, dtype=torch.float64)
    xp[..., :T] = wav
    want = F.conv1d(xp, w.double(), None, stride=hop, padding=hop)
    assert want.shape[-1] == L
    close(enc, want)
    check_stats(st, want.float())


@pytest.mark.parametrize("B,A,T,N_,K,D", [
    (2, 1, 32000, 512, 21, 5), (3, 1, 517, 48, 21, 3), (2, 1, 100, 32, 21, 5),
    (2, 2, 333, 160, 11, 3), (1, 1, 7, 70, 21, 1), (1, 1, 3000, 64, 91, 4), (40, 1, 6400, 256, 21, 5),
])
def test_encoder_tensor_core(B, A, T, N_, K, D):
    """Encoder on the wgmma kernel (window operand, bf16x3)."""
    lib = N.lib()
    g = torch.Generator().manual_seed(3)
    cfg = O.Config(enc_kernel_size=K, upsampling_depth=D)
    Tp = O.padded_length(cfg, T)
    hop = K // 2
    L = Tp // hop
    wav = torch.randn(B, A, T, generator=g).to(DEV)
    w = torch.randn(N_, A, K, generator=g).to(DEV)
    nbytes = lib.sdr_encoder_mma_packed_bytes(N_, A, K)
    assert nbytes > 0
    wpk = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_encoder_mma_pack(p(w), N_, A, K, p(wpk), stream()))
    enc = torch.full((B, N_, L), float("nan"), device=DEV)
    st = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
    N.check(lib.sdr_encoder_mma(p(wav), p(wpk), p(enc), p(st), B, A, T, N_, K, L, stream()))
    xp = torch.zeros(B, A, Tp, device=DEV, dtype=torch.float64)
    xp[..., :T] = wav
    want = F.conv1d(xp, w.double(), None, stride=hop, padding=hop)
    assert want.shape[-1] == L
    close(enc, want, tol=5e-5)
    check_stats(st, want.float(), rtol=3e-5)


OVERLAP_ADD = [
    (2, 2, 21, 3200, 32000, False), (2, 2, 21, 3232, 32079, True), (3, 3, 21, 64, 640, False),
    (2, 4, 11, 72, 333, False), (1, 2, 21, 32, 7, True), (1, 2, 91, 80, 3000, False),
    # filter lengths 3 .. 201 (hop 1 .. 100), 1 / 3 / 5 / 16 outputs, T < K, T not a multiple of the hop, mixture
    # consistency where 1/SA != 0.5
    (2, 1, 3, 40, 37, True), (3, 5, 3, 333, 333, False), (2, 3, 5, 50, 99, True), (1, 5, 7, 30, 89, True),
    (2, 16, 7, 20, 58, False), (2, 16, 41, 8, 30, True), (1, 3, 41, 40, 799, False), (2, 16, 91, 12, 517, True),
    (2, 1, 91, 3, 50, False), (1, 3, 201, 6, 150, True), (2, 1, 201, 20, 1999, False), (1, 16, 201, 4, 399, True),
]


@pytest.mark.parametrize("B,SA,K,L,T,mc", OVERLAP_ADD)
def test_overlap_add(B, SA, K, L, T, mc):
    """Against conv_transpose1d + crop (and mixture consistency) in fp64."""
    g = torch.Generator().manual_seed(4)
    hop = K // 2
    assert T <= hop * L
    C_ = 6
    masked = torch.randn(B, C_, L, generator=g).to(DEV)
    wd = torch.randn(C_, SA, K, generator=g).to(DEV)
    # frames[b, sa*K+j, t] = sum_c wd[c,sa,j] * masked[b,c,t]
    frames = torch.einsum("csj,bct->bsjt", wd, masked).reshape(B, SA * K, L).contiguous()
    mix = torch.randn(B, 1, T, generator=g).to(DEV) if mc else None
    out = torch.full((B, SA, T), float("nan"), device=DEV)
    N.check(N.lib().sdr_overlap_add(p(frames), p(mix), p(out), B, SA, K, L, T, stream()))
    want = F.conv_transpose1d(masked.double(), wd.double(), None, stride=hop, padding=hop,
                              output_padding=hop - 1)[..., :T]
    if mc:
        want = O.mixture_consistency(want, mix.double())
    close(out, want)


@pytest.mark.parametrize("B,G,n,L", [(2, 16, 16, 3200), (2, 4, 8, 100), (3, 8, 4, 33),
                                     (1, 2, 32, 40), (2, 16, 16, 31), (3, 8, 16, 200), (1, 5, 16, 16)])
def test_tac(B, G, n, L):
    g = torch.Generator().manual_seed(5)
    H = 3 * n
    cfg = O.Config(variant="groupcomm", out_channels=G * n, in_channels=2 * G * n, num_blocks=1,
                   upsampling_depth=1, group_size=G)
    sd = {k[len("sm.0.TAC."):]: v.to(DEV) for k, v in O.make_state_dict(cfg, seed=9).items()
          if k.startswith("sm.0.TAC.")}
    x = torch.randn(B, G, n, L, generator=g).to(DEV)
    names = ["TAC_input.0.weight", "TAC_input.0.bias", "TAC_input.1.weight",
             "TAC_mean.0.weight", "TAC_mean.0.bias", "TAC_mean.1.weight",
             "TAC_output.0.weight", "TAC_output.0.bias", "TAC_output.1.weight"]
    assert sd["TAC_mean.0.weight"].shape == (H, H)
    params = (C.c_void_p * 9)(*[sd[k].contiguous().data_ptr() for k in names])
    o = torch.full((B, G, n, L), float("nan"), device=DEV)
    st = torch.zeros(B * G, 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_tac(p(x), params, p(o), p(st), B, G, n, L, stream()))
    taps = {}
    O.tac(x, sd, "", taps)
    want = taps["TAC_output"]
    # n = 16 runs on tensor cores (three chained bf16x3 GEMMs: ~3e-5); the other group widths are exact-fp32 FFMA
    close(o, want, tol=1e-4 if n == 16 else 2e-5)
    check_stats(st, want.reshape(B * G, n, L), rtol=1e-4 if n == 16 else 1e-5)


MIXTURE_CONSISTENCY = [   # kind, S, T, silent estimates; the first two keep their ids
    ("uniform", 2, 32079, "none"), ("magsq", 2, 32079, "none"),
    ("uniform", 1, 2049, "none"), ("magsq", 1, 2048, "none"), ("uniform", 3, 2047, "none"), ("magsq", 3, 2049, "none"),
    ("uniform", 16, 4097, "none"), ("magsq", 16, 2048, "none"), ("magsq", 3, 2049, "one"), ("magsq", 16, 4096, "one"),
    ("magsq", 3, 2047, "all"), ("magsq", 1, 2049, "all"), ("uniform", 16, 2049, "all"),
]


def _mc_id(c):
    return c[0] if c[1:] == (2, 32079, "none") else "-".join(str(v) for v in c)


@pytest.mark.parametrize("kind,S,T,silent", MIXTURE_CONSISTENCY, ids=[_mc_id(c) for c in MIXTURE_CONSISTENCY])
def test_mixture_consistency(kind, S, T, silent):
    """Against mixture_consistency.py in fp64: 1, 2, 3 and 16 sources, both weight types, one or every estimate
    silent ('magsq' then gives it no share of the residual), T on both sides of the power kernel's 2048-sample step."""
    import sudo_rm_rf_b200.mixture_consistency as mc
    g = torch.Generator().manual_seed(6)
    est = torch.randn(3, S, T, generator=g)
    mix = torch.randn(3, 1, T, generator=g)
    if silent == "one":
        est[:, S // 2] = 0
    elif silent == "all":
        est.zero_()
    got = mc.apply(est.to(DEV), mix.to(DEV), kind)
    want = O.mixture_consistency(est.double(), mix.double(), kind)
    close(got, want, tol=1e-5)
    if kind == "uniform":
        assert torch.allclose(got.sum(1, keepdim=True).cpu(), mix, atol=1e-5 * S)
    if silent == "one":
        assert torch.equal(got[:, S // 2].cpu(), torch.zeros(3, T))
    if kind == "magsq" and silent == "all":
        assert torch.equal(got.cpu(), est)


@pytest.mark.parametrize("samples,M,K,L,mode", [
    (2, 256, 512, 3200, "norm"),          # bottleneck (cfg 2)
    (3, 512, 256, 640, "plain_stats"),    # proj_1x1: four 128-wide n-tiles
    (2, 256, 512, 1280, "res"),           # res_conv + in-place skip
    (2, 1024, 256, 384, "mask"),          # mask_net
    (2, 128, 64, 200, "res"),             # single k-block, 128-wide tile, ragged last position tile
    (1, 384, 192, 100, "plain_stats"),    # tile_n = 128 x 3, 3 k-blocks, L < 128
    (5, 256, 128, 132, "norm"),           # positions spill into a 2nd, ragged tile
    (40, 512, 512, 384, "plain_stats"),   # > 132 tiles: persistent CTAs loop over several tiles
    (3, 42, 1024, 200, "plain"),          # decoder GEMM: 42 rows zero-padded to one 128-wide tile
    (2, 300, 128, 332, "res"),            # 300 rows -> padded to 384 = 3 tiles of 128, last one partial
    (2, 160, 64, 64, "plain_stats"),      # padded to 256: two 128-wide tiles, 96 padding columns
    (2, 256, 512, 640, "res_out"),        # skip connection written out of place
    (2, 300, 128, 332, "res_out"),
    (3, 256, 256, 36, "res"),             # L < 128 and not a multiple of 32
    (3, 512, 128, 200, "mask"),           # ragged last position tile: the epilogue's gate reads stop at L
    (20, 512, 64, 1280, "mask"),          # many tiles per CTA, each reading its gate rows straight from global memory
    # per-channel PReLU slopes in the operand transform (the original model, sudormrf.py:33,71)
    (2, 512, 128, 3200, "pc_stats"),      # its proj_1x1 (Co = 128 -> Ci = 512)
    (2, 128, 512, 3200, "pc_stats"),      # its conv_1x1_exp
    (3, 512, 128, 200, "pc"),             # reshape_before_masks, ragged last position tile
    (40, 1024, 512, 384, "pc"),           # the Toeplitz mask GEMM read through module_act; CTAs loop over many tiles
    (1, 256, 64, 100, "pc_stats"),        # a single k-block
])
def test_pointwise_tensor_core(samples, M, K, L, mode):
    """wgmma path (bf16x3 split, fp32 accumulate) against an fp64 reference."""
    lib = N.lib()
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(samples, K, L, generator=g) + 0.5).to(DEV)
    W = (torch.randn(M, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(M, generator=g).to(DEV)
    gamma = (1 + 0.3 * torch.randn(K, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(K, generator=g)).to(DEV)
    slope = torch.tensor([0.2], device=DEV)
    stats_in = raw_stats(x).to(DEV)
    nbytes = lib.sdr_pointwise_mma_packed_bytes(M, K)
    assert nbytes == (M + 127) // 128 * 128 * K * 4
    wpk = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_pointwise_mma_pack(p(W), M, K, p(wpk), stream()))
    y = torch.full((samples, M, L), float("nan"), device=DEV)
    st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    residual = gate = None
    gate_ch, epi = 0, 0
    if mode == "norm":
        nin = norm_in(stats_in, gamma, beta, None, K * L)
        fx = ref_norm(x.double(), gamma.double(), beta.double())
    elif mode in ("res", "res_out"):
        nin = norm_in(stats_in, gamma, beta, slope, K * L)
        fx = ref_norm(x.double(), gamma.double(), beta.double(), slope.double())
        residual = torch.randn(samples, M, L, generator=g).to(DEV)
        if mode == "res":
            y = residual.clone()              # in place: y is its own residual
    elif mode == "mask":
        nin = norm_in(None, None, None, slope, 1.0)
        fx = O.prelu1(x.double(), slope.double())
        gate_ch = M // 2
        gate = torch.randn(samples, gate_ch, L, generator=g).to(DEV)
        epi = 1
    elif mode in ("pc", "pc_stats"):
        slopes = channel_slopes(K, g)
        nin = norm_in(stats_in, gamma, beta, slopes, K * L)
        fx = ref_norm(x.double(), gamma.double(), beta.double(), slopes.double())
    else:
        nin = norm_in()
        fx = x.double()
    want = torch.einsum("mk,skl->sml", W.double(), fx) + bias.double().view(1, -1, 1)
    if mode in ("res", "res_out"):
        want = want + residual.double()
    if mode == "mask":
        idx = torch.arange(M, device=DEV) % gate_ch
        want = torch.relu(want) * gate.double()[:, idx, :]
    want_stats = mode in ("plain_stats", "pc_stats")
    N.check(lib.sdr_pointwise_mma(p(x), C.byref(nin), p(wpk), p(bias), p(y) if mode == "res" else (p(residual) if mode == "res_out" else p(None)),
                                  p(gate), gate_ch, p(y), p(st) if want_stats else p(None),
                                  samples, M, K, L, epi, stream()))
    torch.cuda.synchronize()
    e = O.parity_errors(y, want)
    print("tensor-core pointwise", (samples, M, K, L, mode), "rel_max %.2e rel_l2 %.2e" % e)
    assert max(e) < 5e-5, e
    if want_stats:
        check_stats(st, want.float(), rtol=3e-5)


def test_pointwise_tensor_core_refuses_unaligned_length():
    """The activations' TMA tensor map needs a 16 B row stride, i.e. L % 4 == 0; the forward uses the FFMA kernel for
    other lengths."""
    lib = N.lib()
    x = torch.zeros(1, 64, 130, device=DEV)
    W = torch.zeros(128, 64, device=DEV)
    wpk = torch.empty(lib.sdr_pointwise_mma_packed_bytes(128, 64), dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_pointwise_mma_pack(p(W), 128, 64, p(wpk), stream()))
    y = torch.zeros(1, 128, 130, device=DEV)
    nin = norm_in()
    rc = lib.sdr_pointwise_mma(p(x), C.byref(nin), p(wpk), p(None), p(None), p(None), 0, p(y), p(None),
                               1, 128, 64, 130, 0, stream())
    assert rc == -5


def test_pointwise_tensor_core_eligibility():
    lib = N.lib()
    assert lib.sdr_pointwise_mma_packed_bytes(42, 1024) == 128 * 1024 * 4   # decoder GEMM: rows padded to 128
    assert lib.sdr_pointwise_mma_packed_bytes(16, 64) == 0
    assert lib.sdr_pointwise_mma_packed_bytes(32, 16) == 0         # group-communication blocks
    assert lib.sdr_pointwise_mma_packed_bytes(256, 100) == 0
    assert lib.sdr_pointwise_mma_packed_bytes(512, 256) == 512 * 256 * 4


@pytest.mark.parametrize("samples,C_,L,first", [
    (2, 128, 3200, False), (3, 16, 52, False), (2, 24, 517, True), (1, 7, 3, False), (2, 128, 3200, True),
])
def test_residual_norm(samples, C_, L, first):
    """Tail of the original UBlock (sudormrf.py:184-186): x <- GN(e) + f(x) in place, statistics of the new x;
    f = identity for the first block, else the previous block's module_act (GroupNorm + per-channel PReLU)."""
    g = torch.Generator().manual_seed(21)
    e = (torch.randn(samples, C_, L, generator=g) * 1.7 - 0.4).to(DEV)
    x = (torch.randn(samples, C_, L, generator=g) * 0.8 + 0.2).to(DEV)
    ge = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    be = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    gx = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    bx = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    slopes = channel_slopes(C_, g)
    st_e, st_x = raw_stats(e).to(DEV), raw_stats(x).to(DEV)          # (kept alive: the structs hold raw pointers)
    fe = norm_in(st_e, ge, be, None, C_ * L)
    fx = norm_in() if first else norm_in(st_x, gx, bx, slopes, C_ * L)
    want = ref_norm(e, ge, be) + (x if first else ref_norm(x, gx, bx, slopes))
    st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_residual_norm(p(e), C.byref(fe), p(x), C.byref(fx), p(st), samples, C_, L, stream()))
    close(x, want)
    check_stats(st, want)


SOFTMAX_GATE = [   # B, S, N, L, inplace, logits; the first five keep their ids
    (2, 2, 512, 3200, True, "randn"), (3, 3, 24, 52, False, "randn"), (2, 1, 16, 80, True, "randn"),
    (1, 4, 7, 3, False, "randn"), (2, 16, 8, 10, True, "randn"),
]
# every source count on the vector path (N*L % 4 == 0) and on the scalar path (N*L % 4 != 0)
SOFTMAX_GATE += [(2, S, 8, 12, S % 2 == 0, "randn") for S in range(1, 17)]
SOFTMAX_GATE += [(2, S, 5, 7, S % 2 == 1, "randn") for S in range(1, 17)]
# float4-sized rows behind a pointer that is not 16-byte aligned: the scalar path
SOFTMAX_GATE += [(2, S, 8, 12, False, "offset") for S in (1, 2, 4, 5, 16)]
# logits of +-1e4 (exp underflows to 0 for every source below the largest; the sigmoid saturates), exact ties
SOFTMAX_GATE += [(2, S, 8, 12, True, "1e4") for S in (1, 2, 3, 4, 7, 16)]
SOFTMAX_GATE += [(1, S, 5, 7, False, "1e4") for S in (1, 3, 16)]
SOFTMAX_GATE += [(2, S, 8, 12, False, "ties") for S in (2, 3, 4, 9, 16)]
SOFTMAX_GATE += [(1, S, 5, 7, True, "ties") for S in (3, 16)]


def _sg_id(c):
    return "-".join(str(v) for v in (c[:5] if SOFTMAX_GATE.index(c) < 5 else c))


@pytest.mark.parametrize("B,S,N_,L,inplace,logits", SOFTMAX_GATE, ids=[_sg_id(c) for c in SOFTMAX_GATE])
def test_softmax_gate(B, S, N_, L, inplace, logits):
    """Masks of the original model (sudormrf.py:285-289): softmax over the sources (sigmoid for one) x encoder output,
    against fp64 torch.softmax / torch.sigmoid."""
    g = torch.Generator().manual_seed(22)
    lg = torch.randn(B, S, N_, L, generator=g) * 3
    if logits == "1e4":          # one source at +1e4 and the rest at -1e4, each source in turn; every third position
        pos = torch.arange(N_ * L).view(1, 1, N_, L)              # +-1e4 at random (ties among the largest)
        lg = torch.full((B, S, N_, L), -1e4).scatter_(1, (pos % S).expand(B, 1, N_, L), 1e4)
        rnd = torch.where(torch.rand(B, S, N_, L, generator=g) < 0.5, -1e4, 1e4)
        lg = torch.where(pos % 3 == 2, rnd, lg)
    elif logits == "ties":       # every source ties at each position; on odd positions the first two share the max
        lg = (torch.randn(B, 1, N_, L, generator=g) * 3).expand(B, S, N_, L).clone()
        lg[:, 2:, :, 1::2] -= 1.5
    enc = torch.relu(torch.randn(B, N_, L, generator=g))
    want = (torch.sigmoid(lg.double()) if S == 1 else torch.softmax(lg.double(), dim=1)) * enc.double().unsqueeze(1)
    shift = 1 if logits == "offset" else 0   # one float into a fresh allocation: 4-byte but not 16-byte aligned
    lbuf = torch.empty(lg.numel() + shift, device=DEV)
    ebuf = torch.empty(enc.numel() + shift, device=DEV)
    lbuf[shift:] = lg.reshape(-1).to(DEV)
    ebuf[shift:] = enc.reshape(-1).to(DEV)
    lgd, encd = lbuf[shift:].view(B, S, N_, L), ebuf[shift:].view(B, N_, L)
    if inplace:
        out = lgd
    else:
        obuf = torch.full((lg.numel() + shift,), float("nan"), device=DEV)
        out = obuf[shift:].view(B, S, N_, L)
    N.check(N.lib().sdr_softmax_gate(p(lgd), p(encd), p(out), B, S, N_, L, stream()))
    close(out, want, tol=1e-5)


@pytest.mark.parametrize("B,T,N_,K,D", [(2, 32000, 512, 21, 4), (3, 517, 24, 21, 3), (1, 333, 16, 11, 4)])
def test_original_front_and_back_ends(B, T, N_, K, D):
    """Biased encoder + ReLU and the biased grouped decoder of the original model (sudormrf.py:212-218,245-252,291)
    through the whole-model entry: a model with zero blocks is exactly encoder -> ln -> l1 -> Toeplitz mask GEMM ->
    softmax gate -> decoder GEMM -> overlap-add (tensor-core GEMMs at N = 512, FFMA ones at the small sizes)."""
    import sudo_rm_rf_b200 as P
    kw = dict(out_channels=N_, in_channels=2 * N_, num_blocks=0, upsampling_depth=D, enc_kernel_size=K,
              enc_num_basis=N_, num_sources=2)
    cfg = O.Config(variant="original", **kw)
    sd = O.make_state_dict(cfg, seed=13)
    m = P.OriginalSuDORMRF(**kw)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        y = m(x.to(DEV))
    close(y, O.forward(cfg, sd, x), tol=1e-4)
