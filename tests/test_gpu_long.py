"""The depthwise stage at the frame counts and batch sizes where its dispatch changes, up to 10 s at 16 kHz.

A block's depthwise levels run as the one-pass pyramid (pyramid.cu) while a row fits 32 warp windows and the
per-sample GlobLN table fits 4096 samples, else as D per-level launches plus a merge (levels.cu).  The causal block
always runs causal.cu, which splits rows longer than 4096 frames into windows with a left halo.  Every stage here is
compared with an fp64 torch chain of the same operation; the models with an fp64 run of the oracle (on the GPU, to
keep the long clips cheap).

- every dw_pyramid_kernel<D, threads, minBlocks, per-channel slope> instantiation at 8 and 9 windows (the 256 -> 1024
  thread switch), 17 windows and exactly 32 windows, with shared slopes on both sides of 1 and per-channel slopes;
- exactly 4096 GlobLN samples, and the refusal at 4097;
- the per-level kernels and their merge at L = 16000 / 32000, the shapes the forward hands them past the pyramid;
- the causal pyramid over 4 to 8 windows, with a causality check at every inner window boundary;
- improved / GroupComm / original models on both sides of the 32-window switch, 10 s clips at 16 kHz, GroupComm at
  257 mixtures (4112 samples) and a corpus whose utterances straddle the switch, GroupComm at upsampling_depth 1 on
  both sides of the TAC pre-add fold (L % 4); for each, the kernels one forward enqueues are counted with
  torch.profiler and compared with sdr_forward_launch_count_for.
"""
import collections
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn.functional as F

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
from test_gpu_dispatch import Guards
from test_gpu_stages import channel_slopes, check_stats, norm_in, p, raw_stats, stream

DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---------------------------------------------------------------------------------------------------------------------
# dw_pyramid_kernel: every instantiation at its window-count edges
# ---------------------------------------------------------------------------------------------------------------------
PYR_STEP = {4: 480, 5: 464, 6: 416}      # PyrGeom<D>::kStep: level-0 positions one warp window stores
PYR_MAX_SAMPLES = 4096                   # kPyrMaxSamples


def pyr_windows(D, L):
    return -(-L // PYR_STEP[D])


def pyr_threads(D, L):
    """sdr_depthwise_pyramid's block size: the <= 256-thread instantiation up to 8 windows, else 1024 threads."""
    return 256 if 32 * pyr_windows(D, L) <= 256 else 1024


PYR_LENGTHS = {   # 8 windows (largest 256-thread row), 9 windows (smallest 1024-thread row), 17 windows, 32 windows
    4: (3840, 3856, 8160, 15360),
    5: (3712, 3728, 7888, 14848),
    6: (3328, 3360, 7072, 13312),
}
PYR_PAST_32 = {4: 15376, 5: 14864, 6: 13344}   # the next length the pyramid's alignment allows: 33 windows
PYR_SLOPES = (0.3, 1.7, "pc")                  # shared slope below 1, above 1, one slope per channel
PYR_PARAMS = [(2, 12, D, L, s) for D, Ls in PYR_LENGTHS.items() for L in Ls for s in PYR_SLOPES]
PYR_PARAMS += [
    (2, 512, 5, 14848, 0.3),                 # 1024 rows of 32 windows: every persistent CTA turns its row buffers over
    (2, 512, 4, 15360, "pc"),
    (PYR_MAX_SAMPLES, 4, 4, 448, 0.3),       # the whole per-sample (mean, rstd) table in shared memory is read
]


def _pyr_id(v):
    return str(v)


def pyramid_case(samples, C_, D, L, slope, seed):
    """sdr_depthwise_pyramid + sdr_merge_pyramid on guarded buffers against the fp64 level-by-level chain."""
    lib = N.lib()
    g = torch.Generator().manual_seed(seed)
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.3).to(DEV)
    gy = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    by = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    ws = [torch.randn(C_, 1, 5, generator=g).to(DEV) * 0.6 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    gs = [(1 + 0.3 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    bes = [(0.2 * torch.randn(C_, generator=g)).to(DEV) for _ in range(D)]
    sl = channel_slopes(C_, g) if slope == "pc" else torch.tensor([slope], device=DEV)
    cur = O.glob_ln(y.double(), gy.double(), by.double())
    cur = O.prelu_c(cur, sl.double()) if slope == "pc" else O.prelu1(cur, sl.double())
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
    nbytes = lib.sdr_pyramid_scratch_bytes(samples, C_, D, L)
    assert nbytes > 0
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    gd = Guards()
    yg = gd.input("y", y)
    scratch = gd.output("scratch", torch.zeros(nbytes, dtype=torch.uint8, device=DEV))
    zs = [gd.output(f"z{d}", torch.full((samples, C_, L >> d), float("nan"), device=DEV)) for d in range(D)]
    st0 = gd.output("stats0", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    stm = gd.output("stats_m", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    m = gd.output("m", torch.full((samples, C_, L), float("nan"), device=DEV))
    nin = norm_in(raw_stats(y).to(DEV), gy, by, sl, C_ * L)
    N.check(lib.sdr_depthwise_pyramid(p(yg), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(st0),
                                      p(scratch), D, samples, C_, L, stream()))
    N.check(lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(m), p(stm), samples, C_, L, stream()))
    gd.check()
    e = O.parity_errors(zs[0], z0)
    assert max(e) < 2e-5, e
    check_stats(st0, z0)
    e = O.parity_errors(m, levels[0])
    assert max(e) < 5e-5, e              # (the affine re-composition reorders fp32 roundings over D levels)
    check_stats(stm, levels[0], rtol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,C_,D,L,slope", PYR_PARAMS, ids=_pyr_id)
def test_pyramid_long_rows(samples, C_, D, L, slope):
    pyramid_case(samples, C_, D, L, slope, seed=83)


@pytest.mark.gpu
def test_pyramid_refuses_past_the_sample_table():
    """4097 samples: no scratch, and both pyramid entries refuse the shape before launching anything."""
    lib = N.lib()
    samples, C_, D, L = PYR_MAX_SAMPLES + 1, 4, 4, 448
    assert lib.sdr_pyramid_scratch_bytes(samples, C_, D, L) == 0
    y = torch.zeros(samples, C_, L, device=DEV)
    prm = [torch.zeros(C_, 5, device=DEV) for _ in range(D)]
    zs = [torch.zeros(samples, C_, L >> d, device=DEV) for d in range(D)]
    scratch = torch.zeros(lib.sdr_pyramid_scratch_bytes(PYR_MAX_SAMPLES, C_, D, L), dtype=torch.uint8, device=DEV)
    st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    nin = norm_in(st, prm[0][:, 0], prm[0][:, 1], torch.tensor([0.3], device=DEV), C_ * L)
    assert lib.sdr_depthwise_pyramid(p(y), C.byref(nin), arr(prm), arr(prm), arr(prm), arr(prm), arr(zs), p(st),
                                     p(scratch), D, samples, C_, L, stream()) == -5
    assert lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(y), p(st), samples, C_, L, stream()) == -5
    torch.cuda.synchronize()
    assert not y.any() and not st.any() and not any(z.any() for z in zs)


# ---------------------------------------------------------------------------------------------------------------------
# the per-level kernels past the pyramid's limits
# ---------------------------------------------------------------------------------------------------------------------
DW_LONG = [   # stride, Lin, PReLU: what a block of L = 16000 / 32000 frames hands sdr_depthwise level by level
    (1, 16000, 0.3), (1, 32000, 1.7),        # level 0, shared slope: dw5_wide_kernel<1, true>
    (1, 16000, "pc"), (1, 32000, "pc"),      # level 0 of the original model (per-channel slopes): dw5_vec_kernel<1>
    (2, 32000, None), (2, 16000, None), (2, 8000, None), (2, 4000, None), (2, 2000, None),   # dw5_wide_kernel<2, false>
    (2, 1000, None),                         # Lout = 500: dw5_vec_kernel<2>
    (2, 500, None),                          # Lout = 250: dw5_scalar_kernel
]


@pytest.mark.gpu
@pytest.mark.parametrize("stride,Lin,slope", DW_LONG, ids=_pyr_id)
def test_depthwise_long_rows(stride, Lin, slope):
    samples, C_ = 2, 512
    g = torch.Generator().manual_seed(89)
    x = (torch.randn(samples, C_, Lin, generator=g) * 2 + 0.7).to(DEV)
    gamma = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(C_, generator=g)).to(DEV)
    w = torch.randn(C_, 1, 5, generator=g).to(DEV)
    b = torch.randn(C_, generator=g).to(DEV)
    sl = None if slope is None else (channel_slopes(C_, g) if slope == "pc" else torch.tensor([slope], device=DEV))
    fx = O.glob_ln(x.double(), gamma.double(), beta.double())
    if sl is not None:
        fx = O.prelu_c(fx, sl.double()) if slope == "pc" else O.prelu1(fx, sl.double())
    want = F.conv1d(fx, w.double(), b.double(), stride=stride, padding=2, groups=C_)
    Lout = (Lin - 1) // stride + 1
    gd = Guards()
    xg = gd.input("x", x)
    y = gd.output("y", torch.full((samples, C_, Lout), float("nan"), device=DEV))
    st = gd.output("stats", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    nin = norm_in(raw_stats(x).to(DEV), gamma, beta, sl, C_ * Lin)
    N.check(N.lib().sdr_depthwise(p(xg), C.byref(nin), p(w), p(b), p(y), p(st), samples, C_, Lin, stride, stream()))
    gd.check()
    e = O.parity_errors(y, want)
    assert max(e) < 2e-5, e
    check_stats(st, want)


@pytest.mark.gpu
@pytest.mark.parametrize("depth,L", [(D, L) for D in (4, 5, 6) for L in (16000, 32000)])
def test_merge_long_rows(depth, L):
    samples, C_ = 2, 512
    g = torch.Generator().manual_seed(97)
    zs, gammas, betas = [], [], []
    for d in range(depth):
        zs.append((torch.randn(samples, C_, L >> d, generator=g) + 0.3 * d).to(DEV))
        gammas.append((1 + 0.3 * torch.randn(C_, generator=g)).to(DEV))
        betas.append((0.2 * torch.randn(C_, generator=g)).to(DEV))
    stats = [raw_stats(z).to(DEV) for z in zs]
    levels = [O.glob_ln(z.double(), ga.double(), be.double()) for z, ga, be in zip(zs, gammas, betas)]
    for _ in range(depth - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
    gd = Guards()
    zg = [gd.input(f"z{d}", z) for d, z in enumerate(zs)]
    m = gd.output("m", torch.full((samples, C_, L), float("nan"), device=DEV))
    st = gd.output("stats", torch.zeros(samples, 2, dtype=torch.float64, device=DEV))
    fins = (N.SdrNormIn * depth)(*[norm_in(stats[d], gammas[d], betas[d], None, C_ * (L >> d)) for d in range(depth)])
    zp = (C.c_void_p * depth)(*[z.data_ptr() for z in zg])
    N.check(N.lib().sdr_merge(zp, fins, depth, p(m), p(st), samples, C_, L, stream()))
    gd.check()
    e = O.parity_errors(m, levels[0])
    assert max(e) < 2e-5, e
    check_stats(st, levels[0])


# ---------------------------------------------------------------------------------------------------------------------
# causal pyramid over many windows
# ---------------------------------------------------------------------------------------------------------------------
def causal_window_starts(D, L):
    """First frame of every window launch_causal_pyramid splits a row into (balanced windows of at most 4096 frames,
    rounded up to a float4 boundary of the deepest level)."""
    gran = 4 if D == 1 else 4 << (D - 1)
    tiles = -(-L // 4096)
    W = -(-(-(-L // tiles)) // gran) * gran
    return list(range(0, L, W))


# L = 16000 / 32000: 4 / 8 windows (10 / 20 s at 16 kHz); 28736: 8 windows, the last one 2752 frames at D = 6.
# D = 7, 8 (left halo 756 / 1524 frames): 16384 and 32000, 4 and 8 windows (28736 does not halve 7 times)
CAUSAL_PARAMS = [(D, L) for L in (16000, 28736, 32000) for D in range(1, 7)] + \
                [(D, L) for L in (16384, 32000) for D in (7, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("D,L", CAUSAL_PARAMS)
def test_causal_pyramid_many_windows(D, L):
    lib = N.lib()
    samples, C_ = 2, 16
    g = torch.Generator().manual_seed(101)
    y = (torch.randn(samples, C_, L, generator=g) * 1.3 + 0.1).to(DEV)
    ws = [torch.randn(C_, 1, 21, generator=g).to(DEV) * 0.4 for _ in range(D)]
    bs = [torch.randn(C_, generator=g).to(DEV) * 0.5 for _ in range(D)]
    sp = torch.tensor([0.3], device=DEV)
    sl = [torch.tensor([(0.2, 1.7, -0.4)[d % 3]], device=DEV) for d in range(D)]
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    cur = O.prelu1(y.double(), sp.double())
    levels = []
    for d in range(D):
        cur = O.prelu1(F.conv1d(cur, O.causal_weight(ws[d].double()), bs[d].double(), stride=1 if d == 0 else 2,
                                padding=10, groups=C_), sl[d].double())
        levels.append(cur)
    for _ in range(D - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")

    def run(inp):
        gd = Guards()
        yg = gd.input("y", inp)
        m = gd.output("m", torch.full((samples, C_, L), float("nan"), device=DEV))
        N.check(lib.sdr_causal_pyramid(p(yg), p(sp), arr(ws), arr(bs), arr(sl), p(m), D, samples, C_, L, stream()))
        gd.check()
        return m

    m = run(y)
    e = O.parity_errors(m, levels[0])
    assert max(e) < 2e-5, e
    starts = causal_window_starts(D, L)
    assert len(starts) >= 4
    # causality across every inner window boundary: the frames before t0 do not see the input from t0 on
    for t0 in starts[1:]:
        y2 = y.clone()
        y2[..., t0:] = 7.0
        m2 = run(y2)
        assert torch.equal(m2[..., :t0], m[..., :t0]), t0
        assert not torch.equal(m2[..., t0:], m[..., t0:]), t0


# ---------------------------------------------------------------------------------------------------------------------
# models on both sides of the switch, and the kernels one forward enqueues
# ---------------------------------------------------------------------------------------------------------------------
CLASSES = {"improved": P.SuDORMRF, "groupcomm": P.GroupCommSudoRmRf, "causal": P.CausalSuDORMRF,
           "original": P.OriginalSuDORMRF}
IMPROVED = dict(out_channels=128, in_channels=512, num_blocks=2, upsampling_depth=5, enc_kernel_size=21,
                enc_num_basis=128, num_sources=2)
GROUPCOMM = dict(out_channels=256, in_channels=512, num_blocks=2, upsampling_depth=5, enc_kernel_size=21,
                 enc_num_basis=128, num_sources=2, group_size=16)
ORIGINAL = dict(out_channels=128, in_channels=512, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
                enc_num_basis=128, num_sources=2)
CAUSAL = dict(in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=2, upsampling_depth=4,
              enc_kernel_size=21, enc_num_basis=128, num_sources=2)
GROUPCOMM_D1 = dict(out_channels=64, in_channels=128, num_blocks=3, upsampling_depth=1, enc_kernel_size=21,
                    enc_num_basis=128, num_sources=2, group_size=4)
MODEL_CASES = [   # id, variant, kwargs, T, one-pass pyramid expected (None: the causal block)
    ("improved_L14848_pyramid", "improved", IMPROVED, 148480, True),        # 32 windows
    ("improved_L14880_levels", "improved", IMPROVED, 148481, False),        # 33 windows
    ("groupcomm_L14848_pyramid", "groupcomm", GROUPCOMM, 148480, True),
    ("groupcomm_L14880_levels", "groupcomm", GROUPCOMM, 148481, False),
    ("original_L15360_pyramid", "original", ORIGINAL, 153600, True),        # D = 4: 32 windows
    ("original_L15376_levels", "original", ORIGINAL, 153760, False),        # 33 windows (L % 16 == 0 still)
    ("improved_4src_10s_16k", "improved", dict(IMPROVED, num_sources=4), 160000, False),   # a FUSS clip
    ("causal_10s_16k", "causal", CAUSAL, 160000, None),                     # 4 causal windows per row
    ("groupcomm_D1_L320_folded", "groupcomm", GROUPCOMM_D1, 3200, False),   # TAC pre-add inside proj_1x1
    ("groupcomm_D1_L322_apart", "groupcomm", GROUPCOMM_D1, 3210, False),    # L % 4 == 2: tac_apply, then proj_1x1
]


def build_model(variant, kw, seed):
    cfg = O.Config(variant=variant, **kw)
    sd = O.make_state_dict(cfg, seed=seed)
    m = CLASSES[variant](**kw)
    m.load_state_dict(sd)
    return cfg, sd, m.to(DEV).eval()


def kernels_enqueued(fn):
    """Names of the CUDA kernels `fn` enqueues (memsets and copies excluded), from torch.profiler's device events."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return [n for n in names if not n.startswith(("Memset", "Memcpy", "memset", "memcpy"))]


def check_launch_count(model, B, T, fn):
    lib = N.lib()
    cfg = P._engine.make_config(model)
    want = lib.sdr_forward_launch_count_for(C.byref(cfg), B, T)
    got = kernels_enqueued(fn)
    assert len(got) == want, (want, len(got), collections.Counter(got))


def takes_pyramid(cfg, B, T):
    """Does the forward's plan run this model's depthwise stage as the one-pass pyramid?"""
    G = cfg.group_size if cfg.variant == "groupcomm" else 1
    L = O.padded_length(cfg, T) // cfg.hop
    return N.lib().sdr_pyramid_scratch_bytes(B * G, cfg.in_channels // G, cfg.upsampling_depth, L) > 0


def normalised_input(B, A, T, seed):
    x = torch.randn(B, A, T, generator=torch.Generator().manual_seed(seed))
    return (x - x.mean(-1, keepdim=True)) / (x.std(-1, keepdim=True) + 1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("name,variant,kw,T,pyramid", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_model_at_the_switch(name, variant, kw, T, pyramid):
    cfg, sd, m = build_model(variant, kw, seed=103)
    if pyramid is not None:
        assert takes_pyramid(cfg, 1, T) == pyramid
    x = normalised_input(1, kw.get("in_audio_channels", 1), T, seed=107).to(DEV)
    with torch.no_grad():
        y = m(x)                                  # (packs the weights: the profiled call below is the forward alone)
        check_launch_count(m, 1, T, lambda: m(x))
    ref = O.forward(cfg, {k: v.to(DEV) for k, v in sd.items()}, x, dtype=torch.float64)
    assert y.shape == ref.shape
    e = O.parity_errors(y, ref)
    print(name, "rel_max %.3e rel_l2 %.3e" % e)
    assert max(e) < 1e-4, e


@pytest.mark.gpu
def test_groupcomm_past_the_sample_table():
    """257 mixtures x 16 groups = 4112 GlobLN samples: the blocks run level by level.  Every mixture of the batch
    equals the oracle, and the same mixture run alone (16 samples: the one-pass pyramid)."""
    kw = dict(GROUPCOMM, enc_num_basis=64)
    cfg, sd, m = build_model("groupcomm", kw, seed=109)
    T = 3200                                      # L = 320: one warp window per row
    assert takes_pyramid(cfg, 256, T) and not takes_pyramid(cfg, 257, T)
    x = normalised_input(257, 1, T, seed=113).to(DEV)
    with torch.no_grad():
        y = m(x)
        check_launch_count(m, 257, T, lambda: m(x))
        check_launch_count(m, 256, T, lambda: m(x[:256]))
        # (parity_errors takes the worst sample: every mixture is held to the bound)
        e = O.parity_errors(y, O.forward(cfg, {k: v.to(DEV) for k, v in sd.items()}, x, dtype=torch.float64))
        print("batch of 257 vs oracle: rel_max %.3e rel_l2 %.3e" % e)
        assert max(e) < 1e-4, e
        # alone, a mixture takes the other path: the two agree to fp32 re-association (the pyramid's merge is an
        # affine re-composition of the raw levels, 5e-5 at stage level), not to the last bit as two runs of one path do
        worst = max(max(O.parity_errors(m(x[i:i + 1]), y[i:i + 1])) for i in range(257))
        print("batch of 257 vs each mixture alone: worst %.3e" % worst)
        assert worst < 2e-5, worst


@pytest.mark.gpu
def test_separate_corpus_across_the_switch():
    """One corpus, utterances on both sides of the 32-window switch of an improved D = 5 model (padded to 148480:
    pyramid; 148800 and 160000: level by level; 3200: pyramid): each result equals the utterance separated alone."""
    from sudo_rm_rf_b200.corpus import separate_corpus
    cfg, sd, m = build_model("improved", IMPROVED, seed=127)
    lengths = [148480, 148481, 160000, 148000, 3000, 159999]
    assert [takes_pyramid(cfg, 1, T) for T in lengths] == [True, False, False, True, True, False]
    g = torch.Generator().manual_seed(131)
    wavs = [torch.randn(T, generator=g) * (0.2 + 0.3 * i) + 0.05 * i for i, T in enumerate(lengths)]
    with torch.no_grad():
        got = separate_corpus(m, wavs, max_batch=4)
        for w, yb in zip(wavs, got):
            alone = separate_corpus(m, [w])[0]
            assert yb.shape == (cfg.num_sources, w.shape[0])
            e = O.parity_errors(yb[None], alone[None])
            assert max(e) < 1e-5, (w.shape[0], e)
        for i in (0, 1):                          # one utterance on each side against the oracle
            want = O.separate(cfg, {k: v.to(DEV) for k, v in sd.items()}, wavs[i][None].to(DEV), dtype=torch.float64)
            assert max(O.parity_errors(got[i][None], want)) < 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the parametrisation reaches every pyramid instantiation; plan, scratch and launch count share one predicate
# ---------------------------------------------------------------------------------------------------------------------
def test_pyramid_instantiations_are_all_tested():
    src = open(os.path.join(REPO, "sudo_rm_rf_b200", "csrc", "pyramid.cu")).read()
    compiled = {(int(d), int(t), pc == "true")
                for d, t, pc in re.findall(r"dw_pyramid_kernel<(\d),\s*(\d+),\s*\w+,\s*(true|false)>", src)}
    assert len(compiled) == 12, sorted(compiled)
    tested = {(D, pyr_threads(D, L), slope == "pc") for _, _, D, L, slope in PYR_PARAMS}
    assert compiled == tested, (sorted(compiled - tested), sorted(tested - compiled))
    for D, Ls in PYR_LENGTHS.items():
        assert [pyr_windows(D, L) for L in Ls] == [8, 9, 17, 32]
        assert pyr_windows(D, PYR_PAST_32[D]) == 33


def test_pyramid_limits_agree():
    """Past 32 windows or 4096 samples there is no pyramid scratch; the launch count and the workspace plan then
    follow the per-level path (D depthwise launches per block instead of the pyramid's two)."""
    lib = N.lib()
    for D, Ls in PYR_LENGTHS.items():
        assert lib.sdr_pyramid_scratch_bytes(2, 512, D, Ls[-1]) > 0
        assert lib.sdr_pyramid_scratch_bytes(2, 512, D, PYR_PAST_32[D]) == 0
        for L in range(Ls[-1] + 1, PYR_PAST_32[D]):
            assert lib.sdr_pyramid_scratch_bytes(2, 512, D, L) == 0
    assert lib.sdr_pyramid_scratch_bytes(PYR_MAX_SAMPLES, 4, 4, 448) > 0
    assert lib.sdr_pyramid_scratch_bytes(PYR_MAX_SAMPLES + 1, 4, 4, 448) == 0
    # GroupComm, 16 groups of 32 channels: B * 16 GlobLN samples
    U, D = 2, 5
    m = P.GroupCommSudoRmRf(**dict(GROUPCOMM, num_blocks=U, upsampling_depth=D, enc_num_basis=64))
    cfg = P._engine.make_config(m)
    count = lambda B, T: lib.sdr_forward_launch_count_for(C.byref(cfg), B, T)
    T = 3200
    assert count(1, T) == lib.sdr_forward_launch_count_at(C.byref(cfg), T)
    assert count(256, T) == count(1, T)
    assert count(257, T) == count(256, T) + U * (D - 2)
    ws = lambda B: lib.sdr_workspace_bytes(C.byref(cfg), B, T)
    assert ws(257) < ws(256)                      # the pyramid's row statistics and merge table are not planned
    # one length past 32 windows at B = 1: the same switch
    assert count(1, 148481) == count(1, 148480) + U * (D - 2)
    assert lib.sdr_forward_launch_count_for(C.byref(cfg), 0, T) < 0


def test_tac_fold_follows_the_length():
    """At upsampling_depth 1 a GroupComm model pads to an even frame count only: its blocks fold tac_apply into
    proj_1x1 (one launch fewer each) exactly when L % 4 == 0."""
    cfg = P._engine.make_config(P.GroupCommSudoRmRf(**GROUPCOMM_D1))
    count = lambda T: N.lib().sdr_forward_launch_count_for(C.byref(cfg), 1, T)
    assert count(3200) == count(3210) - GROUPCOMM_D1["num_blocks"]      # L = 320 / 322


def test_benchmark_launch_claim_holds_at_its_batch():
    """bench.py reports the launch count at its clip length for one mixture; every benchmark config's batch stays
    inside the pyramid's sample table, so that is also the count of the forward it times."""
    import bench
    lib = N.lib()
    for name, w in bench.WORKLOADS.items():
        cfg = P._engine.make_config(bench.model_class(w["variant"])(**w["kw"]))
        at = lib.sdr_forward_launch_count_at(C.byref(cfg), w["T"])
        assert at > 0 and lib.sdr_forward_launch_count_for(C.byref(cfg), w["B"], w["T"]) == at, name
