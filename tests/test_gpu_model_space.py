"""Whole models across the geometry around the U-ConvBlocks: source count S, audio-channel count A and filter length K
(hop K // 2), against an fp64 run of the oracle on the GPU.

The blocks themselves are swept elsewhere; what S, A and K shape is the encoder (FFMA below 32 basis functions, else
wgmma with A*K padded to 64-wide k-blocks), the mask GEMM (M = S*A*N, gate row m % N; tensor cores when N % 256 == 0),
the decoder GEMM (M = S*A*K rows, Kc = S*A*N; tensor cores when M >= 32 and Kc % 64 == 0), the overlap-add (tap
window, one bias per source for the original model, 1/SA mixture consistency, the separate() rescale), the original
model's sigmoid / softmax gate, Toeplitz mask and block-diagonal decoder, and the GroupComm TAC.  Every case asserts the
GEMM paths it is there to cover, counts the kernels one forward enqueues, and holds rel_max and rel_L2 below 1e-4.

Then mixture consistency at 1, 3, 5 and 16 sources, separate(normalize=True) at four sources, the refusal boundaries
(S*A = 16 / 17, TAC group width and group count, the FFMA encoder's shared memory, the original model's length rule),
and the FUSS recipe end to end: the four model types as run_fuss_separation.py builds them, 10 s at 16 kHz, through the
validation loop body and its stabilised SI-SDR(i) metric."""
import collections
import ctypes as C
import itertools

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import sisdr as SI
from oracle import sudormrf_oracle as O
from test_gpu_long import CLASSES, normalised_input, takes_pyramid

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4


def build(variant, kw, seed=211):
    cfg = O.Config(variant=variant, **kw)
    sd = O.make_state_dict(cfg, seed=seed, perturbed=True)
    m = CLASSES[variant](**kw)
    m.load_state_dict(sd)
    return cfg, {k: v.to(DEV) for k, v in sd.items()}, m.to(DEV).eval()


def paths(cfg):
    """(encoder, mask, decoder): which of the three run on tensor cores, by the library's own eligibility rules."""
    lib = N.lib()
    S, N_, K, Co = cfg.num_sources, cfg.enc_num_basis, cfg.enc_kernel_size, cfg.out_channels
    A = cfg.in_audio_channels if cfg.variant == "groupcomm" else 1
    enc = lib.sdr_encoder_mma_packed_bytes(N_, A, K) > 0
    if cfg.variant == "original":                       # Toeplitz mask [S*N, N]; block-diagonal decoder [S*K, S*N]
        mask = lib.sdr_pointwise_mma_packed_bytes(S * N_, N_) > 0
    else:                                               # the gated epilogue needs N % 256 == 0 (api.cu make_layout)
        mask = N_ % 256 == 0 and lib.sdr_pointwise_mma_packed_bytes(S * A * N_, Co) > 0
    dec = lib.sdr_pointwise_mma_packed_bytes(S * A * K, S * A * N_) > 0
    return enc, mask, dec


def check_launch_count(model, B, T, fn):
    """The kernels one forward enqueues, counted as the kernel nodes of a CUDA graph captured from it (memsets are
    nodes of another type), against sdr_forward_launch_count_for.  torch.profiler's device records are not used here:
    in a process that has profiled many times they can miss a kernel or a whole window."""
    want = N.lib().sdr_forward_launch_count_for(C.byref(_engine.make_config(model)), B, T)
    cu = C.CDLL("libcuda.so.1")
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(graph, stream=side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = C.c_void_p(graph.raw_cuda_graph())
    n = C.c_size_t(0)
    assert cu.cuGraphGetNodes(g, None, C.byref(n)) == 0
    nodes = (C.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(g, nodes, C.byref(n)) == 0
    types = []
    for node in nodes:
        t = C.c_int(-1)
        assert cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(t)) == 0
        types.append(t.value)
    kernels = types.count(0)                    # CU_GRAPH_NODE_TYPE_KERNEL
    assert kernels == want, (want, collections.Counter(types))


def run_case(variant, kw, T, want_paths, B=2, seed=211):
    cfg, sd, m = build(variant, kw, seed)
    assert paths(cfg) == want_paths, (paths(cfg), want_paths)
    A = kw.get("in_audio_channels", 1) if variant == "groupcomm" else 1
    x = normalised_input(B, A, T, seed=seed + 1).to(DEV)
    with torch.no_grad():
        y = m(x)
        check_launch_count(m, B, T, lambda: m(x))
    ref = O.forward(cfg, sd, x, dtype=torch.float64)
    assert y.shape == ref.shape == (B, cfg.num_sources * A, T)
    e = O.parity_errors(y, ref)
    L = O.padded_length(cfg, T) // cfg.hop
    print(f"{variant} S={cfg.num_sources} A={A} K={cfg.enc_kernel_size} N={cfg.enc_num_basis} T={T} L={L} "
          f"(encoder, mask, decoder) on tensor cores {want_paths}: rel_max {e[0]:.3e} rel_l2 {e[1]:.3e}")
    assert max(e) < TOL, e


# ---------------------------------------------------------------------------------------------------------------------
# the grid: (id, variant, kwargs, T, (encoder, mask, decoder) on tensor cores)
# ---------------------------------------------------------------------------------------------------------------------
def imp(S, K, N_, Co=64, Ci=128, U=1, D=3):
    return dict(out_channels=Co, in_channels=Ci, num_blocks=U, upsampling_depth=D, enc_kernel_size=K,
                enc_num_basis=N_, num_sources=S)


def gc(S, A, K, N_, G, n, Ci=None, U=1, D=3):
    return dict(in_audio_channels=A, out_channels=G * n, in_channels=Ci or 2 * G * n, num_blocks=U,
                upsampling_depth=D, enc_kernel_size=K, enc_num_basis=N_, num_sources=S, group_size=G)


def orig(S, K, N_, Co, Ci=None, U=1, D=3):
    return dict(out_channels=Co, in_channels=Ci or 2 * Co, num_blocks=U, upsampling_depth=D, enc_kernel_size=K,
                enc_num_basis=N_, num_sources=S)


GRID = [
    # improved: S = 1 (the tensor-core mask is M = 256; the 21-row decoder is below the 32-row minimum: FFMA)
    ("imp_S1_K21", "improved", imp(1, 21, 256, D=4), 1601, (True, True, False)),
    # hop 1 (L = padded T); the 9-row decoder is FFMA (M < 32), its Kc = 768 would fill k-blocks
    ("imp_S3_K3", "improved", imp(3, 3, 256), 801, (True, True, False)),
    # two 128-row decoder tiles (164 rows); 41 taps pad to one encoder k-block
    ("imp_S4_K41", "improved", imp(4, 41, 512, D=4), 3201, (True, True, True)),
    # FFMA mask M = 480 (N % 256 != 0) and FFMA decoder (25 rows, Kc = 480 not a multiple of 64)
    ("imp_S5_K5", "improved", imp(5, 5, 96, Co=32, Ci=64), 1001, (True, False, False)),
    # SA = 16 = the overlap-add's kMaxSrc; tensor-core decoder of 112 rows, FFMA mask
    ("imp_S16_K7", "improved", imp(16, 7, 32, Co=32, Ci=64), 1201, (True, False, True)),
    # mask M = 4096 on tensor cores, decoder 1456 rows x Kc 4096, 91 taps in two encoder k-blocks
    ("imp_S16_K91", "improved", imp(16, 91, 256), 3601, (True, True, True)),
    # GroupComm: K = 91, S = 4, G = 16 (n = 16: the tensor-core TAC), as groupcomm_sudormrf_v2.py's __main__ builds it
    ("gc_S4_A1_K91_G16", "groupcomm", gc(4, 1, 91, 256, 16, 16, D=5), 5761, (True, True, True)),
    ("gc_S8_A2_K21_G8", "groupcomm", gc(8, 2, 21, 16, 8, 4), 801, (False, False, True)),     # S*A = 16
    ("gc_S4_A4_K5_G3", "groupcomm", gc(4, 4, 5, 16, 3, 8), 401, (False, False, True)),       # 3 groups
    ("gc_S2_A8_K11_G5", "groupcomm", gc(2, 8, 11, 16, 5, 32), 401, (False, False, True)),    # FFMA encoder at A = 8, n = 32
    ("gc_S1_A16_K3_G12", "groupcomm", gc(1, 16, 3, 16, 12, 4), 201, (False, False, True)),   # A = 16
    # tensor-core TAC (n = 16), proj_1x1 not folded into the TAC pre-add (cib = 128 > 64), mask M = 3072 with Co = 64
    ("gc_S3_A2_K41_G4", "groupcomm", gc(3, 2, 41, 512, 4, 16, Ci=512), 1601, (True, True, True)),
    # original: sigmoid gate, no reshape layer (Co = N); the 5-row decoder is FFMA
    ("orig_S1_K5", "original", orig(1, 5, 64, 64), 1001, (True, True, False)),
    # odd hop 5: lcm(5, 16) = 80 padding; reshape_before_masks 32 -> 48; FFMA mask (Kc = 48) and decoder (Kc = 144)
    ("orig_S3_K11", "original", orig(3, 11, 48, 32, D=4), 1201, (True, False, False)),
    # hop 20: Toeplitz mask M = 1024 on tensor cores; T = 3121 pads to 3200, L = 160 (L % 8 == 0)
    ("orig_S4_K41", "original", orig(4, 41, 256, 128, D=4), 3121, (True, True, True)),
    # generic softmax path (S = 5), hop 1, D = 5
    ("orig_S5_K3", "original", orig(5, 3, 32, 32, D=5), 993, (True, False, False)),
    # generic path at S = 16; block-diagonal decoder 336 x 256 on tensor cores
    ("orig_S16_K21", "original", orig(16, 21, 16, 16), 801, (False, False, True)),
]


@pytest.mark.parametrize("name,variant,kw,T,want", GRID, ids=[c[0] for c in GRID])
def test_geometry(name, variant, kw, T, want):
    cfg = O.Config(variant=variant, **kw)
    if name == "gc_S3_A2_K41_G4":
        # TAC apply stays a launch of its own: the launch count is that of the unfolded plan
        lib = N.lib()
        levels = 2 if takes_pyramid(cfg, 2, T) else cfg.upsampling_depth
        c = _engine.make_config(CLASSES[variant](**kw))
        assert lib.sdr_forward_launch_count_for(C.byref(c), 2, T) == 2 + cfg.num_blocks * (levels + 3 + 2) + 3
    run_case(variant, kw, T, want)


# ---------------------------------------------------------------------------------------------------------------------
# mixture consistency and separate() at S != 2
# ---------------------------------------------------------------------------------------------------------------------
MC_CASES = [c for c in GRID if c[0] in ("imp_S1_K21", "imp_S3_K3", "imp_S5_K5", "imp_S16_K7", "orig_S5_K3",
                                        "orig_S16_K21")]


@pytest.mark.parametrize("name,variant,kw,T,want", MC_CASES, ids=[c[0] for c in MC_CASES])
def test_mixture_consistency_in_the_overlap_add(name, variant, kw, T, want):
    """separate(x, mixture_consistency=True) without normalisation: the 1/SA projection inside the overlap-add against
    O.mixture_consistency on the fp64 forward; at S = 1 it returns the mixture itself."""
    cfg, sd, m = build(variant, kw)
    x = normalised_input(2, 1, T, seed=5).to(DEV) * 0.7 + 0.1
    with torch.no_grad():
        y = m.separate(x, mixture_consistency=True)
    ref = O.mixture_consistency(O.forward(cfg, sd, x, dtype=torch.float64), x.double())
    e = O.parity_errors(y, ref)
    print(f"{name} mixture consistency: rel_max {e[0]:.3e} rel_l2 {e[1]:.3e}")
    assert max(e) < TOL, e
    if cfg.num_sources == 1:
        assert max(O.parity_errors(y, x)) < 1e-6


SEP_CASES = [c for c in GRID if c[0] in ("imp_S4_K41", "orig_S4_K41")]


@pytest.mark.parametrize("mc", [False, True])
@pytest.mark.parametrize("name,variant,kw,T,want", SEP_CASES, ids=[c[0] for c in SEP_CASES])
def test_separate_normalize_four_sources(name, variant, kw, T, want, mc):
    """The README recipe on the device at S = 4: per-utterance normalisation, forward, the rescale inside the
    overlap-add, then optionally mixture consistency against the normalised mixture."""
    cfg, sd, m = build(variant, kw)
    g = torch.Generator().manual_seed(17)
    wav = (torch.randn(2, T, generator=g) * torch.tensor([[0.05], [6.0]]) + torch.tensor([[0.3], [-1.2]])).to(DEV)
    with torch.no_grad():
        y = m.separate(wav, mixture_consistency=mc, normalize=True)
    ref = O.separate(cfg, sd, wav, apply_mixture_consistency=mc, dtype=torch.float64)
    e = O.parity_errors(y, ref)
    print(f"{name} separate(normalize=True, mixture_consistency={mc}): rel_max {e[0]:.3e} rel_l2 {e[1]:.3e}")
    assert max(e) < TOL, e


# ---------------------------------------------------------------------------------------------------------------------
# refusal boundaries: each side
# ---------------------------------------------------------------------------------------------------------------------
def refused(m, x, message):
    with torch.no_grad(), pytest.raises(N.NativeError, match=message):
        m(x)
    torch.cuda.synchronize()                # no CUDA error is left behind


BAD_CONFIG = "bad model configuration"
UNSUPPORTED = "configuration not supported by the sm_90a kernels"


@pytest.mark.parametrize("variant,ok,bad", [
    ("improved", imp(16, 5, 16, Co=16, Ci=32), imp(17, 5, 16, Co=16, Ci=32)),             # S = 16 / 17
    ("groupcomm", gc(8, 2, 5, 16, 4, 4), gc(9, 2, 5, 16, 4, 4)),                           # S*A = 16 / 18
    ("groupcomm", gc(2, 1, 5, 16, 4, 8), gc(2, 1, 5, 16, 4, 12)),                          # group width 8 / 12
    ("groupcomm", gc(2, 1, 5, 16, 4, 32), gc(2, 1, 5, 16, 2, 64)),                         # group width 32 / 64
    ("groupcomm", gc(2, 1, 5, 16, 16, 4), gc(2, 1, 5, 16, 17, 4)),                         # 16 / 17 groups
    ("groupcomm", gc(4, 4, 99, 16, 4, 4), gc(4, 4, 101, 16, 4, 4)),                        # FFMA encoder, A = 4: K 99 / 101
    ("groupcomm", gc(1, 16, 25, 16, 4, 4), gc(1, 16, 27, 16, 4, 4)),                       # FFMA encoder, A = 16: K 25 / 27
], ids=["S17", "SA18", "n12", "n64", "G17", "enc_A4_K101", "enc_A16_K27"])
def test_refusal_boundaries(variant, ok, bad):
    """The refused configuration raises NativeError with the library's message before a forward kernel runs; the
    configuration on the other side of the boundary runs and matches the fp64 oracle."""
    A = bad.get("in_audio_channels", 1)
    cfg_bad = O.Config(variant=variant, **bad)
    T = 2 * cfg_bad.n_least_samples_req + 1
    m_bad = CLASSES[variant](**bad)
    m_bad.load_state_dict(O.make_state_dict(cfg_bad, seed=3))
    m_bad = m_bad.to(DEV).eval()
    x = normalised_input(2, A, T, seed=4).to(DEV)
    c = _engine.make_config(m_bad)
    lib = N.lib()
    if cfg_bad.num_sources * A > 16:
        assert lib.sdr_num_params(C.byref(c)) == -1
        refused(m_bad, x, BAD_CONFIG)
    else:
        assert lib.sdr_num_params(C.byref(c)) > 0
        refused(m_bad, x, UNSUPPORTED)
        # a refusal before anything is enqueued: the null buffers behind it are never reached
        assert lib.sdr_forward(C.byref(c), None, None, None, 2, T, 0, None, 0, None) == -5
        assert lib.sdr_workspace_bytes(C.byref(c), 2, T) > 0
    assert not paths(cfg_bad)[0]            # N = 16: the FFMA encoder
    T_ok = 2 * O.Config(variant=variant, **ok).n_least_samples_req + 1
    run_case(variant, ok, T_ok, paths(O.Config(variant=variant, **ok)))


def test_original_length_rule():
    """K = 41, D = 4: lcm(20, 16) = 80.  T = 240 pads to L = 12 frames, which three stride-2 levels cannot halve
    exactly (the reference fails there too): refused.  The same model object then runs T = 160 (L = 8) and T = 401
    (L = 24) correctly."""
    kw = orig(4, 41, 32, 32, D=4)
    cfg, sd, m = build("original", kw)
    x = normalised_input(2, 1, 240, seed=6).to(DEV)
    refused(m, x, UNSUPPORTED)
    for T in (160, 401):
        x = normalised_input(2, 1, T, seed=T).to(DEV)
        with torch.no_grad():
            y = m(x)
        e = O.parity_errors(y, O.forward(cfg, sd, x, dtype=torch.float64))
        print(f"original K=41 D=4 T={T}: rel_max {e[0]:.3e} rel_l2 {e[1]:.3e}")
        assert max(e) < TOL, e


# ---------------------------------------------------------------------------------------------------------------------
# the FUSS recipe (run_fuss_separation.py) end to end
# ---------------------------------------------------------------------------------------------------------------------
FUSS = dict(out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
            enc_num_basis=512, num_sources=4)                 # the script's defaults (max_num_sources = 4)
FUSS_MODELS = [                                               # run_fuss_separation.py:133-170, model_type ->
    ("relu", "improved", FUSS),
    ("causal", "causal", dict(FUSS, in_audio_channels=1)),
    ("softmax", "original", FUSS),
    ("groupcomm_v2", "groupcomm", dict(FUSS, in_audio_channels=1, group_size=16)),
]
FUSS_T, FUSS_B = 160000, 2                                    # 10 s at 16 kHz


def assignment_scores(pr, tgt, n_est, perms):
    """[B, len(perms)]: the stabilised SI-SDR of every assignment, zero-mean (sisdr.py:508-533), without the SI-SDRi
    baseline (it is the same for every assignment)."""
    pr = pr[:, :n_est] - pr[:, :n_est].mean(-1, keepdim=True)
    tgt = tgt - tgt.mean(-1, keepdim=True)
    tt = (tgt * tgt).sum(-1)
    cols = []
    for p in perms:
        q = pr[:, list(p)]
        rho_sq = (q * tgt).sum(-1) ** 2 / ((q * q).sum(-1) * tt + 1e-9)
        cols.append((10 * torch.log10((rho_sq + 1e-9) / (1. - rho_sq + 1e-9))).mean(-1))
    return torch.stack(cols, -1)


def fuss_metric(n_act):
    """run_fuss_separation.py:105-131."""
    n_est = 1 if n_act == 1 else FUSS["num_sources"]
    return SI.StabilizedPermInvSISDRMetric(zero_mean=True, single_source=False, n_estimated_sources=n_est,
                                           n_actual_sources=n_act, backward_loss=False, improvement=n_act > 1,
                                           return_individual_results=True), n_est


@pytest.mark.parametrize("model_type,variant,kw", FUSS_MODELS, ids=[c[0] for c in FUSS_MODELS])
def test_fuss_validation_loop(model_type, variant, kw):
    """For 1..4 actual sources: seeded clean sources, their sum normalised as at :289-292, model, mixture_consistency
    .apply, the metric on all four estimate rows.  The estimates are held to the fp64 oracle (1e-4), the scores to the
    oracle's metric on the oracle's estimates (2e-3 dB), and the reported assignment must be the oracle's best (or,
    where two assignments are closer than that, score within 2e-3 dB of it in fp64)."""
    cfg, sd, m = build(variant, kw, seed=223)
    g = torch.Generator().manual_seed(227)
    for n_act in range(1, 5):
        clean = (torch.randn(FUSS_B, n_act, FUSS_T, generator=g) * (0.2 + torch.rand(FUSS_B, n_act, 1, generator=g)))
        clean = clean.to(DEV)
        mix = torch.sum(clean, -2, keepdim=True)
        mix = (mix - mix.mean(-1, keepdim=True)) / (mix.std(-1, keepdim=True) + 1e-9)
        with torch.no_grad():
            rec = m(mix)
            if n_act == 1:
                check_launch_count(m, FUSS_B, FUSS_T, lambda: m(mix))
            rec = P.mixture_consistency.apply(rec, mix)
            metric, n_est = fuss_metric(n_act)
            score, best_perm = metric(rec, clean, return_best_permutation=True)
        ref = O.mixture_consistency(O.forward(cfg, sd, mix, dtype=torch.float64), mix.double())
        e = O.parity_errors(rec, ref)
        want, idx = O.stabilized_pit_sisdr(ref, clean.double(), zero_mean=True, improvement=n_act > 1,
                                           n_estimated=n_est)
        # every assignment's fp64 score on the oracle's estimates, to judge near-ties
        perms = list(itertools.permutations(range(n_est), r=n_act))
        cols = assignment_scores(ref, clean.double(), n_est, perms)
        assert torch.equal(cols.argmax(-1), idx)
        got_idx = [perms.index(tuple(int(v) for v in row)) for row in best_perm.cpu()]
        print(f"FUSS {model_type} n_act={n_act}: estimates rel_max {e[0]:.3e} rel_l2 {e[1]:.3e}; "
              f"score {score.cpu().tolist()} vs fp64 {want.cpu().tolist()}")
        assert max(e) < TOL, e
        assert torch.allclose(score.cpu().double(), want.cpu(), atol=2e-3, rtol=0), (score, want)
        for b in range(FUSS_B):
            if got_idx[b] != int(idx[b]):
                assert float(cols[b, int(idx[b])] - cols[b, got_idx[b]]) < 2e-3, (b, got_idx[b], int(idx[b]))
