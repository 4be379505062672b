"""A NaN or an infinity in one mixture stays in that mixture and comes out where the fp64 reference's does.

Callers do pass such data (a corrupt wav in a corpus bucket, a bad stream slot, an upstream stage that overflowed).
Two promises, for a non-finite value (NaN, +inf or -inf) anywhere in mixture j:

- (C) containment: every other mixture's output is what it is on the clean batch: bitwise where no atomics order
  the sums (the causal model, the stream, the stage outputs), within the clean-to-clean spread otherwise (bound 1e-5
  of max |output|, as test_gpu_scratch.compare_runs measures it); the other samples' statistics slots likewise.
  A 1e30 in mixture j (finite, but overflowing any square) is tested for (C) only.
- (P) propagation: element by element, the output is non-finite exactly where the fp64 reference on the same input
  is (NaN and +-inf are not told apart), and within the usual bar where the reference is finite.  The tensor-core
  entries split an operand into three bf16 parts, so an infinite operand is NaN to them (lo = inf - inf): their
  reference takes it as NaN.  The causal model's reference drops its masked taps (oracle.causal_forward
  masked_taps="dropped"); the reference's own arithmetic multiplies them by zero and so leaks a NaN backwards in time,
  which the native code deliberately does not reproduce.

Finite data cannot tell masking by multiplication (0 * x) from masking by selection, so every place where rows meet
(flattened rows, tile edges, halos, padded taps, slot columns) is exercised here with a non-finite neighbour, at the
first and last element of the first, a middle and the last sample, at shapes where samples share a CTA or a tile.

The ReLU sites of the kernels follow torch.relu (NaN stays NaN, -inf -> 0, +inf stays); RELU_SITES names each with the
entry that reaches it, and test_every_relu_site_is_exercised checks the table against the sources and the tests."""
import ctypes as C
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _engine
import sudo_rm_rf_b200.mixture_consistency as MC
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.corpus import separate_corpus
from sudo_rm_rf_b200.streaming import CausalStream
from oracle import sudormrf_oracle as O
from test_gpu_long import normalised_input
from test_gpu_model_space import build
from test_gpu_scratch import CASES
from test_gpu_stages import channel_slopes, norm_in, p, raw_stats, stream

gpu = pytest.mark.gpu
DEV = "cuda"
NAN, INF = float("nan"), float("inf")
BAD = [("nan", NAN), ("+inf", INF), ("-inf", -INF), ("1e30", 1e30)]
SPREAD = 1e-5
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "sudo_rm_rf_b200", "csrc")

# Every ReLU of the kernels, the entry that reaches it and the test here that puts NaN through it.
RELU_SITES = [
    # file, the line's code, the entry that reaches it, the parameter ids here that put NaN through it, a whole-model
    # case (test_gpu_scratch.CASES) that reaches it.  The two float4 lines of pointwise.cu are written the same way in
    # pw_gemm_kernel and pw_small_kernel.
    ("pointwise_mma.cu", "if (MODE == 2) o = relu(o) * *e;", "sdr_pointwise_mma",
     ["test_pointwise_mma_stage[mask]", "test_pointwise_mma_stage[mask_b5]", "test_training_forward[wgmma_mask]"],
     "imp_D4_pyramid_wgmma"),
    ("pointwise_mma.cu", "if constexpr (WINDOW) { if (relu_out) o = relu(o); }", "sdr_encoder_mma_ex",
     ["test_encoder_stage[mma-relu-A1-B5]", "test_encoder_stage[mma-relu-A2-B3]"], "orig_S3_softmax_pyramid"),
    ("pointwise.cu", "o[0] = relu(o[0]) * g.x; o[1] = relu(o[1]) * g.y;", "sdr_pointwise",
     ["test_pointwise_stage[gemm_vec_mask]", "test_pointwise_stage[small_mask]"], "imp_D6_pyramid_mixed"),
    ("pointwise.cu", "o[2] = relu(o[2]) * g.z; o[3] = relu(o[3]) * g.w;", "sdr_pointwise",
     ["test_pointwise_stage[gemm_vec_mask]", "test_pointwise_stage[small_mask]"], "imp_D5_pyramid_ffma"),
    # the forwards' frame counts are multiples of 2^upsampling_depth, so only a depth of 0 or 1 reaches the tail
    ("pointwise.cu", "if (a.epilogue == 1) v = relu(v) * __ldg(grow + l + e);", "sdr_pointwise",
     ["test_pointwise_stage[gemm_tail_mask]", "test_pointwise_stage[gemm_tail_mask_b5]"], None),
    ("frontback.cu", "if (relu_out) o[e] = relu(o[e]);", "sdr_encoder_ex",
     ["test_encoder_stage[ffma-relu-A1-B5]", "test_encoder_stage[ffma-relu-A2-B3]"], "orig_S1_sigmoid"),
    ("backward.cu", "masked[i] = relu(mlog[i]) * __ldg(e + b * NL + r);", "sdr_forward_train",
     ["test_training_forward[wgmma_mask]", "test_training_forward[ffma_mask]"], None),
]


def bits(t):
    return t.contiguous().view(torch.int32)


def sites(shape):
    """(sample, index) pairs: the first element of the first, a middle and the last sample, and the last element of
    each -- the two ends of a sample, where it meets its neighbours in a flattened run."""
    B = shape[0]
    for j in sorted({0, B // 2, B - 1}):
        yield j, (0,) * (len(shape) - 1)
        yield j, tuple(s - 1 for s in shape[1:])


def stats_close(got, clean, n, what):
    """(C) of a statistics slot: fp64 atomics may order the sums differently, nothing more."""
    got, clean = got.reshape(-1, 2), clean.reshape(-1, 2)
    sq = clean[:, 1].abs()
    scale = torch.stack([(n * sq).sqrt(), sq], dim=1) + 1e-30
    err = float(((got - clean).abs() / scale).max()) if got.numel() else 0.0
    assert err < 1e-9, (what, err, got, clean)


def check_class(got, want, what, tol):
    """(P): non-finite exactly where `want` is, and `tol`-close (relative to max |want|) where it is finite."""
    gbad, wbad = ~torch.isfinite(got), ~torch.isfinite(want)
    if not torch.equal(gbad, wbad):
        diff = (gbad != wbad).nonzero()
        raise AssertionError(f"{what}: {diff.shape[0]} elements differ in class, first {diff[:4].tolist()}; "
                             f"got {int(gbad.sum())} non-finite, the reference {int(wbad.sum())}")
    fin = ~wbad
    if fin.any():
        w = want[fin].double()
        err = float((got[fin].double() - w).abs().max() / w.abs().max().clamp_min(1e-30))
        assert err < tol, (what, err)


def check_stage(what, run, ref, ins, key, tc=False, tol=2e-5, values=BAD, where=None):
    """run(ins) -> {name: device output}; fp64 outputs are statistics [B, 2].  ref(ins) -> {name: fp64 reference}
    for the fp32 outputs.  A bad value goes into ins[key] at every site; the clean outputs must be reproducible."""
    clean = run(ins)
    again = run(ins)
    for k, t in clean.items():
        if t.dtype == torch.float64:
            n = max(v[0].numel() for v in clean.values() if v.dtype == torch.float32)
            stats_close(again[k], t, n, (what, k, "clean / clean"))
        else:
            assert torch.equal(bits(again[k]), bits(t)), (what, k, "clean / clean")
    want_clean = ref(ins)
    for k, w in want_clean.items():
        check_class(clean[k], w, (what, k, "clean"), tol)
    x = ins[key]
    for vname, v in values:
        for j, idx in (where or sites(x.shape)):
            bad = dict(ins)
            bad[key] = x.clone()
            bad[key][(j,) + idx] = v
            got = run(bad)
            others = [b for b in range(x.shape[0]) if b != j]
            tag = (what, key, vname, j, idx)
            for k, t in got.items():
                if t.dtype == torch.float64:
                    n = max(u[0].numel() for u in got.values() if u.dtype == torch.float32)
                    stats_close(t[others], clean[k][others], n, tag + (k,))
                else:
                    assert torch.equal(bits(t[others]), bits(clean[k][others])), tag + (k, "(C)")
            if math.isfinite(v):
                continue
            rin = dict(bad)
            if tc:                 # the bf16x3 split: an infinite operand is NaN to the tensor cores
                rin[key] = torch.where(torch.isinf(bad[key]), torch.full_like(bad[key], NAN), bad[key])
            for k, w in ref(rin).items():
                check_class(got[k][j], w[j], tag + (k, "(P)"), tol)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def rnd(g, *shape, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=g) * scale + shift).to(DEV)


def ref_norm(x, gamma, beta, prelu=None):
    y = O.glob_ln(x, gamma, beta) if gamma is not None else x
    if prelu is None:
        return y
    return O.prelu_c(y, prelu) if prelu.numel() > 1 else O.prelu1(y, prelu)


# =====================================================================================================================
# 0. the table of ReLU sites (no device needed)
# =====================================================================================================================
def test_every_relu_site_is_exercised():
    """Every ReLU in the kernels has a row, every row's line is in its file, and the tests it names exist here."""
    srcs = {f: open(os.path.join(CSRC, f)).read() for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))}
    ids = {"test_encoder_stage": ENCODER_IDS, "test_pointwise_stage": [c[0] for c in POINTWISE],
           "test_pointwise_mma_stage": [c[0] for c in POINTWISE_MMA], "test_training_forward": TRAINING_IDS}
    for f, code, entry, tests, case in RELU_SITES:
        assert code in srcs[f], (f, code)
        assert f"int {entry}(" in srcs["api.cu"], entry
        assert case is None or case in [c[0] for c in CASES], case
        for t in tests:
            name, pid = t[:-1].split("[")
            assert pid in ids[name], t
    # nothing outside the table: a ReLU is written relu(...), never as an fmaxf against zero
    found = set()
    for f, s in srcs.items():
        for line in s.splitlines():
            code = line.split("//")[0].strip()
            if "__device__" in code:                      # the helper itself
                continue
            if re.search(r"\brelu\(", code):
                found.add((f, code))
            assert not re.search(r"fmaxf\([^,]+,\s*0(\.0*)?f?\)", code), (f, code, "swallows NaN: use relu()")
    rows = {(f, code) for f, code, *_ in RELU_SITES}
    assert found == rows, (found - rows, rows - found)


# =====================================================================================================================
# 1. stage entries
# =====================================================================================================================
ENCODER = [  # kernel, relu, B, A, T, N, K, L (L odd where the kernel allows it)
    ("ffma", False, 3, 1, 517, 24, 21, 53), ("ffma", True, 5, 1, 203, 20, 11, 41), ("ffma", True, 3, 2, 333, 16, 11, 67),
    ("ffma", False, 5, 2, 97, 8, 5, 49),
    ("mma", False, 3, 1, 517, 64, 21, 53), ("mma", True, 5, 1, 203, 64, 11, 41), ("mma", True, 3, 2, 333, 160, 11, 67),
    ("mma", False, 5, 2, 1280, 32, 21, 129),
]


ENCODER_IDS = [f"{c[0]}-{'relu' if c[1] else 'plain'}-A{c[3]}-B{c[2]}" for c in ENCODER]


@gpu
@pytest.mark.parametrize("kern,relu,B,A,T,N_,K,L", ENCODER, ids=ENCODER_IDS)
def test_encoder_stage(kern, relu, B, A, T, N_, K, L):
    """sdr_encoder_ex / sdr_encoder_mma_ex: the bad sample in the waveform; ReLU on as in the original model."""
    lib = N.lib()
    g = gen(31)
    hop = K // 2
    assert T <= hop * L
    w = rnd(g, N_, A, K)
    bias = rnd(g, N_, scale=0.3) if relu else None
    if kern == "mma":
        wpk = torch.empty(lib.sdr_encoder_mma_packed_bytes(N_, A, K), dtype=torch.uint8, device=DEV)
        assert wpk.numel() > 0
        N.check(lib.sdr_encoder_mma_pack(p(w), N_, A, K, p(wpk), stream()))

    def run(ins):
        enc = torch.full((B, N_, L), NAN, device=DEV)
        st = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
        if kern == "mma":
            rc = lib.sdr_encoder_mma_ex(p(ins["wav"]), p(wpk), p(bias), int(relu), hop, p(enc), p(st), B, A, T, N_, K,
                                        L, stream())
        else:
            rc = lib.sdr_encoder_ex(p(ins["wav"]), p(w), p(bias), int(relu), hop, p(enc), p(st), B, A, T, N_, K, L,
                                    stream())
        N.check(rc)
        torch.cuda.synchronize()
        return {"enc": enc, "stats": st}

    def ref(ins):
        xp = torch.zeros(B, A, hop * L, device=DEV, dtype=torch.float64)
        xp[..., :T] = ins["wav"]
        y = F.conv1d(xp, w.double(), bias.double() if bias is not None else None, stride=hop, padding=hop)
        return {"enc": torch.relu(y) if relu else y}

    check_stage("encoder", run, ref, {"wav": rnd(g, B, A, T)}, "wav", tc=kern == "mma",
                tol=5e-5 if kern == "mma" else 2e-5)


POINTWISE = [  # id, samples, M, K, L, mode; the dispatch rules of launch_pointwise_ffma pick the kernel
    ("gemm_vec_mask", 3, 128, 32, 132, "mask"),      # pw_gemm_kernel<128, true>: the gated epilogue's float4 path
    ("gemm_tail_mask", 3, 128, 32, 131, "mask"),     # pw_gemm_kernel<128, false>: the scalar path (L % 4 != 0)
    ("gemm_tail_mask_b5", 5, 48, 20, 25, "mask"),
    ("small_mask", 5, 32, 16, 132, "mask"),          # pw_small_kernel with the gated epilogue
    ("small_norm", 5, 48, 24, 100, "norm"),          # pw_small_kernel, normalised input, statistics
    ("tile_plain", 5, 32, 16, 132, "plain"),         # pw_tile_kernel (epilogue 0, M <= 32)
    ("tile_res", 3, 16, 8, 1604, "res"),
    ("gemm_norm", 3, 130, 33, 101, "norm"),
]


@gpu
@pytest.mark.parametrize("samples,M,K,L,mode", [c[1:] for c in POINTWISE], ids=[c[0] for c in POINTWISE])
def test_pointwise_stage(samples, M, K, L, mode):
    """sdr_pointwise (FFMA): the bad value in the operand, the residual and the gate."""
    g = gen(32)
    W = rnd(g, M, K, scale=K ** -0.5)
    bias = rnd(g, M)
    gamma, beta, slope = rnd(g, K, scale=0.3, shift=1.0), rnd(g, K, scale=0.2), torch.tensor([0.2], device=DEV)
    gate_ch = M // 2 if mode == "mask" else 0
    ins = {"x": rnd(g, samples, K, L, shift=0.5)}
    if mode == "mask":
        ins["gate"] = rnd(g, samples, gate_ch, L)
    if mode == "res":
        ins["res"] = rnd(g, samples, M, L)

    def run(ins):
        x = ins["x"]
        st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        stats_in = raw_stats(x).to(DEV)
        if mode in ("norm", "res"):
            nin = norm_in(stats_in, gamma, beta, slope if mode == "res" else None, K * L)
        elif mode == "mask":
            nin = norm_in(None, None, None, slope, 1.0)
        else:
            nin = norm_in()
        y = ins["res"].clone() if mode == "res" else torch.full((samples, M, L), NAN, device=DEV)
        N.check(N.lib().sdr_pointwise(p(x), C.byref(nin), p(W), p(bias), p(y) if mode == "res" else p(None),
                                      p(ins.get("gate")), gate_ch, p(y), p(st), samples, M, K, L,
                                      1 if mode == "mask" else 0, stream()))
        torch.cuda.synchronize()
        return {"y": y, "stats": st}

    def ref(ins):
        x = ins["x"].double()
        if mode in ("norm", "res"):
            fx = ref_norm(x, gamma.double(), beta.double(), slope.double() if mode == "res" else None)
        elif mode == "mask":
            fx = O.prelu1(x, slope.double())
        else:
            fx = x
        y = torch.einsum("mk,skl->sml", W.double(), fx) + bias.double().view(1, -1, 1)
        if mode == "res":
            y = y + ins["res"].double()
        if mode == "mask":
            y = torch.relu(y) * ins["gate"].double()[:, torch.arange(M, device=DEV) % gate_ch]
        return {"y": y}

    for key in ins:
        check_stage(f"pointwise {mode}", run, ref, ins, key, tol=3e-5)


POINTWISE_MMA = [  # id, samples, M, K, L, mode
    ("mask", 3, 512, 128, 200, "mask"),              # MODE 2: relu(mlog) * e, ragged last position tile
    ("mask_b5", 5, 256, 64, 36, "mask"),             # several samples in the persistent CTAs' tile sequence
    ("res", 3, 256, 128, 132, "res"),                # MODE 1: in-place residual
    ("plain_stats", 5, 128, 64, 100, "plain"),
    ("norm", 3, 128, 64, 68, "norm"),
]


@gpu
@pytest.mark.parametrize("samples,M,K,L,mode", [c[1:] for c in POINTWISE_MMA], ids=[c[0] for c in POINTWISE_MMA])
def test_pointwise_mma_stage(samples, M, K, L, mode):
    """sdr_pointwise_mma in every epilogue mode: the bad value in the operand (bf16x3: inf counts as NaN), the residual
    and the gate (fp32 epilogue operands: their real value)."""
    lib = N.lib()
    g = gen(33)
    W = rnd(g, M, K, scale=K ** -0.5)
    bias = rnd(g, M)
    gamma, beta, slope = rnd(g, K, scale=0.3, shift=1.0), rnd(g, K, scale=0.2), torch.tensor([0.2], device=DEV)
    wpk = torch.empty(lib.sdr_pointwise_mma_packed_bytes(M, K), dtype=torch.uint8, device=DEV)
    assert wpk.numel() > 0
    N.check(lib.sdr_pointwise_mma_pack(p(W), M, K, p(wpk), stream()))
    gate_ch = M // 2 if mode == "mask" else 0
    ins = {"x": rnd(g, samples, K, L, shift=0.5)}
    if mode == "mask":
        ins["gate"] = rnd(g, samples, gate_ch, L)
    if mode == "res":
        ins["res"] = rnd(g, samples, M, L)

    def run(ins):
        x = ins["x"]
        st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        stats_in = raw_stats(x).to(DEV)
        if mode in ("norm", "res"):
            nin = norm_in(stats_in, gamma, beta, slope if mode == "res" else None, K * L)
        elif mode == "mask":
            nin = norm_in(None, None, None, slope, 1.0)
        else:
            nin = norm_in()
        y = ins["res"].clone() if mode == "res" else torch.full((samples, M, L), NAN, device=DEV)
        want_stats = mode == "plain"
        N.check(lib.sdr_pointwise_mma(p(x), C.byref(nin), p(wpk), p(bias), p(y) if mode == "res" else p(None),
                                      p(ins.get("gate")), gate_ch, p(y), p(st) if want_stats else p(None),
                                      samples, M, K, L, 1 if mode == "mask" else 0, stream()))
        torch.cuda.synchronize()
        return {"y": y, "stats": st} if want_stats else {"y": y}

    def ref(ins):
        x = ins["x"].double()
        if mode in ("norm", "res"):
            fx = ref_norm(x, gamma.double(), beta.double(), slope.double() if mode == "res" else None)
        elif mode == "mask":
            fx = O.prelu1(x, slope.double())
        else:
            fx = x
        y = torch.einsum("mk,skl->sml", W.double(), fx) + bias.double().view(1, -1, 1)
        if mode == "res":
            y = y + ins["res"].double()
        if mode == "mask":
            y = torch.relu(y) * ins["gate"].double()[:, torch.arange(M, device=DEV) % gate_ch]
        return {"y": y}

    for key in ins:
        check_stage(f"pointwise_mma {mode}", run, ref, ins, key, tc=key == "x", tol=5e-5)


DEPTHWISE = [  # samples, C, L, stride, norm: the wide (Lout % 8 == 0), vector and scalar kernels
    (3, 16, 64, 1, True), (5, 16, 64, 1, False), (3, 512, 96, 2, False), (5, 7, 27, 1, False), (3, 9, 18, 2, True),
    (5, 6, 26, 2, False),
]


@gpu
@pytest.mark.parametrize("samples,C_,L,stride,norm", DEPTHWISE)
def test_depthwise_stage(samples, C_, L, stride, norm):
    """sdr_depthwise: without statistics a bad value reaches only its own halo, so any read across a row end shows."""
    g = gen(34)
    gamma, beta, slope = rnd(g, C_, scale=0.3, shift=1.0), rnd(g, C_, scale=0.2), torch.tensor([0.3], device=DEV)
    w, b = rnd(g, C_, 1, 5), rnd(g, C_)
    Lout = (L - 1) // stride + 1

    def run(ins):
        x = ins["x"]
        stats_in = raw_stats(x).to(DEV)
        nin = norm_in(stats_in, gamma, beta, slope, C_ * L) if norm else norm_in(None, None, None, slope, 1.0)
        y = torch.full((samples, C_, Lout), NAN, device=DEV)
        st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        N.check(N.lib().sdr_depthwise(p(x), C.byref(nin), p(w), p(b), p(y), p(st), samples, C_, L, stride, stream()))
        torch.cuda.synchronize()
        return {"y": y, "stats": st}

    def ref(ins):
        x = ins["x"].double()
        fx = ref_norm(x, gamma.double(), beta.double(), slope.double()) if norm else O.prelu1(x, slope.double())
        return {"y": F.conv1d(fx, w.double(), b.double(), stride=stride, padding=2, groups=C_)}

    check_stage("depthwise", run, ref, {"x": rnd(g, samples, C_, L, scale=2.0, shift=0.7)}, "x")


PYRAMID = [(3, 7, 48, 4, False), (5, 9, 96, 5, True), (3, 6, 192, 6, False), (3, 32, 3200, 5, True)]


@gpu
@pytest.mark.parametrize("samples,C_,L,D,fused", PYRAMID)
def test_pyramid_stage(samples, C_, L, D, fused):
    """sdr_depthwise_pyramid (+ sdr_merge_pyramid) and sdr_depthwise_pyramid_fused: overlapping warp windows whose next
    row arrives by bulk TMA.  The level statistics spread a bad value over its sample; no other sample may see it."""
    lib = N.lib()
    g = gen(35)
    gy, by = rnd(g, C_, scale=0.3, shift=1.0), rnd(g, C_, scale=0.2)
    slope = torch.tensor([0.3], device=DEV)
    ws = [rnd(g, C_, 1, 5, scale=0.6) for _ in range(D)]
    bs = [rnd(g, C_, scale=0.5) for _ in range(D)]
    gs = [rnd(g, C_, scale=0.3, shift=1.0) for _ in range(D)]
    bes = [rnd(g, C_, scale=0.2) for _ in range(D)]
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    nbytes = lib.sdr_pyramid_scratch_bytes(samples, C_, D, L)
    assert nbytes > 0

    def run(ins):
        y = ins["x"]
        stats_in = raw_stats(y).to(DEV)              # kept alive: the struct holds a raw pointer
        nin = norm_in(stats_in, gy, by, slope, C_ * L)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        zs = [torch.full((samples, C_, L >> d), NAN, device=DEV) for d in range(D)]
        st0 = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        stm = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        m = torch.full((samples, C_, L), NAN, device=DEV)
        if fused:
            N.check(lib.sdr_depthwise_pyramid_fused(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), p(m),
                                                    p(st0), p(stm), p(scratch), D, samples, C_, L, stream()))
            out = {"m": m, "stats_0": st0, "stats_m": stm}
        else:
            N.check(lib.sdr_depthwise_pyramid(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(st0),
                                              p(scratch), D, samples, C_, L, stream()))
            N.check(lib.sdr_merge_pyramid(arr(zs), p(scratch), D, p(m), p(stm), samples, C_, L, stream()))
            out = {"z0": zs[0], "m": m, "stats_0": st0, "stats_m": stm}
        torch.cuda.synchronize()
        return out

    def ref(ins):
        cur = ref_norm(ins["x"].double(), gy.double(), by.double(), slope.double())
        levels, z0 = [], None
        for d in range(D):
            z = F.conv1d(cur, ws[d].double(), bs[d].double(), stride=1 if d == 0 else 2, padding=2, groups=C_)
            z0 = z if d == 0 else z0
            cur = ref_norm(z, gs[d].double(), bes[d].double())
            levels.append(cur)
        for _ in range(D - 1):
            top = levels.pop()
            levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
        return {"m": levels[0]} if fused else {"z0": z0, "m": levels[0]}

    check_stage("pyramid", run, ref, {"x": rnd(g, samples, C_, L, scale=1.3, shift=0.3)}, "x", tol=1e-4)


CAUSAL_PYRAMID = [(3, 8, 48, 4), (5, 7, 64, 2), (3, 16, 256, 1), (5, 4, 128, 5)]


@gpu
@pytest.mark.parametrize("samples,C_,L,D", CAUSAL_PYRAMID)
def test_causal_pyramid_stage(samples, C_, L, D):
    """sdr_causal_pyramid reads only the 11 surviving taps: a bad value reaches the outputs at and after it, in its
    own channel, and the reference that drops the masked taps says exactly which."""
    lib = N.lib()
    g = gen(36)
    sp = torch.tensor([0.3], device=DEV)
    ws = [rnd(g, C_, 1, 21, scale=0.4) for _ in range(D)]
    bs = [rnd(g, C_, scale=0.5) for _ in range(D)]
    sl = [torch.tensor([0.1 + 0.07 * d], device=DEV) for d in range(D)]
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])

    def run(ins):
        m = torch.full((samples, C_, L), NAN, device=DEV)
        N.check(lib.sdr_causal_pyramid(p(ins["x"]), p(sp), arr(ws), arr(bs), arr(sl), p(m), D, samples, C_, L,
                                       stream()))
        torch.cuda.synchronize()
        return {"m": m}

    def ref(ins):
        cur = O.prelu1(ins["x"].double(), sp.double())
        levels = []
        for d in range(D):
            cur = O.prelu1(O.causal_conv(cur, ws[d].double(), bs[d].double(), stride=1 if d == 0 else 2, padding=10,
                                         groups=C_, masked_taps="dropped"), sl[d].double())
            levels.append(cur)
        for _ in range(D - 1):
            top = levels.pop()
            levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
        return {"m": levels[0]}

    check_stage("causal_pyramid", run, ref, {"x": rnd(g, samples, C_, L, scale=1.3, shift=0.1)}, "x")


@gpu
@pytest.mark.parametrize("samples,C_,L,depth", [(3, 5, 24, 4), (5, 8, 48, 4), (3, 7, 128, 6), (5, 6, 6, 2)])
def test_merge_stage(samples, C_, L, depth):
    """sdr_merge (the per-level path): a bad value in the finest level, whose statistics spread it over its sample."""
    g = gen(41)
    gammas = [rnd(g, C_, scale=0.3, shift=1.0) for _ in range(depth)]
    betas = [rnd(g, C_, scale=0.2) for _ in range(depth)]
    zs = [rnd(g, samples, C_, L >> d, shift=0.3 * d) for d in range(depth)]

    def run(ins):
        levels = [ins["z0"]] + zs[1:]
        stats = [raw_stats(z).to(DEV) for z in levels]          # kept alive: the structs hold raw pointers
        fins = (N.SdrNormIn * depth)(*[norm_in(stats[d], gammas[d], betas[d], None, C_ * (L >> d))
                                      for d in range(depth)])
        zp = (C.c_void_p * depth)(*[z.data_ptr() for z in levels])
        m = torch.full((samples, C_, L), NAN, device=DEV)
        st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        N.check(N.lib().sdr_merge(zp, fins, depth, p(m), p(st), samples, C_, L, stream()))
        torch.cuda.synchronize()
        return {"m": m, "stats": st}

    def ref(ins):
        levels = [ref_norm(z.double(), gammas[d].double(), betas[d].double())
                  for d, z in enumerate([ins["z0"]] + zs[1:])]
        for _ in range(depth - 1):
            top = levels.pop()
            levels[-1] = levels[-1] + F.interpolate(top, scale_factor=2, mode="nearest")
        return {"m": levels[0]}

    check_stage("merge", run, ref, {"z0": zs[0]}, "z0")


@gpu
@pytest.mark.parametrize("B,G,n,L", [(3, 4, 8, 33), (5, 2, 16, 40), (3, 8, 4, 17), (3, 3, 32, 20)])
def test_tac_stage(B, G, n, L):
    """sdr_tac (tac_mma16_kernel at n = 16, tac_kernel otherwise) and sdr_tac_apply: TAC averages over the groups of
    one mixture, so a bad value reaches all of that mixture's groups and no other mixture."""
    g = gen(42)
    cfg = O.Config(variant="groupcomm", out_channels=G * n, in_channels=2 * G * n, num_blocks=1, upsampling_depth=1,
                   group_size=G)
    sd = {k[len("sm.0.TAC."):]: v.to(DEV) for k, v in O.make_state_dict(cfg, seed=9).items()
          if k.startswith("sm.0.TAC.")}
    names = ["TAC_input.0.weight", "TAC_input.0.bias", "TAC_input.1.weight", "TAC_mean.0.weight", "TAC_mean.0.bias",
             "TAC_mean.1.weight", "TAC_output.0.weight", "TAC_output.0.bias", "TAC_output.1.weight"]
    prm = [sd[k].contiguous() for k in names]
    params = (C.c_void_p * 9)(*[t.data_ptr() for t in prm])
    gamma, beta = rnd(g, n, scale=0.3, shift=1.0), rnd(g, n, scale=0.2)

    def run(ins):
        x = ins["x"]
        o = torch.full((B, G, n, L), NAN, device=DEV)
        st = torch.zeros(B * G, 2, dtype=torch.float64, device=DEV)
        N.check(N.lib().sdr_tac(p(x), params, p(o), p(st), B, G, n, L, stream()))
        nin = norm_in(st, gamma, beta, None, n * L)
        out = torch.full((B, G, n, L), NAN, device=DEV)
        N.check(N.lib().sdr_tac_apply(p(x), p(o), C.byref(nin), p(out), B * G, n, L, stream()))
        torch.cuda.synchronize()
        return {"o": o, "out": out, "stats": st.view(B, G, 2)}

    def ref(ins):
        taps = {}
        x = ins["x"].double()
        O.tac(x, {k: v.double() for k, v in sd.items()}, "", taps)
        o = taps["TAC_output"]
        on = O.glob_ln(o.reshape(B * G, n, L), gamma.double(), beta.double()).view(B, G, n, L)
        return {"o": o, "out": x + on}

    check_stage("tac", run, ref, {"x": rnd(g, B, G, n, L)}, "x", tc=n == 16, tol=1e-4)


@gpu
@pytest.mark.parametrize("rows,T", [(3, 517), (5, 8193), (3, 7)])
def test_utterance_stats_stage(rows, T):
    """sdr_utterance_stats: per-row mean and unbiased std."""
    scratch = torch.empty(rows * 2, dtype=torch.float64, device=DEV)

    def run(ins):
        ms = torch.full((rows, 2), NAN, device=DEV)
        N.check(N.lib().sdr_utterance_stats(p(ins["wav"]), p(ms), rows, T, p(scratch), stream()))
        torch.cuda.synchronize()
        return {"ms": ms}

    def ref(ins):
        w = ins["wav"].double()
        return {"ms": torch.stack([w.mean(-1), w.std(-1)], dim=1)}

    check_stage("utterance_stats", run, ref, {"wav": rnd(gen(43), rows, T, scale=0.7, shift=0.1)}, "wav", tol=1e-5)


# The backward stages with per-sample outputs: (C) only (a non-finite mixture's gradients are out of scope, and every
# weight gradient sums over the batch).
@gpu
@pytest.mark.parametrize("samples,C_,L,norm", [(3, 16, 52, True), (5, 7, 33, False), (3, 32, 128, True)])
def test_norm_act_backward_stage(samples, C_, L, norm):
    lib = N.lib()
    g = gen(44)
    gamma, beta, slope = rnd(g, C_, scale=0.3, shift=1.0), rnd(g, C_, scale=0.2), torch.tensor([0.2], device=DEV)
    scratch = torch.empty(lib.sdr_norm_act_backward_scratch_bytes(samples, C_), dtype=torch.uint8, device=DEV)

    def run(ins):
        x = ins["x"]
        stats_in = raw_stats(x).to(DEV)
        nin = norm_in(stats_in, gamma, beta, slope, C_ * L) if norm else norm_in(None, None, None, slope, 1.0)
        dx = torch.full((samples, C_, L), NAN, device=DEV)
        N.check(lib.sdr_norm_act_backward(p(x), C.byref(nin), p(ins["dp"]), p(dx), 0, p(None), p(None), p(None),
                                          p(scratch), samples, C_, L, stream()))
        torch.cuda.synchronize()
        return {"dx": dx}

    ins = {"x": rnd(g, samples, C_, L, shift=0.3), "dp": rnd(g, samples, C_, L)}
    for key in ins:
        check_stage("norm_act_backward", run, lambda ins: {}, ins, key)


@gpu
@pytest.mark.parametrize("samples,C_,Lin,stride", [(3, 16, 52, 1), (5, 7, 34, 2), (3, 9, 64, 2)])
def test_depthwise_backward_stage(samples, C_, Lin, stride):
    lib = N.lib()
    g = gen(45)
    gamma, beta, slope = rnd(g, C_, scale=0.3, shift=1.0), rnd(g, C_, scale=0.2), torch.tensor([0.2], device=DEV)
    w5 = rnd(g, C_, 5)
    Lout = (Lin - 1) // stride + 1
    scratch = torch.empty(lib.sdr_depthwise_backward_scratch_bytes(samples, C_), dtype=torch.uint8, device=DEV)

    def run(ins):
        x = ins["x"]
        stats_in = raw_stats(x).to(DEV)
        nin = norm_in(stats_in, gamma, beta, slope, C_ * Lin)
        dx = torch.full((samples, C_, Lin), NAN, device=DEV)
        dw = torch.empty(C_, 5, device=DEV)
        db = torch.empty(C_, device=DEV)
        N.check(lib.sdr_depthwise_backward(p(ins["dz"]), p(x), C.byref(nin), p(w5), p(None), 1, p(dx), p(dw), p(db),
                                           p(scratch), samples, C_, Lin, stride, stream()))
        torch.cuda.synchronize()
        return {"dx": dx}

    ins = {"x": rnd(g, samples, C_, Lin, shift=0.3), "dz": rnd(g, samples, C_, Lout)}
    for key in ins:
        check_stage("depthwise_backward", run, lambda ins: {}, ins, key)


@gpu
@pytest.mark.parametrize("B,S,N_,L", [(3, 2, 8, 33), (5, 3, 16, 40)])
def test_mask_backward_stage(B, S, N_, L):
    g = gen(46)

    def run(ins):
        dm = ins["dmasked"].clone()
        denc = torch.full((B, N_, L), NAN, device=DEV)
        N.check(N.lib().sdr_mask_backward(p(ins["mlog"]), p(ins["enc"]), p(dm), p(denc), B, S, N_, L, stream()))
        torch.cuda.synchronize()
        return {"dmlog": dm, "denc": denc}

    ins = {"mlog": rnd(g, B, S * N_, L), "enc": rnd(g, B, N_, L), "dmasked": rnd(g, B, S * N_, L)}
    for key in ins:
        check_stage("mask_backward", run, lambda ins: {}, ins, key)


@gpu
@pytest.mark.parametrize("B,SA,K,L,T", [(3, 2, 21, 33, 325), (5, 1, 5, 40, 79)])
def test_overlap_add_backward_stage(B, SA, K, L, T):
    def run(ins):
        gf = torch.full((B, SA * K, L), NAN, device=DEV)
        N.check(N.lib().sdr_overlap_add_backward(p(ins["grad_out"]), p(gf), B, SA, K, L, T, stream()))
        torch.cuda.synchronize()
        return {"grad_frames": gf}

    check_stage("overlap_add_backward", run, lambda ins: {}, {"grad_out": rnd(gen(47), B, SA, T)}, "grad_out")


# The metrics: with a bad estimate or target in item j, every other item's score and permutation are unchanged bit
# for bit (the batch mean is contaminated by definition).
@gpu
@pytest.mark.parametrize("B,S,T", [(3, 2, 517), (5, 3, 64), (3, 4, 33)])
def test_metrics_per_item(B, S, T):
    lib = N.lib()
    g = gen(48)
    scratch = torch.empty(max(lib.sdr_pit_sisdr_scratch_bytes(B, S), lib.sdr_stabilized_sisdr_scratch_bytes(B, S, S)),
                          dtype=torch.uint8, device=DEV)

    def run(ins):
        est, tgt = ins["est"], ins["tgt"]
        best = torch.full((B,), NAN, device=DEV)
        perm = torch.full((B,), -1, dtype=torch.int32, device=DEV)
        N.check(lib.sdr_pit_sisdr(p(est), p(tgt), p(None), p(best), p(perm), B, S, T, 1, 0, 1e-9, p(scratch),
                                  stream()))
        sbest = torch.full((B,), NAN, device=DEV)
        sperm = torch.full((B,), -1, dtype=torch.int32, device=DEV)
        N.check(lib.sdr_stabilized_sisdr(p(est), p(tgt), p(sbest), p(sperm), B, S, S, S, T, 0, 0, 1e-9, p(scratch),
                                         stream()))
        pw = torch.full((B, S, S), NAN, device=DEV)
        N.check(lib.sdr_pairwise_neg_sdr(p(est), p(tgt), p(pw), B, S, T, 1, 1, 1, p(scratch), stream()))
        torch.cuda.synchronize()
        return {"best": best, "perm": perm, "sbest": sbest, "sperm": sperm, "pairwise": pw}

    ins = {"est": rnd(g, B, S, T), "tgt": rnd(g, B, S, T)}
    for key in ins:
        check_stage("metrics", run, lambda ins: {}, ins, key)


@gpu
@pytest.mark.parametrize("samples,C_,L,first", [(3, 16, 52, False), (5, 7, 33, True), (3, 24, 517, False)])
def test_residual_norm_stage(samples, C_, L, first):
    """sdr_residual_norm (the original UBlock's tail): the bad value in either operand."""
    g = gen(37)
    ge, be = rnd(g, C_, scale=0.3, shift=1.0), rnd(g, C_, scale=0.2)
    gx, bx = rnd(g, C_, scale=0.3, shift=1.0), rnd(g, C_, scale=0.2)
    slopes = channel_slopes(C_, g)

    def run(ins):
        e, x = ins["e"], ins["x"].clone()
        st_e, st_x = raw_stats(e).to(DEV), raw_stats(x).to(DEV)
        fe = norm_in(st_e, ge, be, None, C_ * L)
        fx = norm_in() if first else norm_in(st_x, gx, bx, slopes, C_ * L)
        st = torch.zeros(samples, 2, dtype=torch.float64, device=DEV)
        N.check(N.lib().sdr_residual_norm(p(e), C.byref(fe), p(x), C.byref(fx), p(st), samples, C_, L, stream()))
        torch.cuda.synchronize()
        return {"x": x, "stats": st}

    def ref(ins):
        e, x = ins["e"].double(), ins["x"].double()
        fx = x if first else ref_norm(x, gx.double(), bx.double(), slopes.double())
        return {"x": ref_norm(e, ge.double(), be.double()) + fx}

    ins = {"e": rnd(g, samples, C_, L, scale=1.7, shift=-0.4), "x": rnd(g, samples, C_, L, scale=0.8, shift=0.2)}
    for key in ins:
        check_stage("residual_norm", run, ref, ins, key)


@gpu
@pytest.mark.parametrize("B,S,N_,L", [(3, 1, 8, 12), (5, 2, 8, 12), (3, 3, 5, 7), (5, 4, 8, 12), (3, 2, 24, 52)])
def test_softmax_gate_stage(B, S, N_, L):
    """sdr_softmax_gate (the original model's masks): NaN and +-inf logits, sigmoid for one source."""
    g = gen(38)

    def run(ins):
        out = torch.full((B, S, N_, L), NAN, device=DEV)
        N.check(N.lib().sdr_softmax_gate(p(ins["lg"]), p(ins["enc"]), p(out), B, S, N_, L, stream()))
        torch.cuda.synchronize()
        return {"out": out}

    def ref(ins):
        lg = ins["lg"].double()
        gate = torch.sigmoid(lg) if S == 1 else torch.softmax(lg, dim=1)
        return {"out": gate * ins["enc"].double().unsqueeze(1)}

    ins = {"lg": rnd(g, B, S, N_, L, scale=3.0), "enc": torch.relu(rnd(g, B, N_, L))}
    for key in ins:
        check_stage("softmax_gate", run, ref, ins, key, tol=1e-5)


def fold_ref(frames, SA, K, T):
    """overlap-add by selection (no zero weights that would turn a neighbour's NaN into NaN here)."""
    B, _, L = frames.shape
    hop = K // 2
    fr = frames.double().view(B, SA, K, L)
    out = torch.zeros(B, SA, hop * (L + 2) + K, dtype=torch.float64, device=frames.device)
    pos = hop * torch.arange(L, device=frames.device)
    for j in range(K):
        out[:, :, pos + j] += fr[:, :, j, :]
    return out[:, :, hop:hop + T]


@gpu
@pytest.mark.parametrize("B,SA,K,L,T,mc", [(3, 2, 21, 64, 640, False), (5, 2, 21, 33, 325, True),
                                            (3, 3, 5, 50, 99, True), (5, 1, 11, 21, 101, False)])
def test_overlap_add_stage(B, SA, K, L, T, mc):
    """sdr_overlap_add, with and without mixture consistency: the bad value in a frame and in the mixture."""
    g = gen(39)
    hop = K // 2
    assert T <= hop * L

    def run(ins):
        out = torch.full((B, SA, T), NAN, device=DEV)
        N.check(N.lib().sdr_overlap_add(p(ins["frames"]), p(ins.get("mix")), p(out), B, SA, K, L, T, stream()))
        torch.cuda.synchronize()
        return {"out": out}

    def ref(ins):
        y = fold_ref(ins["frames"], SA, K, T)
        return {"out": O.mixture_consistency(y, ins["mix"].double()) if mc else y}

    ins = {"frames": rnd(g, B, SA * K, L)}
    if mc:
        ins["mix"] = rnd(g, B, 1, T)
    for key in ins:
        check_stage("overlap_add", run, ref, ins, key, tol=1e-5)


@gpu
@pytest.mark.parametrize("kind,B,S,T", [("uniform", 3, 2, 2049), ("magsq", 5, 3, 2047), ("magsq", 3, 2, 4097),
                                         ("uniform", 5, 1, 333)])
def test_mixture_consistency_stage(kind, B, S, T):
    """mixture_consistency.apply on the device: the bad value in an estimate and in the mixture."""
    g = gen(40)

    def run(ins):
        out = MC.apply(ins["est"], ins["mix"], kind)
        torch.cuda.synchronize()
        return {"out": out}

    def ref(ins):
        return {"out": O.mixture_consistency(ins["est"].double(), ins["mix"].double(), kind)}

    ins = {"est": rnd(g, B, S, T), "mix": rnd(g, B, 1, T)}
    for key in ins:
        check_stage("mixture_consistency", run, ref, ins, key, tol=1e-5)


# =====================================================================================================================
# 2. whole models, one per dispatch path (test_gpu_scratch.CASES)
# =====================================================================================================================
def model_runs(m, A, entries):
    """name -> (function of the device mixture, mixture consistency)."""
    runs = {"forward": (lambda x: m(x), False)}
    if A == 1:
        runs["forward_mc"] = (lambda x: m.separate(x, mixture_consistency=True), True)
        if "separate" in entries:
            runs["separate_normalize"] = (lambda x: m.separate(x, normalize=True), False)
            runs["separate_normalize_mc"] = (lambda x: m.separate(x, mixture_consistency=True, normalize=True), True)

    def host(x):
        hx = x.cpu().pin_memory()
        out = m.forward_host(hx)
        torch.cuda.synchronize()
        return out.to(DEV)
    if "host" in entries:
        runs["host"] = (host, False)
    return runs


def model_ref(cfg, sd, name, mc, x):
    if name.startswith("separate_normalize"):
        return O.separate(cfg, sd, x[:, 0], apply_mixture_consistency=mc, dtype=torch.float64)
    if cfg.variant == "causal":
        ref = O.causal_forward(cfg, sd, x, dtype=torch.float64, masked_taps="dropped")
    else:
        ref = O.forward(cfg, sd, x, dtype=torch.float64)
    return O.mixture_consistency(ref, x.double()) if mc else ref


def check_model(what, cfg, sd, run, name, mc, x, js, t0, ch=0):
    """(C) and (P) of one entry for a bad value at (j, ch, t0) for j in js."""
    causal = cfg.variant == "causal"
    with torch.no_grad():
        clean = run(x)
        again = run(x)
        spread = float((again - clean).abs().max() / clean.abs().max())
        assert spread == 0.0 if causal else spread <= SPREAD, (what, name, "clean / clean", spread)
        for vname, v in BAD:
            for j in js:
                bad = x.clone()
                bad[j, ch, t0] = v
                got = run(bad)
                others = [b for b in range(x.shape[0]) if b != j]
                tag = (what, name, vname, j, t0)
                if others:
                    if causal:
                        assert torch.equal(bits(got[others]), bits(clean[others])), tag + ("(C)",)
                    else:
                        d = (got[others] - clean[others]).abs().max() / clean[others].abs().max()
                        assert torch.isfinite(got[others]).all() and float(d) <= max(SPREAD, 4 * spread), \
                            tag + ("(C)", float(d))
                if not math.isfinite(v):
                    want = model_ref(cfg, sd, name, mc, bad[j:j + 1])[0]
                    if not causal:
                        check_class(got[j], want, tag + ("(P)",), 1e-4)
                    else:                 # the dropped-tap footprint; outside it, the clean run bit for bit
                        nf = ~torch.isfinite(got[j])
                        assert torch.equal(nf, ~torch.isfinite(want)), tag + ("(P)", int(nf.sum()),
                                                                              int((~torch.isfinite(want)).sum()))
                        assert torch.equal(bits(got[j][~nf]), bits(clean[j][~nf])), tag + ("(P) outside",)


@gpu
@pytest.mark.parametrize("name,variant,kw,B,T,entries,want", CASES, ids=[c[0] for c in CASES])
def test_whole_model(name, variant, kw, B, T, entries, want):
    """model(x), separate(mixture_consistency=True), separate(normalize=True) and forward_host with NaN, +-inf and 1e30
    in the first, a middle and the last mixture (channel 1 of a stereo one)."""
    cfg, sd, m = build(variant, kw, seed=213)
    A = kw.get("in_audio_channels", 1) if variant in ("groupcomm", "causal") else 1
    Bx = max(B, 3)
    x = normalised_input(Bx, A, T, seed=214).to(DEV) if T > 1 else torch.randn(Bx, A, 1, generator=gen(3)).to(DEV)
    js = sorted({0, Bx // 2, Bx - 1})
    for ename, (run, mc) in model_runs(m, A, entries).items():
        xin = x * 1.7 + 0.2 if ename.startswith("separate_normalize") else x
        check_model(name, cfg, sd, run, ename, mc, xin, js, T // 2, ch=A - 1)


@gpu
def test_whole_model_at_benchmark_size():
    """The benchmark's cfg 2 shape: 32 mixtures x 2 s at 16 kHz, NaN in mixture 17."""
    kw = dict(out_channels=256, in_channels=512, num_blocks=4, upsampling_depth=5, enc_kernel_size=21,
              enc_num_basis=512, num_sources=2)
    cfg, sd, m = build("improved", kw, seed=215)
    x = normalised_input(32, 1, 32000, seed=216).to(DEV)
    with torch.no_grad():
        clean = m(x)
        again = m(x)
        bad = x.clone()
        bad[17, 0, 12345] = NAN
        got = m(bad)
    spread = float((again - clean).abs().max() / clean.abs().max())
    assert spread <= SPREAD
    others = [b for b in range(32) if b != 17]
    d = float((got[others] - clean[others]).abs().max() / clean[others].abs().max())
    assert d <= max(SPREAD, 4 * spread), d
    want = O.forward(cfg, sd, bad[17:18], dtype=torch.float64)[0]
    check_class(got[17], want, "cfg 2, mixture 17", 1e-4)


TRAINING = [dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
                 enc_num_basis=256, num_sources=2),
            dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3, enc_kernel_size=11,
                 enc_num_basis=48, num_sources=3)]
TRAINING_IDS = ["wgmma_mask", "ffma_mask"]


@gpu
@pytest.mark.parametrize("kw", TRAINING, ids=TRAINING_IDS)
def test_training_forward(kw):
    """The training forward (sdr_forward_train, which recomputes relu(mlog) * e in mask_apply_kernel): (C) for the other
    mixtures, (P) for the bad one."""
    cfg, sd, m = build("improved", kw, seed=217)
    m.train().enable_training()
    x = normalised_input(3, 1, 1603, seed=218).to(DEV)
    with torch.enable_grad():
        clean = m(x).detach()
        again = m(x).detach()
    spread = float((again - clean).abs().max() / clean.abs().max())
    assert spread <= SPREAD, spread
    for vname, v in BAD:
        for j in (0, 1, 2):
            bad = x.clone()
            bad[j, 0, 800] = v
            with torch.enable_grad():
                got = m(bad).detach()
            others = [b for b in range(3) if b != j]
            d = float((got[others] - clean[others]).abs().max() / clean[others].abs().max())
            assert torch.isfinite(got[others]).all() and d <= max(SPREAD, 4 * spread), (vname, j, d)
            if math.isfinite(v):
                continue
            want = O.forward(cfg, sd, bad[j:j + 1], dtype=torch.float64)[0]
            check_class(got[j], want, ("training forward", vname, j), 1e-4)


# =====================================================================================================================
# 3. ragged buckets and the corpus
# =====================================================================================================================
@gpu
@pytest.mark.parametrize("variant,kw", [
    ("improved", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
                      enc_num_basis=64, num_sources=2)),
    ("causal", dict(in_audio_channels=1, out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=2,
                    enc_kernel_size=21, enc_num_basis=64, num_sources=2))])
def test_corpus_with_one_corrupt_utterance(variant, kw):
    """separate_corpus buckets utterances of different lengths (sdr_separate_ragged): one corrupt utterance is
    non-finite over its whole length, and every other one is what a clean corpus gives."""
    cfg, sd, m = build(variant, kw, seed=219)
    g = gen(220)
    lens = [1601, 1203, 1600, 977, 1550]
    wavs = [torch.randn(n, generator=g) * (0.5 + 0.2 * i) + 0.05 * i for i, n in enumerate(lens)]
    with torch.no_grad():
        clean = separate_corpus(m, wavs, max_batch=8)
        again = separate_corpus(m, wavs, max_batch=8)
        spread = max(float((a - c).abs().max() / c.abs().max()) for a, c in zip(again, clean))
        for vname, v in BAD:
            for i in (0, 2, 4):
                bad = [w.clone() for w in wavs]
                bad[i][lens[i] // 2] = v
                got = separate_corpus(m, bad, max_batch=8)
                for k in range(len(lens)):
                    if k == i:
                        if not math.isfinite(v):
                            assert not torch.isfinite(got[k]).any(), (vname, i, int(torch.isfinite(got[k]).sum()))
                        continue
                    if spread == 0.0:
                        assert torch.equal(bits(got[k]), bits(clean[k])), (vname, i, k)
                    else:
                        d = float((got[k] - clean[k]).abs().max() / clean[k].abs().max())
                        assert d <= max(SPREAD, 4 * spread), (vname, i, k, d)


# =====================================================================================================================
# 4. the stream
# =====================================================================================================================
@gpu
@pytest.mark.parametrize("slots", [3, 300])
def test_stream_with_one_bad_slot(slots):
    """A bad sample in slot j of one chunk (the first chunk, a middle one, its last sample): the other slots are bitwise
    unchanged; slot j equals the offline forward on its clip in class, and bitwise where that is finite; past the
    offline footprint it is the clean stream again; flush() and reset([j]) inside the footprint behave."""
    kw = dict(in_audio_channels=1, out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=3,
              enc_kernel_size=21, enc_num_basis=64, num_sources=2)
    cfg, sd, m = build("causal", kw, seed=221)
    hop = cfg.hop
    granule = N.lib().sdr_stream_granule(C.byref(_engine.make_config(m)))
    Cs = 4 * granule
    n = 10
    x = normalised_input(slots, 1, n * Cs, seed=222).to(DEV)
    j = slots // 2

    def stream_all(xx, stop=None, reset_at=None):
        s = CausalStream(m, slots, Cs)
        outs = []
        for c in range(n if stop is None else stop):
            if reset_at == c:
                s.reset([j])
            outs.append(s.step(xx[..., c * Cs:(c + 1) * Cs]).clone())
        return torch.cat(outs, -1), s

    with torch.no_grad():
        clean, _ = stream_all(x)
        for vname, v in BAD:
            for t0 in (0, 3 * Cs + 17, 4 * Cs - 1):
                bad = x.clone()
                bad[j, 0, t0] = v
                got, _ = stream_all(bad)
                others = [b for b in range(slots) if b != j]
                assert torch.equal(bits(got[others]), bits(clean[others])), (vname, t0, "(C)")
                off = m(bad[j:j + 1])[0]                      # the offline native forward on slot j's clip
                # the stream lags the offline forward by hop samples
                g_j, o_j = got[j][:, hop:], off[:, :n * Cs - hop]
                nf = ~torch.isfinite(g_j)
                assert torch.equal(nf, ~torch.isfinite(o_j)), (vname, t0, int(nf.sum()), int((~torch.isfinite(o_j)).sum()))
                assert torch.equal(bits(g_j[~nf]), bits(o_j[~nf])), (vname, t0, "finite part")
                if math.isfinite(v):
                    continue
                bad_t = (~torch.isfinite(got[j])).any(0).nonzero().flatten()
                assert bad_t.numel() > 0, (vname, t0)
                first, end = int(bad_t.min()), int(bad_t.max()) + 1
                assert end < n * Cs, (vname, t0, "the footprint reaches the end: lengthen the stream")
                # the state carries nothing past the receptive field
                assert torch.equal(bits(got[j][:, end:]), bits(clean[j][:, end:])), (vname, t0, "after the footprint")
                assert torch.equal(bits(got[j][:, :first]), bits(clean[j][:, :first])), (vname, t0, "before it")
                # flush() inside the footprint: non-finite where the offline forward on the streamed clip is
                c_in = t0 // Cs + 1
                assert c_in * Cs % (hop << cfg.upsampling_depth) == 0
                _, s = stream_all(bad, stop=c_in)
                tail = s.flush()[j]
                off_c = m(bad[j:j + 1, :, :c_in * Cs])[0][:, -hop:]
                assert torch.equal(~torch.isfinite(tail), ~torch.isfinite(off_c)), (vname, t0, "flush")
                # reset([j]) inside the footprint: the slot starts over bit for bit
                fresh, _ = stream_all(bad, reset_at=c_in)
                ref_fresh, _ = stream_all(x[..., c_in * Cs:], stop=n - c_in)
                assert torch.equal(bits(fresh[j][:, c_in * Cs:]), bits(ref_fresh[j])), (vname, t0, "reset")
