"""Scale: batches past the 65535 CTAs a grid's y dimension allows, and tensors past 2^31 elements.

Batch.  Every large batch tiles PERIOD = 7 distinct inputs (row b is input b % 7; 7 is coprime to 65536), so a row read
from b mod 65535 / 65536, or written to another row's slot, differs from what its own input gives.  Each row is held to
the same call on the 7-row batch: bitwise where the kernel sums nothing across CTAs, within 1e-6 of max|ref| where the
GlobLN statistics are summed by fp64 atomics.  The 7-row results are held to fp64 torch or the fp64 oracle.  B = 65535,
65536 and 131075 (odd, above 2 x 65536).

Past 2^31 elements.  Each case puts the rows under test at an element offset past 2^31 (past 2^32 where 24 GB allows)
and holds them bitwise to the same call on a small tensor holding only those rows, and to fp64 on a few positions.

Every stage output starts as NaN inside guard bands (tests/guards.py), so a row nobody wrote is non-finite.  A test
that does not find the device memory it needs free is skipped with the amount; its peak is printed."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import mixture_consistency as MC
from sudo_rm_rf_b200.corpus import model_padding_rule, plan_buckets, separate_corpus
from oracle import sudormrf_oracle as O
from guards import Guards
from test_gpu_long import CLASSES, normalised_input
from test_gpu_metric_space import compare_pairwise, compare_pit, compare_stab, separation_batch
from test_gpu_model_space import TOL, build, check_launch_count, gc, imp, orig
from test_gpu_stages import norm_in
from test_gpu_train_space import compare, native_model

DEV = "cuda"
GiB = 2 ** 30
PERIOD = 7
BATCHES = [65535, 65536, 131075]
gpu = pytest.mark.gpu


def p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def need(gib):
    free = torch.cuda.mem_get_info()[0]
    if free < gib * GiB:
        pytest.skip(f"needs {gib:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")


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


def tile(small, B):
    """[PERIOD, ...] -> [B, ...] with row b = small[b % PERIOD]; also returns the row map."""
    idx = torch.arange(B, device=small.device) % small.shape[0]
    return small[idx].contiguous(), idx


def rows_report(bad):
    bad = torch.nonzero(bad).flatten().tolist()
    return f"{len(bad)} rows differ, first {bad[:6]}, last {bad[-3:]}"


def assert_rows_equal(got, want):
    bad = (got != want).reshape(got.shape[0], -1).any(1) | ~torch.isfinite(got).reshape(got.shape[0], -1).all(1)
    assert not bad.any(), rows_report(bad)


def assert_rows_close(got, want, rel=1e-6):
    """Every row within rel * max|want| (the GlobLN statistics are summed by fp64 atomics in no fixed order)."""
    err = (got - want).abs().reshape(got.shape[0], -1)
    bad = ~(err <= rel * want.abs().max())
    assert not bad.any(1).any(), rows_report(bad.any(1)) + f"; max err {float(err.nan_to_num(float('inf')).max()):.3e}"


def selected_rows(B):
    return sorted({0, 65534, 65535, 65536, B - 1} & set(range(B)))


def poison(shape):
    """Best effort, for outputs the library allocates itself: leaves a NaN block of this shape in the caching allocator,
    which usually hands it to the next allocation of the same size, so that an output row the library never writes
    reads NaN rather than a previous call's values.  Nothing guarantees that reuse; the tiling identity, which compares
    every row with the row its own input gives, is what catches an unwritten row."""
    t = torch.full(shape, float("nan"), device=DEV)
    del t


# =====================================================================================================================
# stage entries at large batches
# =====================================================================================================================
def overlap_add(frames, mix, B, SA, K, L, T):
    gd = Guards()
    fr = gd.input("frames", frames)
    mx = gd.input("mix", mix) if mix is not None else None
    out = gd.output("out", torch.full((B, SA, T), float("nan"), device=DEV))
    N.check(N.lib().sdr_overlap_add(p(fr), p(mx), p(out), B, SA, K, L, T, stream()))
    gd.check()
    return out


@gpu
@pytest.mark.parametrize("mc", [False, True])
@pytest.mark.parametrize("B", BATCHES)
def test_overlap_add_batch(B, mc):
    SA, K, L, T = 3, 5, 24, 45
    hop = K // 2
    g = torch.Generator().manual_seed(41)
    masked = torch.randn(PERIOD, 6, L, generator=g).to(DEV)
    wd = torch.randn(6, SA, K, generator=g).to(DEV)
    frames7 = torch.einsum("csj,bct->bsjt", wd, masked).reshape(PERIOD, SA * K, L).contiguous()
    mix7 = torch.randn(PERIOD, 1, T, generator=g).to(DEV) if mc else None
    small = overlap_add(frames7, mix7, PERIOD, SA, K, L, T)
    want = F.conv_transpose1d(masked.double(), wd.double(), None, stride=hop, padding=hop, output_padding=hop - 1)
    want = want[..., :T]
    if mc:
        want = O.mixture_consistency(want, mix7.double())
    assert max(O.parity_errors(small, want)) < 2e-5
    frames, idx = tile(frames7, B)
    out = overlap_add(frames, tile(mix7, B)[0] if mc else None, B, SA, K, L, T)
    assert_rows_equal(out, small[idx])


@gpu
@pytest.mark.parametrize("S", [1, 2, 5])
@pytest.mark.parametrize("B", BATCHES)
def test_softmax_gate_batch(B, S):
    """sdr_softmax_gate (the original model's masks): sigmoid at S = 1, softmax over S sources otherwise."""
    N_, L = 8, 12
    g = torch.Generator().manual_seed(43)
    lg7 = (torch.randn(PERIOD, S, N_, L, generator=g) * 3).to(DEV)
    enc7 = torch.relu(torch.randn(PERIOD, N_, L, generator=g)).to(DEV)

    def run(lg, enc, B):
        gd = Guards()
        a, e = gd.input("logits", lg), gd.input("enc", enc)
        out = gd.output("out", torch.full((B, S, N_, L), float("nan"), device=DEV))
        N.check(N.lib().sdr_softmax_gate(p(a), p(e), p(out), B, S, N_, L, stream()))
        gd.check()
        return out

    small = run(lg7, enc7, PERIOD)
    want = (torch.sigmoid(lg7.double()) if S == 1 else torch.softmax(lg7.double(), 1)) * enc7.double().unsqueeze(1)
    assert max(O.parity_errors(small, want)) < 1e-5
    lg, idx = tile(lg7, B)
    assert_rows_equal(run(lg, tile(enc7, B)[0], B), small[idx])


MC_BATCH = [(S, B) for S, B in ((2, 32767), (2, 32768), (1, 65535), (1, 65536), (3, 131075))]


@gpu
@pytest.mark.parametrize("kind", ["uniform", "magsq"])
@pytest.mark.parametrize("S,B", MC_BATCH, ids=[f"S{S}-B{B}" for S, B in MC_BATCH])
def test_mixture_consistency_batch(S, B, kind):
    """mixture_consistency.apply on both sides of B * S = 65535 (the power kernel has one grid row per (b, s)).
    T = 333 < 2048: one power CTA per row, so the power sums, too, are bitwise reproducible."""
    T = 333
    g = torch.Generator().manual_seed(47)
    est7 = torch.randn(PERIOD, S, T, generator=g).to(DEV)
    mix7 = torch.randn(PERIOD, 1, T, generator=g).to(DEV)
    small = MC.apply(est7, mix7, kind)
    assert max(O.parity_errors(small, O.mixture_consistency(est7.double(), mix7.double(), kind))) < 1e-5
    est, idx = tile(est7, B)
    mix = tile(mix7, B)[0]
    poison((B, S, T))
    assert_rows_equal(MC.apply(est, mix, kind), small[idx])


@gpu
@pytest.mark.parametrize("B", BATCHES)
def test_utterance_stats_batch(B):
    """sdr_utterance_stats: (mean, unbiased std) per row in fp32; one chunk per row at T = 1000."""
    T = 1000
    g = torch.Generator().manual_seed(53)
    wav7 = (torch.randn(PERIOD, T, generator=g) * torch.linspace(0.1, 5, PERIOD).view(-1, 1)
            + torch.linspace(-1, 1, PERIOD).view(-1, 1)).to(DEV)

    def run(wav, rows):
        gd = Guards()
        w = gd.input("wav", wav)
        ms = gd.output("mean_std", torch.full((rows, 2), float("nan"), device=DEV))
        scratch = torch.empty(2 * rows, dtype=torch.float64, device=DEV)
        N.check(N.lib().sdr_utterance_stats(p(w), p(ms), rows, T, p(scratch), stream()))
        gd.check()
        return ms

    small = run(wav7, PERIOD)
    wd = wav7.double()
    want = torch.stack([wd.mean(-1), wd.std(-1)], 1)
    assert torch.allclose(small.double(), want, rtol=1e-6, atol=1e-7), (small, want)
    wav, idx = tile(wav7, B)
    assert_rows_equal(run(wav, B), small[idx])


# =====================================================================================================================
# whole models at large batches: one small configuration per variant
# =====================================================================================================================
CAUSAL = dict(in_audio_channels=1, out_channels=8, in_channels=16, num_blocks=1, upsampling_depth=2, enc_kernel_size=5,
              enc_num_basis=16, num_sources=2)
MODELS = [
    ("improved", imp(2, 5, 16, Co=8, Ci=16, D=2)),
    ("groupcomm", gc(2, 1, 5, 16, 2, 4, D=2)),
    ("causal", CAUSAL),
    ("original", orig(2, 5, 16, 16, D=2)),
]
MODEL_T = 61


def small_and_oracle(variant, kw):
    cfg, sd, m = build(variant, kw, seed=59)
    x7 = normalised_input(PERIOD, 1, MODEL_T, seed=61).to(DEV)
    return cfg, sd, m, x7, O.forward(cfg, sd, x7, dtype=torch.float64)


def check_batch(big, small, ref, idx, what):
    """The tiling identity on every row, then the selected rows against the fp64 oracle."""
    B = big.shape[0]
    assert big.shape == (B,) + tuple(small.shape[1:]), (big.shape, small.shape)
    assert_rows_close(big, small[idx])
    rows = torch.tensor(selected_rows(B), device=DEV)
    e = O.parity_errors(big[rows], ref[idx[rows]])
    print(f"{what} B={B} rows {rows.tolist()}: rel_max {e[0]:.3e} rel_l2 {e[1]:.3e}")
    assert max(e) < TOL, e


@gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("variant,kw", MODELS, ids=[v for v, _ in MODELS])
def test_model_batch(variant, kw, B):
    """model(x) and separate(x, mixture_consistency=True) (the projection inside the overlap-add), and the launch
    count of a captured forward against sdr_forward_launch_count_for at this B."""
    cfg, sd, m, x7, ref = small_and_oracle(variant, kw)
    x, idx = tile(x7, B)
    with torch.no_grad():
        small = m(x7)
        assert max(O.parity_errors(small, ref)) < TOL
        poison((B, cfg.num_sources, MODEL_T))
        check_batch(m(x), small, ref, idx, f"{variant} forward")
        small_mc = m.separate(x7, mixture_consistency=True)
        ref_mc = O.mixture_consistency(ref, x7.double())
        poison((B, cfg.num_sources, MODEL_T))
        check_batch(m.separate(x, mixture_consistency=True), small_mc, ref_mc, idx, f"{variant} mixture consistency")
        check_launch_count(m, B, MODEL_T, lambda: m(x))


@gpu
@pytest.mark.parametrize("variant,kw", MODELS, ids=[v for v, _ in MODELS])
def test_separate_normalize_batch(variant, kw):
    """separate(normalize=True): utterance statistics, normalise_rows, forward and the rescale, at B = 131075."""
    B = BATCHES[-1]
    cfg, sd, m = build(variant, kw, seed=59)
    g = torch.Generator().manual_seed(67)
    wav7 = (torch.randn(PERIOD, MODEL_T, generator=g) * torch.linspace(0.05, 6, PERIOD).view(-1, 1)
            + torch.linspace(-1.2, 0.3, PERIOD).view(-1, 1)).to(DEV)
    ref = O.separate(cfg, sd, wav7, apply_mixture_consistency=False, dtype=torch.float64)
    wav, idx = tile(wav7, B)
    with torch.no_grad():
        small = m.separate(wav7, mixture_consistency=False, normalize=True)
        assert max(O.parity_errors(small, ref)) < TOL
        poison((B, cfg.num_sources, MODEL_T))
        check_batch(m.separate(wav, mixture_consistency=False, normalize=True), small, ref, idx,
                    f"{variant} separate(normalize=True)")


@gpu
@pytest.mark.parametrize("variant,kw", MODELS, ids=[v for v, _ in MODELS])
def test_separate_corpus_batch(variant, kw):
    """sdr_separate_ragged through separate_corpus with max_batch = 131075: one bucket of 131075 utterances, seven
    distinct ones of the lengths that pad to the bucket's width."""
    B = BATCHES[-1]
    cfg, sd, m = build(variant, kw, seed=59)
    Tp = O.padded_length(cfg, MODEL_T)
    lengths = [n for n in range(Tp, Tp - 16, -1) if O.padded_length(cfg, n) == Tp]
    g = torch.Generator().manual_seed(71)
    wav7 = [(torch.randn(lengths[k % len(lengths)], generator=g) * (0.1 + k) + 0.2 * k).to(DEV) for k in range(PERIOD)]
    wavs = [wav7[i % PERIOD] for i in range(B)]
    plan = plan_buckets([int(w.shape[0]) for w in wavs], model_padding_rule(_engine.make_config(m)), B)
    assert len(plan) == 1 and len(plan[0][1]) == B and plan[0][0] == Tp
    with torch.no_grad():
        small = separate_corpus(m, wav7, max_batch=PERIOD)
        got = separate_corpus(m, wavs, max_batch=B)
    for k in range(PERIOD):
        ref = O.separate(cfg, sd, wav7[k].view(1, -1), apply_mixture_consistency=False, dtype=torch.float64)[0]
        assert max(O.parity_errors(small[k], ref)) < TOL
        rows = torch.stack(got[k::PERIOD])
        assert_rows_close(rows, small[k].expand_as(rows).contiguous())
        e = O.parity_errors(rows[-1], ref)
        assert max(e) < TOL, (k, e)


@gpu
@pytest.mark.parametrize("variant,kw", MODELS, ids=[v for v, _ in MODELS])
def test_forward_host_batch(variant, kw):
    """forward_host on pinned host tensors at B = 131075; the host output starts as NaN."""
    B = BATCHES[-1]
    cfg, sd, m, x7, ref = small_and_oracle(variant, kw)
    x, idx = tile(x7, B)
    host_x = x.cpu().pin_memory()
    host_out = torch.full((B, cfg.num_sources, MODEL_T), float("nan")).pin_memory()
    with torch.no_grad():
        small = m(x7)
        m.forward_host(host_x, host_out)
    torch.cuda.synchronize()
    check_batch(host_out.to(DEV), small, ref, idx, f"{variant} forward_host")


@gpu
def test_training_batch_past_65535():
    """Training forward and backward of a one-channel improved model at B = 65537 (the overlap-add of the forward and
    its backward past one grid row per item): the gradient is the sum of the two half batches' gradients."""
    kw = dict(out_channels=1, in_channels=1, num_blocks=1, upsampling_depth=1, enc_kernel_size=3, enc_num_basis=1,
              num_sources=1)
    B, T = 65537, 64
    cfg = O.Config(variant="improved", **kw)
    m = native_model(kw, O.make_state_dict(cfg, seed=8, perturbed=True))
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(3)).to(DEV)
    g = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(4)).to(DEV)
    m.zero_grad(set_to_none=True)
    y = m(x)
    assert torch.isfinite(y).all()
    y.backward(g)
    whole = {n: q.grad.clone() for n, q in m.named_parameters()}
    halves = {}
    for sl in (slice(0, B // 2), slice(B // 2, B)):
        m.zero_grad(set_to_none=True)
        m(x[sl]).backward(g[sl])
        for n, q in m.named_parameters():
            halves[n] = halves.get(n, 0) + q.grad.double()
    compare(whole, halves, {n: halves[n].abs().item() for n in halves if halves[n].numel() == 1},
            "B = 65537 against two half batches", 1e-5)


@gpu
@pytest.mark.parametrize("Sn", [2, 3])
def test_metrics_batch(Sn):
    """PermInvariantSISDR (with and without SI-SDRi), StabilizedPermInvSISDRMetric and PairwiseNegSDR at B = 131075,
    by the comparison rule of test_gpu_metric_space.py."""
    B = BATCHES[-1]
    est, tgt, mix = separation_batch(B, Sn, 257, seed=73 + Sn)
    compare_pit(est, tgt, mix, zero_mean=True, improvement=True, what=f"pit S={Sn} B={B}")
    compare_pit(est, tgt, None, zero_mean=False, improvement=False, what=f"pit S={Sn} B={B} plain")
    compare_stab(est, tgt, Sn, zero_mean=True, improvement=True, what=f"stab S={Sn} B={B}")
    compare_pairwise(est, tgt, "sisdr", True, True, what=f"pairwise S={Sn} B={B}")


# =====================================================================================================================
# tensors past 2^31 elements
# =====================================================================================================================
def norm_none():
    return N.SdrNormIn(0, 0, 0, 0, 1.0, 0)


@gpu
@pytest.mark.parametrize("gated", [False, True])
def test_pointwise_ffma_past_2_32_elements(gated):
    """sdr_pointwise on its generic FFMA kernel (M = 128 > 64): two samples of 128 x 16777220, y has 2^32 + 1024
    elements; sample 0 alone passes 2^31 and sample 1 starts past it.  The last 1028 positions of every row of each
    sample against the same call on those positions alone (the k order of a position does not depend on its tile), and
    fp64 at them."""
    need(20)
    samples, M, K, L, Lr = 2, 128, 4, 16777220, 1028
    g = torch.Generator(device=DEV).manual_seed(79)
    x = torch.randn(samples, K, L, device=DEV, generator=g)
    W = torch.randn(M, K, device=DEV, generator=g) / 2
    bias = torch.randn(M, device=DEV, generator=g)
    gate = torch.randn(samples, 1, L, device=DEV, generator=g) if gated else None
    y = torch.full((samples, M, L), float("nan"), device=DEV)
    nin = norm_none()
    N.check(N.lib().sdr_pointwise(p(x), C.byref(nin), p(W), p(bias), p(None), p(gate), 1 if gated else 0, p(y),
                                  p(None), samples, M, K, L, 1 if gated else 0, stream()))
    xs = x[:, :, -Lr:].contiguous()
    gs = gate[:, :, -Lr:].contiguous() if gated else None
    ys = torch.full((samples, M, Lr), float("nan"), device=DEV)
    N.check(N.lib().sdr_pointwise(p(xs), C.byref(nin), p(W), p(bias), p(None), p(gs), 1 if gated else 0, p(ys),
                                  p(None), samples, M, K, Lr, 1 if gated else 0, stream()))
    torch.cuda.synchronize()
    got = y[:, :, -Lr:]
    assert_rows_equal(got, ys)
    want = torch.einsum("mk,skl->sml", W.double(), xs.double()) + bias.double().view(1, -1, 1)
    if gated:
        want = torch.relu(want) * gs.double()
    assert max(O.parity_errors(got, want)) < 3e-5
    assert torch.isfinite(y[:, :, :4]).all()     # the wrapped-index targets of the last rows


MMA_BIG = [("plain", 256, 64, 0), ("gated", 128, 64, 128)]


@gpu
@pytest.mark.parametrize("mode,M,K,gate_ch", MMA_BIG, ids=[c[0] for c in MMA_BIG])
def test_pointwise_mma_past_2_31_elements(mode, M, K, gate_ch):
    """sdr_pointwise_mma, one sample of M x 16777220: 2^32 + 1024 (plain, M = 256) or 2^31 + 512 (gated, M = 128,
    gate rows through the same TMA tensor map) output elements, read and written by TMA at coordinates past 2^31.  The
    last 1028 positions (tile aligned) against the same call on those positions alone, and fp64 at them."""
    need(23)
    L, Lr = 16777220, 1028
    lib = N.lib()
    g = torch.Generator(device=DEV).manual_seed(83)
    x = torch.randn(1, K, L, device=DEV, generator=g)
    W = torch.randn(M, K, device=DEV, generator=g) / K ** 0.5
    bias = torch.randn(M, device=DEV, generator=g)
    gate = torch.randn(1, gate_ch, L, device=DEV, generator=g) if gate_ch else None
    wpk = torch.empty(lib.sdr_pointwise_mma_packed_bytes(M, K), dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_pointwise_mma_pack(p(W), M, K, p(wpk), stream()))
    nin = norm_none()
    epi = 1 if gate_ch else 0
    y = torch.full((1, M, L), float("nan"), device=DEV)
    N.check(lib.sdr_pointwise_mma(p(x), C.byref(nin), p(wpk), p(bias), p(None), p(gate), gate_ch, p(y), p(None),
                                  1, M, K, L, epi, stream()))
    xs = x[:, :, -Lr:].contiguous()
    gs = gate[:, :, -Lr:].contiguous() if gate_ch else None
    ys = torch.full((1, M, Lr), float("nan"), device=DEV)
    N.check(lib.sdr_pointwise_mma(p(xs), C.byref(nin), p(wpk), p(bias), p(None), p(gs), gate_ch, p(ys), p(None),
                                  1, M, K, Lr, epi, stream()))
    torch.cuda.synchronize()
    got = y[:, :, -Lr:]
    assert_rows_equal(got[0], ys[0])
    want = torch.einsum("mk,skl->sml", W.double(), xs.double()) + bias.double().view(1, -1, 1)
    if gate_ch:
        want = torch.relu(want) * gs.double()
    assert max(O.parity_errors(got, want)) < 5e-5
    assert torch.isfinite(y[:, :, :4]).all()


@gpu
def test_overlap_add_past_2_31_elements():
    """sdr_overlap_add with mixture consistency, B = 513, SA = 16, T = 262145: 2^31 + 4202512 output elements, the
    last item's rows start past 2^31.  Frames that span every output position would be 2x the output, so they span the
    first half (K = 2001, hop 1000, L = 131): the second half of each row is the mixture-consistency correction alone,
    which still differs from row to row.  The last two items against the same call on them alone, and fp64 on the
    last (the transposed convolution zero-padded to T)."""
    need(18)
    B, SA, K, T = 513, 16, 2001, 262145
    hop = K // 2
    L = -(-T // hop) // 2
    g = torch.Generator(device=DEV).manual_seed(89)
    frames = torch.randn(B, SA * K, L, device=DEV, generator=g)
    mix = torch.randn(B, 1, T, device=DEV, generator=g)
    out = torch.full((B, SA, T), float("nan"), device=DEV)
    assert out.numel() > 2 ** 31 and (B - 1) * SA * T > 2 ** 31
    N.check(N.lib().sdr_overlap_add(p(frames), p(mix), p(out), B, SA, K, L, T, stream()))
    fs, ms = frames[-2:].contiguous(), mix[-2:].contiguous()
    os_ = torch.full((2, SA, T), float("nan"), device=DEV)
    N.check(N.lib().sdr_overlap_add(p(fs), p(ms), p(os_), 2, SA, K, L, T, stream()))
    torch.cuda.synchronize()
    assert_rows_equal(out[-2:], os_)
    assert torch.isfinite(out[:2]).all()
    del frames, out
    # frames[b, s*K + j, t] as a transposed convolution: an identity "masked" of SA*K channels through a one-hot wd
    f = fs[-1:].double().view(1, SA * K, L)
    wd = torch.zeros(SA * K, SA, K, dtype=torch.float64, device=DEV)
    for s in range(SA):
        wd[s * K + torch.arange(K), s, torch.arange(K)] = 1.0
    # past the frames' span the overlap-add is not cropped: frame L - 1's last tap lands on position hop * L
    f = F.pad(f, (0, 1))
    want = F.conv_transpose1d(f, wd, None, stride=hop, padding=hop, output_padding=hop - 1)
    want = F.pad(want, (0, T - want.shape[-1]))
    want = O.mixture_consistency(want, ms[-1:].double())
    assert max(O.parity_errors(os_[-1:], want)) < 2e-5


# The depthwise, merge, TAC-apply and residual-norm kernels count one sample's items (channels x positions) in int:
# 33 samples of 64 channels x ~2^20 positions, so sample 32 starts past 2^31 while each sample stays below it.  The
# last four channels of the last sample are held bitwise to the same call on them alone (the kernels are per channel
# once the sample's statistics are given), and to fp64.
BIG_S, BIG_C, SUB = 33, 64, 4


def norm_parts(C_, count, g):
    """Raw (sum, sumsq) statistics per sample (mean in [-1, 1], variance in [0.5, 2]), gamma and beta."""
    mean = torch.rand(BIG_S, dtype=torch.float64, device=DEV, generator=g) * 2 - 1
    var = torch.rand(BIG_S, dtype=torch.float64, device=DEV, generator=g) * 1.5 + 0.5
    stats = torch.stack([mean * count, (var + mean * mean) * count], 1).contiguous()
    gamma = 1 + 0.3 * torch.randn(C_, device=DEV, generator=g)
    beta = 0.2 * torch.randn(C_, device=DEV, generator=g)
    return stats, gamma, beta


def ref_glob(x, stats, gamma, beta, count, slope=None):
    """fp64 GlobLN of x (one sample, [C, L]) from its raw statistics (eps 1e-8, as the kernels), then PReLU."""
    mean = stats[0] / count
    var = (stats[1] / count - mean * mean).clamp_min(0)
    y = (x.double() - mean) / torch.sqrt(var + 1e-8) * gamma.double().view(-1, 1) + beta.double().view(-1, 1)
    if slope is None:
        return y
    sl = slope.double().view(-1, 1)
    return torch.where(y >= 0, y, y * sl)


def last_sample_parts(*ts):
    """Copies of the last SUB channels of the last sample of each [samples, C, ...] tensor (that slice is contiguous
    already, so .contiguous() would return a view of the big tensor)."""
    return [t[-1:, -SUB:].clone() for t in ts]


def check_last_stats(st, y_last):
    yd = y_last.double()
    want = torch.stack([yd.sum(), (yd * yd).sum()])
    n = y_last.numel()
    assert abs(float(st[-1, 0] - want[0])) <= 1e-5 * float((n * want[1]).sqrt()), (st[-1], want)
    assert abs(float(st[-1, 1] - want[1])) <= 1e-5 * float(want[1]), (st[-1], want)


DW_BIG = [("wide", 1048584), ("vec", 1048580), ("scalar", 1048583)]     # Lout % 8 == 0, % 4 == 0, odd


@gpu
@pytest.mark.parametrize("path,L", DW_BIG, ids=[c[0] for c in DW_BIG])
def test_depthwise_past_2_31_elements(path, L):
    """sdr_depthwise, stride 1, read through GlobLN + PReLU, on each of its three kernels."""
    need(18)
    assert (BIG_S - 1) * BIG_C * L > 2 ** 31 and BIG_C * L < 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(107)
    count = BIG_C * L
    x = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    w5 = torch.randn(BIG_C, 5, device=DEV, generator=g) / 2
    bias = torch.randn(BIG_C, device=DEV, generator=g)
    stats, gamma, beta = norm_parts(BIG_C, count, g)
    slope = torch.tensor([0.2], device=DEV)
    y = torch.full_like(x, float("nan"))
    st = torch.zeros(BIG_S, 2, dtype=torch.float64, device=DEV)
    nin = norm_in(stats, gamma, beta, slope, count)
    N.check(N.lib().sdr_depthwise(p(x), C.byref(nin), p(w5), p(bias), p(y), p(st), BIG_S, BIG_C, L, 1, stream()))
    xs, = last_sample_parts(x)
    ss, gs, bs = stats[-1:].contiguous(), gamma[-SUB:].contiguous(), beta[-SUB:].contiguous()
    ws, bis = w5[-SUB:].contiguous(), bias[-SUB:].contiguous()
    ys = torch.full_like(xs, float("nan"))
    sts = torch.zeros(1, 2, dtype=torch.float64, device=DEV)
    ns = norm_in(ss, gs, bs, slope, count)
    N.check(N.lib().sdr_depthwise(p(xs), C.byref(ns), p(ws), p(bis), p(ys), p(sts), 1, SUB, L, 1, stream()))
    torch.cuda.synchronize()
    assert_rows_equal(y[-1, -SUB:], ys[0])
    assert torch.isfinite(y[0, :SUB]).all()
    check_last_stats(st, y[-1])
    f = ref_glob(xs[0], ss[0], gs, bs, count, slope)
    want = F.conv1d(f.unsqueeze(0), ws.double().view(SUB, 1, 5), bis.double(), padding=2, groups=SUB)
    assert max(O.parity_errors(ys, want)) < 2e-5


# L % 4 == 0 and L % 2 == 0; the wide kernel needs depth >= 4, whose four levels would take 24 GiB here
MERGE_BIG = [("vec", 1048584), ("scalar", 1048582)]


@gpu
@pytest.mark.parametrize("path,L", MERGE_BIG, ids=[c[0] for c in MERGE_BIG])
def test_merge_past_2_31_elements(path, L):
    """sdr_merge at depth 2 (z0 [samples, C, L], z1 [samples, C, L/2], each read through its GlobLN), on its vector
    and scalar kernels."""
    need(22)
    assert (BIG_S - 1) * BIG_C * L > 2 ** 31 and BIG_C * L < 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(109)
    z0 = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    z1 = torch.randn(BIG_S, BIG_C, L // 2, device=DEV, generator=g)
    parts = [norm_parts(BIG_C, BIG_C * L >> d, g) for d in range(2)]
    m = torch.full_like(z0, float("nan"))
    st = torch.zeros(BIG_S, 2, dtype=torch.float64, device=DEV)
    nins = (N.SdrNormIn * 2)(*[norm_in(s_, g_, b_, None, BIG_C * L >> d) for d, (s_, g_, b_) in enumerate(parts)])
    zs = (C.c_void_p * 2)(z0.data_ptr(), z1.data_ptr())
    N.check(N.lib().sdr_merge(zs, nins, 2, p(m), p(st), BIG_S, BIG_C, L, stream()))
    z0s, z1s = last_sample_parts(z0, z1)
    sub_parts = [(s_[-1:].contiguous(), g_[-SUB:].contiguous(), b_[-SUB:].contiguous()) for s_, g_, b_ in parts]
    ms = torch.full_like(z0s, float("nan"))
    sts = torch.zeros(1, 2, dtype=torch.float64, device=DEV)
    nss = (N.SdrNormIn * 2)(*[norm_in(s_, g_, b_, None, BIG_C * L >> d) for d, (s_, g_, b_) in enumerate(sub_parts)])
    zss = (C.c_void_p * 2)(z0s.data_ptr(), z1s.data_ptr())
    N.check(N.lib().sdr_merge(zss, nss, 2, p(ms), p(sts), 1, SUB, L, stream()))
    torch.cuda.synchronize()
    assert_rows_equal(m[-1, -SUB:], ms[0])
    assert torch.isfinite(m[0, :SUB]).all()
    check_last_stats(st, m[-1])
    want = ref_glob(z0s[0], sub_parts[0][0][0], sub_parts[0][1], sub_parts[0][2], BIG_C * L)
    want = want + ref_glob(z1s[0], sub_parts[1][0][0], sub_parts[1][1], sub_parts[1][2], BIG_C * L >> 1) \
        .repeat_interleave(2, -1)
    assert max(O.parity_errors(ms[0], want)) < 2e-5


@gpu
def test_tac_apply_past_2_31_elements():
    """sdr_tac_apply: out = x + GlobLN(o), with o read from x's buffer (both inputs) to keep two 8 GiB tensors."""
    need(18)
    L = 1048584
    g = torch.Generator(device=DEV).manual_seed(113)
    x = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    stats, gamma, beta = norm_parts(BIG_C, BIG_C * L, g)
    out = torch.full_like(x, float("nan"))
    nin = norm_in(stats, gamma, beta, None, BIG_C * L)
    N.check(N.lib().sdr_tac_apply(p(x), p(x), C.byref(nin), p(out), BIG_S, BIG_C, L, stream()))
    xs, = last_sample_parts(x)
    ss, gs, bs = stats[-1:].contiguous(), gamma[-SUB:].contiguous(), beta[-SUB:].contiguous()
    outs = torch.full_like(xs, float("nan"))
    ns = norm_in(ss, gs, bs, None, BIG_C * L)
    N.check(N.lib().sdr_tac_apply(p(xs), p(xs), C.byref(ns), p(outs), 1, SUB, L, stream()))
    torch.cuda.synchronize()
    assert_rows_equal(out[-1, -SUB:], outs[0])
    assert torch.isfinite(out[0, :SUB]).all()
    want = xs[0].double() + ref_glob(xs[0], ss[0], gs, bs, BIG_C * L)
    assert max(O.parity_errors(outs[0], want)) < 2e-5


@gpu
def test_residual_norm_past_2_31_elements():
    """sdr_residual_norm (the original UBlock's tail): x <- GN(e) + module_act(x) in place, per-channel PReLU."""
    need(18)
    L = 1048584
    g = torch.Generator(device=DEV).manual_seed(127)
    e = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    x = torch.randn(BIG_S, BIG_C, L, device=DEV, generator=g)
    se, ge, be = norm_parts(BIG_C, BIG_C * L, g)
    sx, gx, bx = norm_parts(BIG_C, BIG_C * L, g)
    slopes = 0.1 + 0.5 * torch.rand(BIG_C, device=DEV, generator=g)
    es, xs = last_sample_parts(e, x)                  # before the in-place call
    st = torch.zeros(BIG_S, 2, dtype=torch.float64, device=DEV)
    fe, fx = norm_in(se, ge, be, None, BIG_C * L), norm_in(sx, gx, bx, slopes, BIG_C * L)
    N.check(N.lib().sdr_residual_norm(p(e), C.byref(fe), p(x), C.byref(fx), p(st), BIG_S, BIG_C, L, stream()))
    sub = [t[-1:].contiguous() for t in (se, sx)] + [t[-SUB:].contiguous() for t in (ge, be, gx, bx, slopes)]
    ses, sxs, ges, bes, gxs, bxs, sls = sub
    want = ref_glob(es[0], ses[0], ges, bes, BIG_C * L) + ref_glob(xs[0], sxs[0], gxs, bxs, BIG_C * L, sls)
    sts = torch.zeros(1, 2, dtype=torch.float64, device=DEV)
    fes, fxs = norm_in(ses, ges, bes, None, BIG_C * L), norm_in(sxs, gxs, bxs, sls, BIG_C * L)
    N.check(N.lib().sdr_residual_norm(p(es), C.byref(fes), p(xs), C.byref(fxs), p(sts), 1, SUB, L, stream()))
    torch.cuda.synchronize()
    assert_rows_equal(x[-1, -SUB:], xs[0])
    assert torch.isfinite(x[0, :SUB]).all()
    check_last_stats(st, x[-1])
    assert max(O.parity_errors(xs[0], want)) < 2e-5


@gpu
def test_per_sample_items_past_int_are_refused():
    """One sample of 512 channels x 4194305 positions (2^31 + 512 items): the kernels that count a sample's items in
    int refuse it before anything is launched (the buffers are never read)."""
    lib = N.lib()
    t = torch.zeros(1024, device=DEV)
    st = torch.zeros(2, dtype=torch.float64, device=DEV)
    nin = norm_in()
    C_, L = 512, 4194305
    assert C_ * L > 2 ** 31 - 1
    assert lib.sdr_depthwise(p(t), C.byref(nin), p(t), p(t), p(t), p(st), 1, C_, L, 1, stream()) == -5
    assert lib.sdr_depthwise(p(t), C.byref(nin), p(t), p(t), p(t), p(st), 1, C_, L + 1, 2, stream()) == -5
    zs = (C.c_void_p * 2)(t.data_ptr(), t.data_ptr())
    ns = (N.SdrNormIn * 2)(norm_in(), norm_in())
    assert lib.sdr_merge(zs, ns, 2, p(t), p(st), 1, C_, L + 1, stream()) == -5
    gln = norm_in(st.view(1, 2), t, t, None, 1.0)
    assert lib.sdr_tac_apply(p(t), p(t), C.byref(gln), p(t), 1, C_, L, stream()) == -5
    assert lib.sdr_residual_norm(p(t), C.byref(nin), p(t), C.byref(nin), p(st), 1, C_, L, stream()) == -5
    torch.cuda.synchronize()


BIG_MODELS = [
    ("improved", imp(4, 5, 64, Co=8, Ci=16, D=2)),
    ("groupcomm", gc(4, 1, 5, 64, 2, 4, D=2)),
    ("causal", dict(CAUSAL, enc_num_basis=64, num_sources=4)),
    ("original", orig(4, 5, 64, 16, D=2)),
]


@gpu
@pytest.mark.parametrize("variant,kw", BIG_MODELS, ids=[v for v, _ in BIG_MODELS])
def test_model_workspace_past_2_31_elements(variant, kw):
    """A whole model whose masked tensor (B x S*N x L) passes 2^31 elements: its last item against a B = 1 run and the
    fp64 oracle."""
    cfg = O.Config(variant=variant, **kw)
    T = MODEL_T
    L = O.padded_length(cfg, T) // cfg.hop
    B = 2 ** 31 // (cfg.num_sources * cfg.enc_num_basis * L) + 2
    assert B * cfg.num_sources * cfg.enc_num_basis * L > 2 ** 31
    c = _engine.make_config(CLASSES[variant](**kw))
    ws = N.lib().sdr_workspace_bytes(C.byref(c), B, T)
    need(ws / GiB + 1.5)
    cfg, sd, m = build(variant, kw, seed=97)
    x1 = normalised_input(1, 1, T, seed=101).to(DEV)
    x = torch.randn(B, 1, T, device=DEV, generator=torch.Generator(device=DEV).manual_seed(103))
    x[-1] = x1[0]
    with torch.no_grad():
        one = m(x1)
        big = m(x)
    assert torch.isfinite(big[0]).all()
    last = big[-1:].clone()
    del big
    print(f"{variant}: B = {B}, workspace {ws / GiB:.1f} GiB")
    assert_rows_close(last, one)
    e = O.parity_errors(last, O.forward(cfg, sd, x1, dtype=torch.float64))
    assert max(e) < TOL, e


# =====================================================================================================================
# size and launch-count queries (no GPU)
# =====================================================================================================================
QUERY_BATCHES = [65535, 65536, 2 ** 27, 2 ** 31 - 1]
QUERY_MODELS = [
    ("improved", imp(2, 21, 128, Co=128, Ci=512, D=5)),
    ("groupcomm", gc(2, 1, 21, 128, 16, 16, D=5)),
    ("causal", dict(CAUSAL, out_channels=128, in_channels=512, upsampling_depth=5, enc_kernel_size=21,
                    enc_num_basis=128)),
    ("original", orig(2, 21, 128, 128, D=4)),
]


def plan_bytes(cfg, variant, B, T):
    """The forward workspace of make_plan (csrc/api.cu), recomputed: 256-byte aligned segments in order."""
    seg = lambda n: (n + 255) // 256 * 256
    S, A, N_, K = cfg.num_sources, cfg.in_audio_channels if variant == "groupcomm" else 1, cfg.enc_num_basis, \
        cfg.enc_kernel_size
    Co, Ci, U, D = cfg.out_channels, cfg.in_channels, cfg.num_blocks, cfg.upsampling_depth
    G = cfg.group_size if variant == "groupcomm" else 1
    L = O.padded_length(cfg, T) // cfg.hop
    causal, gcm, og = variant == "causal", variant == "groupcomm", variant == "original"
    block_slots = 0 if causal else D + 2 + (1 if gcm else 0) + (2 if og else 0)
    BL = B * L * 4
    total = seg((1 + U * block_slots) * B * G * 2 * 8)                   # statistics
    total += seg(BL * N_) + seg(BL * Co)                                 # e, x
    if gcm or og:
        total += seg(BL * Co)                                            # xt
    if gcm:
        total += seg(BL * Co)                                            # o
    elif og and Co != N_:
        total += seg(BL * N_)                                            # reshape_before_masks output
    total += seg(BL * Ci)                                                # y
    for d in range(D):
        if not (causal and d > 0):
            total += seg((BL * Ci) >> d)                                 # z[d]
    # the one-pass depthwise pyramid keeps per-sample tables; it is never taken past its sample limit (asserted below)
    total += seg(BL * S * A * N_) + seg(BL * S * A * K)                  # masked, frames
    return total


@pytest.mark.parametrize("B", QUERY_BATCHES)
@pytest.mark.parametrize("variant,kw", QUERY_MODELS, ids=[v for v, _ in QUERY_MODELS])
def test_size_queries_at_scale(variant, kw, B):
    """sdr_workspace_bytes, sdr_separate_workspace_bytes, sdr_train_saved_bytes and the launch-count query at large B:
    the exact figure recomputed from the plan, or 0 / an error where B * group_size passes 2^31 - 1; never a wrapped
    value."""
    lib = N.lib()
    cfg = O.Config(variant=variant, **kw)
    c = _engine.make_config(CLASSES[variant](**kw))
    T = 32000
    G = cfg.group_size if variant == "groupcomm" else 1
    ws = lib.sdr_workspace_bytes(C.byref(c), B, T)
    sep = lib.sdr_separate_workspace_bytes(C.byref(c), B, T)
    n = lib.sdr_forward_launch_count_for(C.byref(c), B, T)
    if B * G > 2 ** 31 - 1:
        assert ws == 0 and sep == 0 and n == -5, (ws, sep, n)
        return
    want = plan_bytes(cfg, variant, B, T)
    assert ws == want, (ws, want)
    extra = (B * T * 4 + 255) // 256 * 256 + (B * 16 + 255) // 256 * 256 + (B * 8 + 255) // 256 * 256
    assert sep == want + extra, (sep, want + extra)
    D, U = cfg.upsampling_depth, cfg.num_blocks
    if variant == "causal":
        want_n = 2 + 3 * U + 3
    elif variant == "original":
        want_n = 2 + U * (D + 4) + (1 if cfg.out_channels != cfg.enc_num_basis else 0) + 4
    elif variant == "groupcomm":
        want_n = 2 + U * (D + 3 + 1) + 3                 # 16 -> 32 channels per group: tac_apply rides on proj_1x1
    else:
        want_n = 2 + U * (D + 3) + 3
    assert n == want_n, (n, want_n)                      # the one-pass pyramid is never taken at these batches
    saved = lib.sdr_train_saved_bytes(C.byref(c), B, T)
    if variant != "improved":
        assert saved == 0
    else:
        L = O.padded_length(cfg, T) // cfg.hop
        BL = B * L * 4
        seg = lambda k: (k + 255) // 256 * 256
        want_saved = seg((1 + U * (D + 2)) * B * 2 * 8) + seg(BL * cfg.enc_num_basis) \
            + seg(seg(BL * cfg.out_channels) * (U + 1))
        assert saved == want_saved, (saved, want_saved)


def test_forward_refuses_wrapped_sample_count():
    """GroupComm at B * G past 2^31 - 1: the forward refuses before it reads a buffer."""
    kw = QUERY_MODELS[1][1]
    c = _engine.make_config(CLASSES["groupcomm"](**kw))
    B = (2 ** 31 - 1) // 16 + 1
    assert N.lib().sdr_forward(C.byref(c), None, None, None, B, 32000, 0, None, 0, None) == -5
    assert N.lib().sdr_forward(C.byref(c), None, None, None, B - 1, 32000, 0, None, 0, None) == -2


def test_forward_refuses_items_past_int_per_sample():
    """An improved model with 512 channels at 4194304 frames per mixture (2^31 items in one GlobLN sample): the size
    queries answer 0 / SDR_ERR_UNSUPPORTED and the forward refuses before it reads a buffer; 4194300 frames pass."""
    kw = imp(2, 21, 128, Co=128, Ci=512, D=1)
    cfg = O.Config(variant="improved", **kw)
    c = _engine.make_config(CLASSES["improved"](**kw))
    lib = N.lib()
    T_bad, T_ok = cfg.hop * 4194304, cfg.hop * 4194300
    assert O.padded_length(cfg, T_bad) // cfg.hop == 4194304 and O.padded_length(cfg, T_ok) // cfg.hop == 4194300
    assert lib.sdr_workspace_bytes(C.byref(c), 1, T_bad) == 0
    assert lib.sdr_separate_workspace_bytes(C.byref(c), 1, T_bad) == 0
    assert lib.sdr_train_saved_bytes(C.byref(c), 1, T_bad) == 0
    assert lib.sdr_forward_launch_count_for(C.byref(c), 1, T_bad) == -5
    assert lib.sdr_forward(C.byref(c), None, None, None, 1, T_bad, 0, None, 0, None) == -5
    assert lib.sdr_workspace_bytes(C.byref(c), 1, T_ok) > 0
    assert lib.sdr_forward_launch_count_for(C.byref(c), 1, T_ok) > 0
    assert lib.sdr_forward(C.byref(c), None, None, None, 1, T_ok, 0, None, 0, None) == -2
