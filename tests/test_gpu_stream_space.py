"""Streaming of CausalSuDORMRF across what the C-ABI accepts, and the stream object's promised behaviour.

Whole-model streams at every depth the stage takes beyond the ones test_gpu_stream.py runs, the shortest and longest
filters (hop 1 and 127), one to sixteen output channels (S*A), every 1x1 convolution on the wgmma kernel and all on
FFMA, the longest chunk (4096 frames), 300 and 65535 slots, and mixture consistency at one and three sources.  Every
case streams at least six chunks at a length that is a multiple of hop * 2^D (the flush tail is compared too) and,
where the depth allows one, at a length that is not.  Each is compared with
- the native offline forward on the same weights (<= 1e-5, printed whether bitwise),
- the fp64 oracle on the whole clip (<= 1e-3 max|ref| per sample and rel-L2 <= 1e-3),
- the fp64 chunked restatement (tests/stream_oracle.py), step by step with its flush tail, at the same bar.

Then the lifecycle: flush() keeps the state, flush() of a fresh or reset stream is zero, reset() and reset([j]) touch
exactly the slots they name, model(x) and a second stream of the same model can run between steps, changed weights
are picked up on the next step, and steps give the same bits on a side CUDA stream and for fp64, fp16 and strided
chunks."""
import pytest
import torch

from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
from stream_oracle import CausalStreamOracle, causal_stream_forward, granule
from test_gpu_stream import DEV, TOL, build, mixture, streamed

pytestmark = pytest.mark.gpu

BASE = dict(in_audio_channels=1, out_channels=16, in_channels=24, num_blocks=2, upsampling_depth=4,
            enc_kernel_size=21, enc_num_basis=16, num_sources=2)      # every GEMM on FFMA (K < 64)
WGMMA = dict(in_audio_channels=1, out_channels=64, in_channels=64, num_blocks=2, upsampling_depth=4,
             enc_kernel_size=21, enc_num_basis=64, num_sources=2)     # every GEMM and the encoder on wgmma


def compare_stream(cfg, sd, m, x, chunk):
    """Stream x [B, A, n*chunk] and compare with the offline forward, the whole-clip oracle and the restatement."""
    hop, T, q = cfg.hop, x.shape[-1], cfg.n_least_samples_req
    xd = x.to(DEV)
    out, tail = streamed(m, xd, chunk)
    with torch.no_grad():
        nat = m(xd)
    assert torch.equal(out[..., :hop], torch.zeros_like(out[..., :hop]))
    got = torch.cat([out[..., hop:], tail], -1)
    aligned = T % q == 0
    n_cmp = T if aligned else T - hop
    e_nat = O.parity_errors(got[..., :n_cmp], nat[..., :n_cmp])
    bitwise = torch.equal(got[..., :n_cmp], nat[..., :n_cmp])
    ref = O.causal_forward(cfg, sd, x, dtype=torch.float64)
    e = O.parity_errors(got[..., :n_cmp], ref[..., :n_cmp])
    s_out, s_tail = causal_stream_forward(cfg, sd, x.double(), chunk)
    e_s = O.parity_errors(torch.cat([out, tail], -1), torch.cat([s_out, s_tail], -1))
    print(f"  B={x.shape[0]} chunk={chunk} ({chunk // hop} frames) x {T // chunk} "
          f"{'aligned' if aligned else 'unaligned'}: native rel_max {e_nat[0]:.2e} rel_l2 {e_nat[1]:.2e} "
          f"bitwise {bitwise}; fp64 oracle {max(e):.2e}; restatement {max(e_s):.2e}")
    assert max(e_nat) <= 1e-5, e_nat
    assert max(e) < TOL, e
    assert max(e_s) < TOL, e_s


def check_model(kw, B, g=1, seed=21):
    """Six chunks of g granules (n*C a multiple of hop * 2^D: the flush tail is compared), then seven chunks of an odd
    number of granules (not a multiple, D >= 3; at D <= 2 every granule multiple is one)."""
    cfg, sd, m = build(kw, seed=seed)
    G, q, A = granule(cfg), cfg.n_least_samples_req, cfg.in_audio_channels
    print(f"{kw}: granule {G}")
    runs = [(g, 6)]
    go = g if g % 2 else g - 1
    if (7 * go * G) % q:
        runs.append((go, 7))
    else:
        print("  every chunk count is a multiple of hop * 2^D at this depth: no unaligned length")
    for gg, n in runs:
        assert (n * gg * G) % q == 0 or n == 7
        compare_stream(cfg, sd, m, mixture(B, A, n * gg * G, seed=seed + gg), gg * G)
    return cfg, m


# ---- depth, filter length, sources, GEMM kernels, chunk length, slots ----
@pytest.mark.parametrize("D", [1, 2, 6, 7, 8])
def test_depths(D):
    check_model(dict(BASE, upsampling_depth=D), B=3)


def test_depth8_longest_chunk_crosses_offline_windows():
    """4096 frames per step at D = 8; the offline forward splits its 24576-frame rows into causal windows."""
    check_model(dict(BASE, upsampling_depth=8), B=2, g=32)


@pytest.mark.parametrize("k,A,g", [(3, 1, 5), (5, 1, 3), (63, 2, 1), (255, 1, 1)])
def test_filter_lengths(k, A, g):
    """hop 1, 2, 31 and 127 (the longest the overlap-add takes); N = 32 puts the encoder on wgmma, whose operand
    pads A*k taps to a 64-row k-block: 3 -> 64, 5 -> 64, 126 -> 128, 255 -> 256."""
    kw = dict(BASE, enc_kernel_size=k, in_audio_channels=A, enc_num_basis=32)
    assert N.lib().sdr_encoder_mma_packed_bytes(32, A, k) > 0
    check_model(kw, B=2, g=g)


@pytest.mark.parametrize("S,A", [(1, 1), (3, 1), (8, 2), (16, 1)])
def test_source_counts(S, A):
    check_model(dict(BASE, num_sources=S, in_audio_channels=A), B=2)


def _gemm_shapes(kw):
    S, A, k, N_, Co, Ci = (kw[n] for n in ("num_sources", "in_audio_channels", "enc_kernel_size", "enc_num_basis",
                                           "out_channels", "in_channels"))
    return [(Co, N_), (Ci, Co), (Co, Ci), (S * A * N_, Co), (S * A * k, S * A * N_)]   # bottleneck, proj, res, mask, dec


def test_every_gemm_on_wgmma():
    lib = N.lib()
    assert lib.sdr_encoder_mma_packed_bytes(WGMMA["enc_num_basis"], 1, WGMMA["enc_kernel_size"]) > 0
    assert all(lib.sdr_pointwise_mma_packed_bytes(M, K) > 0 for M, K in _gemm_shapes(WGMMA))
    check_model(WGMMA, B=3)


def test_every_gemm_on_ffma():
    lib = N.lib()
    assert lib.sdr_encoder_mma_packed_bytes(BASE["enc_num_basis"], 1, BASE["enc_kernel_size"]) == 0
    assert all(lib.sdr_pointwise_mma_packed_bytes(M, K) == 0 for M, K in _gemm_shapes(BASE))
    check_model(dict(BASE, upsampling_depth=3), B=3)


def test_300_slots_share_gemm_tiles():
    """8 frames per slot: one 128-column GEMM tile spans 16 slots."""
    check_model(WGMMA, B=300)


TINY = dict(in_audio_channels=1, out_channels=8, in_channels=8, num_blocks=1, upsampling_depth=2, enc_kernel_size=5,
            enc_num_basis=8, num_sources=2)


def test_65535_slots():
    """Slot j streams mixture j mod 7: every slot equals that slot of a 7-slot stream, bit for bit."""
    cfg, sd, m = build(TINY)
    G = granule(cfg)
    B = 65535
    base = mixture(7, 1, 2 * G, seed=4).to(DEV)
    x = base.repeat(-(-B // 7), 1, 1)[:B]
    with torch.no_grad():
        big = m.stream(B, G)
        small = m.stream(7, G)
        for c in range(2):
            got = big.step(x[..., c * G:(c + 1) * G])
            want = small.step(base[..., c * G:(c + 1) * G])
            assert torch.equal(got, want.repeat(-(-B // 7), 1, 1)[:B]), c
        assert torch.equal(big.flush(), small.flush().repeat(-(-B // 7), 1, 1)[:B])
    compare_stream(cfg, sd, m, mixture(7, 1, 6 * G, seed=4), G)


@pytest.mark.parametrize("S", [1, 3])
def test_mixture_consistency_other_source_counts(S):
    """The projection divides the residual by S; at S = 2 a divisor of 1/2 hides any other constant."""
    cfg, sd, m = build(dict(BASE, num_sources=S))
    G = granule(cfg)
    x = mixture(2, 1, 10 * G, seed=9).to(DEV)
    out, tail = streamed(m, x, G, mc=True)
    with torch.no_grad():
        ref = m.separate(x, mixture_consistency=True)
    hop = cfg.hop
    got = torch.cat([out[..., hop:], tail], -1)
    e = O.parity_errors(got, ref)
    print("S=%d mixture consistency vs separate: rel_max %.2e rel_l2 %.2e bitwise %s" % ((S,) + e
                                                                                        + (torch.equal(got, ref),)))
    assert max(e) <= 1e-5, e
    # the projected estimates add up to the mixture, delayed by hop, flush tail included
    assert torch.allclose(got.sum(1), x[:, 0], atol=1e-5)


# ---- lifecycle and API semantics ----
MID = dict(BASE, out_channels=64, in_channels=64, enc_num_basis=64)


def chunks_of(x, C):
    return [x[..., c:c + C] for c in range(0, x.shape[-1], C)]


@pytest.mark.parametrize("mc", [False, True])
def test_flush_keeps_the_state(mc):
    cfg, sd, m = build(MID)
    G = granule(cfg)
    x = mixture(2, 1, 6 * G, seed=31).to(DEV)
    with torch.no_grad():
        a, b = m.stream(2, G, mixture_consistency=mc), m.stream(2, G, mixture_consistency=mc)
        outs_a, outs_b = [], []
        for i, c in enumerate(chunks_of(x, G)):
            outs_a.append(a.step(c))
            outs_b.append(b.step(c))
            if i in (0, 2):
                a.flush()
                a.flush()
        assert torch.equal(torch.cat(outs_a, -1), torch.cat(outs_b, -1))
        assert torch.equal(a.flush(), b.flush())
        assert torch.equal(a._state, b._state)


@pytest.mark.parametrize("mc", [False, True])
def test_flush_of_a_fresh_or_reset_stream_is_zero(mc):
    cfg, sd, m = build(MID)
    G = granule(cfg)
    with torch.no_grad():
        s = m.stream(3, G, mixture_consistency=mc)
        zero = torch.zeros(3, 2, cfg.hop, device=DEV)
        assert torch.equal(s.flush(), zero)
        s.step(mixture(3, 1, G, seed=32).to(DEV))
        assert not torch.equal(s.flush(), zero)
        s.reset()
        assert torch.equal(s.flush(), zero)


def test_reset_touches_exactly_the_named_slots():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    B = 4
    x1 = mixture(B, 1, 3 * G, seed=33).to(DEV)
    x2 = mixture(B, 1, 3 * G, seed=34).to(DEV)
    with torch.no_grad():
        s = m.stream(B, G)
        for c in chunks_of(x1, G):
            s.step(c)
        before = s._state.clone()
        s.reset([])
        assert torch.equal(s._state, before)
        s.reset([2])
        per_slot = s._state.view(B, -1)
        assert not torch.equal(before.view(B, -1)[2], per_slot[2])
        assert torch.equal(per_slot[2], torch.zeros_like(per_slot[2]))
        for j in (0, 1, 3):
            assert torch.equal(per_slot[j], before.view(B, -1)[j]), j
        s.reset()
        fresh = m.stream(B, G)
        assert torch.equal(s._state, fresh._state)
        got = torch.cat([s.step(c) for c in chunks_of(x2, G)], -1)
        want = torch.cat([fresh.step(c) for c in chunks_of(x2, G)], -1)
        assert torch.equal(got, want)
        assert torch.equal(s.flush(), fresh.flush())


def test_model_calls_between_steps():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    x = mixture(2, 1, 6 * G, seed=35).to(DEV)
    other = mixture(5, 1, 3001, seed=36).to(DEV)
    with torch.no_grad():
        a, b = m.stream(2, G), m.stream(2, G)
        got, want = [], []
        for c in chunks_of(x, G):
            m(other)                                      # another batch and length on the model's own workspace
            got.append(a.step(c))
            m(other[:1, :, :777])
        for c in chunks_of(x, G):
            want.append(b.step(c))
    assert torch.equal(torch.cat(got, -1), torch.cat(want, -1))
    assert torch.equal(a.flush(), b.flush())


def test_two_streams_of_one_model():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    x = mixture(2, 1, 6 * 3 * G, seed=37).to(DEV)
    with torch.no_grad():
        fine, coarse = m.stream(2, G), m.stream(2, 3 * G)
        out_f, out_c = [], []
        for i, c in enumerate(chunks_of(x, 3 * G)):       # alternate: three fine steps, one coarse step
            out_f += [fine.step(cc) for cc in chunks_of(c, G)]
            out_c.append(coarse.step(c))
        nat = m(x)
    hop = cfg.hop
    for name, outs, s in (("G", out_f, fine), ("3G", out_c, coarse)):
        got = torch.cat([torch.cat(outs, -1)[..., hop:], s.flush()], -1)
        e = O.parity_errors(got, nat)
        print(f"chunk {name}: vs native rel_max {e[0]:.2e} rel_l2 {e[1]:.2e} bitwise {torch.equal(got, nat)}")
        assert max(e) <= 1e-5, e


def test_weights_changed_mid_stream():
    cfg, sd, m = build(BASE, seed=11)
    sd2 = O.make_state_dict(cfg, seed=12)
    G = granule(cfg)
    x = mixture(2, 1, 6 * G, seed=38)
    ref = CausalStreamOracle(cfg, sd, 2)
    s = m.stream(2, G)
    got, want = [], []
    with torch.no_grad():
        for i, c in enumerate(chunks_of(x, G)):
            if i == 3:
                m.load_state_dict(sd2)
                ref.set_weights(sd2)
            got.append(s.step(c.to(DEV)))
            want.append(ref.step(c))
        got.append(s.flush())
    want.append(ref.flush())
    for i, (g_, w_) in enumerate(zip(got, want)):
        e = O.parity_errors(g_, w_)
        print(f"step {i}: vs restatement rel_max {e[0]:.2e} rel_l2 {e[1]:.2e}")
        assert max(e) < TOL, (i, e)
    # the swap changed the output: a stream that kept the old weights differs from step 3 on
    old = CausalStreamOracle(cfg, sd, 2)
    kept = [old.step(c) for c in chunks_of(x, G)]
    assert max(O.parity_errors(got[3], kept[3])) > 1e-2


def test_side_stream_and_input_forms():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    B, T = 3, 6 * G
    x = mixture(B, 1, T, seed=39).to(DEV)
    with torch.no_grad():
        base = m.stream(B, G)
        want = torch.cat([base.step(c.contiguous()) for c in chunks_of(x, G)], -1)
        # a side CUDA stream
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            s = m.stream(B, G)
            got = torch.cat([s.step(c) for c in chunks_of(x, G)], -1)
        torch.cuda.current_stream().wait_stream(side)
        assert torch.equal(got, want)
        # strided chunks: slices of a [T, A, B] buffer seen as [B, A, T]
        xt = x.permute(2, 1, 0).contiguous().permute(2, 1, 0)
        assert not xt[..., :G].is_contiguous()
        s = m.stream(B, G)
        assert torch.equal(torch.cat([s.step(c) for c in chunks_of(xt, G)], -1), want)
        # fp64 and fp16 chunks: the same bits as their fp32 casts
        for dt in (torch.float64, torch.float16):
            xd = x.to(dt)
            s, r = m.stream(B, G), m.stream(B, G)
            a = torch.cat([s.step(c) for c in chunks_of(xd, G)], -1)
            b = torch.cat([r.step(c.float()) for c in chunks_of(xd, G)], -1)
            assert a.dtype == torch.float32 and torch.equal(a, b), dt
