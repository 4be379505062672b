"""Windowed separation of a corpus on the GPU (DESIGN.md section 7i).

Stage entries on synthetic estimates: the ragged merge is bitwise the single-recording merge run on each recording
alone, for every batch size, and matches the fp64 oracle; a NaN, an infinity or a silent overlap stays in its
recording; poisoned and guarded buffers.  Whole calls: every recording equals ``separate_long`` on it alone, for every
model variant; memory does not grow with the corpus; a flat output past 2^31 elements; a side stream."""
import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
import windowed_oracle as WO
from guards import POISON_HUGE, POISON_NAN, check_bands, guarded_copy, poisoned, poisoned_like
from oracle import sudormrf_oracle as O
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import windowed

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPREAD = 1e-5      # run-to-run spread of the non-causal forwards, whose fp64 statistics are summed by atomics
MARGIN = 1e-6

# ---------------------------------------------------------------------------------------------------------------------
# stages
# ---------------------------------------------------------------------------------------------------------------------
SW, SH = 64, 40
# W + 1, W + H, exact window multiples, one-sample tails and a recording of 8 windows, mixed; with M = 3 the long one
# spans three batches, with M >= 7 a batch holds three recordings or more
STAGE_LENGTHS = [SW + 3 * SH, SW + 1, SW + 7 * SH, SW + SH, SW + 5 * SH + 1, SW + 2 * SH + 1,
                 SW + 1]


def estimates(lengths, S, A, seed):
    """Per recording, est [K, S, A, W]: windows of random sources in a random order plus noise (clear margins)."""
    gen = np.random.default_rng(seed)
    out = []
    for T in lengths:
        src = gen.standard_normal((S, A, T)).astype(np.float32)
        K = WO.plan(T, SW, SH)[0]
        win = WO.windows(src.reshape(1, S * A, T), SW, SH).reshape(K, S, A, SW)
        est = np.stack([win[k][gen.permutation(S)] for k in range(K)])
        out.append((est + 0.3 * gen.standard_normal(est.shape)).astype(np.float32))
    return out


def descriptors(plan, lengths):
    return torch.tensor([[o, lengths[i], g] for i, o, g in zip(plan.long, plan.offsets, plan.firsts)],
                        dtype=torch.int64).to(DEV)


def run_ragged(est, lengths, S, A, M, pattern=0, check=False):
    """Ragged merge of the estimates of every recording (all longer than SW) in batches of M global windows;
    ([S A, T] per recording, [K, S] per recording)."""
    lib = N.lib()
    plan = windowed.corpus_plan(lengths, SW, SH, M)
    desc = descriptors(plan, lengths)
    if check:
        desc = guarded_copy(desc)
        desc_before = desc.clone()
    allest = torch.from_numpy(np.concatenate([e.reshape(-1, S * A, SW) for e in est])).to(DEV)
    carry = poisoned(lib.sdr_window_ragged_carry_bytes(S, A, SW), pattern)
    Mb = plan.batches[0][1]
    scratch = poisoned(lib.sdr_window_ragged_scratch_bytes(S, Mb), pattern)
    out = poisoned_like(torch.empty(S * A * plan.samples, device=DEV), pattern)
    perm = poisoned_like(torch.empty(plan.windows, S, dtype=torch.int32, device=DEV), pattern)
    for g0, m in plan.batches:
        chunk = allest[g0:g0 + m].contiguous()
        sc = scratch if m == Mb else poisoned(lib.sdr_window_ragged_scratch_bytes(S, m), pattern)
        if check:
            chunk = guarded_copy(chunk)
            before = chunk.clone()
        windowed.merge(chunk, carry, perm, out, S, A, SW, SH, g0, m, sc, desc=desc)
        if check:
            check_bands(chunk, "estimates")
            check_bands(sc, "scratch")
            assert torch.equal(chunk, before), "the estimates were modified"
    if check:
        for t, what in ((carry, "carry"), (scratch, "scratch"), (out, "out"), (perm, "perm"), (desc, "desc")):
            check_bands(t, what)
        assert torch.equal(desc, desc_before)
    torch.cuda.synchronize()
    outs = [out[S * A * o:S * A * (o + lengths[i])].view(S * A, lengths[i]) for i, o in zip(plan.long, plan.offsets)]
    perms = [perm[g:g + K] for g, K in zip(plan.firsts, plan.counts)]
    return outs, perms


def run_single(est, T, S, A):
    """sdr_window_merge with B = 1 on one recording's estimates [K, S, A, W], one batch."""
    lib = N.lib()
    K = est.shape[0]
    carry = poisoned(lib.sdr_window_carry_bytes(1, S, A, SW), 0)
    scratch = poisoned(lib.sdr_window_merge_scratch_bytes(1, S, K), 0)
    out = torch.empty(1, S * A, T, device=DEV)
    perm = torch.empty(1, K, S, dtype=torch.int32, device=DEV)
    windowed.merge(torch.from_numpy(est).to(DEV).reshape(1, K, S * A, SW), carry, perm, out, S, A, SW, SH, 0, K,
                   scratch)
    torch.cuda.synchronize()
    return out[0], perm[0]


@pytest.mark.parametrize("S,A", [(2, 1), (3, 2), (4, 1)])
def test_ragged_merge_is_the_merge_of_each_recording(S, A):
    est = estimates(STAGE_LENGTHS, S, A, 10 * S + A)
    singles = [run_single(e, T, S, A) for e, T in zip(est, STAGE_LENGTHS)]
    for r, (e, T) in enumerate(zip(est, STAGE_LENGTHS)):
        pi, margin = WO.align(e[None], T, SW, SH)
        assert (margin[0, 1:] > MARGIN).all(), r
        assert np.array_equal(singles[r][1].cpu().numpy(), pi[0]), r
        assert np.array_equal(singles[r][0].cpu().numpy(), WO.overlap_add(e[None], pi, T, SW, SH)[0]), r
    for M in (1, 2, 3, 7, 32):
        outs, perms = run_ragged(est, STAGE_LENGTHS, S, A, M)
        for r in range(len(STAGE_LENGTHS)):
            assert torch.equal(perms[r], singles[r][1]), (M, r)
            assert torch.equal(outs[r].view(torch.int32), singles[r][0].view(torch.int32)), (M, r)


def test_nonfinite_and_silent_overlaps_stay_in_their_recording():
    S, A = 3, 1
    clean = estimates(STAGE_LENGTHS, S, A, 3)
    est = [e.copy() for e in clean]
    est[0][1, :, :, SH:] = 0                  # recording 0: overlap 2 silent in both windows, rho_2 = id
    est[0][2, :, :, :SW - SH] = 0
    est[2][3, 1, 0, 5] = np.nan               # recording 2: NaN in overlap 3
    est[4][2, 2, 0, SW - 1] = np.inf          # recording 4: inf in overlap 3 (window 2's tail)
    hit = {0: 2, 2: 3, 4: 3}
    for M in (2, 7):
        ref_out, ref_perm = run_ragged(clean, STAGE_LENGTHS, S, A, M)
        out, perm = run_ragged(est, STAGE_LENGTHS, S, A, M)
        for r in range(len(STAGE_LENGTHS)):
            if r in hit:
                p = perm[r].cpu().numpy()
                assert np.array_equal(p[hit[r]], p[hit[r] - 1]), (M, r)
                pi, _ = WO.align(est[r][None], STAGE_LENGTHS[r], SW, SH)
                assert np.array_equal(p, pi[0]), (M, r)
            else:
                assert torch.equal(perm[r], ref_perm[r]), (M, r)
                assert torch.equal(out[r].view(torch.int32), ref_out[r].view(torch.int32)), (M, r)
        assert torch.isfinite(out[0]).all()


@pytest.mark.parametrize("S,A", [(2, 1), (4, 2)])
def test_entries_on_poisoned_and_guarded_buffers(S, A):
    gen = np.random.default_rng(5)
    lengths = STAGE_LENGTHS
    plan = windowed.corpus_plan(lengths, SW, SH, 3)
    xs = [gen.standard_normal((A, T)).astype(np.float32) for T in lengths]
    x = torch.from_numpy(np.concatenate([v.reshape(-1) for v in xs])).to(DEV)
    want = np.concatenate([WO.windows(v[None], SW, SH)[0] for v in xs])          # [G, A, W]
    desc = guarded_copy(descriptors(plan, lengths))
    for pattern in (0, POISON_NAN, POISON_HUGE):
        xg = guarded_copy(x)
        for g0, m in [(0, plan.windows), (0, 1), (2, 3), (plan.windows - 2, 2)] + plan.batches:
            batch = poisoned_like(torch.empty(m, A, SW, device=DEV), pattern)
            windowed.gather(xg, batch, SW, SH, g0, m, desc=desc)
            check_bands(batch, "batch")
            assert np.array_equal(batch.cpu().numpy(), want[g0:g0 + m]), (g0, m)
        check_bands(xg, "mixture")
        check_bands(desc, "desc")
        assert torch.equal(xg, x)
    est = [gen.standard_normal(e.shape).astype(np.float32) for e in estimates(lengths, S, A, 6)]
    clean = run_ragged(est, lengths, S, A, 3, 0, check=True)
    for pattern in (POISON_NAN, POISON_HUGE):
        got = run_ragged(est, lengths, S, A, 3, pattern, check=True)
        for r in range(len(lengths)):
            assert torch.equal(got[1][r], clean[1][r]), pattern
            assert torch.equal(got[0][r].view(torch.int32), clean[0][r].view(torch.int32)), pattern


def test_ragged_refusals():
    lib = N.lib()
    S, A = 2, 1
    est = torch.zeros(2, S * A, SW, device=DEV)
    desc = torch.tensor([[0, SW + 1, 0]], dtype=torch.int64, device=DEV)
    carry = torch.empty(1 << 16, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(1024, dtype=torch.uint8, device=DEV)
    out = torch.empty(S * A * (SW + 1), device=DEV)
    with pytest.raises(N.NativeError, match="code -5"):
        windowed.merge(est, carry, None, out, 5, A, SW, SH, 0, 2, scratch, desc=desc)
    with pytest.raises(N.NativeError, match="code -2"):                   # misaligned carry
        windowed.merge(est, carry[8:], None, out, S, A, SW, SH, 0, 2, scratch, desc=desc)
    with pytest.raises(N.NativeError, match="code -2"):                   # H < W / 2
        windowed.merge(est, carry, None, out, S, A, SW, SW // 2 - 1, 0, 2, scratch, desc=desc)
    assert lib.sdr_window_ragged_carry_bytes(5, 1, 16) == 0


# ---------------------------------------------------------------------------------------------------------------------
# whole calls
# ---------------------------------------------------------------------------------------------------------------------
MODELS = {
    "improved": (P.SuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                  enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    "improved3": (P.SuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=3,
                                   enc_kernel_size=11, enc_num_basis=64, num_sources=3)),
    "groupcomm": (P.GroupCommSudoRmRf, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                            enc_kernel_size=21, enc_num_basis=64, num_sources=2, group_size=4)),
    "groupcomm_stereo": (P.GroupCommSudoRmRf, dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3,
                                                   enc_kernel_size=11, enc_num_basis=16, num_sources=2, group_size=8,
                                                   in_audio_channels=2)),
    "causal": (P.CausalSuDORMRF, dict(in_audio_channels=1, out_channels=64, in_channels=128, num_blocks=2,
                                      upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    "original": (P.OriginalSuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                          enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
}
_cache = {}


def model(name):
    if name not in _cache:
        cls, kw = MODELS[name]
        variant = name.rstrip("3").replace("_stereo", "")
        sd = O.make_state_dict(O.Config(variant=variant, **kw), seed=11)
        m = cls(**kw)
        m.load_state_dict(sd)
        _cache[name] = m.to(DEV).eval()
    return _cache[name]


def recording(A, T, seed):
    """[A, T]: two well-separated synthetic sources (a slow chirp and a pulsed tone) and a little noise."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64) / 8000.0
    a = torch.sin(2 * np.pi * (150.0 + 40.0 * t) * t)
    b = 0.7 * torch.sin(2 * np.pi * 1300.0 * t) * (torch.sin(2 * np.pi * 0.7 * t) > 0)
    x = a + b + 0.05 * torch.randn(A, T, generator=g, dtype=torch.float64)
    return (x + 0.1).float().to(DEV)


W, H = 4000, 2000
LENGTHS = [W + 5 * H + 123, 1000, W + 1, W - 1, W + H, W, W + 3 * H, 7, W + 2 * H + 1, W + 9 * H + 777]


def cases():
    for name in MODELS:
        mono = MODELS[name][1].get("in_audio_channels", 1) == 1
        for normalize in (True, False):
            for mc in (True, False):
                if mono or not (normalize or mc):
                    yield pytest.param(name, normalize, mc, id=f"{name}-norm{int(normalize)}-mc{int(mc)}")


def clear_windows(m, x, normalize, mc):
    """The number of leading windows of x's separate_long whose alignment margins are all clear."""
    T = x.shape[-1]
    K = WO.plan(T, W, H)[0]
    if K == 1:
        return 1
    A = x.shape[0]
    wins = torch.from_numpy(WO.windows(x[None].cpu().numpy(), W, H)).to(DEV).reshape(K, A, W)
    est = m.separate(wins, mixture_consistency=mc, normalize=normalize).cpu().numpy()
    _, margin = WO.align(est.reshape(1, K, m.num_sources, A, W), T, W, H)
    close = np.nonzero(margin[0, 1:] <= 100 * SPREAD)[0]
    return K if close.size == 0 else 1 + int(close[0])


@pytest.mark.parametrize("name,normalize,mc", list(cases()))
def test_each_recording_is_separate_long_alone(name, normalize, mc):
    m = model(name)
    A = getattr(m, "in_audio_channels", 1)
    xs = [recording(A, T, 100 + i) for i, T in enumerate(LENGTHS)]
    bitwise = name == "causal"
    with torch.no_grad():
        for mw in (5, 32):
            outs, perms = windowed.separate_long_corpus(m, [x if A > 1 or i % 2 else x[0] for i, x in enumerate(xs)],
                                                        W, H, normalize=normalize, mixture_consistency=mc,
                                                        max_windows=mw, return_permutations=True)
            assert len(outs) == len(perms) == len(xs)
            for i, x in enumerate(xs):
                want, wperm = windowed.separate_long(m, x[None], W, H, normalize=normalize, mixture_consistency=mc,
                                                     return_permutations=True)
                got, T = outs[i], x.shape[-1]
                assert got.shape == (m.num_sources * A, T) and got.dtype == torch.float32, i
                if wperm is None:
                    assert perms[i] is None, i
                else:
                    assert perms[i].shape == wperm[0].shape and perms[i].dtype == torch.int32, i
                if bitwise:
                    assert torch.equal(got.view(torch.int32), want[0].view(torch.int32)), (mw, i)
                    assert wperm is None or torch.equal(perms[i], wperm[0]), (mw, i)
                    continue
                kc = clear_windows(m, x, normalize, mc)
                K = 1 if wperm is None else wperm.shape[1]
                if wperm is not None:
                    assert torch.equal(perms[i][:kc], wperm[0, :kc]), (mw, i)
                end = T if kc == K else kc * H
                scale = want[0].abs().max().clamp_min(1e-30)
                assert float((got[:, :end] - want[0, :, :end]).abs().max() / scale) <= 2 * SPREAD, (mw, i)


def test_surface_method_and_class_defaults():
    m = model("groupcomm")                      # GroupComm separates with mixture consistency by default
    xs = [recording(1, T, i)[0] for i, T in enumerate(LENGTHS[:4])]
    with torch.no_grad():
        got = m.separate_long_corpus(xs, W, H)
        want = windowed.separate_long_corpus(m, xs, W, H, mixture_consistency=True)
        off = windowed.separate_long_corpus(m, xs, W, H, mixture_consistency=False)
    for g, w, o in zip(got, want, off):
        assert float((g - w).abs().max() / w.abs().max()) <= 2 * SPREAD
    assert any(float((w - o).abs().max()) > 1e-3 for w, o in zip(want, off))
    c = model("causal")
    with torch.no_grad():
        outs, perms = c.separate_long_corpus(xs, W, H, return_permutations=True)
    assert perms[0] is not None and perms[1] is None and len(outs) == 4


def test_a_nonfinite_recording_leaves_the_others_bitwise():
    m = model("causal")
    xs = [recording(1, T, 200 + i) for i, T in enumerate(LENGTHS)]
    with torch.no_grad():
        clean = windowed.separate_long_corpus(m, xs, W, H, max_windows=4)
        for r, bad in ((0, float("nan")), (8, float("inf")), (6, 0.0)):
            ys = [x.clone() for x in xs]
            if bad == 0.0:                       # a silent stretch across overlap 2
                ys[r][:, 2 * H - 10:W + H + 10] = 0
            else:
                ys[r][0, 2 * H + 17] = bad
            got = windowed.separate_long_corpus(m, ys, W, H, max_windows=4)
            for i in range(len(xs)):
                if i != r:
                    assert torch.equal(got[i].view(torch.int32), clean[i].view(torch.int32)), (r, i)


def test_memory_is_set_by_the_window_batch():
    m = model("improved")
    gen = np.random.default_rng(1)
    corpora = {n: [recording(1, int(T), n + i)[0] for i, T in enumerate(gen.integers(5 * 8000, 30 * 8000, n))]
               for n in (10, 100)}
    peaks, sizes = {}, {}
    with torch.no_grad():
        windowed.separate_long_corpus(m, corpora[10], 32000, 16000, max_windows=8)    # workspace, allocator warm
        for n, xs in corpora.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            outs = windowed.separate_long_corpus(m, xs, 32000, 16000, max_windows=8)
            torch.cuda.synchronize()
            peaks[n] = torch.cuda.max_memory_allocated() - base
            sizes[n] = sum(x.numel() for x in xs)
            del outs
    # what grows with the corpus: the flat copy of its input and its output (S = 2)
    grows = (1 + 2) * 4 * (sizes[100] - sizes[10])
    assert peaks[100] - peaks[10] <= grows + (4 << 20), (peaks, grows)


def test_flat_output_past_2_31_elements():
    kw = dict(in_audio_channels=2, out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=3,
              enc_kernel_size=11, enc_num_basis=16, num_sources=4)
    sd = O.make_state_dict(O.Config(variant="causal", **kw), seed=4)
    m = P.CausalSuDORMRF(**kw)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    Wl, Hl = 1 << 22, 1 << 21
    S, A = 4, 2
    big = 1 << 28                                # S A big = 2^31: everything after it lies past 2^31 elements
    lengths = [big, Wl + Hl + 5, 3000, 3 * Wl + 11]
    xs = []
    for i, T in enumerate(lengths):
        g = torch.Generator(device=DEV).manual_seed(i)
        xs.append(torch.randn(A, T, generator=g, device=DEV))
    with torch.no_grad():
        outs, perms = windowed.separate_long_corpus(m, xs, Wl, Hl, normalize=False, max_windows=4,
                                                    return_permutations=True)
        assert all(bool(torch.isfinite(o).all()) for o in outs)
        for i in (1, 2, 3):
            want, wperm = windowed.separate_long(m, xs[i][None], Wl, Hl, normalize=False, return_permutations=True)
            assert torch.equal(outs[i].view(torch.int32), want[0].view(torch.int32)), i
            assert (wperm is None and perms[i] is None) or torch.equal(perms[i], wperm[0]), i
        out0 = outs[0]
    assert out0.shape == (S * A, big)


def test_side_stream_gives_the_default_streams_bits():
    m = model("causal")
    xs = [recording(1, T, 300 + i)[0] for i, T in enumerate(LENGTHS)]
    with torch.no_grad():
        want, wperm = windowed.separate_long_corpus(m, xs, W, H, max_windows=3, return_permutations=True)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            got, gperm = windowed.separate_long_corpus(m, xs, W, H, max_windows=3, return_permutations=True)
        torch.cuda.current_stream().wait_stream(side)
    for i in range(len(xs)):
        assert torch.equal(got[i].view(torch.int32), want[i].view(torch.int32)), i
        assert (wperm[i] is None and gperm[i] is None) or torch.equal(gperm[i], wperm[i]), i
