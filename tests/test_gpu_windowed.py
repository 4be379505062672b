"""Windowed separation on the GPU (DESIGN.md section 7e).

Stage entries on synthetic estimates: windows holding the true sources in a random order come back as the sources;
the permutations and the output are bitwise independent of the batch size; a silent or non-finite overlap keeps the
previous order and stays in its recording; every source and channel count; poisoned and guarded buffers.
Whole calls: a clip that fits one window is ``separate``; longer clips match the fp64 oracle's alignment and the fp32
cross-fade of the same window estimates, for every model variant; memory does not grow with the length; a clip the
whole-clip forward refuses runs."""
import itertools
import threading

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


def run_merge(est, T, W, H, M, pattern=0, check=False):
    """Merges est [B, K, S, A, W] (device) in batches of M windows; (out [B, S A, T], perm [B, K, S])."""
    B, K, S, A, _ = est.shape
    lib = N.lib()
    carry = poisoned(lib.sdr_window_carry_bytes(B, S, A, W), pattern)
    scratch = poisoned(lib.sdr_window_merge_scratch_bytes(B, S, M), pattern)
    out = poisoned_like(torch.empty(B, S * A, T, device=DEV), pattern)
    perm = poisoned_like(torch.empty(B, K, S, dtype=torch.int32, device=DEV), pattern)
    for k0 in range(0, K, M):
        m = min(M, K - k0)
        chunk = est[:, k0:k0 + m].reshape(B, m, S * A, W).contiguous()
        if check:
            chunk = guarded_copy(chunk)
            before = chunk.clone()
        sc = scratch if m == M else poisoned(lib.sdr_window_merge_scratch_bytes(B, S, m), pattern)
        windowed.merge(chunk, carry, perm, out, S, A, W, H, k0, m, sc)
        if check:
            check_bands(chunk, "estimates")
            check_bands(sc, "scratch")
            assert torch.equal(chunk, before), "the estimates were modified"
    if check:
        for t, what in ((carry, "carry"), (scratch, "scratch"), (out, "out"), (perm, "perm")):
            check_bands(t, what)
    torch.cuda.synchronize()
    return out, perm


def permuted_windows(src, W, H, gen):
    """src [B, S, A, T] -> (est [B, K, S, A, W] with every window's sources in a random order, orders [B, K, S])."""
    B, S, A, T = src.shape
    K = WO.plan(T, W, H)[0]
    win = WO.windows(src.reshape(B, S * A, T), W, H).reshape(B, K, S, A, W)
    orders = np.array([[gen.permutation(S) for _ in range(K)] for _ in range(B)])
    est = np.stack([np.stack([win[b, k][orders[b, k]] for k in range(K)]) for b in range(B)])
    return est, orders          # est[b, k][q] is true source orders[b, k][q]


@pytest.mark.parametrize("S", [1, 2, 3, 4])
@pytest.mark.parametrize("A", [1, 2])
def test_merge_recovers_permuted_sources(S, A):
    gen = np.random.default_rng(10 * S + A)
    B, W, H = 3, 96, 60
    T = W + 9 * H + 7
    src = gen.standard_normal((B, S, A, T)).astype(np.float32)
    est, orders = permuted_windows(src, W, H, gen)
    K = est.shape[1]
    out, perm = run_merge(torch.from_numpy(est).to(DEV), T, W, H, K)
    out, perm = out.cpu().numpy(), perm.cpu().numpy()
    for b in range(B):
        for k in range(K):
            # output source s of window k is the true source output s of window 0 is
            assert np.array_equal(orders[b, k][perm[b, k]], orders[b, 0]), (b, k)
    want = src[np.arange(B)[:, None], orders[:, 0]].reshape(B, S * A, T)
    assert np.allclose(out, want, rtol=1e-6, atol=1e-6)
    assert np.array_equal(out, WO.overlap_add(est, perm.astype(np.int64), T, W, H))


@pytest.mark.parametrize("S,A", [(2, 1), (3, 2), (4, 1)])
def test_merge_bitwise_independent_of_batch_size(S, A):
    gen = np.random.default_rng(S * 7 + A)
    B, W, H = 2, 200, 130
    T = W + 11 * H + 1
    K = WO.plan(T, W, H)[0]
    # estimates that share a slowly varying part with their neighbours: the scores have a clear winner
    base = gen.standard_normal((B, S, A, T)).astype(np.float32)
    est, _ = permuted_windows(base, W, H, gen)
    est = (est + 0.5 * gen.standard_normal(est.shape)).astype(np.float32)
    dev = torch.from_numpy(est).to(DEV)
    ref_out, ref_perm = run_merge(dev, T, W, H, K)
    for M in (1, 2, K - 1, K + 1):
        out, perm = run_merge(dev, T, W, H, min(M, K))
        assert torch.equal(perm, ref_perm), M
        assert torch.equal(out.view(torch.int32), ref_out.view(torch.int32)), M
    pi, margin = WO.align(est, T, W, H)
    clear = margin > MARGIN
    assert clear[:, 1:].all()
    assert np.array_equal(ref_perm.cpu().numpy(), pi)
    assert np.array_equal(ref_out.cpu().numpy(), WO.overlap_add(est, pi, T, W, H))


def test_silent_and_nonfinite_overlaps_keep_the_order_and_their_recording():
    gen = np.random.default_rng(3)
    B, S, A, W, H = 3, 3, 1, 64, 40
    T = W + 6 * H
    src = gen.standard_normal((B, S, A, T)).astype(np.float32)
    clean, _ = permuted_windows(src, W, H, gen)
    est = clean.copy()
    est[0, 1, :, :, H:] = 0          # overlap 2 silent in both windows: C_2 = 0, rho_2 = id
    est[0, 2, :, :, :W - H] = 0
    est[1, 3, 1, 0, 5] = np.nan      # NaN in overlap 3: rho_3 = id
    est[1, 4, 2, 0, W - 1] = np.inf  # inf in overlap 5 (window 4's tail): rho_5 = id
    out, perm = run_merge(torch.from_numpy(est).to(DEV), T, W, H, 2)
    perm = perm.cpu().numpy()
    assert np.array_equal(perm[0, 2], perm[0, 1])
    assert np.array_equal(perm[1, 3], perm[1, 2])
    assert np.array_equal(perm[1, 5], perm[1, 4])
    # the oracle agrees on every window, and recording 2 is bitwise the clean run's
    pi, _ = WO.align(est, T, W, H)
    assert np.array_equal(perm, pi)
    clean_out, clean_perm = run_merge(torch.from_numpy(clean).to(DEV), T, W, H, 2)
    assert np.array_equal(clean_perm[2].cpu().numpy(), perm[2])
    assert torch.equal(out[2].view(torch.int32), clean_out[2].view(torch.int32))
    o = out.cpu().numpy()
    assert np.isfinite(o[0]).all() and np.isfinite(o[2]).all()


@pytest.mark.parametrize("S,A", [(2, 1), (4, 2)])
def test_entries_on_poisoned_and_guarded_buffers(S, A):
    gen = np.random.default_rng(5)
    B, W, H = 2, 128, 80
    T = W + 7 * H + 3
    K = WO.plan(T, W, H)[0]
    x = torch.from_numpy(gen.standard_normal((B, A, T)).astype(np.float32)).to(DEV)
    want = WO.windows(x.cpu().numpy(), W, H)
    for pattern in (0, POISON_NAN, POISON_HUGE):
        xg = guarded_copy(x)
        for k0, m in ((0, K), (0, 1), (2, 3), (K - 2, 2)):
            batch = poisoned_like(torch.empty(B * m, A, W, device=DEV), pattern)
            windowed.gather(xg, batch, W, H, k0, m)
            check_bands(batch, "batch")
            assert np.array_equal(batch.cpu().numpy().reshape(B, m, A, W), want[:, k0:k0 + m])
        check_bands(xg, "mixture")
        assert torch.equal(xg, x)
    est = gen.standard_normal((B, K, S, A, W)).astype(np.float32)
    dev = torch.from_numpy(est).to(DEV)
    clean = run_merge(dev, T, W, H, 3, 0, check=True)
    for pattern in (POISON_NAN, POISON_HUGE):
        got = run_merge(dev, T, W, H, 3, pattern, check=True)
        assert torch.equal(got[1], clean[1]), pattern
        assert torch.equal(got[0].view(torch.int32), clean[0].view(torch.int32)), pattern


def test_merge_refusals():
    lib = N.lib()
    est = torch.zeros(1, 2, 5, 1, 16, device=DEV)
    carry = torch.empty(1 << 16, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(1024, dtype=torch.uint8, device=DEV)
    out = torch.empty(1, 5, 30, device=DEV)
    with pytest.raises(N.NativeError, match="not implemented|unsupported|SDR|code -5"):
        windowed.merge(est, carry, None, out, 5, 1, 16, 8, 0, 2, scratch)
    with pytest.raises(N.NativeError):                      # k0 + M past K
        windowed.merge(est, carry, None, out, 2, 1, 16, 8, 2, 2, scratch)
    with pytest.raises(N.NativeError):                      # misaligned carry
        windowed.merge(est, carry[8:], None, out, 2, 1, 16, 8, 0, 2, scratch)
    assert lib.sdr_window_carry_bytes(1, 5, 1, 16) == 0


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


def mixture(B, A, T, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64) / 8000.0
    tone = torch.sin(2 * np.pi * 220.0 * t) * torch.sin(2 * np.pi * 0.3 * t)
    x = 0.3 * torch.randn(B, A, T, generator=g, dtype=torch.float64) + tone
    return (x + 0.1).float().to(DEV)


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def cases():
    for name in MODELS:
        mono = MODELS[name][1].get("in_audio_channels", 1) == 1
        for normalize, mc in itertools.product((True, False), (True, False)):
            if mono or not (normalize or mc):
                yield pytest.param(name, normalize, mc, id=f"{name}-norm{int(normalize)}-mc{int(mc)}")


@pytest.mark.parametrize("name,normalize,mc", list(cases()))
def test_single_window_is_separate(name, normalize, mc):
    m = model(name)
    A = m.in_audio_channels if hasattr(m, "in_audio_channels") else 1
    W = 4000
    bitwise = name == "causal"
    with torch.no_grad():
        for T in (W - 1, W, 1000):
            x = mixture(2, A, T, T)
            got = m.separate_long(x, W, normalize=normalize, mixture_consistency=mc)
            ref = m.separate(x, mixture_consistency=mc, normalize=normalize)
            assert got.shape == ref.shape and got.dtype == torch.float32
            if bitwise:
                assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), T
            else:
                assert rel(got, ref) <= SPREAD, T
        if A == 1 and normalize:
            x = mixture(2, 1, W, 5)[:, 0]                 # [B, T] as separate() takes it
            got = m.separate_long(x, W, normalize=True, mixture_consistency=mc)
            assert got.shape == (2, m.num_sources, W)


@pytest.mark.parametrize("name,normalize,mc", list(cases()))
def test_windows_match_the_oracle(name, normalize, mc):
    m = model(name)
    A = m.in_audio_channels if hasattr(m, "in_audio_channels") else 1
    S = m.num_sources
    B, W, H = 2, 4000, 2500
    T = W + 5 * H + 123
    K = WO.plan(T, W, H)[0]
    x = mixture(B, A, T, 7)
    with torch.no_grad():
        out, perm = windowed.separate_long(m, x, W, H, normalize=normalize, mixture_consistency=mc,
                                           max_windows=K + 3, return_permutations=True)
        batch = torch.from_numpy(WO.windows(x.cpu().numpy(), W, H)).to(DEV).reshape(B * K, A, W)
        est = m.separate(batch, mixture_consistency=mc, normalize=normalize)
        again = m.separate(batch, mixture_consistency=mc, normalize=normalize)
    spread = rel(again, est)
    assert spread == 0.0 if name == "causal" else spread <= SPREAD
    est = est.cpu().numpy().reshape(B, K, S, A, W)
    pi, margin = WO.align(est, T, W, H)
    want = WO.overlap_add(est, pi, T, W, H)
    got, perm = out.cpu().numpy(), perm.cpu().numpy()
    scale = np.abs(want).max()
    for b in range(B):
        close = np.nonzero(margin[b, 1:] <= MARGIN)[0]
        kbad = K if close.size == 0 else 1 + int(close[0])
        assert np.array_equal(perm[b, :kbad], pi[b, :kbad]), b
        end = T if kbad == K else kbad * H
        assert np.abs(got[b, :, :end] - want[b, :, :end]).max() <= (MARGIN + spread) * scale, b


def test_memory_is_set_by_the_window_batch():
    m = model("improved")
    W, mw = 16000, 4
    xs = {T: mixture(1, 1, T, T % 1000) for T in (2_000_000, 8_000_000)}
    peaks = {}
    with torch.no_grad():
        m.separate_long(xs[2_000_000], W, max_windows=mw)       # workspace, kernels, allocator warm
        for T, x in xs.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            out = m.separate_long(x, W, max_windows=mw)
            torch.cuda.synchronize()
            peaks[T] = torch.cuda.max_memory_allocated()
            del out
    larger_out = 8_000_000 * m.num_sources * 4
    assert abs(peaks[8_000_000] - peaks[2_000_000]) <= larger_out + (1 << 20), peaks


def test_past_the_whole_clip_limit():
    kw = dict(out_channels=64, in_channels=128, num_blocks=1, upsampling_depth=4, enc_kernel_size=21,
              enc_num_basis=4096, num_sources=2)
    sd = O.make_state_dict(O.Config(variant="improved", **kw), seed=2)
    m = P.SuDORMRF(**kw)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    B, T, W, H, mw = 1, 6_000_000, 32000, 16000, 16
    x = mixture(B, 1, T, 9)
    with torch.no_grad():
        with pytest.raises(N.NativeError):
            m(x)
        out, perm = windowed.separate_long(m, x, W, H, normalize=False, max_windows=mw, return_permutations=True)
        K = WO.plan(T, W, H)[0]
        wins = torch.from_numpy(WO.windows(x.cpu().numpy(), W, H)).to(DEV)
        # the driver's batches, so that every window estimate comes from the same forward shape
        est = torch.cat([m(wins[:, k0:k0 + mw].reshape(-1, 1, W)) for k0 in range(0, K, mw)])
    est = est.cpu().numpy().reshape(B, K, 2, 1, W)
    pi, margin = WO.align(est, T, W, H)
    want = WO.overlap_add(est, pi, T, W, H)
    got = out.cpu().numpy()
    assert np.isfinite(got).all()
    clear = margin[0, 1:] > MARGIN
    assert np.array_equal(perm.cpu().numpy()[0, 1:][clear], pi[0, 1:][clear])
    if clear.all():
        assert np.abs(got - want).max() <= (MARGIN + SPREAD) * np.abs(want).max()


def test_side_streams_and_threads():
    """Calls on a side stream and from two host threads sharing the model give the default stream's result."""
    m = model("causal")                 # no atomics in the forward: every run is bitwise the same
    W, H = 4000, 2000
    xs = [mixture(2, 1, W + 9 * H + 11, 20 + i) for i in range(2)]
    with torch.no_grad():
        want = [m.separate_long(x, W, H, max_windows=3) for x in xs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            got = m.separate_long(xs[0], W, H, max_windows=3)
        torch.cuda.current_stream().wait_stream(side)
        assert torch.equal(got, want[0])
    results, errs = {}, []

    def worker(i):
        try:
            st = torch.cuda.Stream()
            with torch.no_grad(), torch.cuda.stream(st):
                for _ in range(3):
                    r = m.separate_long(xs[i], W, H, max_windows=3)
                st.synchronize()
                results[i] = r
        except Exception as e:          # noqa: BLE001  (reported below)
            errs.append(e)
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(120)
    assert not errs, errs
    for i in range(2):
        assert torch.equal(results[i], want[i]), i
