"""Windowed streams on the GPU (DESIGN.md section 7f).

Stage level: fed the same window estimates, the stream merge and flush are bitwise ``sdr_window_merge`` over the
whole input, permutations included.  Model level: ``cat(steps) + flush`` is ``separate_long`` on the concatenated
input (bitwise for the causal model, within the spread of the fp64-atomic forwards elsewhere), at n = H, W, W + H
and many windows; flush rules; resets; CUDA-graph capture; NaN containment and guarded buffers; weight updates and
stream hand-over; one hour through U16/512 with constant memory."""
import itertools

import ctypes as C
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


def ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None else None)


def cur():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------------------------
# 1. stage level
# ---------------------------------------------------------------------------------------------------------------------
def offline(est, T, W, H):
    """sdr_window_merge over est [B, K, S, A, W] in one batch: (out [B, S A, T], perm [B, K, S])."""
    B, K, S, A, _ = est.shape
    lib = N.lib()
    carry = torch.empty(lib.sdr_window_carry_bytes(B, S, A, W), dtype=torch.uint8, device=DEV)
    scratch = torch.empty(lib.sdr_window_merge_scratch_bytes(B, S, K), dtype=torch.uint8, device=DEV)
    out = torch.empty(B, S * A, T, device=DEV)
    perm = torch.empty(B, K, S, dtype=torch.int32, device=DEV)
    windowed.merge(est.reshape(B, K, S * A, W).contiguous(), carry, perm, out, S, A, W, H, 0, K, scratch)
    return out, perm


def staged(x, est, S, C_, W, H, pattern=0, check=False):
    """The stream's stages on chunks of x [B, A, N] with window k's estimate est[:, k] (zeros for k = -1): (steps
    [B, S A, N], flush [B, S A, H], the carry's pi after every step [steps, B, S])."""
    B, A, Ntot = x.shape
    q = C_ // H
    lib = N.lib()
    state = poisoned(lib.sdr_window_stream_state_bytes(B, S, A, W, H), pattern)
    scratch = poisoned(lib.sdr_window_stream_merge_scratch_bytes(B, S, C_, H), pattern)
    N.check(lib.sdr_window_stream_reset(ptr(state), B, S, A, W, H, None, 0, cur()), "reset")
    outs, pis = [], []
    zero = torch.zeros(B, 1, S * A, W, device=DEV)
    flat = est.reshape(B, est.shape[1], S * A, W)
    for j in range(Ntot // C_):
        n = j * C_
        chunk = x[..., n:n + C_].contiguous()
        batch = poisoned_like(torch.empty(B * q, A, W, device=DEV), pattern)
        if check:
            chunk = guarded_copy(chunk)
        N.check(lib.sdr_window_stream_gather(ptr(state), ptr(chunk), ptr(batch), B, S, A, C_, W, H, cur()), "gather")
        k0 = n // H - 1
        e = torch.cat(([zero] if k0 < 0 else []) + [flat[:, max(k0, 0):k0 + q]], dim=1).contiguous()
        out = poisoned_like(torch.empty(B, S * A, C_, device=DEV), pattern)
        if check:
            e = guarded_copy(e)
        N.check(lib.sdr_window_stream_merge(ptr(e), ptr(state), ptr(out), B, S, A, C_, W, H, ptr(scratch), cur()),
                "merge")
        if check:
            for t, what in ((chunk, "chunk"), (batch, "batch"), (e, "estimates"), (out, "out")):
                check_bands(t, what)
        outs.append(out.clone())
        pis.append(state[:B * S * 4].view(torch.int32).view(B, S).clone())
    n = Ntot
    single = torch.zeros(B, S * A, H, device=DEV)
    fest = flat[:, n // H - 1].contiguous() if W < 2 * H else None
    fscratch = poisoned(lib.sdr_window_stream_flush_scratch_bytes(B, S), pattern)
    tail = poisoned_like(torch.empty(B, S * A, H, device=DEV), pattern)
    before = state.clone()
    N.check(lib.sdr_window_stream_flush(ptr(single), ptr(fest), ptr(state), ptr(tail), B, S, A, W, H, ptr(fscratch),
                                        cur()), "flush")
    assert torch.equal(state, before), "the flush changed the state"
    if check:
        for t, what in ((state, "state"), (scratch, "scratch"), (fscratch, "flush scratch"), (tail, "tail")):
            check_bands(t, what)
    torch.cuda.synchronize()
    return torch.cat(outs, dim=-1), tail, torch.stack(pis)


STAGE_CASES = [(S, A, W, H, q) for (S, A), (W, H), q in itertools.product(
    [(1, 1), (2, 1), (3, 2), (4, 1)], [(64, 32), (96, 60), (101, 51), (77, 40)], [1, 2, 5])]


@pytest.mark.parametrize("S,A,W,H,q", STAGE_CASES)
def test_stages_are_the_offline_merge_bitwise(S, A, W, H, q):
    gen = np.random.default_rng(S * 1000 + A * 100 + W + q)
    B, C_ = 3, q * H
    steps = max(2, -(-12 * H // C_))
    Ntot = steps * C_
    K = WO.plan(Ntot, W, H)[0]
    # windows that share a slowly varying part with their neighbours, sources in random orders
    base = gen.standard_normal((B, S, A, Ntot)).astype(np.float32)
    win = WO.windows(base.reshape(B, S * A, Ntot), W, H).reshape(B, K, S, A, W)
    est = np.stack([np.stack([win[b, k][gen.permutation(S)] for k in range(K)]) for b in range(B)])
    est = torch.from_numpy((est + 0.5 * gen.standard_normal(est.shape)).astype(np.float32)).to(DEV)
    x = torch.from_numpy(gen.standard_normal((B, A, Ntot)).astype(np.float32)).to(DEV)
    want, perm = offline(est, Ntot, W, H)
    got, tail, pis = staged(x, est, S, C_, W, H)
    assert torch.equal(got[..., H:].view(torch.int32), want[..., :Ntot - H].view(torch.int32))
    assert not got[..., :H].any()
    assert torch.equal(tail.view(torch.int32), want[..., Ntot - H:].view(torch.int32))
    for j in range(steps):
        last = (j + 1) * q - 2                          # the last window step j completes (-1: none yet)
        if last >= 0:
            assert torch.equal(pis[j], perm[:, last]), j


@pytest.mark.parametrize("pattern", [POISON_NAN, POISON_HUGE])
def test_stages_on_poisoned_and_guarded_buffers(pattern):
    gen = np.random.default_rng(8)
    B, S, A, W, H, q = 2, 3, 2, 96, 60, 2
    Ntot = 8 * q * H
    K = WO.plan(Ntot, W, H)[0]
    est = torch.from_numpy(gen.standard_normal((B, K, S, A, W)).astype(np.float32)).to(DEV)
    x = torch.from_numpy(gen.standard_normal((B, A, Ntot)).astype(np.float32)).to(DEV)
    clean = staged(x, est, S, q * H, W, H)
    got = staged(x, est, S, q * H, W, H, pattern, check=True)
    for a, b in zip(got, clean):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_gather_windows_and_history():
    gen = np.random.default_rng(2)
    B, S, A, W, H, q = 2, 2, 2, 50, 30, 3
    C_ = q * H
    lib = N.lib()
    x = torch.from_numpy(gen.standard_normal((B, A, 4 * C_)).astype(np.float32)).to(DEV)
    state = torch.empty(lib.sdr_window_stream_state_bytes(B, S, A, W, H), dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_window_stream_reset(ptr(state), B, S, A, W, H, None, 0, cur()), "reset")
    wins = WO.windows(x.cpu().numpy(), W, H)
    est = torch.zeros(B, q, S * A, W, device=DEV)
    out = torch.empty(B, S * A, C_, device=DEV)
    scratch = torch.empty(lib.sdr_window_stream_merge_scratch_bytes(B, S, C_, H), dtype=torch.uint8, device=DEV)
    for j in range(4):
        batch = torch.full((B, q, A, W), 7.0, device=DEV)
        chunk = x[..., j * C_:(j + 1) * C_].contiguous()
        N.check(lib.sdr_window_stream_gather(ptr(state), ptr(chunk), ptr(batch), B, S, A, C_, W, H, cur()), "g")
        for m in range(q):
            k = j * q - 1 + m
            want = wins[:, k] if k >= 0 else np.zeros((B, A, W), np.float32)
            assert np.array_equal(batch[:, m].cpu().numpy(), want), (j, m)
        N.check(lib.sdr_window_stream_merge(ptr(est), ptr(state), ptr(out), B, S, A, C_, W, H, ptr(scratch), cur()),
                "m")
        fb = torch.full((B, A, W), 7.0, device=DEV)
        N.check(lib.sdr_window_stream_gather(ptr(state), None, ptr(fb), B, S, A, 0, W, H, cur()), "flush gather")
        n = (j + 1) * C_
        want = np.zeros((B, A, W), np.float32)
        want[..., :H] = x[..., n - H:n].cpu().numpy()
        assert np.array_equal(fb.cpu().numpy(), want), j


# ---------------------------------------------------------------------------------------------------------------------
# 2-3. model level and flush
# ---------------------------------------------------------------------------------------------------------------------
SMALL = dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64,
             num_sources=2)
MODELS = {
    "improved": (P.SuDORMRF, "improved", SMALL),
    "groupcomm": (P.GroupCommSudoRmRf, "groupcomm", dict(SMALL, group_size=4)),
    "causal": (P.CausalSuDORMRF, "causal", dict(SMALL, in_audio_channels=1)),
    "causal_stereo": (P.CausalSuDORMRF, "causal", dict(SMALL, in_audio_channels=2)),
    "original": (P.OriginalSuDORMRF, "original", SMALL),
}
_cache = {}


def model(name, seed=11):
    if (name, seed) not in _cache:
        cls, variant, kw = MODELS[name]
        sd = O.make_state_dict(O.Config(variant=variant, **kw), seed=seed)
        m = cls(**kw)
        m.load_state_dict(sd)
        _cache[name, seed] = m.to(DEV).eval()
    return _cache[name, seed]


def mixture(B, A, T, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64) / 8000.0
    tone = torch.sin(2 * np.pi * 220.0 * t) * torch.sin(2 * np.pi * 0.3 * t)
    x = 0.3 * torch.randn(B, A, T, generator=g, dtype=torch.float64) + tone
    return (x + 0.1).float().to(DEV)


def run_stream(st, x):
    C_ = st.chunk_samples
    return torch.cat([st.step(x[..., j:j + C_]) for j in range(0, x.shape[-1], C_)], dim=-1)


def clear_end(m, x, W, H, normalize, mc):
    """The first sample of x's windowed separation that a near-tie of the alignment may change (T when none)."""
    B, A, T = x.shape
    if T <= W:
        return T
    K = WO.plan(T, W, H)[0]
    batch = torch.from_numpy(WO.windows(x.cpu().numpy(), W, H)).to(DEV).reshape(B * K, A, W)
    est = m.separate(batch, mixture_consistency=mc, normalize=normalize).cpu().numpy()
    _, margin = WO.align(est.reshape(B, K, -1, A, W), T, W, H)
    close = np.nonzero((margin[:, 1:] <= MARGIN).any(axis=0))[0]
    return T if close.size == 0 else (1 + int(close[0])) * H


def agree(got, want, exact, end=None):
    end = want.shape[-1] if end is None else end
    if exact:
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    else:
        g, w = got[..., :end], want[..., :end]
        assert float((g - w).abs().max()) <= (MARGIN + SPREAD) * float(want.abs().max())


def cases():
    for name in ("causal", "improved", "groupcomm", "original"):
        for normalize, mc in itertools.product((True, False), (True, False)):
            yield pytest.param(name, normalize, mc, id=f"{name}-norm{int(normalize)}-mc{int(mc)}")
    yield pytest.param("causal_stereo", False, False, id="causal_stereo-norm0-mc0")


@pytest.mark.parametrize("W,H,q", [(4000, 2000, 1), (3000, 2000, 2)])
@pytest.mark.parametrize("name,normalize,mc", list(cases()))
def test_steps_and_flush_are_separate_long(name, normalize, mc, W, H, q):
    m = model(name)
    A = MODELS[name][2].get("in_audio_channels", 1)
    exact = name.startswith("causal")
    C_ = q * H
    x = mixture(2, A, 12 * H, 3)
    marks = {n for n in (H, W, W + H, 12 * H) if n % C_ == 0}
    with torch.no_grad():
        st = m.stream_windows(2, C_, W, H, normalize=normalize, mixture_consistency=mc)
        assert st.latency == H and st.batch_size == 2
        assert not st.flush().any()                         # no step since the reset: zeros
        outs = []
        for n in range(0, x.shape[-1], C_):
            outs.append(st.step(x[..., n:n + C_]))
            if n + C_ in marks:
                end = n + C_
                got = torch.cat(outs + [st.flush()], dim=-1)[..., H:]
                want = m.separate_long(x[..., :end], W, H, normalize=normalize, mixture_consistency=mc)
                lim = end if exact else clear_end(m, x[..., :end], W, H, normalize, mc)
                agree(got, want, exact, lim)


def test_flush_single_window_rules_and_an_idle_slot():
    """n = H is separated unpadded; n = W = 2H is window 0; a slot reset before the flush gives zeros."""
    m = model("causal")
    W, H = 4000, 2000
    x = mixture(3, 1, 2 * H, 9)
    with torch.no_grad():
        st = m.stream_windows(3, H, W, H)
        st.step(x[..., :H])
        assert torch.equal(st.flush(), m.separate(x[..., :H], normalize=True))
        st.step(x[..., H:])
        st.reset([1])
        tail = st.flush()
        want = m.separate(x, normalize=True)[..., H:]
        assert torch.equal(tail[[0, 2]], want[[0, 2]]) and not tail[1].any()


# ---------------------------------------------------------------------------------------------------------------------
# 4. reset
# ---------------------------------------------------------------------------------------------------------------------
def test_reset_starts_slots_over_and_leaves_the_others():
    m = model("causal")
    W, H, q = 3000, 2000, 2
    C_ = q * H
    x = mixture(4, 1, 10 * C_, 4)
    with torch.no_grad():
        ref = run_stream(m.stream_windows(4, C_, W, H), x)
        st = m.stream_windows(4, C_, W, H)
        a = run_stream(st, x[..., :4 * C_])
        st.reset([1, 3])
        b = run_stream(st, x[..., 4 * C_:])
        got = torch.cat([a, b], dim=-1)
        assert torch.equal(got[[0, 2]], ref[[0, 2]])
        for s in (1, 3):
            fresh = run_stream(m.stream_windows(1, C_, W, H), x[s:s + 1, :, 4 * C_:])
            assert torch.equal(b[s:s + 1], fresh), s


# ---------------------------------------------------------------------------------------------------------------------
# 5. capture
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["causal", "improved"])
def test_captured_step_is_the_eager_step(name):
    m = model(name)
    W, H = 4000, 2000
    B, C_, steps = 3, 2 * H, 30
    x = mixture(B, 1, steps * C_, 12)
    with torch.no_grad():
        st = m.stream_windows(B, C_, W, H, normalize=False)
        eager = run_stream(st, x)
        st.reset()
        chunk = torch.empty(B, 1, C_, device=DEV)
        out = torch.empty(B, 2, C_, device=DEV)
        chunk.copy_(x[..., :C_])
        st.step(chunk, out=out)                              # warms the workspace and the packed weights
        first = out.clone()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            st.step(chunk, out=out)
        got = [first]
        for j in range(1, steps):
            chunk.copy_(x[..., j * C_:(j + 1) * C_])
            g.replay()
            got.append(out.clone())
        torch.cuda.synchronize()
    got = torch.cat(got, dim=-1)
    if name == "causal":
        assert torch.equal(got.view(torch.int32), eager.view(torch.int32))
    else:
        with torch.no_grad():
            end = clear_end(m, x, W, H, False, False)
        agree(got[..., H:], eager[..., H:], False, end - H)


# ---------------------------------------------------------------------------------------------------------------------
# 6. contained bad values
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_a_bad_value_stays_in_its_slot(bad):
    m = model("causal")
    W, H = 3000, 2000
    C_ = 2 * H
    x = mixture(3, 1, 8 * C_, 6)
    y = x.clone()
    y[1, 0, 3 * C_ + 17] = bad
    with torch.no_grad():
        clean = run_stream(m.stream_windows(3, C_, W, H), x)
        got = run_stream(m.stream_windows(3, C_, W, H), y)
    assert torch.equal(got[[0, 2]].view(torch.int32), clean[[0, 2]].view(torch.int32))
    assert not torch.isfinite(got[1]).all()


@pytest.mark.parametrize("pattern", [POISON_NAN, POISON_HUGE])
def test_poisoned_outputs_and_guarded_chunks(pattern):
    m = model("causal")
    W, H = 3000, 2000
    C_ = 2 * H
    x = mixture(2, 1, 6 * C_, 8)
    with torch.no_grad():
        want = run_stream(m.stream_windows(2, C_, W, H), x)
        st = m.stream_windows(2, C_, W, H)
        outs = []
        for j in range(6):
            chunk = guarded_copy(x[..., j * C_:(j + 1) * C_].contiguous())
            before = chunk.clone()
            out = poisoned_like(torch.empty(2, 2, C_, device=DEV), pattern)
            st.step(chunk, out=out)
            check_bands(chunk, "chunk")
            check_bands(out, "out")
            assert torch.equal(chunk, before)
            outs.append(out.clone())
    assert torch.equal(torch.cat(outs, dim=-1), want)


def test_step_refusals():
    m = model("causal")
    with torch.no_grad():
        st = m.stream_windows(2, 2000, 4000, 2000)
        with pytest.raises(RuntimeError, match="CUDA"):
            st.step(torch.zeros(2, 1, 2000))
        with pytest.raises(RuntimeError, match="shape"):
            st.step(torch.zeros(2, 1, 4000, device=DEV))
        with pytest.raises(RuntimeError, match="out must be"):
            st.step(torch.zeros(2, 1, 2000, device=DEV), out=torch.empty(2, 2, 1999, device=DEV))
    with pytest.raises(RuntimeError, match="requires grad"):
        st.step(torch.zeros(2, 1, 2000, device=DEV, requires_grad=True))
    with pytest.raises(IndexError):
        st.reset([2])


# ---------------------------------------------------------------------------------------------------------------------
# 7. weights and CUDA streams
# ---------------------------------------------------------------------------------------------------------------------
def test_weights_changed_between_steps_are_used_by_the_next():
    W, H = 4000, 2000
    cls, variant, kw = MODELS["causal"]
    sd1 = O.make_state_dict(O.Config(variant=variant, **kw), seed=21)
    sd2 = O.make_state_dict(O.Config(variant=variant, **kw), seed=22)
    m = cls(**kw)
    m.load_state_dict(sd1)
    m = m.to(DEV).eval()
    m2 = cls(**kw)
    m2.load_state_dict(sd2)
    m2 = m2.to(DEV).eval()
    x = mixture(2, 1, 10 * H, 13)
    with torch.no_grad():
        st = m.stream_windows(2, H, W, H)
        run_stream(st, x[..., :5 * H])
        other = m2.stream_windows(2, H, W, H)
        other._state.copy_(st._state)
        m.load_state_dict(sd2)                              # in place: the packed weights are stale from here on
        got = run_stream(st, x[..., 5 * H:])
        want = run_stream(other, x[..., 5 * H:])
        assert torch.equal(got, want)
        st.reset()
        assert torch.equal(run_stream(st, x), run_stream(m2.stream_windows(2, H, W, H), x))


def test_steps_alternating_between_cuda_streams():
    m = model("causal")
    W, H = 3000, 2000
    C_ = 2 * H
    x = mixture(2, 1, 12 * C_, 14)
    with torch.no_grad():
        want = run_stream(m.stream_windows(2, C_, W, H), x)
        st = m.stream_windows(2, C_, W, H)
        sides = [torch.cuda.Stream(), torch.cuda.Stream()]
        for s in sides:
            s.wait_stream(torch.cuda.current_stream())
        outs = []
        for j in range(12):
            with torch.cuda.stream(sides[j % 2]):
                if j == 6:
                    st.reset([1])                           # slot 1 starts over on chunk 6
                outs.append(st.step(x[..., j * C_:(j + 1) * C_]))
        with torch.cuda.stream(sides[0]):
            tail = st.flush()
        for s in sides:
            torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        got = torch.cat(outs, dim=-1)
        assert torch.equal(got[0], want[0])
        assert torch.equal(got[1, :, :6 * C_], want[1, :, :6 * C_])
        fresh = m.stream_windows(1, C_, W, H)
        assert torch.equal(got[1:, :, 6 * C_:], run_stream(fresh, x[1:, :, 6 * C_:]))
        assert torch.equal(tail[1:], fresh.flush())


# ---------------------------------------------------------------------------------------------------------------------
# 8. one hour through U16/512
# ---------------------------------------------------------------------------------------------------------------------
def test_one_hour_at_8k_through_u16_512():
    kw = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5, enc_kernel_size=21,
              enc_num_basis=512, num_sources=2)
    m = P.SuDORMRF(**kw)
    m.load_state_dict(O.make_state_dict(O.Config(variant="improved", **kw), seed=3))
    m = m.to(DEV).eval()
    fs, W, H = 8000, 32000, 16000
    T = 3600 * fs
    steps = T // H
    x = mixture(1, 1, T, 15)
    out = torch.empty(steps, 1, 2, H, device=DEV)
    with torch.no_grad():
        st = m.stream_windows(1, H, W, H)
        st.step(x[..., :H], out=out[0])
        st.step(x[..., H:2 * H], out=out[1])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.max_memory_allocated()
        for j in range(2, steps):
            st.step(x[..., j * H:(j + 1) * H], out=out[j])
            if j == 100:
                torch.cuda.synchronize()
                early = torch.cuda.max_memory_allocated()
        torch.cuda.synchronize()
        late = torch.cuda.max_memory_allocated()
        tail = st.flush()
        got = torch.cat([out.permute(1, 2, 0, 3).reshape(1, 2, T), tail], dim=-1)[..., H:]
        want, perm = windowed.separate_long(m, x, W, H, return_permutations=True)
        K = perm.shape[1]
        wins = torch.from_numpy(WO.windows(x.cpu().numpy(), W, H)).to(DEV).reshape(K, 1, W)
        est = torch.cat([m.separate(wins[k:k + 32], normalize=True) for k in range(0, K, 32)])
    assert late == early, (base, early, late)
    _, margin = WO.align(est.cpu().numpy().reshape(1, K, 2, 1, W), T, W, H)
    close = np.nonzero(margin[0, 1:] <= MARGIN)[0]
    end = T if close.size == 0 else (1 + int(close[0])) * H
    print(f"one hour: clear up to {end / fs:.0f} s of {T / fs:.0f} s")
    agree(got, want, False, end)
