"""BSS-eval on the GPU across its whole input space, against fp64: every source count with and without the mixture
and with either assignment, every filter length edge (warp edges, the solve CTA's 256-thread boundary, F = 2), the
correlation and energy chunk edges up to 30 s items, near-degenerate references (windowed tones, DC, AR(0.999),
band-limited noise with silent ends, one source 80 dB below another, amplitudes 1e-30 and 1e30, fp32 denormals),
poisoned and guarded workspaces through the C-ABI, non-finite inputs, batches past 65535 items and 2^31 elements,
and graph replay.

On white and AR references the oracle is bss_eval, the normal equations as mir_eval solves them.  On
near-degenerate references the normal equations' condition number reaches 1e15 and np.linalg.solve, and so mir_eval,
is off by dB; there the oracle is QR (bss_eval_span).  Where the GPU's recursion drops delayed references
(kept_delays), its values are those of its own fp64 restatement (bss_eval_recursion) within the usual bands, and
within SPAN_TOL of QR onto the kept delays: the generalised inverses let a little of the dropped directions into
the predictors, so the recursion is not exactly that projection.  What the SIR then measures depends on where the cut
falls (how many delays of a tone survive); these tests pin the cut to the restated rule and check that SDR <= SIR and
SDR <= SAR, which hold wherever it falls."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.signal import butter, lfilter, sosfilt

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from bss_oracle import (PROJECTION_DEFECT, bss_eval, bss_eval_mixture, bss_eval_recursion, bss_eval_span, kept_delays,
                        recursion_defect, span_defect)
from guards import POISON_HUGE, POISON_NAN, Guards, check_bands, poisoned
from test_gpu_bss_eval import DEV, check_values, make_item, run

pytestmark = pytest.mark.gpu
GiB = 1 << 30
# where the recursion drops delays: dB, GPU against its fp64 restatement (worst seen 8.3e-3 on an H100: the pivots
# next to the tolerance differ in rounding) and against QR onto the kept delays (worst seen 0.029)
RECURSION_TOL = 0.02
SPAN_TOL = 0.05
WORST = {}                  # "kind band" -> (largest |GPU - oracle| in dB, where)


@pytest.fixture(autouse=True)
def device_memory():
    """Frees the cached blocks after each test: the 2^31-element case needs most of the device."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def compare(kind, got, want, label, amp_db=None):
    """check_values, and the worst error per band recorded under `kind`."""
    check_values(got, want, label, amp_db)
    g, w = np.asarray(got, np.float64), np.asarray(want, np.float64)
    ok = np.isfinite(g) & np.isfinite(w)
    for band, sel in (("< -20 dB", w < -20), ("[-20, 60] dB", (w >= -20) & (w <= 60)),
                      ("(60, 120] dB", (w > 60) & (w <= 120))):
        m = ok & sel
        if m.any():
            err = float(np.max(np.abs(g - w)[m]))
            if err > WORST.get(f"{kind} {band}", (-1.0, ""))[0]:
                WORST[f"{kind} {band}"] = (err, label)


def check(got, refs, ests, perm, F, kind, label, oracle):
    """The permutation where the oracle's best mean SIR wins by more than 1e-3 dB below 120 dB, and the three
    criteria wherever the permutations agree.  -> the oracle's (sdr, sir, sar, perm)."""
    r64, e64 = refs.astype(np.float64), ests.astype(np.float64)
    sdr, sir, sar, p, gap = oracle(r64, e64, perm, F, margin=True)
    if gap > 1e-3 and np.mean(sir) <= 120:
        assert np.array_equal(got[3], p), (label, got[3], p)
    if np.array_equal(got[3], p):
        for g, w, name in zip(got[:3], (sdr, sir, sar), ("sdr", "sir", "sar")):
            compare(kind, g, w, f"{label} {name}", sdr if name == "sir" else None)
    return sdr, sir, sar, p


def batch(rng, S, T, F, B):
    items = [make_item(rng, S, T, F, coloured=(b % 2 == 1)) for b in range(B)]
    return np.stack([i[0] for i in items]), np.stack([i[1] for i in items])


def mixture_of(rng, refs):
    return (refs.sum(-2) + 0.01 * rng.standard_normal(refs.shape[:-2] + refs.shape[-1:])).astype(np.float32)


def item_slice(out, b):
    return [o[b] for o in out]


# ---------------------------------------------------------------------------------------------------------------------
# source counts x mixture x assignment
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("perm", [True, False], ids=["perm", "fixed"])
@pytest.mark.parametrize("mixture", [False, True], ids=["plain", "mixture"])
@pytest.mark.parametrize("S", [1, 2, 3, 4])
def test_sources_mixture_assignment(S, mixture, perm):
    """Every instantiation bss_eval_launch<S, S> and <S, S + 1> at F = 512; with the mixture, its scores and the
    improvements against the oracle, and the estimates' scores bitwise those of the call without it.  S = 4 with the
    mixture is the largest solve footprint (208 KiB of dynamic shared memory)."""
    F, T = 512, 6000
    B = 3 if S == 4 and mixture else 2
    rng = np.random.default_rng(100 * S + 10 * mixture + perm)
    refs, ests = batch(rng, S, T, F, B)
    if not mixture:
        got = run(refs, ests, perm, F)
        for b in range(B):
            check(item_slice(got, b), refs[b], ests[b], perm, F, "sources", f"S{S} perm{perm} item {b}", bss_eval)
        return
    mix = mixture_of(rng, refs)
    got = run(refs, ests, perm, F, mixture=torch.from_numpy(mix).to(DEV))
    plain = run(refs, ests, perm, F)
    for a, b in zip(got[:4], plain):
        assert np.array_equal(a, b, equal_nan=True)
    extra = got[4]
    for b in range(B):
        o = check(item_slice(got[:4], b), refs[b], ests[b], perm, F, "sources", f"S{S} mixture item {b}", bss_eval)
        m = bss_eval_mixture(refs[b].astype(np.float64), mix[b].astype(np.float64), F)
        for k, name in enumerate(("sdr", "sir", "sar")):
            compare("mixture", extra[name][b], m[k], f"S{S} mixture {name} item {b}", m[0] if k == 1 else None)
            if np.array_equal(got[3][b], o[3]):
                d = o[k] - m[k]
                ok = np.isfinite(d) & (np.abs(o[k]) <= 60) & (np.abs(m[k]) <= 60)
                err = np.abs(extra[name + "i"][b] - d)[ok]
                assert np.all(err <= 2e-3), (S, name, extra[name + "i"][b], d)


# ---------------------------------------------------------------------------------------------------------------------
# filter lengths
# ---------------------------------------------------------------------------------------------------------------------
FS = [1, 2, 31, 33, 255, 256, 257, 511, 512]


@pytest.mark.parametrize("shortest", [True, False], ids=["shortest", "T4000"])
@pytest.mark.parametrize("S", [2, 4])
@pytest.mark.parametrize("F", FS)
def test_filter_lengths(F, S, shortest):
    """Warp edges (31, 33), the solve CTA's 256 threads (257 and 511: a thread owns two lags), F = 1 and 2, at the
    shortest item allowed, (S - 1) F + 1 samples, where the delays fill all but F - 1 of the dimensions, and at 4000."""
    T = (S - 1) * F + 1 if shortest else 4000
    rng = np.random.default_rng(1000 * F + 10 * S + shortest)
    refs, ests = batch(rng, S, T, F, 2)
    got = run(refs, ests, True, F)
    for b in range(2):
        check(item_slice(got, b), refs[b], ests[b], True, F, "filter lengths", f"F{F} S{S} T{T} item {b}", bss_eval)


# ---------------------------------------------------------------------------------------------------------------------
# lengths: chunk edges, the 16-chunk clamp, whole utterances
# ---------------------------------------------------------------------------------------------------------------------
# correlation chunks ceil(T / 4096) and energy chunks ceil((T + F - 1) / 4096), both clamped to 1..16: 4096k - F + 1
# and + 2 change the energy chunks alone; 61440 / 61441 reach the clamp
LENGTHS = [(2, 4095, 512), (2, 4096, 512), (2, 4097, 512), (3, 4097, 33), (2, 7681, 512), (2, 7682, 512),
           (4, 7681, 512), (4, 7682, 512), (2, 4096 * 15 - 511, 512), (2, 4096 * 15 - 510, 512), (2, 61440, 512),
           (2, 61441, 512), (3, 61441, 256), (1, 61441, 1), (2, 160000, 512), (4, 160000, 512), (2, 480000, 512)]


@pytest.mark.parametrize("S,T,F", LENGTHS)
def test_length_edges(S, T, F):
    rng = np.random.default_rng(T + 7 * S + F)
    B = 1 if T > 100000 else 2
    refs, ests = batch(rng, S, T, F, B)
    got = run(refs, ests, True, F)
    for b in range(B):
        check(item_slice(got, b), refs[b], ests[b], True, F, "lengths", f"S{S} T{T} F{F} item {b}", bss_eval)
    if T > 100000:                                      # zero padded by 1000 and next to another item: equal values
        pad = np.zeros((1, S, 1000), np.float32)
        other = lambda: rng.standard_normal((1, S, T + 1000)).astype(np.float32)      # noqa: E731
        refs2 = np.concatenate([np.concatenate([refs, pad], 2), other()])
        ests2 = np.concatenate([np.concatenate([ests, pad], 2), other()])
        padded = run(refs2, ests2, True, F)
        for a, p in zip(got[:3], padded[:3]):
            assert np.all(np.abs(a[0] - p[0]) <= 1e-6), (a[0], p[0])
        assert np.array_equal(got[3][0], padded[3][0])


@pytest.mark.parametrize("T", [4097, 61441, 160001])
def test_error_in_the_last_sample(T):
    """F = 1 and an estimate that equals its reference but in its last sample: the whole of |e - P e|^2 sits in the
    last energy chunk's last sample, which every chunk split here leaves over (T mod chunks = 1)."""
    rng = np.random.default_rng(T)
    refs = rng.standard_normal((1, 2, T)).astype(np.float32)
    ests = refs[:, ::-1].copy()
    ests[0, :, -1] += 0.05
    got = run(refs, ests, True, 1)
    assert np.all(np.isfinite(got[0])) and np.all(got[0] < 100), got[0]
    check(item_slice(got, 0), refs[0], ests[0], True, 1, "lengths", f"last sample T{T}", bss_eval)


# ---------------------------------------------------------------------------------------------------------------------
# conditioning
# ---------------------------------------------------------------------------------------------------------------------
def tones(rng, T):
    t = np.arange(T)
    f = rng.uniform(60, 2000, 3)
    return sum(np.sin(2 * np.pi * f[i] / 16000 * t + rng.uniform(0, 6)) for i in range(3)) * np.hanning(T)


def dc_noise(rng, T):
    return 1.0 + 1e-3 * rng.standard_normal(T)


def ar999(rng, T):
    return lfilter([1.0], [1.0, -0.999], rng.standard_normal(T))


def band_silent_ends(rng, T):
    x = sosfilt(butter(8, rng.uniform(0.05, 0.2), output="sos"), rng.standard_normal(T))
    x[:T // 8] = 0
    x[-T // 8:] = 0
    return x


def white(rng, T):
    return rng.standard_normal(T)


KINDS = {"tones": tones, "dc": dc_noise, "ar999": ar999, "band": band_silent_ends, "white": white}
CONDITIONING = [("tones",), ("dc",), ("ar999",), ("band",), ("tones", "white"), ("white", "band"),
                ("ar999", "tones"), ("dc", "white")]



def conditioned_item(rng, S, T, kinds, loud=None):
    """References of the given kinds (cycled), estimates = a mixing matrix with 0.05..0.3 off-diagonals x references
    + white noise at 20 dB + a short FIR; `loud` scales reference 0 by that many dB."""
    refs = np.stack([KINDS[kinds[i % len(kinds)]](rng, T) for i in range(S)])
    refs /= np.sqrt(np.mean(refs ** 2, axis=1, keepdims=True))
    if loud is not None:
        refs[0] *= 10 ** (loud / 20)
    ests = (np.eye(S) + rng.uniform(0.05, 0.3) * rng.standard_normal((S, S))) @ refs
    for i in range(S):
        noise = rng.standard_normal(T)
        ests[i] += noise * np.sqrt(np.sum(ests[i] ** 2) / np.sum(noise ** 2) / 100)
        ests[i] = lfilter([1.0, 0.3, -0.1], [1.0], ests[i])
    return refs.astype(np.float32), ests.astype(np.float32)


def check_ordered(got, label):
    """Cut-independent: |e - P_j e|^2 = |e - P_all e|^2 + |P_all e - P_j e|^2 and |P_all e| >= |P_j e|, so SDR is at
    most SIR and at most SAR (up to the 1e-3 dB rounding allowance), and nothing is NaN."""
    sdr, sir, sar = (np.asarray(g, np.float64) for g in got[:3])
    assert not (np.isnan(sdr).any() or np.isnan(sir).any() or np.isnan(sar).any()), (label, got)
    assert np.all(sdr <= sir + 1e-3) and np.all(sdr <= sar + 1e-3), (label, sdr, sir, sar)


def conditioning_case(S, T, F, kinds, kind_label, scale=1.0, loud=None, seed=0):
    rng = np.random.default_rng(seed)
    refs, ests = conditioned_item(rng, S, T, kinds, loud)
    refs = (refs.astype(np.float64) * scale).astype(np.float32)
    ests = (ests.astype(np.float64) * scale).astype(np.float32)
    got = run(refs, ests, True, F)
    r64, e64 = refs.astype(np.float64), ests.astype(np.float64)
    if max(recursion_defect(r64, e, F) for e in e64) > PROJECTION_DEFECT:
        # The recursion's joint solution is no projection (it lost definiteness): the item is reported NaN, perm -1.
        # QR shows the projection itself is well defined, so the breakdown is the normal equations' alone.
        assert all(np.isnan(g).all() for g in got[:3]) and (got[3] == -1).all(), (kind_label, got)
        assert max(span_defect(r64, e, F) for e in e64) < 1e-9
        return got, True
    check_ordered(got, kind_label)
    dropped = not kept_delays(r64, F).all()
    if not dropped:
        check(got, refs, ests, True, F, f"conditioning QR {kinds[0]}", kind_label, bss_eval_span)
        return got, dropped
    for oracle, tol, kind in ((bss_eval_recursion, RECURSION_TOL, "conditioning GPU - restated recursion"),
                              (bss_eval_span, SPAN_TOL, "conditioning GPU - QR onto kept delays")):
        want = oracle(r64, e64, True, F, margin=True)
        if want[4] > 1e-3:
            assert np.array_equal(got[3], want[3]), (kind, kind_label, got[3], want[3])
        if not np.array_equal(got[3], want[3]):
            continue
        for g, w, name in zip(got[:3], want[:3], ("sdr", "sir", "sar")):
            assert np.array_equal(np.isinf(g), np.isinf(w)), (kind_label, name, g, w)
            d = np.abs(g - w)[np.isfinite(w)]
            assert np.all(d <= tol), (kind, kind_label, name, g, w)
            if d.size and d.max() > WORST.get(kind, (-1.0, ""))[0]:
                WORST[kind] = (float(d.max()), f"{kind_label} {name}")
    return got, dropped


@pytest.mark.parametrize("kinds", CONDITIONING, ids=["-".join(k) for k in CONDITIONING])
@pytest.mark.parametrize("S", [1, 2, 3, 4])
def test_conditioning(S, kinds):
    """Near-degenerate references and mixed sets: against QR where nothing is dropped, against the restated
    recursion and QR onto the kept delays where something is (the SIR then depends on where the cut falls: the
    oracles restate that cut, and check_ordered holds whatever it is).  Three or four band-limited references
    (8th-order Butterworth, cutoffs 0.05..0.2) break the recursion: NaN and perm -1 there."""
    if S == 1 and len(kinds) > 1:
        pytest.skip("a mixed set needs two references")
    conditioning_case(S, 4000, 512, kinds, f"S{S} {'-'.join(kinds)}", seed=S * 31 + len(kinds[0]))


@pytest.mark.parametrize("S", [2, 3, 4])
def test_one_source_80_db_below_another(S):
    conditioning_case(S, 6000, 512, ("white", "ar999"), f"S{S} loud", loud=80.0, seed=S)


@pytest.mark.parametrize("scale", [1e-30, 1e30, 1e-39], ids=["1e-30", "1e30", "denormal"])
@pytest.mark.parametrize("S", [1, 2, 4])
def test_amplitude_extremes(S, scale):
    """Amplitudes 1e-30 and 1e30 and fp32 denormals (|x| < 1.2e-38): the fp64 products and sums absorb them, so the
    values are the oracle's on the same fp32 inputs.  Denormal inputs are coarsely quantised, so they are compared
    with the oracle of the quantised values, not with the unscaled run."""
    got, _ = conditioning_case(S, 5000, 256, ("white", "tones"), f"S{S} scale {scale:g}", scale=scale, seed=3 * S)
    if scale != 1e-39:
        unit, _ = conditioning_case(S, 5000, 256, ("white", "tones"), f"S{S} scale 1", seed=3 * S)
        for a, b in zip(got[:3], unit[:3]):
            assert np.all((a == b) | (np.abs(a - b) <= 1e-3)), (scale, a, b)


# ---------------------------------------------------------------------------------------------------------------------
# the C-ABI on poisoned scratch, guarded buffers
# ---------------------------------------------------------------------------------------------------------------------
def ptr(t):
    return C.c_void_p(t.data_ptr())


def abi_call(refs, ests, mix, B, S, T, F, perm, pattern):
    """One sdr_bss_eval(_mixture) call with every buffer guarded and a scratch of exactly the queried size filled with
    `pattern` (0: clean).  -> the outputs, after checking the bands and that no input changed."""
    lib = N.lib()
    nbytes = lib.sdr_bss_eval_scratch_bytes(B, S, T, F)
    scratch = poisoned(nbytes, pattern)
    g = Guards()
    r, e = g.input("reference", refs), g.input("estimate", ests)
    nan = torch.full((B, S), float("nan"), dtype=torch.float64, device=DEV)
    outs = [g.output(n, nan) for n in ("sdr", "sir", "sar")]
    pm = g.output("perm", torch.full((B, S), -7, dtype=torch.int32, device=DEV))
    st = N.stream(DEV)
    if mix is None:
        rc = lib.sdr_bss_eval(ptr(r), ptr(e), *map(ptr, outs), ptr(pm), B, S, T, F, int(perm), ptr(scratch), st)
    else:
        m = g.input("mixture", mix)
        mouts = [g.output("mix_" + n, nan) for n in ("sdr", "sir", "sar")]
        rc = lib.sdr_bss_eval_mixture(ptr(r), ptr(e), ptr(m), *map(ptr, outs), ptr(pm), *map(ptr, mouts), B, S, T, F,
                                      int(perm), ptr(scratch), st)
        outs += mouts
    assert rc == 0, rc
    g.check()
    check_bands(scratch, "scratch")
    return [o.clone() for o in outs] + [pm.clone()]


@pytest.mark.parametrize("with_mixture", [False, True], ids=["sdr_bss_eval", "sdr_bss_eval_mixture"])
@pytest.mark.parametrize("S,T,F", [(2, 9000, 512), (4, 7682, 512), (3, 61441, 33)])
def test_poisoned_scratch_and_guards(S, T, F, with_mixture):
    """Scratch of exactly sdr_bss_eval_scratch_bytes filled with NaN and with 1e30: bitwise the clean run's results,
    no byte written outside any buffer, no input changed."""
    rng = np.random.default_rng(S + T)
    B = 3
    refs, ests = batch(rng, S, T, F, B)
    r, e = torch.from_numpy(refs).to(DEV), torch.from_numpy(ests).to(DEV)
    m = torch.from_numpy(mixture_of(rng, refs)).to(DEV) if with_mixture else None
    for perm in (True, False):
        clean = abi_call(r, e, m, B, S, T, F, perm, 0)
        assert not any(torch.isnan(o).any() for o in clean[:-1])
        for pattern in (POISON_NAN, POISON_HUGE):
            got = abi_call(r, e, m, B, S, T, F, perm, pattern)
            for a, b in zip(got, clean):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), (perm, hex(pattern))


# ---------------------------------------------------------------------------------------------------------------------
# non-finite inputs stay in their item
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")], ids=["nan", "inf", "-inf"])
@pytest.mark.parametrize("where", ["reference", "estimate", "mixture"])
@pytest.mark.parametrize("at", ["start", "halo", "end"])
def test_nonfinite_stays_in_its_item(where, value, at):
    """A NaN or inf in one sample of item 2.  In a reference: every score of the item NaN, perm -1.  In an estimate:
    its scores NaN and perm -1, its mixture scores unchanged.  In the mixture: its mixture scores NaN, nothing else
    changed.  Every other item bitwise unchanged.  "halo" puts the fault 10 samples into the second correlation
    chunk, inside the first chunk's F - 1 sample halo."""
    S, T, F, B, bad = 2, 9000, 512, 5, 2
    rng = np.random.default_rng(17)
    refs, ests = batch(rng, S, T, F, B)
    mix = mixture_of(rng, refs)
    per = -(-T // -(-T // 4096))                        # the correlation chunk length
    t = {"start": 0, "halo": per + 10, "end": T - 1}[at]
    clean = run(refs, ests, True, F, mixture=torch.from_numpy(mix).to(DEV))
    arr = {"reference": refs, "estimate": ests, "mixture": mix}[where].copy()
    if where == "mixture":
        arr[bad, t] = value
    else:
        arr[bad, 1, t] = value
    args = {"reference": refs, "estimate": ests, "mixture": mix}
    args[where] = arr
    got = run(args["reference"], args["estimate"], True, F, mixture=torch.from_numpy(args["mixture"]).to(DEV))
    others = [b for b in range(B) if b != bad]
    scores = ("sdr", "sir", "sar")
    for k in range(4):
        assert np.array_equal(got[k][others], clean[k][others])
    for n in scores + ("sdri", "siri", "sari"):
        assert np.array_equal(got[4][n][others], clean[4][n][others]), n
    est_nan = where != "mixture"
    mix_nan = where != "estimate"
    for k in range(3):
        if est_nan:
            assert np.isnan(got[k][bad]).all(), (k, got[k][bad])
        else:
            assert np.array_equal(got[k][bad], clean[k][bad])
    assert (got[3][bad] == -1).all() if est_nan else np.array_equal(got[3][bad], clean[3][bad])
    for n in scores:
        if mix_nan:
            assert np.isnan(got[4][n][bad]).all(), (n, got[4][n][bad])
        else:
            assert np.array_equal(got[4][n][bad], clean[4][n][bad]), n


# ---------------------------------------------------------------------------------------------------------------------
# batch and size limits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,T", [(2, 6), (4, 16)])
def test_batch_past_grid_limit_with_mixture(S, T):
    B, F = 65537, 4
    g = torch.Generator(device=DEV).manual_seed(S)
    refs = torch.randn(B, S, T, device=DEV, generator=g)
    ests = torch.randn(B, S, T, device=DEV, generator=g)
    mix = torch.randn(B, T, device=DEV, generator=g)
    with torch.no_grad():
        full = P.bss_eval_sources(refs, ests, True, F, mixture=mix)
        h = B // 2 + 3
        lo = P.bss_eval_sources(refs[:h], ests[:h], True, F, mixture=mix[:h])
        hi = P.bss_eval_sources(refs[h:], ests[h:], True, F, mixture=mix[h:])
    for f, a, b in zip(full[:4], lo[:4], hi[:4]):
        assert torch.equal(f, torch.cat([a, b]))
    for n in full[4]:
        assert torch.equal(full[4][n], torch.cat([lo[4][n], hi[4][n]])), n
    r, e, m = refs.cpu().numpy(), ests.cpu().numpy(), mix.cpu().numpy()
    for b in (0, 65535, B - 1):
        got = [x[b].cpu().numpy() for x in full[:4]]
        check(got, r[b], e[b], True, F, "batch", f"B{B} item {b}", bss_eval)
        want = bss_eval_mixture(r[b].astype(np.float64), m[b].astype(np.float64), F)
        for k, name in enumerate(("sdr", "sir", "sar")):
            compare("batch", full[4][name][b].cpu().numpy(), want[k], f"B{B} item {b} mixture {name}",
                    want[0] if k == 1 else None)


def test_past_2_31_elements():
    """B S T = 2 x 13423 x 80000 > 2^31 at F = 4 (16 chunks per item): bitwise the two sub-batches' results, and the
    last item (whose rows start past 2^31) against the oracle."""
    S, T, F = 2, 80000, 4
    B = (1 << 31) // (S * T) + 2
    need = 2 * B * S * T * 4 + N.lib().sdr_bss_eval_scratch_bytes(B, S, T, F) + 2 * GiB
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")
    g = torch.Generator(device=DEV).manual_seed(5)
    refs = torch.randn(B, S, T, device=DEV, generator=g)
    ests = torch.randn(B, S, T, device=DEV, generator=g).mul_(0.3)      # in place: no 8.6 GiB temporaries
    ests[:, 0].add_(refs[:, 1])
    ests[:, 1].add_(refs[:, 0])
    with torch.no_grad():
        full = P.bss_eval_sources(refs, ests, True, F)
        h = B // 2
        lo = P.bss_eval_sources(refs[:h], ests[:h], True, F)
        hi = P.bss_eval_sources(refs[h:], ests[h:], True, F)
    for f, a, b in zip(full, lo, hi):
        assert torch.equal(f, torch.cat([a, b]))
    got = [x[B - 1].cpu().numpy() for x in full]
    check(got, refs[B - 1].cpu().numpy(), ests[B - 1].cpu().numpy(), True, F, "batch", "2^31 last item", bss_eval)


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
def test_graph_replay_four_sources_with_mixture():
    """S = 4, F = 512 with the mixture captured once and replayed on new inputs copied into the captured buffers."""
    rng = np.random.default_rng(21)
    S, T, F, B = 4, 5000, 512, 2
    refs, ests = batch(rng, S, T, F, B)
    r, e = torch.from_numpy(refs).to(DEV), torch.from_numpy(ests).to(DEV)
    m = torch.from_numpy(mixture_of(rng, refs)).to(DEV)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            P.bss_eval_sources(r, e, True, F, mixture=m)      # warm-up: sets the kernels' shared-memory limits
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap = P.bss_eval_sources(r, e, True, F, mixture=m)
        refs2, ests2 = batch(rng, S, T, F, B)
        for dst, src in ((r, refs2), (e, ests2), (m, mixture_of(rng, refs2))):
            dst.copy_(torch.from_numpy(src))
        graph.replay()
        torch.cuda.synchronize()
        eager = P.bss_eval_sources(r, e, True, F, mixture=m)
    for a, b in zip(cap[:4], eager[:4]):
        assert torch.equal(a, b)
    for n in eager[4]:
        assert torch.equal(cap[4][n], eager[4][n]), n


def test_zz_print_worst_errors():
    for kind, (err, label) in sorted(WORST.items()):
        print(f"worst {kind}: {err:.2e} dB at {label}")
