"""Every entry is a pure function of its inputs: what the caller-owned scratch memory holds on entry changes nothing.

The library works inside buffers its caller owns (workspaces, the training forward's `saved`, the host entry's device
staging, packed weights, outputs) and neither allocates nor clears them wholesale.  Here every such buffer is exactly
as large as its size query says, sits between guard bands (tests/guards.py), and starts as zeros (the clean run), as
0x7FA5A5A5 words (NaN in fp32, 7.6e306 as an fp64: propagates through arithmetic) or as 0x7149F2CA words (1e30 in
fp32, 5.3e237 as an fp64: survives what swallows a NaN: fmaxf-style ReLU, max, comparisons, the PReLU select).

- whole-model entries at the C-ABI, one model per dispatch path: the result is finite everywhere, no band is touched,
  the mixture and the packed weights are bitwise unchanged, the poisoned result equals the clean one (bitwise for the
  causal model, which has no atomics; within the run-to-run spread of the fp64 statistics atomics otherwise, measured
  here between two clean runs, printed, and bounded by 1e-5), and the clean result is the fp64 oracle's to 1e-4;
- the size and alignment refusals of the same entries: each returns before anything is enqueued, the output keeps its
  poison;
- call order on one workspace through the Python modules: long / short / long shapes across the pyramid switch, four
  variants through one buffer, a captured graph replayed on a poisoned workspace, a stream whose step workspace is
  poisoned between steps, CorpusSeparator with every buffer it owns poisoned between passes;
- the training forward and backward with `saved`, both workspaces and the gradient buffer poisoned;
- the metric kernels and the stage entries that take their own scratch, and the stage `stats` contract (the caller
  zeroes them: a pre-loaded slot comes back as pre-load + sums)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.corpus import CorpusSeparator, separate_corpus
from oracle import sudormrf_oracle as O
from guards import (POISON_HUGE, POISON_NAN, check_bands, guarded_copy, poisoned, poisoned_like, repoison)
from stream_oracle import granule
from test_gpu_long import normalised_input, takes_pyramid
from test_gpu_model_space import build, gc, imp, orig, paths

gpu = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4              # clean result against the fp64 oracle (rel_max and rel_L2)
SPREAD = 1e-5           # bound on clean-to-clean and clean-to-poisoned differences where fp64 atomics order the sums
PATTERNS = [("nan", POISON_NAN), ("1e30", POISON_HUGE)]
OK, BAD_ARGUMENT, WORKSPACE = 0, -2, -3


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel(a, b):
    """max |a - b| / max |b|; inf when a is not finite."""
    if not torch.isfinite(a).all():
        return float("inf")
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


# =====================================================================================================================
# 1. the helper itself (no device needed)
# =====================================================================================================================
@pytest.mark.parametrize("nbytes", [1, 6, 4096, 1000003])
@pytest.mark.parametrize("pattern", [0, POISON_NAN, POISON_HUGE])
def test_poisoned_helper_reports_writes_outside(nbytes, pattern):
    t = poisoned(nbytes, pattern, device="cpu")
    assert t.numel() == nbytes and t.dtype == torch.uint8 and t.data_ptr() % 256 == 0
    if nbytes >= 4:
        word = int(t[:4].view(torch.int32)[0]) & 0xFFFFFFFF
        assert word == pattern
        f = t[:4].view(torch.float32)[0]
        assert (pattern == POISON_NAN) == bool(torch.isnan(f)) and (pattern == POISON_HUGE) == bool(f > 9e29)
    t.fill_(7)                                              # the interior is the caller's
    check_bands(t, "interior writes")
    for where in range(4):                                  # either end of either band
        t2 = poisoned(nbytes, pattern, device="cpu")
        buf, off = t2._bands[0], t2._bands[1]
        buf[(0, off - 1, off + nbytes, buf.numel() - 1)[where]] ^= 1
        with pytest.raises(AssertionError, match="written"):
            check_bands(t2, "stray write")
    v = poisoned_like(torch.empty(3, 5), POISON_HUGE)
    assert v.shape == (3, 5) and bool((v > 9e29).all())
    check_bands(v, "typed view")


# =====================================================================================================================
# 2. whole-model entries at the C-ABI
# =====================================================================================================================
def flat_params(m, c):
    """The parameters in state_dict order as sdr_pack_weights takes them (fp32, contiguous, the model's constant folds)."""
    transform = getattr(m, "_b200_param_transform", None)
    out = []
    for name in _engine.state_dict_names(c):
        t = _engine._fetch(m, name).detach().to(torch.float32)
        out.append((transform(name, t) if transform else t).contiguous())
    return out


def pack(c, params, pattern=POISON_NAN):
    """sdr_pack_weights into a poisoned, guarded buffer of exactly sdr_packed_weight_bytes."""
    lib = N.lib()
    nbytes = lib.sdr_packed_weight_bytes(C.byref(c))
    assert nbytes > 0
    buf = poisoned(nbytes, pattern)
    ptrs = (C.c_void_p * len(params))(*[t.data_ptr() for t in params])
    N.check(lib.sdr_pack_weights(C.byref(c), ptrs, len(params), p(buf), nbytes, stream()), "sdr_pack_weights")
    check_bands(buf, "packed weights after sdr_pack_weights")
    return buf


class Model:
    """One model, its guarded packed weights, and every whole-model entry on guarded, exactly-sized buffers."""

    def __init__(self, variant, kw, seed=211):
        self.variant, self.kw = variant, kw
        self.cfg, self.sd, self.m = build(variant, kw, seed)
        self.c = _engine.make_config(self.m)
        self.A = kw.get("in_audio_channels", 1) if variant in ("groupcomm", "causal") else 1
        self.SA = self.cfg.num_sources * self.A
        self.packed = pack(self.c, flat_params(self.m, self.c))
        self.packed_before = self.packed.clone()

    def ws_bytes(self, entry, B, T):
        lib = N.lib()
        q = lib.sdr_separate_workspace_bytes if entry in ("separate", "ragged") else lib.sdr_workspace_bytes
        n = q(C.byref(self.c), B, T)
        assert n > 0
        return n

    def run(self, entry, x, pattern, mc=0, lengths=None, ws=None):
        """entry in forward / separate / ragged / host.  x [B, A, T] on the device.  Returns a copy of the output
        after checking the return code, the bands, the inputs and that every output element was written."""
        lib, c = N.lib(), self.c
        B, A, T = x.shape
        xg = guarded_copy(x)
        own_ws = ws is None
        if own_ws:
            ws = poisoned(self.ws_bytes(entry, B, T), pattern)
        out = poisoned_like(torch.empty(B, self.SA, T, device=DEV), pattern or POISON_NAN)
        extra = []
        if entry == "forward":
            rc = lib.sdr_forward(C.byref(c), p(self.packed), p(xg), p(out), B, T, mc, p(ws), ws.numel(), stream())
        elif entry == "separate":
            rc = lib.sdr_separate(C.byref(c), p(self.packed), p(xg), p(out), B, T, mc, p(ws), ws.numel(), stream())
        elif entry == "ragged":
            lens = guarded_copy(torch.tensor(lengths, dtype=torch.int64, device=DEV))
            extra.append(("lengths", lens))
            rc = lib.sdr_separate_ragged(C.byref(c), p(self.packed), p(xg), p(lens), p(out), B, T, mc, 1, p(ws),
                                         ws.numel(), stream())
        else:
            nio = lib.sdr_host_staging_bytes(C.byref(c), B, T)
            staging = poisoned(nio, pattern)
            extra.append(("staging", staging))
            hx = x.cpu().pin_memory()
            hout = torch.empty(B, self.SA, T).pin_memory()
            repoison(hout.view(torch.uint8), pattern or POISON_NAN)
            rc = lib.sdr_forward_host(C.byref(c), p(self.packed), p(hx), p(hout), B, T, mc, p(staging), nio, p(ws),
                                      ws.numel(), stream())
        assert rc == OK, (entry, rc)
        torch.cuda.synchronize()
        for name, t in [("workspace", ws), ("out", out), ("mixture", xg), ("packed", self.packed)] + extra:
            check_bands(t, f"{entry} {name}")
        assert torch.equal(xg.view(torch.int32), x.view(torch.int32)), "the mixture was modified"
        assert torch.equal(self.packed, self.packed_before), "the packed weights were modified"
        res = hout.to(DEV) if entry == "host" else out.clone()
        rows = [b for b in range(B) if lengths is None or lengths[b] > 1]      # torch's std of one sample is NaN
        assert torch.isfinite(res[rows]).all(), f"{entry}: output elements left unwritten or not finite"
        return res

    def oracle(self, entry, x, mc, lengths=None):
        cfg, sd = self.cfg, self.sd
        if entry in ("forward", "host"):
            ref = O.forward(cfg, sd, x, dtype=torch.float64)
            return O.mixture_consistency(ref, x.double()) if mc else ref
        if entry == "separate":
            return O.separate(cfg, sd, x[:, 0], apply_mixture_consistency=bool(mc), dtype=torch.float64)
        rows = []
        for b, n in enumerate(lengths):          # each utterance alone, padded to the bucket's width
            w = x[b, 0, :n].double()
            mean, std = w.mean(), w.std()
            xn = torch.zeros(1, 1, x.shape[-1], dtype=torch.float64, device=x.device)
            xn[0, 0, :n] = (w - mean) / (std + 1e-9)
            ref = O.forward(cfg, sd, xn, dtype=torch.float64) * std + mean
            rows.append(O.mixture_consistency(ref, xn) if mc else ref)
        return torch.cat(rows)

    def gemm_paths(self):
        """Which 1x1 convolutions have a tensor-core image: (bottleneck, proj_1x1, res_conv / conv_1x1_exp)."""
        f = N.lib().sdr_pointwise_mma_packed_bytes
        cfg = self.cfg
        G = cfg.group_size if self.variant == "groupcomm" else 1
        Co, Ci = cfg.out_channels // G, cfg.in_channels // G
        return f(cfg.out_channels, cfg.enc_num_basis) > 0, f(Ci, Co) > 0, f(Co, Ci) > 0

    def launches(self, B, T):
        return N.lib().sdr_forward_launch_count_for(C.byref(self.c), B, T)


def causal(S, A, K, N_, Co, Ci, U=2, D=4):
    return dict(in_audio_channels=A, out_channels=Co, in_channels=Ci, num_blocks=U, upsampling_depth=D,
                enc_kernel_size=K, enc_num_basis=N_, num_sources=S)


# id, variant, kwargs, B, T, entries, expectations:
#   pyramid: the depthwise stage runs as the one-pass pyramid; gemms: (bottleneck, proj, res) on wgmma;
#   io: (encoder, mask, decoder) on wgmma (test_gpu_model_space.paths); folded: tac_apply rides on proj_1x1
CASES = [
    # every 1x1 on wgmma, the window encoder with 21 taps padded to 64, the decoder's 42 rows in a 128-row tile;
    # T a multiple of hop * 2^D, B = 1
    ("imp_D4_pyramid_wgmma", "improved", imp(2, 21, 256, Co=128, Ci=128, U=2, D=4), 1, 1600, ("forward", "host", "separate"),
     dict(pyramid=True, gemms=(True, True, True), io=(True, True, True))),
    # every 1x1 and the encoder on FFMA; T % hop != 0; B = 3
    ("imp_D5_pyramid_ffma", "improved", imp(2, 5, 16, Co=8, Ci=16, U=2, D=5), 3, 193, ("forward", "separate"),
     dict(pyramid=True, gemms=(False, False, False), io=(False, False, False))),
    # D = 6; the block's 1x1 convolutions on wgmma, the mask and the decoder on FFMA
    ("imp_D6_pyramid_mixed", "improved", imp(2, 11, 64, Co=64, Ci=128, U=1, D=6), 2, 967, ("forward",),
     dict(pyramid=True, gemms=(True, True, True), io=(True, False, False))),
    # D = 3: level by level; T = 1, B = 5
    ("imp_D3_levels_T1", "improved", imp(2, 21, 64, Co=32, Ci=64, U=2, D=3), 5, 1, ("forward", "host"),
     dict(pyramid=False, gemms=(True, False, True), io=(True, False, True))),
    # D = 4 and T < hop * 2^D: one padded quantum, 2 frames at the deepest level, too short for the pyramid
    ("imp_D4_short_row", "improved", imp(3, 21, 64, Co=32, Ci=64, U=1, D=4), 2, 157, ("forward", "separate"),
     dict(pyramid=False, gemms=(True, False, True), io=(True, False, True))),
    # GroupComm, 16 channels per group (tac_mma16_kernel), stereo, tac_apply folded into proj_1x1, pyramid over B * G
    ("gc_n16_stereo_folded", "groupcomm", gc(2, 2, 21, 64, 2, 16, U=2, D=4), 2, 1600, ("forward", "host"),
     dict(pyramid=True, folded=True, gemms=(True, False, False), io=(True, False, True))),
    # 8 channels per group (tac_kernel), 128 proj_1x1 rows: tac_apply is a launch of its own; level by level
    ("gc_n8_unfolded", "groupcomm", gc(2, 1, 11, 32, 2, 8, Ci=256, U=2, D=3), 3, 403, ("forward", "separate"),
     dict(pyramid=False, folded=False)),
    ("gc_n4_folded", "groupcomm", gc(3, 1, 5, 16, 3, 4, U=1, D=2), 3, 61, ("forward",), dict(pyramid=False, folded=True)),
    ("gc_n32_folded", "groupcomm", gc(2, 1, 21, 32, 2, 32, U=1, D=4), 1, 1603, ("forward",),
     dict(pyramid=True, folded=True)),
    # the original model: sigmoid gate, no reshape_before_masks (Co == N)
    ("orig_S1_sigmoid", "original", orig(1, 5, 64, 64, U=2, D=3), 3, 1001, ("forward", "separate"), dict(pyramid=False)),
    # reshape_before_masks; hop 20, D = 4: lcm(20, 16) = 80 pads 401 to 480, L = 24 (L % 16 != 0): level by level
    ("orig_S2_lcm_remainder", "original", orig(2, 41, 48, 32, U=2, D=4), 2, 401, ("forward",), dict(pyramid=False)),
    # softmax over three sources; L = 160: the pyramid with per-channel PReLU slopes
    ("orig_S3_softmax_pyramid", "original", orig(3, 21, 32, 32, U=1, D=4), 2, 1600, ("forward", "host"),
     dict(pyramid=True)),
    # the causal model (no statistics, no atomics: bitwise) at D = 1 and at its default depth
    ("causal_D1", "causal", causal(2, 1, 21, 64, 32, 64, U=2, D=1), 3, 395, ("forward", "separate", "host"), dict()),
    ("causal_default_depth", "causal", causal(2, 1, 21, 128, 128, 128, U=2, D=4), 2, 1601, ("forward", "separate"),
     dict(gemms=(True, True, True))),
    ("causal_stereo", "causal", causal(2, 2, 11, 32, 16, 32, U=1, D=3), 1, 7, ("forward",), dict()),
]


def assert_dispatch(M, B, T, want):
    cfg, D, U = M.cfg, M.cfg.upsampling_depth, M.cfg.num_blocks
    if M.variant == "causal":
        assert M.launches(B, T) == 2 + 3 * U + 3
    else:
        pyr = takes_pyramid(cfg, B, T)
        assert pyr == want["pyramid"], ("pyramid", pyr)
        levels = 2 if pyr else D
        if M.variant == "original":
            count = 2 + U * (levels + 4) + (1 if cfg.out_channels != cfg.enc_num_basis else 0) + 4
        elif M.variant == "groupcomm":
            count = 2 + U * (levels + 3 + (1 if want["folded"] else 2)) + 3
        else:
            count = 2 + U * (levels + 3) + 3
        assert M.launches(B, T) == count, (M.launches(B, T), count)
    if "gemms" in want:
        assert M.gemm_paths() == want["gemms"], M.gemm_paths()
    if "io" in want:
        assert paths(cfg) == want["io"], paths(cfg)


def compare_runs(M, entry, x, mc, lengths=None, what=""):
    """Two clean runs, the oracle, then both poisons."""
    bitwise = M.variant == "causal"
    clean = M.run(entry, x, 0, mc, lengths)
    again = M.run(entry, x, 0, mc, lengths)
    rows = [b for b in range(x.shape[0]) if lengths is None or lengths[b] > 1]
    spread = rel(again[rows], clean[rows])
    ref = M.oracle(entry, x, mc, lengths)
    if lengths is None:
        e = O.parity_errors(clean, ref)
    else:                                        # a ragged row is valid up to its length
        e = tuple(max(v) for v in zip(*[O.parity_errors(clean[b:b + 1, :, :lengths[b]], ref[b:b + 1, :, :lengths[b]])
                                        for b in rows]))
    assert max(e) < TOL, (what, e)
    assert spread == 0.0 if bitwise else spread <= SPREAD, (what, spread)
    diffs = []
    for pname, pattern in PATTERNS:
        got = M.run(entry, x, pattern, mc, lengths)
        if lengths is not None and 1 in lengths:     # the one-sample row is NaN in every run, and only that row
            b = lengths.index(1)
            assert torch.isnan(got[b, :, 0]).all() and torch.isnan(clean[b, :, 0]).all()
        d = rel(got[rows], clean[rows])
        same = torch.equal(got[rows].view(torch.int32), clean[rows].view(torch.int32))
        diffs.append(f"{pname}: {d:.2e}{' (bitwise)' if same else ''}")
        if bitwise:
            assert same, (what, pname, d)
        else:
            assert d <= SPREAD, (what, pname, d)
    print(f"{what} {entry} mc={mc}: oracle rel_max {e[0]:.2e}; clean / clean {spread:.2e}"
          f"{' (bitwise)' if spread == 0.0 else ''}; clean / poisoned " + ", ".join(diffs))


@gpu
@pytest.mark.parametrize("name,variant,kw,B,T,entries,want", CASES, ids=[c[0] for c in CASES])
def test_whole_model_on_poisoned_scratch(name, variant, kw, B, T, entries, want):
    M = Model(variant, kw)
    assert_dispatch(M, B, T, want)
    x = (normalised_input(B, M.A, T, seed=212) if T > 1 else torch.tensor([[[0.7]], [[-1.3]], [[0.0]], [[2.5]], [[1e-3]]])).to(DEV)
    wav = x * torch.linspace(0.3, 2.0, B, device=DEV).view(B, 1, 1) + 0.2        # separate() normalises it itself
    with torch.no_grad():
        for entry in entries:
            if entry == "separate" and M.A != 1:
                continue
            for mc in ((0, 1) if M.A == 1 else (0,)):
                compare_runs(M, entry, wav if entry == "separate" else x, mc, what=name)


RAGGED = [("improved", imp(2, 21, 64, Co=32, Ci=64, U=2, D=4)), ("causal", causal(2, 1, 21, 64, 32, 64, U=2, D=2))]


@gpu
@pytest.mark.parametrize("variant,kw", RAGGED, ids=[v for v, _ in RAGGED])
def test_separate_ragged_on_poisoned_scratch(variant, kw):
    """Lengths 1, mid and full in one bucket whose padding is zero, as the contract requires."""
    M = Model(variant, kw)
    T = 3 * O.padded_length(M.cfg, 1)
    lengths = [1, T // 2 + 3, T]
    g = torch.Generator().manual_seed(5)
    wav = torch.zeros(3, 1, T)
    for b, n in enumerate(lengths):
        wav[b, 0, :n] = torch.randn(n, generator=g) * (0.4 + b) + 0.1 * b
    with torch.no_grad():
        for mc in (0, 1):
            compare_runs(M, "ragged", wav.to(DEV), mc, lengths, what=f"{variant} ragged")


# =====================================================================================================================
# 3. size and alignment contract: every refusal returns before anything is enqueued
# =====================================================================================================================
SMALL = imp(2, 21, 64, Co=32, Ci=64, U=1, D=2)


def spare(nbytes, extra=256):
    """A poisoned buffer with `extra` spare bytes, to take misaligned views of; the base is 256 B aligned."""
    return poisoned(nbytes + extra, POISON_NAN)


@gpu
def test_refusals_of_the_forward_entries():
    lib = N.lib()
    M = Model("improved", SMALL)
    c, B, T = M.c, 2, 200
    x = guarded_copy(normalised_input(B, 1, T, seed=3).to(DEV))
    lens = torch.full((B,), T, dtype=torch.int64, device=DEV)
    out = poisoned_like(torch.empty(B, 2, T, device=DEV), POISON_HUGE)
    out_before = out.clone()
    npk = M.packed.numel()
    pk2 = spare(npk)
    pk2[16:16 + npk].copy_(M.packed)              # the same image 16 B further on: an aligned, valid packed buffer
    nws, nsep = M.ws_bytes("forward", B, T), M.ws_bytes("separate", B, T)
    ws = spare(nsep)
    Tr = O.padded_length(M.cfg, T)
    xr = guarded_copy(torch.zeros(B, 1, Tr, device=DEV))
    outr = poisoned_like(torch.empty(B, 2, Tr, device=DEV), POISON_HUGE)
    nrag = M.ws_bytes("ragged", B, Tr)
    wsr = spare(nrag)

    def fwd(pk=M.packed, w=ws, n=nws):
        return lib.sdr_forward(C.byref(c), p(pk), p(x), p(out), B, T, 0, p(w), n, stream())

    def sep(pk=M.packed, w=ws, n=nsep):
        return lib.sdr_separate(C.byref(c), p(pk), p(x), p(out), B, T, 0, p(w), n, stream())

    def rag(pk=M.packed, w=wsr, n=nrag):
        return lib.sdr_separate_ragged(C.byref(c), p(pk), p(xr), p(lens), p(outr), B, Tr, 0, 1, p(w), n, stream())

    for call, n, w in ((fwd, nws, ws), (sep, nsep, ws), (rag, nrag, wsr)):
        assert call(n=n - 1) == WORKSPACE
        assert call(n=0) == WORKSPACE
        for skew in (4, 128):
            assert call(w=w[skew:]) == BAD_ARGUMENT, skew
        for skew in (4, 8):
            assert call(pk=pk2[16 + skew:]) == BAD_ARGUMENT, skew
        assert call(w=None) == BAD_ARGUMENT and call(pk=None) == BAD_ARGUMENT
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), out_before.view(torch.int32)), "a refused call wrote the output"
    assert bool((outr > 9e29).all())
    for t, what in ((out, "out"), (outr, "ragged out"), (ws, "workspace"), (wsr, "ragged workspace"), (x, "mixture")):
        check_bands(t, what)
    # the same buffers are accepted as they are, and from the aligned copy of the weights
    assert fwd() == OK and fwd(pk=pk2[16:]) == OK and sep() == OK and rag() == OK
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(outr).all()


@gpu
def test_refusals_of_forward_host():
    """sdr_forward_host checks the staging buffer and the forward's workspace before its first copy: after a refusal
    the staging buffer still holds its poison, so the mixture was not copied in."""
    lib = N.lib()
    M = Model("improved", SMALL)
    c, B, T = M.c, 2, 200
    hx = normalised_input(B, 1, T, seed=3).pin_memory()
    hout = torch.empty(B, 2, T).pin_memory()
    repoison(hout.view(torch.uint8), POISON_HUGE)
    nio, nws = lib.sdr_host_staging_bytes(C.byref(c), B, T), M.ws_bytes("forward", B, T)
    io, ws = spare(nio), spare(nws)
    io_before = io.clone()

    def host(pk=M.packed, s=io, ns=nio, w=ws, n=nws):
        return lib.sdr_forward_host(C.byref(c), p(pk), p(hx), p(hout), B, T, 0, p(s), ns, p(w), n, stream())

    assert host(ns=nio - 1) == WORKSPACE and host(n=nws - 1) == WORKSPACE
    for skew in (4, 128):
        assert host(s=io[skew:]) == BAD_ARGUMENT and host(w=ws[skew:]) == BAD_ARGUMENT
    assert host(s=None) == BAD_ARGUMENT and host(w=None) == BAD_ARGUMENT and host(pk=None) == BAD_ARGUMENT
    torch.cuda.synchronize()
    assert torch.equal(io, io_before), "a refused sdr_forward_host copied into the staging buffer"
    assert bool((hout > 9e29).all()), "a refused sdr_forward_host wrote the host output"
    assert host() == OK
    torch.cuda.synchronize()
    assert torch.isfinite(hout).all()
    check_bands(io, "staging")
    check_bands(ws, "workspace")


@gpu
def test_refusals_of_pack_weights_and_image_is_fully_written():
    """A buffer one byte short or 4 bytes off 16 B alignment is refused untouched; two packs into differently poisoned
    buffers of exactly sdr_packed_weight_bytes are bitwise equal, so the derived regions, the bf16 hi/lo images and
    the padded decoder rows are all written."""
    lib = N.lib()
    for variant, kw in (("improved", imp(2, 21, 256, Co=128, Ci=128, U=1, D=4)), ("original", orig(3, 21, 32, 32, U=1, D=4)),
                        ("causal", causal(2, 1, 21, 128, 128, 128, U=1, D=2)), ("groupcomm", gc(2, 2, 21, 64, 2, 16, U=1))):
        cfg, sd, m = build(variant, kw)
        c = _engine.make_config(m)
        params = flat_params(m, c)
        a, b, z = pack(c, params, POISON_NAN), pack(c, params, POISON_HUGE), pack(c, params, 0)
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(a, z), variant
        nbytes = a.numel()
        buf = spare(nbytes)
        before = buf.clone()
        ptrs = (C.c_void_p * len(params))(*[t.data_ptr() for t in params])
        assert lib.sdr_pack_weights(C.byref(c), ptrs, len(params), p(buf), nbytes - 1, stream()) == WORKSPACE
        assert lib.sdr_pack_weights(C.byref(c), ptrs, len(params), p(buf[4:]), nbytes, stream()) == BAD_ARGUMENT
        assert lib.sdr_pack_weights(C.byref(c), ptrs, len(params), None, nbytes, stream()) == BAD_ARGUMENT
        torch.cuda.synchronize()
        assert torch.equal(buf, before)


@gpu
def test_refusals_of_the_stream_entries():
    lib = N.lib()
    M = Model("causal", causal(2, 1, 21, 64, 32, 64, U=1, D=2))
    c, B = M.c, 3
    Cs = 2 * granule(M.cfg)
    nst, nws = lib.sdr_stream_state_bytes(C.byref(c), B), lib.sdr_stream_workspace_bytes(C.byref(c), B, Cs)
    assert nst > 0 and nws > 0
    state, ws = spare(nst), spare(nws)
    chunk = guarded_copy(normalised_input(B, 1, Cs, seed=4).to(DEV))
    out = poisoned_like(torch.empty(B, 2, Cs, device=DEV), POISON_HUGE)
    tail = poisoned_like(torch.empty(B, 2, M.cfg.hop, device=DEV), POISON_HUGE)
    before = state.clone()

    def step(s=state, w=ws, n=nws, pk=M.packed):
        return lib.sdr_stream_step(C.byref(c), p(pk), p(s), p(chunk), p(out), B, Cs, 0, p(w), n, stream())

    assert step(n=nws - 1) == WORKSPACE
    for skew in (4, 128):
        assert step(w=ws[skew:]) == BAD_ARGUMENT
    for skew in (4, 8):
        assert step(s=state[skew:]) == BAD_ARGUMENT
        assert lib.sdr_stream_reset(C.byref(c), p(state[skew:]), B, None, 0, stream()) == BAD_ARGUMENT
        assert lib.sdr_stream_flush(C.byref(c), p(state[skew:]), p(tail), B, 0, stream()) == BAD_ARGUMENT
    assert step(s=None) == BAD_ARGUMENT and step(w=None) == BAD_ARGUMENT
    torch.cuda.synchronize()
    assert torch.equal(state, before) and bool((out > 9e29).all()) and bool((tail > 9e29).all())
    assert lib.sdr_stream_reset(C.byref(c), p(state), B, None, 0, stream()) == OK and step() == OK
    assert lib.sdr_stream_flush(C.byref(c), p(state), p(tail), B, 0, stream()) == OK
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(tail).all()
    for t, what in ((state, "state"), (ws, "workspace"), (out, "out"), (tail, "tail")):
        check_bands(t, what)


@gpu
def test_refusals_of_the_training_entries_and_metrics():
    lib = N.lib()
    M = Model("improved", SMALL)
    c, B, T = M.c, 2, 200
    x = guarded_copy(normalised_input(B, 1, T, seed=3).to(DEV))
    out = poisoned_like(torch.empty(B, 2, T, device=DEV), POISON_HUGE)
    nsv, nws = lib.sdr_train_saved_bytes(C.byref(c), B, T), M.ws_bytes("forward", B, T)
    nbw = lib.sdr_backward_workspace_bytes(C.byref(c), B, T)
    saved, ws, bws = spare(nsv), spare(nws), spare(nbw)
    ngrad = sum(lib.sdr_param_numel(C.byref(c), i) for i in range(lib.sdr_num_params(C.byref(c))))
    grads = poisoned_like(torch.empty(ngrad, device=DEV), POISON_HUGE)
    gout = guarded_copy(torch.randn(B, 2, T, device=DEV))

    def train(sv=saved, ns=nsv, w=ws, n=nws):
        return lib.sdr_forward_train(C.byref(c), p(M.packed), p(x), p(out), B, T, p(sv), ns, p(w), n, stream())

    def back(sv=saved, w=bws, n=nbw):
        return lib.sdr_backward(C.byref(c), p(M.packed), p(x), p(sv), p(gout), p(grads), B, T, p(w), n, stream())

    assert train(ns=nsv - 1) == WORKSPACE and train(n=nws - 1) == WORKSPACE and back(n=nbw - 1) == WORKSPACE
    for skew in (4, 128):
        assert train(sv=saved[skew:]) == BAD_ARGUMENT and train(w=ws[skew:]) == BAD_ARGUMENT
        assert back(sv=saved[skew:]) == BAD_ARGUMENT and back(w=bws[skew:]) == BAD_ARGUMENT
    # the metrics take 8 B aligned scratch (fp64 accumulators)
    est, tgt = torch.randn(2, 2, 100, device=DEV), torch.randn(2, 2, 100, device=DEV)
    best, perm = torch.empty(2, device=DEV), torch.empty(2, dtype=torch.int32, device=DEV)
    pw = torch.empty(2, 2, 2, device=DEV)
    sc = spare(max(lib.sdr_pit_sisdr_scratch_bytes(2, 2), lib.sdr_stabilized_sisdr_scratch_bytes(2, 2, 2)))
    assert lib.sdr_pit_sisdr(p(est), p(tgt), None, p(best), p(perm), 2, 2, 100, 1, 0, 1e-9, p(sc[4:]), stream()) == BAD_ARGUMENT
    assert lib.sdr_stabilized_sisdr(p(est), p(tgt), p(best), p(perm), 2, 2, 2, 2, 100, 1, 0, 1e-9, p(sc[4:]),
                                    stream()) == BAD_ARGUMENT
    assert lib.sdr_pairwise_neg_sdr(p(est), p(tgt), p(pw), 2, 2, 100, 1, 1, 1, p(sc[4:]), stream()) == BAD_ARGUMENT
    torch.cuda.synchronize()
    assert bool((out > 9e29).all()) and bool((grads > 9e29).all())
    assert train() == OK and back() == OK
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(grads).all()
    for t, what in ((saved, "saved"), (ws, "workspace"), (bws, "backward workspace"), (grads, "grads"), (out, "out")):
        check_bands(t, what)


# =====================================================================================================================
# 4. call order on one workspace, through the Python modules
# =====================================================================================================================
def poison_state(m, pattern):
    """Poisons, in place, the workspace (and staging buffer) the module keeps for its next calls."""
    torch.cuda.synchronize()
    st = _engine._state(m, torch.device(DEV, torch.cuda.current_device()))
    for buf in (st.workspace, st.staging):
        if buf is not None:
            repoison(buf, pattern)
    return st


def assert_same(got, want, bitwise, what):
    d = rel(got, want)
    same = torch.equal(got.view(torch.int32), want.view(torch.int32))
    print(f"{what}: {d:.2e}{' (bitwise)' if same else ''}")
    assert same if bitwise else d <= SPREAD, (what, d)


ABA = [("improved", imp(2, 21, 64, Co=32, Ci=64, U=2, D=4)), ("original", orig(2, 21, 32, 32, U=2, D=4)),
       ("groupcomm", gc(2, 1, 21, 64, 2, 16, U=2, D=4)), ("causal", causal(2, 1, 21, 64, 32, 64, U=2, D=4))]


@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
@pytest.mark.parametrize("variant,kw", ABA, ids=[v for v, _ in ABA])
def test_long_short_long_on_one_workspace(variant, kw, pname, pattern):
    """model(x_A) on the pyramid path, model(x_B) on the per-level path inside the same buffer, model(x_A) again without
    re-poisoning: the third result is the first.  Then with separate(), mixture consistency toggled and forward_host
    in the middle."""
    cfg, sd, m = build(variant, kw)
    bitwise = variant == "causal"
    TA, TB = 1600, 150
    if variant != "causal":
        assert takes_pyramid(cfg, 2, TA) and not takes_pyramid(cfg, 3, TB)
    xa, xb = normalised_input(2, 1, TA, seed=6).to(DEV), normalised_input(3, 1, TB, seed=7).to(DEV)
    hb, hout = xb.cpu().pin_memory(), torch.empty(3, 2, TB).pin_memory()
    with torch.no_grad():
        first = m(xa)
        assert max(O.parity_errors(first, O.forward(cfg, sd, xa, dtype=torch.float64))) < TOL
        short = m(xb)
        assert max(O.parity_errors(short, O.forward(cfg, sd, xb, dtype=torch.float64))) < TOL
        st = poison_state(m, pattern)
        ws_ptr = st.workspace.data_ptr()
        a1 = m(xa)
        b1 = m(xb)
        a2 = m(xa)
        assert st.workspace.data_ptr() == ws_ptr, "the module replaced its workspace"
        assert_same(a1, first, bitwise, f"{variant} {pname} A on a poisoned workspace")
        assert_same(b1, short, bitwise, f"{variant} {pname} B inside A's leftovers")
        assert_same(a2, first, bitwise, f"{variant} {pname} A after B")
        # separate(normalize=True) needs a larger workspace: poison it once it exists, then A / B / A again
        sep_first = m.separate(xa * 0.5 + 0.1, normalize=True)
        poison_state(m, pattern)
        s1 = m.separate(xa * 0.5 + 0.1, normalize=True)
        mc_b = m.separate(xb, mixture_consistency=True)
        repoison(hout.view(torch.uint8), pattern)
        m.forward_host(hb, hout)
        torch.cuda.synchronize()
        s2 = m.separate(xa * 0.5 + 0.1, normalize=True)
        a3 = m(xa)
        assert_same(s1, sep_first, bitwise, f"{variant} {pname} separate on a poisoned workspace")
        assert_same(s2, sep_first, bitwise, f"{variant} {pname} separate after B with mixture consistency and forward_host")
        assert_same(a3, first, bitwise, f"{variant} {pname} A at the end")
        assert_same(hout.to(DEV), short, bitwise, f"{variant} {pname} forward_host of B")
        want_mc = O.mixture_consistency(O.forward(cfg, sd, xb, dtype=torch.float64), xb.double())
        assert max(O.parity_errors(mc_b, want_mc)) < TOL
        poison_state(m, pattern)                      # the staging buffer too, then the graph path of forward_host
        for _ in range(3):                            # eager, capture, replay
            repoison(hout.view(torch.uint8), pattern)
            m.forward_host(hb, hout)
            torch.cuda.synchronize()
            assert_same(hout.to(DEV), short, bitwise, f"{variant} {pname} forward_host")
            poison_state(m, pattern)


@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
def test_one_buffer_four_variants(pname, pattern):
    """One poisoned buffer, sized for the largest, handed to sdr_forward of four models in turn, twice round."""
    models = [Model(v, kw) for v, kw in ABA]
    B, T = 2, 1603
    x = normalised_input(B, 1, T, seed=8).to(DEV)
    with torch.no_grad():
        clean = [M.run("forward", x, 0) for M in models]
        for M, y in zip(models, clean):
            assert max(O.parity_errors(y, M.oracle("forward", x, 0))) < TOL
        ws = poisoned(max(M.ws_bytes("forward", B, T) for M in models), pattern)
        for rnd in range(2):
            for M, y in zip(models, clean):
                got = M.run("forward", x, pattern, ws=ws)
                assert_same(got, y, M.variant == "causal", f"{M.variant} {pname} round {rnd}")


@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
@pytest.mark.parametrize("variant,kw", ABA[:2] + ABA[3:], ids=["improved", "original", "causal"])
def test_captured_graph_replays_on_a_poisoned_workspace(variant, kw, pname, pattern):
    """The clear of the statistics is part of the captured forward."""
    cfg, sd, m = build(variant, kw)
    x = normalised_input(2, 1, 1600, seed=9).to(DEV)
    with torch.no_grad():
        eager = m(x)
        assert max(O.parity_errors(eager, O.forward(cfg, sd, x, dtype=torch.float64))) < TOL
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.graph(graph, stream=side):
            y = m(x)
        torch.cuda.current_stream().wait_stream(side)
        for k in range(2):
            poison_state(m, pattern)
            y.fill_(float("nan"))
            graph.replay()
            torch.cuda.synchronize()
            assert_same(y, eager, variant == "causal", f"{variant} {pname} replay {k}")


@gpu
@pytest.mark.parametrize("mc", [False, True])
@pytest.mark.parametrize("kw", [causal(2, 1, 21, 64, 32, 64, U=2, D=3), causal(2, 1, 5, 16, 8, 16, U=1, D=2)],
                         ids=["window_encoder", "ffma_encoder"])
def test_stream_with_poisoned_step_workspace(kw, mc):
    """Six chunks; the step workspace is poisoned between steps, the state lives in a guarded buffer.  Bitwise the
    unpoisoned stream, and model(x) delayed by hop."""
    cfg, sd, m = build("causal", kw)
    enc_mma = N.lib().sdr_encoder_mma_packed_bytes(cfg.enc_num_basis, 1, cfg.enc_kernel_size) > 0
    assert enc_mma == (cfg.enc_num_basis >= 32)
    B, Cs, hop = 3, 2 * granule(cfg), cfg.hop
    x = normalised_input(B, 1, 6 * Cs, seed=10).to(DEV)
    with torch.no_grad():
        plain, s = m.stream(B, Cs, mixture_consistency=mc), m.stream(B, Cs, mixture_consistency=mc)
        s._state = poisoned(s._state.numel(), POISON_NAN)
        s._ws = poisoned(s._ws.numel(), POISON_NAN)
        s.reset()
        want, got = [], []
        for k in range(6):
            chunk = x[..., k * Cs:(k + 1) * Cs]
            want.append(plain.step(chunk))
            torch.cuda.synchronize()
            repoison(s._ws, PATTERNS[k % 2][1])
            got.append(s.step(chunk))
        want, got = torch.cat(want, -1), torch.cat(got, -1)
        assert torch.isfinite(got).all()
        assert torch.equal(got, want) and torch.equal(s.flush(), plain.flush())
        check_bands(s._state, "stream state")
        check_bands(s._ws, "step workspace")
        whole = m.separate(x, mixture_consistency=mc)
        assert torch.equal(got[..., hop:], whole[..., :6 * Cs - hop])
        # reset([j]) on the guarded state: slot j is zero, the others and the bands are as they were
        before = s._state.clone().view(B, -1)
        s.reset([1])
        torch.cuda.synchronize()
        after = s._state.view(B, -1)
        assert not after[1].any() and torch.equal(after[0], before[0]) and torch.equal(after[2], before[2])
        s.reset([B - 1])
        check_bands(s._state, "stream state after reset of the last slot")


@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
def test_corpus_separator_with_every_buffer_poisoned_between_passes(pname, pattern):
    """Buckets in increasing padded length alternate between two slots, and the batches of one slot differ in size: a
    slot serves a large batch, then a small one.  The zero padding of the ragged contract comes from the packing."""
    kw = imp(2, 21, 48, Co=32, Ci=64, U=2, D=4)
    cfg, sd, m = build("improved", kw)
    g = torch.Generator().manual_seed(8)
    lengths = [4000, 3999, 3850, 4001, 2000, 2100, 4000, 3900, 160, 90, 4100, 3841, 30, 2050, 2060]
    wavs = [torch.randn(n, generator=g) * (0.2 + 0.1 * i) + 0.05 * i for i, n in enumerate(lengths)]
    want = separate_corpus(m, wavs, max_batch=4)
    sep = CorpusSeparator(m, max_batch=4)
    for k in range(3):                                   # eager, capture, replay
        got = sep.run(wavs)
        for a, b in zip(got, want):
            assert torch.isfinite(a).all() and torch.equal(a, b.cpu()), f"{pname} pass {k}"
        torch.cuda.synchronize()
        for buf in [sep._ws] + sep._d_in + sep._d_out + sep._d_len + sep._h_in + sep._h_out:
            repoison(buf.view(torch.uint8), pattern)
    assert sep.launches["captured"] > 0 and sep.launches["replayed"] > 0


# =====================================================================================================================
# 5. training: sdr_forward_train and sdr_backward
# =====================================================================================================================
TRAIN = [("D3_levels_B1_pads", imp(2, 21, 64, Co=32, Ci=64, U=2, D=3), 1, 1001),
         ("D4_pyramid_B3", imp(2, 21, 64, Co=32, Ci=64, U=2, D=4), 3, 1600),
         ("D4_pyramid_wgmma_B3_pads", imp(2, 21, 256, Co=128, Ci=128, U=1, D=4), 3, 1443)]


@gpu
@pytest.mark.parametrize("name,kw,B,T", TRAIN, ids=[c[0] for c in TRAIN])
def test_training_on_poisoned_scratch(name, kw, B, T):
    """With one `saved`, a backward on a poisoned workspace into a poisoned gradient buffer is bitwise the clean one
    (every gradient is written, every reduction has a fixed order); with `saved` and the forward's workspace poisoned
    before the forward, the gradients are the clean run's within the forward's run-to-run spread."""
    lib = N.lib()
    M = Model("improved", kw)
    c = M.c
    assert takes_pyramid(M.cfg, B, T) == ("pyramid" in name)
    x = guarded_copy(normalised_input(B, 1, T, seed=11).to(DEV))
    gout = guarded_copy(torch.randn(B, 2, T, generator=torch.Generator().manual_seed(12)).to(DEV))
    nsv, nws = lib.sdr_train_saved_bytes(C.byref(c), B, T), M.ws_bytes("forward", B, T)
    nbw = lib.sdr_backward_workspace_bytes(C.byref(c), B, T)
    ngrad = sum(lib.sdr_param_numel(C.byref(c), i) for i in range(lib.sdr_num_params(C.byref(c))))

    def forward(pattern):
        saved, ws = poisoned(nsv, pattern), poisoned(nws, pattern)
        out = poisoned_like(torch.empty(B, 2, T, device=DEV), pattern or POISON_NAN)
        assert lib.sdr_forward_train(C.byref(c), p(M.packed), p(x), p(out), B, T, p(saved), nsv, p(ws), nws, stream()) == OK
        for t, what in ((saved, "saved"), (ws, "workspace"), (out, "out"), (x, "mixture"), (M.packed, "packed")):
            check_bands(t, f"forward_train {what}")
        assert torch.isfinite(out).all()
        return saved, out

    def backward(saved, pattern):
        ws = poisoned(nbw, pattern)
        grads = poisoned_like(torch.empty(ngrad, device=DEV), pattern or POISON_NAN)
        sv_before = saved.clone()
        assert lib.sdr_backward(C.byref(c), p(M.packed), p(x), p(saved), p(gout), p(grads), B, T, p(ws), nbw, stream()) == OK
        for t, what in ((saved, "saved"), (ws, "workspace"), (grads, "grads"), (gout, "grad_out"), (M.packed, "packed")):
            check_bands(t, f"backward {what}")
        assert torch.equal(saved, sv_before), "the backward wrote `saved`"
        assert torch.isfinite(grads).all(), "a gradient element is not finite or was never written"
        return grads.clone()

    saved, out = forward(0)
    assert max(O.parity_errors(out, O.forward(M.cfg, M.sd, x, dtype=torch.float64))) < TOL
    clean = backward(saved, 0)
    assert torch.equal(backward(saved, 0), clean), "two clean backwards differ"
    for pname, pattern in PATTERNS:
        assert torch.equal(backward(saved, pattern), clean), f"{name}: backward on {pname} scratch"
    saved2, out2 = forward(0)
    spread = rel(backward(saved2, 0), clean)
    assert spread <= SPREAD, spread
    for pname, pattern in PATTERNS:
        sv, o = forward(pattern)
        d_out, d = rel(o, out), rel(backward(sv, pattern), clean)
        print(f"{name}: forward_train on {pname} scratch: out {d_out:.2e}, gradients {d:.2e} (clean / clean {spread:.2e})")
        assert d_out <= SPREAD and d <= SPREAD, (pname, d_out, d)
    # the clean gradients are the autograd module's
    m = M.m
    m.enable_training()
    m.train()
    m.zero_grad(set_to_none=True)
    m(x.clone()).backward(gout.clone())
    flat = torch.cat([_engine._fetch(m, n).grad.reshape(-1) for n in _engine.state_dict_names(c)])
    assert rel(flat, clean) <= SPREAD


# =====================================================================================================================
# 6. entries with their own scratch
# =====================================================================================================================
@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
def test_metrics_on_poisoned_scratch(pname, pattern):
    lib = N.lib()
    B, S, T = 5, 3, 8191
    g = torch.Generator().manual_seed(13)
    tgt = (torch.randn(B, S, T, generator=g) * (0.2 + torch.rand(B, S, 1, generator=g)) + 0.05).to(DEV)
    est = (0.8 * tgt.flip(1) + 0.1 * torch.randn(B, S, T, generator=g).to(DEV)).contiguous()
    mix = tgt.sum(1, keepdim=True).contiguous()
    e, t, mx = guarded_copy(est), guarded_copy(tgt), guarded_copy(mix)
    best = poisoned_like(torch.empty(B, device=DEV), pattern)
    perm = poisoned_like(torch.empty(B, dtype=torch.int32, device=DEV), pattern)
    sc = poisoned(lib.sdr_pit_sisdr_scratch_bytes(B, S), pattern)
    assert lib.sdr_pit_sisdr(p(e), p(t), p(mx), p(best), p(perm), B, S, T, 1, 1, 1e-9, p(sc), stream()) == OK
    want, wi = O.pit_sisdr(est.double(), tgt.double(), mix.double(), zero_mean=True, improvement=True, eps=1e-9)
    for buf, what in ((sc, "pit scratch"), (best, "best"), (perm, "perm"), (e, "est"), (t, "target"), (mx, "mixture")):
        check_bands(buf, what)
    assert torch.allclose(best.double(), want, atol=1e-3, rtol=0) and torch.equal(perm.long(), wi.to(DEV).long())
    # pairwise: the same Gram pass, its own finalize
    pw = poisoned_like(torch.empty(B, S, S, device=DEV), pattern)
    sc = poisoned(lib.sdr_pit_sisdr_scratch_bytes(B, S), pattern)
    assert lib.sdr_pairwise_neg_sdr(p(e), p(t), p(pw), B, S, T, 1, 1, 1, p(sc), stream()) == OK
    check_bands(sc, "pairwise scratch")
    check_bands(pw, "pairwise out")
    assert torch.allclose(pw.double(), O.pairwise_neg_sdr(est.double(), tgt.double(), "sisdr", True, True), atol=1e-3, rtol=0)
    # stabilised: 3 estimates against 2 actual sources
    best = poisoned_like(torch.empty(B, device=DEV), pattern)
    perm = poisoned_like(torch.empty(B, dtype=torch.int32, device=DEV), pattern)
    t2 = guarded_copy(tgt[:, :2].contiguous())
    sc = poisoned(lib.sdr_stabilized_sisdr_scratch_bytes(B, S, 2), pattern)
    assert lib.sdr_stabilized_sisdr(p(e), p(t2), p(best), p(perm), B, S, S, 2, T, 1, 1, 1e-9, p(sc), stream()) == OK
    want, wi = O.stabilized_pit_sisdr(est.double(), tgt[:, :2].double(), zero_mean=True, improvement=True, n_estimated=S)
    for buf, what in ((sc, "stabilised scratch"), (best, "best"), (perm, "perm"), (t2, "target")):
        check_bands(buf, what)
    assert torch.allclose(best.double(), want, atol=1e-3, rtol=0) and torch.equal(perm.long(), wi.to(DEV).long())


def stats_of(x):
    x64 = x.double().reshape(x.shape[0], -1)
    return torch.stack([x64.sum(1), (x64 * x64).sum(1)], 1).contiguous()


def close(got, want, what, tol=1e-4):
    d = float((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-30))
    assert torch.isfinite(got).all() and d <= tol, (what, d)


@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
def test_backward_stage_entries_on_poisoned_scratch(pname, pattern):
    """sdr_pointwise_wgrad, sdr_norm_act_backward, sdr_depthwise_backward and sdr_encoder_wgrad on exactly-sized
    poisoned scratch and poisoned outputs, against fp64 autograd of the single operation."""
    lib = N.lib()
    g = torch.Generator().manual_seed(14)
    rand = lambda *s: torch.randn(*s, generator=g).to(DEV)
    B = 3
    # weight gradient of a 1x1 convolution read through GlobLN + PReLU; 1000 positions: two partial sums per sample
    M_, K_, L = 65, 63, 1000
    dy, x = guarded_copy(rand(B, M_, L)), guarded_copy(rand(B, K_, L) * 2 + 0.3)
    gamma, beta, slope = rand(K_) * 0.3 + 1, rand(K_) * 0.2, torch.tensor([0.3], device=DEV)
    st = stats_of(x)
    fin = N.SdrNormIn(p(st), p(gamma), p(beta), p(slope), float(K_ * L), 0)
    dw, db = poisoned_like(torch.empty(M_, K_, device=DEV), pattern), poisoned_like(torch.empty(M_, device=DEV), pattern)
    sc = poisoned(lib.sdr_pointwise_wgrad_scratch_bytes(B, M_, K_, L), pattern)
    assert lib.sdr_pointwise_wgrad(p(dy), p(x), C.byref(fin), p(dw), p(db), p(sc), B, M_, K_, L, stream()) == OK
    for buf, what in ((sc, "wgrad scratch"), (dw, "dw"), (db, "db"), (dy, "dy"), (x, "x")):
        check_bands(buf, what)
    W = torch.zeros(M_, K_, dtype=torch.float64, device=DEV, requires_grad=True)
    bias = torch.zeros(M_, dtype=torch.float64, device=DEV, requires_grad=True)
    xx = F.prelu(O.glob_ln(x.double(), gamma.double(), beta.double()), slope.double())
    (F.conv1d(xx, W.unsqueeze(-1), bias) * dy.double()).sum().backward()
    close(dw, W.grad, "wgrad dw")
    close(db, bias.grad, "wgrad db")
    # backward of PReLU(GlobLN(x))
    C_, L = 48, 1001
    x, dp = guarded_copy(rand(B, C_, L) * 1.5 + 0.2), guarded_copy(rand(B, C_, L))
    gamma, beta, slope = rand(C_) * 0.3 + 1, rand(C_) * 0.2, torch.tensor([0.27], device=DEV)
    st = stats_of(x)
    fin = N.SdrNormIn(p(st), p(gamma), p(beta), p(slope), float(C_ * L), 0)
    dx = poisoned_like(torch.empty(B, C_, L, device=DEV), pattern)
    dg, dbe, da = (poisoned_like(torch.empty(n, device=DEV), pattern) for n in (C_, C_, 1))
    sc = poisoned(lib.sdr_norm_act_backward_scratch_bytes(B, C_), pattern)
    assert lib.sdr_norm_act_backward(p(x), C.byref(fin), p(dp), p(dx), 0, p(dg), p(dbe), p(da), p(sc), B, C_, L, stream()) == OK
    for buf, what in ((sc, "norm scratch"), (dx, "dx"), (dg, "dgamma"), (dbe, "dbeta"), (da, "dslope"), (x, "x"), (dp, "dp")):
        check_bands(buf, what)
    x64, g64, b64, a64 = (v.double().requires_grad_(True) for v in (x, gamma, beta, slope))
    (F.prelu(O.glob_ln(x64, g64, b64), a64) * dp.double()).sum().backward()
    for got, want, what in ((dx, x64.grad, "dx"), (dg, g64.grad, "dgamma"), (dbe, b64.grad, "dbeta"), (da, a64.grad, "dslope")):
        close(got, want, "norm/act " + what)
    # backward of a stride-2 depthwise level with the pooled merge gradient added
    C_, Lin, pool = 48, 64, 4
    x, dz = guarded_copy(rand(B, C_, Lin) + 0.1), guarded_copy(rand(B, C_, Lin // 2))
    gamma, beta, w5 = rand(C_) * 0.3 + 1, rand(C_) * 0.2, rand(C_, 5) * 0.4
    dm = guarded_copy(rand(B, C_, Lin * pool))
    st = stats_of(x)
    fin = N.SdrNormIn(p(st), p(gamma), p(beta), None, float(C_ * Lin), 0)
    dx = poisoned_like(torch.empty(B, C_, Lin, device=DEV), pattern)
    dw, db = poisoned_like(torch.empty(C_, 5, device=DEV), pattern), poisoned_like(torch.empty(C_, device=DEV), pattern)
    sc = poisoned(lib.sdr_depthwise_backward_scratch_bytes(B, C_), pattern)
    assert lib.sdr_depthwise_backward(p(dz), p(x), C.byref(fin), p(w5), p(dm), pool, p(dx), p(dw), p(db), p(sc), B, C_,
                                      Lin, 2, stream()) == OK
    for buf, what in ((sc, "depthwise scratch"), (dx, "dx"), (dw, "dw5"), (db, "dbias"), (x, "x"), (dz, "dz"), (dm, "pool")):
        check_bands(buf, what)
    n64 = O.glob_ln(x.double(), gamma.double(), beta.double()).requires_grad_(True)
    w64 = w5.double().requires_grad_(True)
    b64 = torch.zeros(C_, dtype=torch.float64, device=DEV, requires_grad=True)
    (F.conv1d(n64, w64.unsqueeze(1), b64, stride=2, padding=2, groups=C_) * dz.double()).sum().backward()
    close(dx, n64.grad + dm.double().reshape(B, C_, Lin, pool).sum(-1), "depthwise dx")
    close(dw, w64.grad, "dw5")
    close(db, b64.grad, "dbias")
    # encoder weight gradient: the gathered windows and the partial sums share one scratch
    K, T, Nb = 21, 999, 64
    cfg = O.Config(variant="improved", enc_kernel_size=K, upsampling_depth=2)
    L = O.padded_length(cfg, T) // cfg.hop
    wav, de = guarded_copy(rand(B, 1, T)), guarded_copy(rand(B, Nb, L))
    dw = poisoned_like(torch.empty(Nb, K, device=DEV), pattern)
    sc = poisoned(lib.sdr_encoder_wgrad_scratch_bytes(B, Nb, K, L), pattern)
    assert lib.sdr_encoder_wgrad(p(de), p(wav), p(dw), p(sc), B, Nb, K, L, T, stream()) == OK
    for buf, what in ((sc, "encoder wgrad scratch"), (dw, "dw"), (wav, "wav"), (de, "denc")):
        check_bands(buf, what)
    W = torch.zeros(Nb, 1, K, dtype=torch.float64, device=DEV, requires_grad=True)
    (F.conv1d(O.pad_wave(cfg, wav, torch.float64), W, None, stride=cfg.hop, padding=cfg.hop) * de.double()).sum().backward()
    close(dw, W.grad.reshape(Nb, K), "encoder wgrad")


@gpu
@pytest.mark.parametrize("pname,pattern", PATTERNS, ids=[n for n, _ in PATTERNS])
@pytest.mark.parametrize("D,L", [(4, 160), (5, 3728)])
def test_pyramid_entries_on_poisoned_scratch_and_preloaded_stats(D, L, pname, pattern):
    """sdr_depthwise_pyramid + sdr_merge_pyramid and sdr_depthwise_pyramid_fused on exactly-sized poisoned scratch (row
    statistics and coefficient table) against the fp64 level-by-level chain, m of the two bitwise equal.  `stats0` and
    `stats_m` are the caller's to zero: pre-loaded slots come back as pre-load + the sums."""
    lib = N.lib()
    samples, C_ = 3, 12
    g = torch.Generator().manual_seed(15)
    rand = lambda *s: torch.randn(*s, generator=g).to(DEV)
    y = guarded_copy(rand(samples, C_, L) * 1.3 + 0.3)
    gy, by, slope = 1 + 0.3 * rand(C_), 0.2 * rand(C_), torch.tensor([0.3], device=DEV)
    ws = [rand(C_, 1, 5) * 0.6 for _ in range(D)]
    bs = [rand(C_) * 0.5 for _ in range(D)]
    gs = [1 + 0.3 * rand(C_) for _ in range(D)]
    bes = [0.2 * rand(C_) for _ in range(D)]
    cur = O.prelu1(O.glob_ln(y.double(), gy.double(), by.double()), slope.double())
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
    want_m = levels[0]
    nbytes = lib.sdr_pyramid_scratch_bytes(samples, C_, D, L)
    assert nbytes > 0
    arr = lambda ts: (C.c_void_p * D)(*[t.data_ptr() for t in ts])
    st_y = stats_of(y)
    nin = N.SdrNormIn(p(st_y), p(gy), p(by), p(slope), float(C_ * L), 0)
    preload = torch.tensor([[3.0, 5.0], [-7.0, 11.0], [0.5, 2.0]], dtype=torch.float64, device=DEV)

    def stats(pre):
        return guarded_copy(preload.clone() if pre else torch.zeros(samples, 2, dtype=torch.float64, device=DEV))

    # stats0 is also read, by the solve, as level 0's statistics: a pre-loaded stats0 changes m, so m and stats_m are
    # compared in the runs that zero it
    results = {}
    for pre0, prem in ((False, False), (False, True), (True, False)):
        # two launches, the levels in HBM
        sc = poisoned(nbytes, pattern)
        zs = [poisoned_like(torch.empty(samples, C_, L >> d, device=DEV), pattern) for d in range(D)]
        m2 = poisoned_like(torch.empty(samples, C_, L, device=DEV), pattern)
        s0, sm = stats(pre0), stats(prem)
        assert lib.sdr_depthwise_pyramid(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), arr(zs), p(s0), p(sc),
                                         D, samples, C_, L, stream()) == OK
        assert lib.sdr_merge_pyramid(arr(zs), p(sc), D, p(m2), p(sm), samples, C_, L, stream()) == OK
        for buf, what in [(sc, "scratch"), (m2, "m"), (s0, "stats0"), (sm, "stats_m"), (y, "y")] + [(z, "z") for z in zs]:
            check_bands(buf, f"pyramid {what}")
        # one fused stage
        scf = poisoned(nbytes, pattern)
        mf = poisoned_like(torch.empty(samples, C_, L, device=DEV), pattern)
        s0f, smf = stats(pre0), stats(prem)
        assert lib.sdr_depthwise_pyramid_fused(p(y), C.byref(nin), arr(ws), arr(bs), arr(gs), arr(bes), p(mf), p(s0f),
                                               p(smf), p(scf), D, samples, C_, L, stream()) == OK
        for buf, what in ((scf, "scratch"), (mf, "m"), (s0f, "stats0"), (smf, "stats_m"), (y, "y")):
            check_bands(buf, f"fused pyramid {what}")
        assert torch.isfinite(mf).all() and torch.equal(mf, m2), "the fused stage's merge is not the two-launch one"
        if not pre0:
            close(mf, want_m, "merge")
        results[(pre0, prem)] = (s0.clone(), sm.clone(), s0f.clone(), smf.clone(), mf.clone())
    zero, loaded_m, loaded_0 = results[(False, False)], results[(False, True)], results[(True, False)]
    assert torch.equal(loaded_m[4], zero[4]), "a pre-loaded stats_m changed m"
    for k, want, what in ((0, stats_of(z0), "stats0"), (1, stats_of(want_m), "stats_m"), (2, stats_of(z0), "fused stats0"),
                          (3, stats_of(want_m), "fused stats_m")):
        assert torch.allclose(zero[k], want, rtol=1e-4, atol=1e-2), what
        loaded = loaded_0 if k % 2 == 0 else loaded_m
        assert torch.allclose(loaded[k] - preload, zero[k], rtol=1e-9, atol=1e-6), f"{what}: not pre-load + sums"
