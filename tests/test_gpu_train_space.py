"""The improved model's native backward across every depth, source count, filter length, block count, channel count,
length and batch it accepts, at bars that see one wrong position per (sample, channel) row.

Whole-model gradients are compared with fp64 autograd through the oracle in two tiers:

- Tier A, a model with no branch point near zero: every shared PReLU slope is 1.0 (the identity, whose slope gradient
  sum dp * min(v, 0) the kernels still compute) and each row of ``mask_net.1.bias`` is shifted so that the fp64 mask
  logits of that row sit at least 5% of the logits' RMS above zero at every (sample, position), far beyond the ~1e-5
  error of the tensor-core forward.  The native gradient then differs from fp64 only by rounding: every tensor and
  the whole gradient are held (rel-L2 and rel-max) to 1e-4 when all 1x1 convolutions of the forward run on FFMA, and
  to max(1e-3, 3x the fp32 eager error) when any runs on the tensor cores.
- Tier B, models whose every GEMM runs on FFMA (by the library's own eligibility queries), with perturbed slopes and
  the real ReLU mask, under the projection loss and the PIT SI-SDR loss: 1e-3 per tensor and for the whole gradient.

A scalar PReLU slope's gradient is a sum over B * C * L terms that cancels; it is held to tol * sum |dp * min(v, 0)|,
dp and v captured in the fp64 oracle at the PReLU.  Each case asserts which GEMMs run on the tensor cores, and
prints the native and fp32 eager (TF32 off) errors.  One missing position per row moves a gradient by about
1/sqrt(L) (2e-2 at L = 3200, 8e-3 at L = 16000), a slope gradient by about 1/L of its scale.

Measured worst cases on an H100 80GB HBM3 at a 700 W power limit (per tensor, slopes scaled as above):
- tier A, tensor-core forward: 1.2e-4 (t161, proj_1x1.norm.beta); whole gradient 1.7e-5 rel-L2, 3.4e-5 rel-max;
- tier A, FFMA forward: 1.3e-6;
- tier B: 3.0e-6 (PIT loss at K = 3, D = 1).
Removing one term per row (the last position of the depthwise backward, of a weight-gradient chunk, of the frame
gather or of a slope sum, or one pooled position at P >= 64) fails tier A at 1.2e-3 to 1.5e-1.

Then the stage entries in the modes the backward calls them, the contracts (bitwise reproducibility, the launch count,
training at more than 65535 weight-gradient partials), and the autograd plumbing."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as NAT
from oracle import sudormrf_oracle as O
from test_gpu_train import (_kernel_nodes, check, grad_errors, make_batch, native_model, norm_in, pit_loss,
                            projection_loss, ptr, rand, ref_norm_act, stats_of, stream)

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
TOL = 1e-3              # stages, tier B, and tier A with a tensor-core forward
TOL_FFMA = 1e-4         # tier A with every 1x1 convolution on FFMA
MARGIN = 0.05           # tier A: mask logits at least this fraction of their RMS above zero
CONVS = ("enc", "bn", "proj", "res", "mask", "dec")


def imp(S=2, K=21, N=128, Co=64, Ci=128, U=2, D=4):
    return dict(out_channels=Co, in_channels=Ci, num_blocks=U, upsampling_depth=D, enc_kernel_size=K,
                enc_num_basis=N, num_sources=S)


def frames(kw, T):
    cfg = O.Config(variant="improved", **kw)
    return O.padded_length(cfg, T) // cfg.hop


def tc_convs(kw, T):
    """The 1x1 convolutions (and the encoder) the forward runs on the tensor cores, by the library's own rules: a
    packed image (M >= 32, Kc a multiple of 64; the encoder: N >= 32), L % 4 == 0 for the GEMMs, and the mask GEMM's
    gated epilogue only when N % 256 == 0."""
    lib = NAT.lib()
    S, N, K = kw["num_sources"], kw["enc_num_basis"], kw["enc_kernel_size"]
    Co, Ci, U = kw["out_channels"], kw["in_channels"], kw["num_blocks"]
    L = frames(kw, T)

    def mma(M, Kc):
        return L % 4 == 0 and lib.sdr_pointwise_mma_packed_bytes(M, Kc) > 0
    on = {"enc": lib.sdr_encoder_mma_packed_bytes(N, 1, K) > 0, "bn": mma(Co, N), "proj": U > 0 and mma(Ci, Co),
          "res": U > 0 and mma(Co, Ci), "mask": N % 256 == 0 and mma(S * N, Co), "dec": mma(S * K, S * N)}
    return tuple(c for c in CONVS if on[c])


def batch(B, T, seed=1):
    """B >= 3: sample 1 silent, sample 2 a DC offset with a little signal."""
    return make_batch(B, T, seed=seed, silent_dc=B >= 3)


def oracle_grads(cfg, sd, x, loss_fn, dtype=F64, taps=None):
    """Autograd through the oracle (PReLU as nn.PReLU, F.prelu) -> (gradients, slope scales, loss).  The scale of a
    scalar slope is sum |dp * min(v, 0)| over its input v and output gradient dp."""
    sdd = {k: v.to(DEV, dtype).requires_grad_(True) for k, v in sd.items()}
    names = {id(v): k for k, v in sdd.items()}
    scale = {}

    def prelu(v, slope):
        out = F.prelu(v, slope.reshape(1))
        name, neg = names[id(slope)], v.detach().clamp(max=0.0)
        out.register_hook(lambda g: scale.__setitem__(name, (g * neg).abs().sum().item()))
        return out
    old = O.prelu1
    O.prelu1 = prelu
    try:
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            y = O.forward(cfg, sdd, x.to(DEV, dtype), taps=taps, dtype=dtype)
            loss = loss_fn(y)
            loss.backward()
    finally:
        O.prelu1 = old
    return {k: v.grad for k, v in sdd.items()}, scale, loss.item()


def native_grads(m, x, loss_fn):
    m.zero_grad(set_to_none=True)
    y = m(x.to(DEV))
    loss = loss_fn(y)
    loss.backward()
    return {n: p.grad for n, p in m.named_parameters()}, loss.item()


def mask_input(cfg, taps):
    return taps[f"sm.{cfg.num_blocks - 1}.out"] if cfg.num_blocks else taps["bottleneck"]


def mask_logits(cfg, sd, taps):
    return F.conv1d(mask_input(cfg, taps), sd["mask_net.1.weight"].to(DEV, F64), sd["mask_net.1.bias"].to(DEV, F64))


def smooth_state_dict(cfg, x, seed):
    """Tier A weights: perturbed, every scalar PReLU slope 1.0, and each mask-logit row shifted above zero by at
    least MARGIN times the logits' RMS over every (sample, position) of x.  Returns (state_dict, margin)."""
    sd = O.make_state_dict(cfg, seed=seed, perturbed=True)
    for k in sd:
        if k.endswith("act.weight") or k == "mask_net.0.weight":
            sd[k] = torch.ones_like(sd[k])
    taps = {}
    with torch.no_grad():
        O.forward(cfg, {k: v.to(DEV, F64) for k, v in sd.items()}, x.to(DEV, F64), taps=taps, dtype=F64)
    logits = mask_logits(cfg, sd, taps)
    margin = MARGIN * logits.pow(2).mean().sqrt().item()
    low = logits.amin(dim=(0, 2))
    b = sd["mask_net.1.bias"].to(DEV, F64)
    sd["mask_net.1.bias"] = (b + (1.01 * margin - low).clamp_min(0.0)).float().cpu()
    return sd, margin


def compare(got, ref, scale, label, tol, eager=None, eager_factor=None):
    """Every tensor and the whole flattened gradient within the bar, rel-L2 and rel-max; a scalar slope within
    bar * its scale.  With `eager_factor` the bar is max(tol, eager_factor x the fp32 eager error of the same
    measure).  Prints the worst native and fp32 eager errors."""
    bad = []
    worst, worst_e = ("", 0.0), ("", 0.0)
    acc = {"n": [0.0, 0.0], "e": [0.0, 0.0]}                 # native / eager: sum d^2, max |d|
    rmax = rsq = 0.0
    for name, r in ref.items():
        g = got[name]
        assert g is not None, name
        e = eager[name] if eager is not None else None
        rsq += (r ** 2).sum().item()
        rmax = max(rmax, r.abs().max().item())
        for key, t in (("n", g), ("e", e)):
            if t is None:
                continue
            d = t.double() - r
            acc[key][0] += (d ** 2).sum().item()
            acc[key][1] = max(acc[key][1], d.abs().max().item())
        if r.numel() == 1:
            s = max(scale[name], 1e-300)
            errs = (abs(g.double().item() - r.item()) / s,) * 2
            errs_e = (abs(e.double().item() - r.item()) / s,) * 2 if e is not None else (0.0, 0.0)
        else:
            errs = grad_errors(g, r)
            errs_e = grad_errors(e, r) if e is not None else (0.0, 0.0)
        bars = [max(tol, eager_factor * x) if eager_factor else tol for x in errs_e]
        if max(errs) > worst[1]:
            worst = (name, max(errs))
        if max(errs_e) > worst_e[1]:
            worst_e = (name, max(errs_e))
        if not (errs[0] <= bars[0] and errs[1] <= bars[1]):
            bad.append((name, errs, bars))
    whole = ((acc["n"][0] / rsq) ** 0.5, acc["n"][1] / rmax)
    whole_e = ((acc["e"][0] / rsq) ** 0.5, acc["e"][1] / rmax)
    print(f"{label}: native worst {worst[0]} {worst[1]:.2e}, whole rel_l2={whole[0]:.2e} rel_max={whole[1]:.2e}; "
          f"fp32 eager worst {worst_e[0]} {worst_e[1]:.2e}, whole rel_l2={whole_e[0]:.2e} rel_max={whole_e[1]:.2e}")
    assert not bad, bad
    for x, xe in zip(whole, whole_e):
        assert x <= (max(tol, eager_factor * xe) if eager_factor else tol), (label, whole, whole_e)


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 3. tier A: every axis around a small base, one at a time
# ---------------------------------------------------------------------------------------------------------------------
ALL = CONVS
NO_MASK = ("enc", "bn", "proj", "res", "dec")          # N % 256 != 0: the mask GEMM runs on FFMA
U16 = imp(K=21, N=512, Co=256, Ci=512, U=16, D=5)
FFMA_KW = imp(N=24, Co=48, Ci=96)                       # N < 32, no Kc a multiple of 64, N % 256 != 0
AXES = [
    # id, kwargs, B, T, GEMMs on the tensor cores
    ("base", imp(), 3, 2000, NO_MASK),
    ("ffma", FFMA_KW, 3, 2000, ()),
    # depth: L = 200 (D 1-3), 208, 224, 256 (D 6-8: the deepest level is 2 frames at D = 8)
    *[(f"depth{D}", imp(D=D), 3, 2000, NO_MASK) for D in (1, 2, 3, 5, 6, 7, 8)],
    # sources; S = 16 at N = 16 runs the FFMA encoder and bottleneck
    ("sources1", imp(S=1), 3, 2000, ("enc", "bn", "proj", "res")),           # 21 decoder rows
    *[(f"sources{S}", imp(S=S), 3, 2000, NO_MASK) for S in (3, 4, 8)],
    ("sources16_n16", imp(S=16, N=16), 3, 2000, ("proj", "res", "dec")),
    # filter length: hop 1, 2, 10, 20, 31
    ("kernel3", imp(K=3), 3, 2000, ("enc", "bn", "proj", "res")),
    ("kernel5", imp(K=5), 3, 2000, ("enc", "bn", "proj", "res")),
    ("kernel41", imp(K=41), 3, 2000, NO_MASK),
    ("kernel63", imp(K=63), 3, 2000, NO_MASK),
    # blocks: none (the mask reads the bottleneck), one, three, and sixteen at full width
    ("blocks0", imp(U=0), 3, 2000, ("enc", "bn", "dec")),
    ("blocks1", imp(U=1), 3, 2000, NO_MASK),
    ("blocks3", imp(U=3), 3, 2000, NO_MASK),
    ("u16_512", U16, 2, 8000, ALL),
    # channel counts at the 64-wide wgrad tile edges (base Co = 64, Ci = 128, N = 128)
    ("co16", imp(Co=16), 3, 2000, ("enc", "dec")),
    ("co31", imp(Co=31), 3, 2000, ("enc", "dec")),
    *[(f"co{c}", imp(Co=c), 3, 2000, ("enc", "bn", "res", "dec")) for c in (32, 63, 65)],
    *[(f"co{c}", imp(Co=c), 3, 2000, NO_MASK) for c in (128, 192, 256)],
    *[(f"ci{c}", imp(Ci=c), 3, 2000, ("enc", "bn", "dec")) for c in (16, 31)],
    *[(f"ci{c}", imp(Ci=c), 3, 2000, ("enc", "bn", "proj", "dec")) for c in (32, 63, 65)],
    *[(f"ci{c}", imp(Ci=c), 3, 2000, NO_MASK) for c in (64, 192, 256)],
    *[(f"n{c}", imp(N=c), 3, 2000, ("proj", "res")) for c in (16, 31)],
    ("n32", imp(N=32), 3, 2000, ("enc", "proj", "res", "dec")),
    *[(f"n{c}", imp(N=c), 3, 2000, ("enc", "proj", "res")) for c in (63, 65)],
    *[(f"n{c}", imp(N=c), 3, 2000, NO_MASK) for c in (64, 192)],
    ("n256", imp(N=256), 3, 2000, ALL),
    ("n256_s3", imp(S=3, N=256), 3, 2000, ALL),
    # lengths: hop * 2^D = 160; L = 16 (below, at and one past one multiple), 160 / 176, 512, 528, 1040
    *[(f"t{T}", imp(), 3, T, NO_MASK) for T in (159, 160, 161, 1599, 1601)],
    ("l512", imp(), 3, 5120, NO_MASK),
    ("l528", imp(), 3, 5280, NO_MASK),
    ("l1040", imp(), 3, 10400, NO_MASK),
    ("l102_d1", imp(D=1), 3, 1001, ("enc",)),             # L = 102 is not a multiple of 4: every GEMM on FFMA
    ("u16_512_10s", U16, 1, 160000, ALL),                  # 10 s at 16 kHz: L = 16000
    # batch
    *[(f"batch{B}", imp(), B, 2000, NO_MASK) for B in (1, 2, 5, 33)],
]


@pytest.mark.parametrize("name,kw,B,T,want", AXES, ids=[a[0] for a in AXES])
def test_tier_a_smooth_model(name, kw, B, T, want):
    cfg = O.Config(variant="improved", **kw)
    paths = tc_convs(kw, T)
    assert paths == want, (paths, want)
    x = batch(B, T)
    sd, margin = smooth_state_dict(cfg, x, seed=31)
    loss = projection_loss(B, kw["num_sources"], T)
    taps = {}
    ref, scale, _ = oracle_grads(cfg, sd, x, loss, taps=taps)
    low = mask_logits(cfg, sd, taps).min().item()
    assert low >= margin, (low, margin)
    eager, _, _ = oracle_grads(cfg, sd, x, loss, dtype=torch.float32)
    got, _ = native_grads(native_model(kw, sd), x, loss)
    label = f"tier A {name} L={frames(kw, T)} tensor cores {paths or 'none'}"
    if paths:
        compare(got, ref, scale, label, TOL, eager, eager_factor=3)
    else:
        compare(got, ref, scale, label, TOL_FFMA, eager)


# ---------------------------------------------------------------------------------------------------------------------
# 2. tier B: every GEMM on FFMA, perturbed slopes, the real ReLU mask
# ---------------------------------------------------------------------------------------------------------------------
FFMA = [
    # N < 32: FFMA encoder; Co = 48 / Ci = 96 / S*N = 48: no k-block multiple of 64; N % 256 != 0: FFMA mask
    ("ffma_base", imp(N=24, Co=48, Ci=96), 3, 2000),
    ("ffma_s3_k41_d6", imp(S=3, K=41, N=24, Co=48, Ci=96, D=6), 2, 3001),
    ("ffma_s1_k3_d1_odd", imp(S=1, K=3, N=24, Co=48, Ci=96, D=1), 1, 1001),
    ("ffma_k5_d8", imp(K=5, N=24, Co=48, Ci=96, D=8), 2, 3000),
    ("ffma_b5_u3", imp(N=24, Co=48, Ci=96, U=3), 5, 1500),
]


@pytest.mark.parametrize("loss_kind", ["projection", "pit"])
@pytest.mark.parametrize("name,kw,B,T", FFMA, ids=[f[0] for f in FFMA])
def test_tier_b_ffma_model(name, kw, B, T, loss_kind):
    assert tc_convs(kw, T) == (), tc_convs(kw, T)
    cfg = O.Config(variant="improved", **kw)
    sd = O.make_state_dict(cfg, seed=41, perturbed=True)
    x = batch(B, T, seed=2)
    if loss_kind == "projection":
        loss = projection_loss(B, kw["num_sources"], T)
    else:
        loss = pit_loss(torch.randn(B, kw["num_sources"], T, generator=torch.Generator().manual_seed(5)))
    ref, scale, lr = oracle_grads(cfg, sd, x, loss)
    eager, _, _ = oracle_grads(cfg, sd, x, loss, dtype=torch.float32)
    got, ln = native_grads(native_model(kw, sd), x, loss)
    assert abs(ln - lr) <= 1e-4 * max(1.0, abs(lr)), (ln, lr)
    compare(got, ref, scale, f"tier B {name} {loss_kind} L={frames(kw, T)}", TOL, eager)


# ---------------------------------------------------------------------------------------------------------------------
# 4. stage entries, in the modes the backward calls them
# ---------------------------------------------------------------------------------------------------------------------
FINS = ("none", "gln", "prelu", "gln_prelu")      # how the wgrad operand is read: the mask reads x_U through PReLU,
WG_MK = [(1, 129), (63, 64), (64, 65), (65, 63), (129, 1)]   # the bottleneck e through GLN, res_conv through both
WG_L = (1, 15, 16, 17, 511, 512, 513, 16000)
WG_CASES = [(fin, L, *WG_MK[(i + j) % len(WG_MK)]) for i, fin in enumerate(FINS) for j, L in enumerate(WG_L)]


def fin_of(fin, x, C_, L, gamma, beta, slope):
    """(sdr_norm_in, fp64 values the kernel should read, the statistics tensor the sdr_norm_in points to)."""
    norm, act = "gln" in fin, "prelu" in fin
    if fin == "none":
        return None, x.double(), None
    st = stats_of(x) if norm else None
    nin = norm_in(st, gamma if norm else None, beta if norm else None, slope if act else None, C_ * L)
    v = ref_norm_act(x.double(), gamma.double() if norm else None, beta.double(), slope.double() if act else None)
    return nin, v, st


def run_wgrad(samples, M, K, L, fin, bias=True, seed=0):
    dy, x = rand(samples, M, L, seed=seed + 1), rand(samples, K, L, seed=seed + 2, scale=2.0) + 0.3
    gamma, beta = rand(K, seed=seed + 3) * 0.3 + 1, rand(K, seed=seed + 4) * 0.2
    slope = torch.tensor([0.3], device=DEV)
    nin, xx, _st = fin_of(fin, x, K, L, gamma, beta, slope)
    dw = torch.full((M, K), float("nan"), device=DEV)
    db = torch.full((M,), float("nan"), device=DEV) if bias else None
    lib = NAT.lib()
    scratch = torch.empty(lib.sdr_pointwise_wgrad_scratch_bytes(samples, M, K, L), dtype=torch.uint8, device=DEV)
    NAT.check(lib.sdr_pointwise_wgrad(ptr(dy), ptr(x), C.byref(nin) if nin else None, ptr(dw), ptr(db), ptr(scratch),
                                      samples, M, K, L, stream()), "sdr_pointwise_wgrad")
    check(dw, torch.einsum("bml,bkl->mk", dy.double(), xx), f"wgrad {samples}x{M}x{K} L={L} {fin}")
    if bias:
        check(db, dy.double().sum((0, 2)), "bias")


@pytest.mark.parametrize("fin,L,M,K", WG_CASES)
def test_stage_wgrad_input_modes(fin, L, M, K):
    run_wgrad(2, M, K, L, fin)


@pytest.mark.parametrize("samples,M,K,L,bias", [(64, 65, 63, 513, False), (64, 129, 64, 17, True),
                                                 (33, 64, 65, 1040, False)])
def test_stage_wgrad_many_samples(samples, M, K, L, bias):
    run_wgrad(samples, M, K, L, "gln_prelu", bias=bias)


def test_stage_wgrad_past_65535_partials():
    """samples * ceil(L / 512) = 66000 * 2 partials: more than a grid's y or z dimension holds."""
    run_wgrad(66000, 3, 2, 513, "gln_prelu")


def run_norm_act(B, C_, L, norm, act, mode="plain", outs=(True, True, True), x=None, seed=0):
    """sdr_norm_act_backward against fp64 autograd.  mode: "plain", "accumulate" (dx += over a nonzero dx), or
    "alias" (dx is dp, as every block calls it)."""
    if x is None:
        x = rand(B, C_, L, seed=seed + 5, scale=1.5) + 0.2
    dp = rand(B, C_, L, seed=seed + 6)
    gamma, beta = rand(C_, seed=seed + 7) * 0.3 + 1, rand(C_, seed=seed + 8) * 0.2
    slope = torch.tensor([0.27], device=DEV)
    st = stats_of(x) if norm else None
    fin = norm_in(st, gamma if norm else None, beta if norm else None, slope if act else None, C_ * L)
    dp0 = dp.clone()
    base = rand(B, C_, L, seed=seed + 9) if mode == "accumulate" else None
    dx = dp if mode == "alias" else (base.clone() if base is not None else torch.empty_like(x))
    nan = float("nan")
    dg, dbeta, da = (torch.full(s, nan, device=DEV) if o else None for s, o in zip(((C_,), (C_,), (1,)), outs))
    lib = NAT.lib()
    scratch = torch.empty(lib.sdr_norm_act_backward_scratch_bytes(B, C_), dtype=torch.uint8, device=DEV)
    NAT.check(lib.sdr_norm_act_backward(ptr(x), C.byref(fin), ptr(dp), ptr(dx), int(mode == "accumulate"), ptr(dg),
                                        ptr(dbeta), ptr(da), ptr(scratch), B, C_, L, stream()),
              "sdr_norm_act_backward")
    x64 = x.double().requires_grad_(True)
    g64, b64, a64 = (t.double().requires_grad_(True) for t in (gamma, beta, slope))
    v = ref_norm_act(x64, g64 if norm else None, b64, a64 if act else None)
    (v * dp0.double()).sum().backward()
    want = x64.grad + (base.double() if base is not None else 0.0)
    label = f"norm/act B={B} C={C_} L={L} norm={norm} act={act} {mode}"
    check(dx, want, label)
    if norm and dg is not None:
        check(dg, g64.grad, label + " dgamma")
    if norm and dbeta is not None:
        check(dbeta, b64.grad, label + " dbeta")
    if act and da is not None:
        # the slope gradient cancels: scale it by sum |dp * min(v, 0)|
        pre = ref_norm_act(x.double(), gamma.double() if norm else None, beta.double(), None)
        s = (dp0.double() * pre.clamp(max=0.0)).abs().sum().item()
        err = abs(da.double().item() - a64.grad.item()) / s
        print(f"{label} dslope: err/scale={err:.2e}")
        assert err <= TOL, (label, err)
    return dx


NA_MODES = [(True, False), (False, True), (True, True)]


@pytest.mark.parametrize("mode", ["accumulate", "alias"])
@pytest.mark.parametrize("norm,act", NA_MODES, ids=["gln", "prelu", "gln_prelu"])
def test_stage_norm_act_accumulate_and_alias(norm, act, mode):
    run_norm_act(3, 96, 333, norm, act, mode)


@pytest.mark.parametrize("outs", [(g, b, a) for g in (True, False) for b in (True, False) for a in (True, False)],
                         ids=lambda o: "".join("gbs"[i] if v else "-" for i, v in enumerate(o)))
def test_stage_norm_act_null_outputs(outs):
    run_norm_act(2, 64, 201, True, True, "alias", outs)


@pytest.mark.parametrize("B,C_,L", [(2, 2048, 150), (300, 3, 40), (257, 5, 17)])
def test_stage_norm_act_wide_and_many_samples(B, C_, L):
    run_norm_act(B, C_, L, True, True)


@pytest.mark.parametrize("mean,spread", [(10.0, 1.0), (1e3, 10.0), (1e3, 1.0), (1e3, 1e-2)])
def test_stage_norm_act_ill_conditioned(mean, spread):
    """Rows at |mean| / std up to 1e5 (the sign alternating over samples), against a two-pass fp64 GLN."""
    B, C_, L = 4, 32, 500
    g = torch.Generator().manual_seed(17)
    x = torch.randn(B, C_, L, generator=g, dtype=F64)
    x = (x - x.mean((1, 2), keepdim=True)) / x.std((1, 2), keepdim=True)
    sign = torch.tensor([1.0, -1.0, 1.0, -1.0], dtype=F64).view(B, 1, 1)
    run_norm_act(B, C_, L, True, True, "alias", x=(mean * sign + spread * x).float().to(DEV))


def run_depthwise(B, C_, Lin, stride, fin, pool, seed=0):
    """sdr_depthwise_backward against fp64 autograd; fin None = pool only (dz NULL)."""
    Lout = Lin // stride
    x, dz = rand(B, C_, Lin, seed=seed + 9) + 0.1, rand(B, C_, Lout, seed=seed + 10)
    gamma, beta = rand(C_, seed=seed + 11) * 0.3 + 1, rand(C_, seed=seed + 12) * 0.2
    slope = torch.tensor([0.31], device=DEV)
    w5 = rand(C_, 5, seed=seed + 13) * 0.4
    dm = rand(B, C_, Lin * pool, seed=seed + 14) if pool else None
    dx = torch.full_like(x, float("nan"))
    lib = NAT.lib()
    if fin is None:
        NAT.check(lib.sdr_depthwise_backward(None, None, None, None, ptr(dm), pool, ptr(dx), None, None, None,
                                             B, C_, Lin, stride, stream()), "sdr_depthwise_backward (pool only)")
        check(dx, dm.double().reshape(B, C_, Lin, pool).sum(-1), f"depthwise pool only P={pool} Lin={Lin}")
        return
    nin, n, _st = fin_of(fin, x, C_, Lin, gamma, beta, slope)
    dw, db = torch.full((C_, 5), float("nan"), device=DEV), torch.full((C_,), float("nan"), device=DEV)
    scratch = torch.empty(lib.sdr_depthwise_backward_scratch_bytes(B, C_), dtype=torch.uint8, device=DEV)
    NAT.check(lib.sdr_depthwise_backward(ptr(dz), ptr(x), C.byref(nin) if nin else None, ptr(w5), ptr(dm), pool,
                                         ptr(dx), ptr(dw), ptr(db), ptr(scratch), B, C_, Lin, stride, stream()),
              "sdr_depthwise_backward")
    n = n.detach().requires_grad_(True)
    w64 = w5.double().requires_grad_(True)
    b64 = torch.zeros(C_, dtype=F64, device=DEV, requires_grad=True)
    z = F.conv1d(n, w64.unsqueeze(1), b64, stride=stride, padding=2, groups=C_)
    assert z.shape[-1] == Lout
    (z * dz.double()).sum().backward()
    want = n.grad + (dm.double().reshape(B, C_, Lin, pool).sum(-1) if pool else 0.0)
    label = f"depthwise {fin} s={stride} P={pool} C={C_} Lin={Lin}"
    check(dx, want, label)
    check(dw, w64.grad, label + " dw5")
    check(db, b64.grad, label + " dbias")


@pytest.mark.parametrize("stride,pool,Lin", [(1, 0, 1000), (1, 0, 17), (2, 2, 64), (2, 1, 1000)])
def test_stage_depthwise_through_gln_prelu(stride, pool, Lin):
    """Level 0 reads PReLU_p(GLN_p(y))."""
    run_depthwise(2, 48, Lin, stride, "gln_prelu", pool)


@pytest.mark.parametrize("Lin", [2, 126])
@pytest.mark.parametrize("pool", [2, 4, 8, 16, 32, 64, 128])
def test_stage_depthwise_pool_only(pool, Lin):
    """The deepest level's gradient: dm pooled by 2^(D-1), with no depthwise term."""
    run_depthwise(2, 24, Lin, 2, None, pool)


@pytest.mark.parametrize("L", [256, 768])
@pytest.mark.parametrize("d", range(1, 8))
def test_stage_depthwise_pyramid_pairs(d, L):
    """The (level d-1, level d) launch of a depth-8 block: stride 2 over L >> (d-1) frames read through GLN, with
    dm pooled by 2^(d-1) (at L = 256, level 7 has 2 frames)."""
    run_depthwise(2, 16, L >> (d - 1), 2, "gln", 1 << (d - 1))


@pytest.mark.parametrize("S,N,L", [(1, 24, 37), (4, 31, 100), (8, 16, 33), (16, 24, 37), (16, 256, 17)])
def test_stage_mask_backward_sources(S, N, L):
    """S up to 16, N * L not a multiple of 256, and exact zeros in the logits (derivative 0, as torch.relu)."""
    B = 3
    mlog, e, dmk = rand(B, S * N, L, seed=15), rand(B, N, L, seed=16), rand(B, S * N, L, seed=17)
    mlog.view(-1)[::7] = 0.0
    dml, de = dmk.clone(), torch.full((B, N, L), float("nan"), device=DEV)
    NAT.check(NAT.lib().sdr_mask_backward(ptr(mlog), ptr(e), ptr(dml), ptr(de), B, S, N, L, stream()))
    m64, e64 = mlog.double().requires_grad_(True), e.double().requires_grad_(True)
    masked = torch.relu(m64.view(B, S, N, L)) * e64.unsqueeze(1)
    (masked.reshape(B, S * N, L) * dmk.double()).sum().backward()
    check(dml, m64.grad, f"mask dmlog S={S} N={N} L={L}")
    check(de, e64.grad, "mask de")


@pytest.mark.parametrize("SA,K,D,T", [(16, 21, 2, 801), (16, 3, 3, 17), (5, 41, 2, 1603), (3, 63, 1, 125),
                                      (1, 5, 4, 66)])
def test_stage_overlap_add_and_encoder_wgrad_sources(SA, K, D, T):
    """SA up to 16 at B = 5, T at most one hop past a multiple of hop * 2^D (the last frame mostly padding)."""
    B, N = 5, 40
    hop = K // 2
    assert 0 < T % (hop << D) <= hop
    cfg = O.Config(variant="improved", enc_kernel_size=K, upsampling_depth=D)
    L = O.padded_length(cfg, T) // hop
    lib = NAT.lib()
    gout = rand(B, SA, T, seed=18)
    dF = torch.full((B, SA * K, L), float("nan"), device=DEV)
    NAT.check(lib.sdr_overlap_add_backward(ptr(gout), ptr(dF), B, SA, K, L, T, stream()))
    fr = torch.zeros(B, SA * K, L, dtype=F64, device=DEV, requires_grad=True)
    eye = torch.eye(SA * K, dtype=F64, device=DEV).reshape(SA * K, SA, K)
    ola = F.conv_transpose1d(fr, eye, None, stride=hop, padding=hop, output_padding=hop - 1)[..., :T]
    (ola * gout.double()).sum().backward()
    check(dF, fr.grad, f"overlap-add backward SA={SA} K={K} T={T}")
    wav, de = rand(B, 1, T, seed=19), rand(B, N, L, seed=20)
    dw = torch.full((N, K), float("nan"), device=DEV)
    scratch = torch.empty(lib.sdr_encoder_wgrad_scratch_bytes(B, N, K, L), dtype=torch.uint8, device=DEV)
    NAT.check(lib.sdr_encoder_wgrad(ptr(de), ptr(wav), ptr(dw), ptr(scratch), B, N, K, L, T, stream()))
    W = torch.zeros(N, 1, K, dtype=F64, device=DEV, requires_grad=True)
    e = F.conv1d(O.pad_wave(cfg, wav, F64), W, None, stride=hop, padding=hop)
    assert e.shape[-1] == L
    (e * de.double()).sum().backward()
    check(dw, W.grad.reshape(N, K), f"encoder wgrad K={K} T={T}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. contracts
# ---------------------------------------------------------------------------------------------------------------------
CONTRACT = [("ffma", FFMA_KW, ()), ("tensor_cores", imp(N=256), ALL)]


def flat_grads(m):
    return torch.cat([p.grad.reshape(-1) for _, p in m.named_parameters()])


@pytest.mark.parametrize("name,kw,want", CONTRACT, ids=[c[0] for c in CONTRACT])
def test_backward_bitwise_reproducible(name, kw, want):
    """sdr_backward twice on one saved buffer and gradient, then model(x).backward(g) twice: byte-identical."""
    B, T = 3, 2000
    assert tc_convs(kw, T) == want
    cfg = O.Config(variant="improved", **kw)
    m = native_model(kw, O.make_state_dict(cfg, seed=5, perturbed=True))
    x = batch(B, T).to(DEV)
    g = torch.randn(B, kw["num_sources"], T, generator=torch.Generator().manual_seed(6)).to(DEV)
    y = m(x)
    ctx = y.grad_fn                      # the autograd node of the native training function holds its buffers
    lib = NAT.lib()
    ws = torch.empty(lib.sdr_backward_workspace_bytes(C.byref(ctx.cfg), B, T), dtype=torch.uint8, device=DEV)
    numel = sum(p.numel() for p in m.parameters())
    outs = []
    for _ in range(2):
        flat = torch.full((numel,), float("nan"), device=DEV)
        ws.fill_(0xA5)
        NAT.check(lib.sdr_backward(C.byref(ctx.cfg), C.c_void_p(ctx.packed.data_ptr()), C.c_void_p(x.data_ptr()),
                                   C.c_void_p(ctx.saved.data_ptr()), C.c_void_p(g.data_ptr()),
                                   C.c_void_p(flat.data_ptr()), B, T, C.c_void_p(ws.data_ptr()), ws.numel(),
                                   stream()), "sdr_backward")
        outs.append(flat.cpu())
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    y.backward(g)
    first = flat_grads(m).cpu()
    assert torch.equal(first.view(torch.int32), outs[0].view(torch.int32))
    m.zero_grad(set_to_none=True)
    m(x).backward(g)
    assert torch.equal(flat_grads(m).cpu().view(torch.int32), first.view(torch.int32))


LAUNCH = [("depth1", imp(D=1)), ("depth8", imp(D=8)), ("blocks0", imp(U=0)), ("ffma", FFMA_KW),
          ("tensor_cores_s3", imp(S=3, N=256))]


@pytest.mark.parametrize("name,kw", LAUNCH, ids=[c[0] for c in LAUNCH])
def test_backward_launch_count_across_configs(name, kw):
    """The kernel nodes of a CUDA graph captured from y.backward(g) equal sdr_backward_launch_count."""
    B, T = 2, 2000
    cfg = O.Config(variant="improved", **kw)
    m = native_model(kw, O.make_state_dict(cfg, seed=0))
    x = make_batch(B, T).to(DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m(x).backward(torch.randn(B, kw["num_sources"], T, device=DEV))     # packs the weights, sizes the workspace
        m.zero_grad(set_to_none=True)
        y = m(x)
        g = torch.randn_like(y)
    side.synchronize()
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph, stream=side):
        y.backward(g)
    torch.cuda.current_stream().wait_stream(side)
    got = _kernel_nodes(graph)
    want = NAT.lib().sdr_backward_launch_count(C.byref(_engine.make_config(m)), B, T)
    U, D = kw["num_blocks"], kw["upsampling_depth"]
    print(f"{name}: {got} graph kernel nodes, C-ABI {want}, tensor cores {tc_convs(kw, T) or 'none'}")
    assert want == 22 + U * (14 + 5 * D + (D > 1))
    assert got == want
    assert all(p.grad is not None for p in m.parameters())


def test_training_past_65535_weight_gradient_partials():
    """A 1-channel model at B = 32769, L = 1024: B * ceil(L / 512) = 65538 partials per weight gradient.  Where the
    library sizes the saved buffer, the forward and the backward both run, and the gradient is the sum of the two
    half batches' gradients."""
    kw = dict(out_channels=1, in_channels=1, num_blocks=1, upsampling_depth=1, enc_kernel_size=3, enc_num_basis=1,
              num_sources=1)
    B, T = 32769, 1024
    cfg = O.Config(variant="improved", **kw)
    assert frames(kw, T) == 1024
    m = native_model(kw, O.make_state_dict(cfg, seed=8, perturbed=True))
    c = _engine.make_config(m)
    lib = NAT.lib()
    assert lib.sdr_train_saved_bytes(C.byref(c), B, T) > 0
    assert lib.sdr_backward_workspace_bytes(C.byref(c), B, T) > 0
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(3)).to(DEV)
    g = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(4)).to(DEV)
    m.zero_grad(set_to_none=True)
    m(x).backward(g)
    whole = {n: p.grad.clone() for n, p in m.named_parameters()}
    halves = {}
    for sl in (slice(0, B // 2), slice(B // 2, B)):
        m.zero_grad(set_to_none=True)
        m(x[sl]).backward(g[sl])
        for n, p in m.named_parameters():
            halves[n] = halves.get(n, 0) + p.grad.double()
    compare(whole, halves, {n: halves[n].abs().item() for n in halves if halves[n].numel() == 1},
            "B = 32769 against two half batches", 1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# autograd plumbing
# ---------------------------------------------------------------------------------------------------------------------
PLUMB = imp(S=2, U=1, D=3)


def plumbing_model():
    cfg = O.Config(variant="improved", **PLUMB)
    return native_model(PLUMB, O.make_state_dict(cfg, seed=12, perturbed=True))


def test_frozen_encoder_gets_no_gradient():
    m = plumbing_model()
    x = make_batch(2, 2000).to(DEV)
    g = torch.randn(2, 2, 2000, generator=torch.Generator().manual_seed(9)).to(DEV)
    m(x).backward(g)
    full = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    dict(m.named_parameters())["encoder.weight"].requires_grad_(False)
    m(x).backward(g)
    for n, p in m.named_parameters():
        if n == "encoder.weight":
            assert p.grad is None
        else:
            assert torch.equal(p.grad, full[n]), n


@pytest.mark.parametrize("kind", ["sum", "flip", "transpose"])
def test_expanded_and_strided_output_gradients(kind):
    """y.sum() hands the backward a stride-0 gradient, y.flip(-1) and y.transpose(1, 2) strided ones: the same
    gradients as the explicit contiguous one."""
    m = plumbing_model()
    B, S, T = 2, 2, 2000
    x = make_batch(B, T).to(DEV)
    G = torch.randn(B, S, T, generator=torch.Generator().manual_seed(10)).to(DEV)
    y = m(x)
    if kind == "sum":
        y.sum().backward()
        g = torch.ones(B, S, T, device=DEV)
    elif kind == "flip":
        (y.flip(-1) * G).sum().backward()
        g = G.flip(-1).contiguous()
    else:
        (y.transpose(1, 2) * G.transpose(1, 2).contiguous()).sum().backward()
        g = G
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    m(x).backward(g)
    for n, p in m.named_parameters():
        assert torch.equal(got[n], p.grad), n
