"""The FUSS training step after the model on the native path: the differentiable ``mixture_consistency.apply`` and
``PermInvariantSNRwithZeroRefs`` (``sudo_rm_rf_b200.snr``), against the fp64 oracle run on the GPU on the same fp32
values (``O.mixture_consistency`` and ``snr_oracle.snr_zero_refs`` under autograd), inside CUDA graphs, and in ten steps of
run_fuss_separation.py's training loop.

Bars: gradients within 1e-5 of each row's max |grad| (plus the rounding of the input dtype for fp16 / bf16 inputs,
whose gradients come back in that dtype); loss values within 1e-3 dB, with the oracle's permutation unless the
oracle's score of the native permutation is within 1e-3 dB of its best; repeated calls and graph replays bitwise
equal."""
import contextlib
import itertools

import pytest
import torch
import torch.nn.functional as F

import sudo_rm_rf_b200 as P
from oracle import sudormrf_oracle as O
from snr_oracle import snr_zero_refs

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRAD_TOL = 1e-5
DB_TOL = 1e-3


def row_rel_err(got, ref):
    """max over rows (all but the last axis) of max|got - ref| / max|ref| (rows of zeros must be matched exactly)."""
    d = (got.double() - ref.double()).abs().reshape(-1, ref.shape[-1]).amax(1)
    m = ref.double().abs().reshape(-1, ref.shape[-1]).amax(1)
    return float(torch.where(m > 0, d / m.clamp_min(1e-300), d * 1e300).max())


# ---------------------------------------------------------------------------
# mixture consistency
# ---------------------------------------------------------------------------
def mc_inputs(B, S, T, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    est = torch.randn(B, S, T, generator=g) * (0.1 + torch.rand(B, S, 1, generator=g))
    mix = est.sum(1, keepdim=True) + 0.3 * torch.randn(B, 1, T, generator=g)
    gout = torch.randn(B, S, T, generator=g)
    return est.to(DEV, dtype), mix.to(DEV, dtype), gout.to(DEV)


def mc_native(est, mix, gout, kind, mix_grad):
    e = est.clone().requires_grad_(True)
    m = mix.clone().requires_grad_(mix_grad)
    out = P.mixture_consistency.apply(e, m, kind)
    assert out.grad_fn is not None
    (out * gout).sum().backward()
    return out.detach(), e.grad, (m.grad if mix_grad else None)


def mc_oracle(est, mix, gout, kind):
    e = est.to(torch.float32).double().requires_grad_(True)
    m = mix.to(torch.float32).double().requires_grad_(True)
    (O.mixture_consistency(e, m, kind) * gout.double()).sum().backward()
    return e.grad, m.grad


MC_GRID = [(kind, S, B, T) for kind in ("uniform", "magsq") for S, B, T in (
    (1, 3, 1), (2, 2, 1001), (3, 2, 4096), (4, 3, 4097), (4, 2, 8193), (2, 1, 64 * 4096 + 3), (3, 1000, 777),
    (4, 257, 130))]


@pytest.mark.parametrize("kind,S,B,T", MC_GRID)
def test_mixture_consistency_grad_matches_fp64_autograd(kind, S, B, T):
    est, mix, gout = mc_inputs(B, S, T, seed=S * 7 + T % 97)
    _, ge, gm = mc_native(est, mix, gout, kind, mix_grad=True)
    re, rm = mc_oracle(est, mix, gout, kind)
    ee, em = row_rel_err(ge, re), row_rel_err(gm, rm)
    print(f"mc {kind} S={S} B={B} T={T}: grad_est {ee:.2e}, grad_mix {em:.2e}")
    assert ge.dtype == torch.float32 and gm.shape == mix.shape
    assert ee <= GRAD_TOL and em <= GRAD_TOL


@pytest.mark.parametrize("kind", ["uniform", "magsq"])
def test_mixture_consistency_grad_at_ten_minutes_of_audio(kind):
    est, mix, gout = mc_inputs(1, 4, 9_600_000, seed=5)
    _, ge, gm = mc_native(est, mix, gout, kind, mix_grad=True)
    re, rm = mc_oracle(est, mix, gout, kind)
    ee, em = row_rel_err(ge, re), row_rel_err(gm, rm)
    print(f"mc {kind} T=9.6M: grad_est {ee:.2e}, grad_mix {em:.2e}")
    assert ee <= GRAD_TOL and em <= GRAD_TOL


@pytest.mark.parametrize("kind", ["uniform", "magsq"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_mixture_consistency_grad_in_input_dtype(kind, dtype):
    est, mix, gout = mc_inputs(3, 4, 3001, seed=11, dtype=dtype)
    _, ge, gm = mc_native(est, mix, gout, kind, mix_grad=True)
    assert ge.dtype == dtype and gm.dtype == dtype
    re, rm = mc_oracle(est, mix, gout, kind)
    tol = GRAD_TOL + (torch.finfo(dtype).eps if dtype != torch.float64 else 0.0)
    ee, em = row_rel_err(ge, re), row_rel_err(gm, rm)
    print(f"mc {kind} {dtype}: grad_est {ee:.2e}, grad_mix {em:.2e} (bar {tol:.1e})")
    assert ee <= tol and em <= tol


@pytest.mark.parametrize("kind", ["uniform", "magsq"])
@pytest.mark.parametrize("S", [1, 2, 3, 4])
def test_mixture_consistency_forward_bitwise_with_and_without_grad(kind, S):
    est, mix, _ = mc_inputs(4, S, 5003, seed=S)
    with torch.no_grad():
        plain = P.mixture_consistency.apply(est, mix, kind)
    assert plain.grad_fn is None
    plain2 = P.mixture_consistency.apply(est, mix, kind)          # grad mode on, nothing requires grad
    assert plain2.grad_fn is None
    for e_grad, m_grad in ((True, False), (False, True), (True, True)):
        out = P.mixture_consistency.apply(est.clone().requires_grad_(e_grad), mix.clone().requires_grad_(m_grad), kind)
        assert out.grad_fn is not None
        assert torch.equal(out.detach(), plain)
    assert torch.equal(plain2, plain)


@pytest.mark.parametrize("kind", ["uniform", "magsq"])
def test_mixture_consistency_backward_is_bitwise_reproducible(kind):
    est, mix, gout = mc_inputs(5, 4, 70001, seed=3)
    a = mc_native(est, mix, gout, kind, mix_grad=True)
    b = mc_native(est, mix, gout, kind, mix_grad=True)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_mixture_consistency_grad_to_the_estimates_only():
    est, mix, gout = mc_inputs(2, 3, 999, seed=8)
    _, ge, _ = mc_native(est, mix, gout, "magsq", mix_grad=False)
    re, _ = mc_oracle(est, mix, gout, "magsq")
    assert row_rel_err(ge, re) <= GRAD_TOL


# ---------------------------------------------------------------------------
# PermInvariantSNRwithZeroRefs
# ---------------------------------------------------------------------------
def snr_inputs(B, S, T, seed, Tp=None):
    g = torch.Generator().manual_seed(seed)
    n = max(T, Tp or T)
    tgt = torch.randn(B, S, n, generator=g) * (0.2 + torch.rand(B, S, 1, generator=g)) + 0.05
    est = torch.stack([tgt[b, torch.randperm(S, generator=g)] for b in range(B)])
    est = est * 0.8 + torch.randn(B, S, n, generator=g) * torch.logspace(-2.5, 0, B).view(B, 1, 1)
    return est[:, :, :(Tp or T)].contiguous().to(DEV), tgt[:, :, :T].contiguous().to(DEV)


def perm_scores(pr, tgt, zero_mean, thr, eps):
    """fp64 score of every permutation [B, S!] (the columns snr_zero_refs takes the max of)."""
    S = pr.shape[1]
    n = min(pr.shape[-1], tgt.shape[-1])
    p, t = pr[..., :n].double(), tgt[..., :n].double()
    if zero_mean:
        p, t = p - p.mean(-1, keepdim=True), t - t.mean(-1, keepdim=True)
    tp = (t * t).sum(-1, keepdim=True)
    mix = t.sum(1, keepdim=True)
    mp = (mix * mix).sum(-1, keepdim=True)
    act = (10. * torch.log10(tp / (mp + eps))).ge(thr)
    stab = 0.001 * torch.where(act, tp, mp.expand_as(tp))
    cols = []
    for perm in itertools.permutations(range(S)):
        err = p[:, list(perm)] - t
        cols.append((10. * act * torch.log10((tp + eps) / ((err * err).sum(-1, keepdim=True) + stab + eps) + eps))
                    .sum(1) * act.sum(1))
    return torch.cat(cols, -1)


def native_snr(pr, tgt, S, zero_mean, thr=-40., eps=1e-9):
    fn = P.snr.PermInvariantSNRwithZeroRefs(zero_mean=zero_mean, n_sources=S, backward_loss=False,
                                            inactivity_threshold=thr, return_individual_results=True)
    with torch.no_grad():
        val, perms = fn(pr, tgt, eps=eps, return_best_permutation=True)
    table = {p: i for i, p in enumerate(itertools.permutations(range(S)))}
    return val, torch.tensor([table[tuple(r)] for r in perms.tolist()])


def check_snr_against_oracle(pr, tgt, S, zero_mean, thr=-40., eps=1e-9, label=""):
    val, idx = native_snr(pr, tgt, S, zero_mean, thr, eps)
    with torch.no_grad():
        ref, ridx = snr_zero_refs(pr.double(), tgt.double(), zero_mean, thr, eps)
    ref, ridx = ref.cpu(), ridx.cpu()
    val = val.double().cpu()
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isnan(val), torch.isnan(ref)), label
    err = (val[fin] - ref[fin]).abs().max().item() if fin.any() else 0.0
    print(f"snr {label}: max |native - fp64| = {err:.2e} dB")
    assert err <= DB_TOL, label
    differ = (idx != ridx) & fin
    if differ.any():
        scores = perm_scores(pr, tgt, zero_mean, thr, eps).cpu()
        rows = differ.nonzero().flatten()
        gap = (scores[rows, ridx[rows]] - scores[rows, idx[rows]]).abs()
        assert bool((gap <= DB_TOL).all()), (label, rows, gap)
    return val, idx


SNR_GRID = [(S, zm, B, T) for S in (1, 2, 3, 4) for zm in (False, True) for B, T in ((3, 1), (2, 4096), (3, 4097))] + \
    [(4, False, 255, 300), (4, True, 256, 301), (3, False, 257, 500), (4, False, 1000, 257),
     (2, True, 2, 64 * 4096), (4, False, 2, 64 * 4096 + 5), (4, True, 3, 160000), (4, False, 3, 160000)]


@pytest.mark.parametrize("S,zero_mean,B,T", SNR_GRID)
def test_snr_forward_matches_fp64_oracle(S, zero_mean, B, T):
    pr, tgt = snr_inputs(B, S, T, seed=S * 100 + B + T % 89)
    check_snr_against_oracle(pr, tgt, S, zero_mean, label=f"S={S} zm={zero_mean} B={B} T={T}")


@pytest.mark.parametrize("thr,eps", [(-20., 1e-9), (-60., 1e-6), (-40., 0.0), (-10., 1e-3)])
def test_snr_forward_threshold_and_eps(thr, eps):
    pr, tgt = snr_inputs(6, 4, 3000, seed=17)
    tgt[0, 3] *= 0.03
    tgt[1, 2] *= 0.003
    check_snr_against_oracle(pr, tgt, 4, False, thr, eps, label=f"thr={thr} eps={eps}")


def degenerate(S, zero_mean):
    pr, tgt = snr_inputs(5, S, 2000, seed=40 + S)
    tgt[0, 0] = 0.0                                     # a silent target
    tgt[1, S - 1] *= 1e-3                               # a target 60 dB below the others
    tgt[2] = 0.0                                        # all silent: num_active = 0, every permutation scores 0
    pr[3, 1] = pr[3, 0]                                 # two identical estimates: the first maximum wins
    return pr, tgt


@pytest.mark.parametrize("S", [2, 3, 4])
@pytest.mark.parametrize("zero_mean", [False, True])
def test_snr_degenerate_rows(S, zero_mean):
    pr, tgt = degenerate(S, zero_mean)
    val, idx = check_snr_against_oracle(pr, tgt, S, zero_mean, label=f"degenerate S={S} zm={zero_mean}")
    assert float(val[2]) == 0.0 and int(idx[2]) == 0


@pytest.mark.parametrize("Tp,T", [(5000, 4321), (4321, 5000)])
def test_snr_forward_crops_to_the_shorter(Tp, T):
    pr, tgt = snr_inputs(3, 4, T, seed=2, Tp=Tp)
    check_snr_against_oracle(pr, tgt, 4, True, label=f"crop pr {Tp} t {T}")


def test_snr_nan_stays_in_its_item():
    pr, tgt = snr_inputs(4, 4, 3000, seed=9)
    clean, _ = native_snr(pr, tgt, 4, False)
    pr[1, 2, 1234] = float("nan")
    val, _ = native_snr(pr, tgt, 4, False)
    assert torch.isnan(val[1])
    keep = torch.tensor([0, 2, 3])
    assert torch.equal(val[keep], clean[keep])


def test_snr_return_conventions():
    pr, tgt = snr_inputs(5, 3, 2000, seed=4)
    ind, _ = native_snr(pr, tgt, 3, True)
    for backward_loss in (False, True):
        for individual in (False, True):
            fn = P.snr.PermInvariantSNRwithZeroRefs(zero_mean=True, n_sources=3, backward_loss=backward_loss,
                                                    return_individual_results=individual)
            with torch.no_grad():
                v = fn(pr, tgt)
            want = ind.to(DEV) if individual else ind.to(DEV).mean()
            assert torch.equal(v, -want if backward_loss else want)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_snr_casts_inputs_and_strided_views(dtype):
    pr, tgt = snr_inputs(3, 4, 2001, seed=6)
    pr_v = pr.to(dtype).transpose(0, 1).contiguous().transpose(0, 1)        # a strided view
    tgt_v = tgt.to(dtype)[:, :, ::1]
    check_snr_against_oracle(pr_v, tgt_v, 4, False, label=f"{dtype} strided")
    p = pr_v.detach().clone().requires_grad_(True)
    P.snr.PermInvariantSNRwithZeroRefs(n_sources=4)(p, tgt_v).backward()
    assert p.grad.dtype == dtype and p.grad.shape == p.shape


def snr_grads(pr, tgt, S, zero_mean, thr, eps, w):
    p = pr.clone().requires_grad_(True)
    fn = P.snr.PermInvariantSNRwithZeroRefs(zero_mean=zero_mean, n_sources=S, backward_loss=True,
                                            inactivity_threshold=thr, return_individual_results=w is not None)
    v = fn(p, tgt, eps=eps)
    (v * w).sum().backward() if w is not None else v.backward()
    q = pr.double().requires_grad_(True)
    best, _ = snr_zero_refs(q, tgt.double(), zero_mean, thr, eps)
    rv = -best if w is not None else -best.mean()
    (rv * w.double()).sum().backward() if w is not None else rv.backward()
    return p.grad, q.grad


GRAD_GRID = [(S, zm, B, T, ind) for S in (1, 2, 3, 4) for zm in (False, True) for B, T, ind in (
    (3, 1000, False), (2, 4097, True))] + [(4, False, 257, 300, True), (4, True, 3, 160000, False),
                                          (4, False, 2, 64 * 4096 + 1, True)]


@pytest.mark.parametrize("S,zero_mean,B,T,individual", GRAD_GRID)
def test_snr_grad_matches_fp64_autograd(S, zero_mean, B, T, individual):
    pr, tgt = snr_inputs(B, S, T, seed=S + 3 * B + T % 31)
    w = (torch.rand(B, device=DEV) + 0.5) if individual else None
    g, r = snr_grads(pr, tgt, S, zero_mean, -40., 1e-9, w)
    e = row_rel_err(g, r)
    print(f"snr grad S={S} zm={zero_mean} B={B} T={T} individual={individual}: {e:.2e}")
    assert e <= GRAD_TOL


@pytest.mark.parametrize("S", [2, 4])
@pytest.mark.parametrize("zero_mean", [False, True])
def test_snr_grad_degenerate_rows_and_crop(S, zero_mean):
    pr, tgt = degenerate(S, zero_mean)
    g, r = snr_grads(pr, tgt, S, zero_mean, -40., 1e-9, torch.rand(5, device=DEV) + 0.5)
    assert float(g[2].abs().max()) == 0.0                 # num_active = 0: no gradient
    assert row_rel_err(g, r) <= GRAD_TOL
    pr, tgt = snr_inputs(3, S, 3000, seed=12, Tp=3500)
    g, r = snr_grads(pr, tgt, S, zero_mean, -40., 1e-9, None)
    assert g.shape == pr.shape and float(g[..., 3000:].abs().max()) == 0.0
    assert row_rel_err(g, r) <= GRAD_TOL


def test_snr_backward_is_bitwise_reproducible():
    pr, tgt = snr_inputs(7, 4, 90001, seed=21)
    a, _ = snr_grads(pr, tgt, 4, True, -40., 1e-9, None)
    b, _ = snr_grads(pr, tgt, 4, True, -40., 1e-9, None)
    assert torch.equal(a, b)
    v1, _ = native_snr(pr, tgt, 4, True)
    v2, _ = native_snr(pr, tgt, 4, True)
    assert torch.equal(v1, v2)


# ---------------------------------------------------------------------------
# both in a captured graph
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["uniform", "magsq"])
def test_projection_and_loss_forward_backward_in_a_cuda_graph(kind):
    pr, tgt = snr_inputs(3, 4, 20001, seed=30)
    mix = tgt.sum(1, keepdim=True)
    est = pr.clone().requires_grad_(True)
    fn = P.snr.PermInvariantSNRwithZeroRefs(n_sources=4, zero_mean=False, backward_loss=True)

    def step():
        est.grad = None
        loss = fn(P.mixture_consistency.apply(est, mix, kind), tgt)
        loss.backward()
        return loss

    eager_loss = step().detach().clone()
    eager_grad = est.grad.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    est.grad = None
    with torch.cuda.graph(graph):
        loss = fn(P.mixture_consistency.apply(est, mix, kind), tgt)
        loss.backward()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(loss, eager_loss) and torch.equal(est.grad, eager_grad)


# ---------------------------------------------------------------------------
# the FUSS training step (run_fuss_separation.py:232-265)
# ---------------------------------------------------------------------------
FUSS = dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=3, enc_kernel_size=21,
            enc_num_basis=128, num_sources=4)


@contextlib.contextmanager
def nn_prelu_oracle():
    """nn.PReLU's derivative at 0 is the slope; the oracle's torch.where form gives 1 there (same forward values)."""
    old = O.prelu1
    O.prelu1 = lambda x, slope: F.prelu(x, slope.reshape(1))
    try:
        yield
    finally:
        O.prelu1 = old


def fuss_clean():
    g = torch.Generator().manual_seed(44)
    clean = torch.randn(2, 4, 4000, generator=g) * torch.tensor([1.0, 0.5, 0.2, 0.05]).view(1, 4, 1)
    clean[1, 3] = 0.0                                   # a mixture with three sources, as FUSS has
    return clean.to(DEV)


def normalise(mixture):                                 # run_fuss_separation.py:237-243
    return (mixture - mixture.mean(-1, keepdim=True)) / (mixture.std(-1, keepdim=True) + 1e-9)


def fuss_loop(forward, project, loss_fn, params, clean, steps=10):
    opt = torch.optim.Adam(params, lr=1e-3)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        x = normalise(torch.sum(clean, -2, keepdim=True))
        est = project(forward(x), x)
        loss = loss_fn(est, clean)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 5.0)
        opt.step()
        losses.append(loss.item())
    return losses


def fuss_model(sd):
    m = P.SuDORMRF(**FUSS)
    m.load_state_dict(sd)
    return m.to(DEV).enable_training().train()


def test_fuss_step_tracks_oracle():
    cfg = O.Config(variant="improved", **FUSS)
    sd = O.make_state_dict(cfg, seed=14)
    clean = fuss_clean()
    m = fuss_model(sd)
    native_loss = P.snr.PermInvariantSNRwithZeroRefs(n_sources=4, zero_mean=False, backward_loss=True,
                                                     inactivity_threshold=-40.)
    ln = fuss_loop(lambda x: m(x), P.mixture_consistency.apply, native_loss, list(m.parameters()), clean)
    p64 = {k: v.to(DEV, torch.float64).clone().requires_grad_(True) for k, v in sd.items()}

    def fwd(x):
        with nn_prelu_oracle():
            return O.forward(cfg, p64, x.double(), dtype=torch.float64)

    lo = fuss_loop(fwd, O.mixture_consistency,
                   lambda e, c: -snr_zero_refs(e, c.double(), False, -40.)[0].mean(), list(p64.values()), clean)
    dist = max(((p.detach().double() - p64[n].detach()).norm() / p64[n].detach().norm()).item()
               for n, p in m.named_parameters())
    print("native loss", [f"{v:.4f}" for v in ln])
    print("oracle loss", [f"{v:.4f}" for v in lo])
    print(f"largest parameter distance after 10 Adam steps: {dist:.2e}")
    assert ln[-1] < ln[0]
    for a, b in zip(ln, lo):
        assert abs(a - b) <= 1e-2 * abs(b)


def test_fuss_native_loss_grads_match_torch_autograd_loss():
    """One step: the native loss and the loss restated in torch autograd (fp64) on the same native estimates give the
    same parameter gradients."""
    cfg = O.Config(variant="improved", **FUSS)
    sd = O.make_state_dict(cfg, seed=15)
    clean = fuss_clean()
    m = fuss_model(sd)
    x = normalise(torch.sum(clean, -2, keepdim=True))
    grads = []
    for loss_fn in (P.snr.PermInvariantSNRwithZeroRefs(n_sources=4, zero_mean=False, backward_loss=True,
                                                       inactivity_threshold=-40.),
                    lambda e, c: -snr_zero_refs(e.double(), c.double(), False, -40.)[0].mean()):
        m.zero_grad(set_to_none=True)
        loss_fn(P.mixture_consistency.apply(m(x), x), clean).backward()
        grads.append({n: p.grad.clone() for n, p in m.named_parameters()})
    worst = 0.0
    for n, g in grads[0].items():
        r = grads[1][n].double()
        e = ((g.double() - r).norm() / r.norm().clamp_min(1e-300)).item()
        worst = max(worst, e)
        assert e <= 1e-2, (n, e)
    print(f"native loss vs torch autograd loss: worst parameter gradient rel-L2 {worst:.2e}")
