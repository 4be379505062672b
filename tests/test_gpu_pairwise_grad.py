"""The improved model's training loss on the native path: the differentiable ``PairwiseNegSDR`` and
``PITLossWrapper`` on top of it (``sudo_rm_rf_b200.sisdr``) against fp64 autograd of the oracle run on the GPU on the
same fp32 values (``O.pairwise_neg_sdr``, ``O.pit_from_pairwise``), the training forward against the evaluation
forward, a whole improved-model step in one CUDA graph, ten steps of run_improved_sudormrf.py's training loop, the
entries on poisoned and guarded buffers, and a non-finite input's reach.

Bars: each gradient row within 1e-5 of that row's max |grad| (plus the rounding of the input dtype for fp16 / bf16
inputs, whose gradients come back in that dtype); values in dB by ``test_gpu_metric_space.check_scores``' rule;
repeated calls, graph replays and poisoned workspaces bitwise equal to the clean run."""
import ctypes as C
import itertools

import pytest
import torch

from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import sisdr as S
from oracle import sudormrf_oracle as O
from guards import POISON_HUGE, POISON_NAN, check_bands, guarded_copy, poisoned, poisoned_like
from test_gpu_metric_space import B_EDGES, check_scores, f64, pw_db, separation_batch
from test_gpu_train import RUNNER, _oracle_step_params, native_model, nn_prelu_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRAD_TOL = 1e-5
TYPES = ("snr", "sisdr", "sdsdr")
FLAGS = list(itertools.product((False, True), (False, True)))              # (zero_mean, take_log)
T_EDGES = [1, 2, 255, 257, 4095, 4096, 4097, 262145, 160000]               # chunk edges; 160000 = 10 s at 16 kHz
PATTERNS = [("nan", POISON_NAN), ("1e30", POISON_HUGE)]
TYPE_CODE = {"snr": 0, "sisdr": 1, "sdsdr": 2}
WORST = {}


def row_rel_err(got, ref):
    """max over rows (all but the last axis) of max|got - ref| / max|ref| (rows of zeros must be matched exactly)."""
    d = (got.double() - ref.double()).abs().reshape(-1, ref.shape[-1]).amax(1)
    m = ref.double().abs().reshape(-1, ref.shape[-1]).amax(1)
    return float(torch.where(m > 0, d / m.clamp_min(1e-300), d * 1e300).max())


def note(kind, err, label):
    if err > WORST.get(kind, (0.0, ""))[0]:
        WORST[kind] = (err, label)
    print(f"{label}: {kind} {err:.2e} (worst so far {WORST[kind][0]:.2e} at {WORST[kind][1]})")


def native(est, tgt, sdr_type, zero_mean, take_log, gout):
    """-> (values [B, S, S] fp32, gradient of sum(values * gout) with respect to est)."""
    e = est.detach().clone().requires_grad_(True)
    out = S.PairwiseNegSDR(sdr_type, zero_mean=zero_mean, take_log=take_log)(e, tgt)
    assert out.grad_fn is not None and out.dtype == torch.float32
    (out * gout).sum().backward()
    return out.detach(), e.grad


def oracle(est, tgt, sdr_type, zero_mean, take_log, gout):
    e = f64(est).requires_grad_(True)
    out = O.pairwise_neg_sdr(e, f64(tgt), sdr_type, zero_mean, take_log)
    (out * gout.double()).sum().backward()
    return out.detach(), e.grad


def compare(est, tgt, sdr_type, zero_mean, take_log, label, seed=0):
    B, Sn, _ = est.shape
    gout = torch.rand(B, Sn, Sn, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV) + 0.5
    got, grad = native(est, tgt, sdr_type, zero_mean, take_log, gout)
    want, ref = oracle(est, tgt, sdr_type, zero_mean, take_log, gout)
    assert grad.shape == est.shape and grad.dtype == est.dtype
    e_in, e_out = check_scores(pw_db(got, take_log), pw_db(want, take_log), what=label)
    note("value dB", max(e_in, e_out), label)
    err = row_rel_err(grad, ref)
    note("gradient", err, label)
    assert err <= GRAD_TOL, (label, err)
    return got, grad


# ---------------------------------------------------------------------------------------------------------------------
# gradient parity: every sdr_type x (zero_mean, take_log) x S = 1..4, length and batch edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("Sn", [1, 2, 3, 4])
def test_grad_matches_fp64_autograd_at_length_edges(sdr_type, Sn):
    for T in T_EDGES:
        est, tgt, _ = separation_batch(3 if T < 100000 else 2, Sn, T, seed=T + 10 * Sn)
        for zm, tl in FLAGS:
            compare(est, tgt, sdr_type, zm, tl, f"{sdr_type} S={Sn} T={T} zm={zm} log={tl}", seed=T)


@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("Sn", [2, 4])
@pytest.mark.parametrize("B", B_EDGES)
def test_grad_matches_fp64_autograd_at_batch_edges(sdr_type, Sn, B):
    est, tgt, _ = separation_batch(B, Sn, 777, seed=B + Sn)
    for zm, tl in FLAGS:
        compare(est, tgt, sdr_type, zm, tl, f"{sdr_type} S={Sn} B={B} zm={zm} log={tl}", seed=B)


@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("zero_mean,take_log", FLAGS)
def test_grad_degenerate_rows(sdr_type, zero_mean, take_log):
    """A silent target and an estimate equal to its target against fp64 autograd.  The latter's |noise|^2 is 0 in
    the reference; for sisdr, whose projection rescales the target, the one-pass Gram form gets rounding of a few ulp
    of <t, t> beside the 1e-8 floor.  It is tested at <t, t> ~ 1, where that rounding is 1e-8 of the floor (at
    <t, t> ~ 1e3 it is ~1e-4 of it, and so is the error of that pair's gradient without take_log).  The backward forms
    each pair's noise vector before weighting it, so an exactly zero noise gives an exactly zero term whatever its
    weight (~1e16 here).  A constant estimate row under zero_mean is the one place the two forms
    legitimately differ outright (its mean-removed energies are rounding noise, not 0:
    test_gpu_metric_space.check_constant): there the gradient is finite and every other item matches."""
    est, tgt, _ = separation_batch(4, 3, 3001, seed=77)
    tgt[0, 0] = 0.0
    est[2], tgt[2] = est[2] * 0.02, tgt[2] * 0.02
    est[2, 2] = tgt[2, 2]
    est[3, 1] = 0.375
    keep = [0, 1, 2] if zero_mean else [0, 1, 2, 3]
    label = f"degenerate {sdr_type} zm={zero_mean} log={take_log}"
    compare(est[keep].contiguous(), tgt[keep].contiguous(), sdr_type, zero_mean, take_log, label, seed=3)
    if zero_mean:
        gout = torch.rand(4, 3, 3, device=DEV) + 0.5
        got, grad = native(est, tgt, sdr_type, zero_mean, take_log, gout)
        assert torch.isfinite(got).all() and torch.isfinite(grad).all()
        sub, gsub = native(est[keep].contiguous(), tgt[keep].contiguous(), sdr_type, zero_mean, take_log, gout[keep])
        assert torch.equal(got[keep], sub) and torch.equal(grad[keep], gsub)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64, "strided"])
def test_grad_in_input_dtype_and_strided_views(dtype):
    est, tgt, _ = separation_batch(3, 4, 3001, seed=11)
    if dtype == "strided":
        est = est.transpose(0, 1).contiguous().transpose(0, 1)
        tgt = torch.stack([tgt, -tgt], -1)[..., 0]
        tol = GRAD_TOL
    else:
        est, tgt = est.to(dtype), tgt.to(dtype)
        tol = GRAD_TOL + (torch.finfo(dtype).eps if dtype != torch.float64 else 0.0)
    gout = torch.rand(3, 4, 4, device=DEV) + 0.5
    _, grad = native(est, tgt, "sisdr", True, True, gout)
    assert grad.dtype == est.dtype and grad.shape == est.shape
    _, ref = oracle(est, tgt, "sisdr", True, True, gout)
    err = row_rel_err(grad, ref)
    note(f"gradient, {dtype} input", err, f"dtype {dtype}")
    assert err <= tol, (dtype, err)


# ---------------------------------------------------------------------------------------------------------------------
# the training forward against the evaluation forward; reproducibility
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("Sn", [1, 2, 3, 4])
def test_train_forward_matches_eval_forward(sdr_type, Sn):
    est, tgt, _ = separation_batch(5, Sn, 70001, seed=Sn)
    worst = 0.0
    for zm, tl in FLAGS:
        fn = S.PairwiseNegSDR(sdr_type, zero_mean=zm, take_log=tl)
        with torch.no_grad():
            ev = fn(est, tgt)
        assert ev.grad_fn is None
        tr = fn(est.clone().requires_grad_(True), tgt)
        assert tr.grad_fn is not None
        d = ((tr.detach().double() - ev.double()).abs() / ev.double().abs().clamp_min(1.0)).max().item()
        worst = max(worst, d)
        assert d <= 1e-6, (zm, tl, d)
        with torch.enable_grad():
            assert torch.equal(fn(est, tgt), ev)                          # nothing requires grad: the eval path
    print(f"train vs eval forward {sdr_type} S={Sn}: {worst:.2e} relative (of max(|value|, 1))")


def test_forward_and_backward_are_bitwise_reproducible():
    est, tgt, _ = separation_batch(7, 4, 262145, seed=21)
    gout = torch.rand(7, 4, 4, device=DEV) + 0.5
    for sdr_type in TYPES:
        a = native(est, tgt, sdr_type, True, True, gout)
        b = native(est, tgt, sdr_type, True, True, gout)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), sdr_type


# ---------------------------------------------------------------------------------------------------------------------
# through PITLossWrapper
# ---------------------------------------------------------------------------------------------------------------------
def perm_avg_of(pairwise):
    """A perm_avg callable built on a pairwise loss: the mean of the diagonal, [batch]."""
    return lambda e, t: pairwise(e, t).diagonal(dim1=1, dim2=2).mean(-1)


@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("Sn", [1, 2, 3, 4])
def test_pit_wrapper_backpropagates(sdr_type, Sn):
    est, tgt, _ = separation_batch(6, Sn, 16001, seed=5 * Sn)
    for zm, tl in FLAGS:
        nat = S.PairwiseNegSDR(sdr_type, zero_mean=zm, take_log=tl)
        ref = lambda e, t: O.pairwise_neg_sdr(e, t, sdr_type, zm, tl)             # noqa: E731
        for mode, fn_n, fn_r in (("pw_mtx", nat, ref), ("perm_avg", perm_avg_of(nat), perm_avg_of(ref))):
            e = est.clone().requires_grad_(True)
            loss, reordered = S.PITLossWrapper(fn_n, pit_from=mode)(e, tgt, return_est=True)
            loss.backward()
            r = f64(est).requires_grad_(True)
            want, want_re = S.PITLossWrapper(fn_r, pit_from=mode)(r, f64(tgt), return_est=True)
            want.backward()
            label = f"wrapper {mode} {sdr_type} S={Sn} zm={zm} log={tl}"
            check_scores(pw_db(loss.detach().view(1), tl), pw_db(want.detach().view(1), tl), what=label)
            assert torch.equal(reordered.detach().double(), want_re.detach()), label     # the same permutations
            err = row_rel_err(e.grad, r.grad)
            note("wrapper gradient", err, label)
            assert err <= GRAD_TOL, (label, err)


# ---------------------------------------------------------------------------------------------------------------------
# the improved model's step: one CUDA graph; ten steps of run_improved_sudormrf.py's loop
# ---------------------------------------------------------------------------------------------------------------------
def runner_batch():
    gen = torch.Generator().manual_seed(33)
    tgt = torch.randn(2, 2, 4000, generator=gen)
    return tgt.sum(1, keepdim=True), tgt


def test_improved_step_in_one_cuda_graph():
    """Native forward, PITLossWrapper(PairwiseNegSDR('sisdr')), backward: captured once and replayed, the loss and
    every parameter gradient bitwise equal to the eager step's."""
    cfg = O.Config(variant="improved", **RUNNER)
    m = native_model(RUNNER, O.make_state_dict(cfg, seed=12)).train()
    x, tgt = (t.to(DEV) for t in runner_batch())
    loss_fn = S.PITLossWrapper(S.PairwiseNegSDR("sisdr"), pit_from="pw_mtx")
    params = list(m.parameters())

    def step():
        for q in params:
            q.grad = None
        loss = loss_fn(m(x), tgt)
        loss.backward()
        return loss

    eager_loss = step().detach().clone()
    eager = [q.grad.clone() for q in params]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    for q in params:
        q.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = loss_fn(m(x), tgt)
        loss.backward()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(loss, eager_loss)
        for q, g in zip(params, eager):
            assert torch.equal(q.grad, g)
    print(f"graph step: loss {eager_loss.item():.4f}, {len(params)} parameter gradients bitwise equal on replay")


def runner_loop(forward, loss_fn, params, steps=10):
    """run_improved_sudormrf.py's step: PIT(neg SI-SDR) -> backward -> clip_grad_norm_(5.0) -> Adam(1e-3)."""
    opt = torch.optim.Adam(params, lr=1e-3)
    x, tgt = runner_batch()
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = loss_fn(forward(x), tgt)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 5.0)
        opt.step()
        losses.append(loss.item())
    return losses


def test_runner_loop_on_native_loss_tracks_oracle():
    """test_gpu_train.test_runner_loop_adam_clip_tracks_oracle's loop and bars, with the native loss on the native
    side: every loss within 1e-2 of fp64's, and the loss falls."""
    cfg = O.Config(variant="improved", **RUNNER)
    sd = O.make_state_dict(cfg, seed=10)
    m = native_model(RUNNER, sd).train()
    native_loss = S.PITLossWrapper(S.PairwiseNegSDR("sisdr"), pit_from="pw_mtx")
    ln = runner_loop(lambda x: m(x.to(DEV)), lambda y, t: native_loss(y, t.to(DEV)), list(m.parameters()))
    p64 = _oracle_step_params(sd)

    def fwd(x):
        with nn_prelu_oracle():
            return O.forward(cfg, p64, x.to(DEV, torch.float64), dtype=torch.float64)
    lo = runner_loop(fwd, lambda y, t: O.pit_from_pairwise(O.pairwise_neg_sdr(y, t.to(y)))[0].mean(),
                     list(p64.values()))
    dist = max(((q.detach().double() - p64[n].detach()).norm() / p64[n].detach().norm()).item()
               for n, q in m.named_parameters())
    print("native loss", [f"{v:.4f}" for v in ln])
    print("oracle loss", [f"{v:.4f}" for v in lo])
    print(f"largest parameter distance after 10 Adam steps: {dist:.2e}")
    assert ln[-1] < ln[0]
    for a, b in zip(ln, lo):
        assert abs(a - b) <= 1e-2 * abs(b)


# ---------------------------------------------------------------------------------------------------------------------
# the entries on poisoned scratch, coefficients and outputs between guard bands
# ---------------------------------------------------------------------------------------------------------------------
def ptr(t):
    return C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def run_entries(est, tgt, gout, sdr_type, pattern):
    """sdr_pairwise_neg_sdr_train then sdr_pairwise_neg_sdr_backward with every buffer they write poisoned."""
    lib = N.lib()
    B, Sn, T = est.shape
    e, t, g = guarded_copy(est), guarded_copy(tgt), guarded_copy(gout)
    out = poisoned_like(torch.empty(B, Sn, Sn, device=DEV), pattern)
    coef = poisoned(lib.sdr_pairwise_neg_sdr_coef_bytes(B, Sn), pattern)
    sc = poisoned(lib.sdr_pairwise_neg_sdr_train_scratch_bytes(B, Sn, T), pattern)
    grad = poisoned_like(torch.empty(B, Sn, T, device=DEV), pattern)
    assert lib.sdr_pairwise_neg_sdr_train(ptr(e), ptr(t), ptr(out), ptr(coef), B, Sn, T, TYPE_CODE[sdr_type], 1, 1,
                                          ptr(sc), stream()) == 0
    assert lib.sdr_pairwise_neg_sdr_backward(ptr(e), ptr(t), ptr(coef), ptr(g), ptr(grad), B, Sn, T, stream()) == 0
    for buf, what in ((e, "est"), (t, "target"), (g, "grad_out"), (out, "out"), (coef, "coef"), (sc, "scratch"),
                      (grad, "grad_est")):
        check_bands(buf, what)
    assert torch.equal(e, est) and torch.equal(t, tgt) and torch.equal(g, gout)
    return out.clone(), grad.clone()


@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("Sn", [1, 3, 4])
def test_entries_on_poisoned_and_guarded_buffers(sdr_type, Sn):
    est, tgt, _ = separation_batch(5, Sn, 8193, seed=13 + Sn)
    gout = torch.rand(5, Sn, Sn, device=DEV) + 0.5
    clean = run_entries(est, tgt, gout, sdr_type, 0)
    _, ref = oracle(est, tgt, sdr_type, True, True, gout)
    assert row_rel_err(clean[1], ref) <= GRAD_TOL
    for pname, pattern in PATTERNS:
        got = run_entries(est, tgt, gout, sdr_type, pattern)
        assert torch.equal(got[0], clean[0]) and torch.equal(got[1], clean[1]), pname


# ---------------------------------------------------------------------------------------------------------------------
# a non-finite value stays in its own item
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sdr_type", TYPES)
@pytest.mark.parametrize("where", ["est", "target"])
def test_nonfinite_stays_in_its_item(sdr_type, where):
    B, Sn, T = 4, 3, 5001
    est, tgt, _ = separation_batch(B, Sn, T, seed=19)
    gout = torch.rand(B, Sn, Sn, device=DEV) + 0.5
    for zm, tl in FLAGS:
        clean = native(est, tgt, sdr_type, zm, tl, gout)
        wrapper = S.PITLossWrapper(S.PairwiseNegSDR(sdr_type, zero_mean=zm, take_log=tl), pit_from="pw_mtx")
        e0 = est.clone().requires_grad_(True)
        wrapper(e0, tgt).backward()
        for bad in (0, 2, B - 1):
            for v in (float("nan"), float("inf"), -float("inf"), 1e30):
                e, t = est.clone(), tgt.clone()
                x = e if where == "est" else t
                x[bad, 1, 0] = v
                x[bad, Sn - 1, T - 1] = v
                got = native(e, t, sdr_type, zm, tl, gout)
                keep = [b for b in range(B) if b != bad]
                label = f"{sdr_type} zm={zm} log={tl} {where}[{bad}] = {v}"
                assert torch.equal(got[0][keep], clean[0][keep]), label
                assert torch.equal(got[1][keep], clean[1][keep]), label
                if v != 1e30:
                    assert not torch.isfinite(got[1][bad]).all(), label
                e1 = e.clone().requires_grad_(True)
                wrapper(e1, t).backward()
                assert torch.equal(e1.grad[keep], e0.grad[keep]), label


def test_zz_print_worst_errors():
    for kind, (err, label) in sorted(WORST.items()):
        print(f"worst {kind}: {err:.2e} at {label}")
