"""The FUSS training step after the model, without a GPU: the fp64 oracle (``snr_oracle.snr_zero_refs``,
``O.mixture_consistency``) against goldens from the unmodified reference (tests/golden/make_golden_snr.py) in values,
permutations and autograd gradients, the new C-ABI symbols, and the refusals that fire before any device work."""
import itertools
import json
import os

import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
from snr_oracle import snr_zero_refs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prepost_snr_zero_refs.npz")
SYMBOLS = ("sdr_mixture_consistency_backward", "sdr_mixture_consistency_backward_scratch_bytes", "sdr_snr_zero_refs",
           "sdr_snr_zero_refs_backward", "sdr_snr_zero_refs_scratch_bytes", "sdr_snr_zero_refs_coef_bytes")


def load():
    z = np.load(GOLDEN)
    meta = json.loads(bytes(z["meta"]).decode())
    # the fp32 inputs are computed on in fp64, as the reference was
    pick = lambda prefix: {k[len(prefix):]: torch.from_numpy(z[k]).to(torch.float64 if z[k].dtype.kind == "f" else None)   # noqa
                           for k in z.files if k.startswith(prefix)}
    return ([(c, pick(f"snr{i}/")) for i, c in enumerate(meta["snr"])],
            [(c, pick(f"mc{i}/")) for i, c in enumerate(meta["mc"])])


SNR, MC = load()


def assert_close_rows(got, ref, tol, label):
    """max |got - ref| per item within tol of that item's max |ref|."""
    d = (got - ref).abs().reshape(ref.shape[0], -1).amax(1)
    m = ref.abs().reshape(ref.shape[0], -1).amax(1).clamp_min(1e-300)
    assert bool((d <= tol * m).all()), (label, (d / m).max().item())


@pytest.mark.parametrize("ci", range(len(SNR)), ids=[f"{i}-{c['name']}-S{c['S']}" for i, (c, _) in enumerate(SNR)])
def test_snr_zero_refs_oracle_matches_reference_golden(ci):
    c, t = SNR[ci]
    est = t["est"].clone().requires_grad_(True)
    best, idx = snr_zero_refs(est, t["tgt"], zero_mean=c["zero_mean"], inactivity_threshold=c["thr"], eps=c["eps"])
    value = best if c["individual"] else best.mean()
    if c["backward_loss"]:
        value = -value
    assert torch.allclose(value.detach(), t["value"], atol=1e-12, rtol=0), (value, t["value"])
    perms = list(itertools.permutations(range(c["S"])))
    assert [perms[int(i)] for i in idx] == [tuple(int(v) for v in row) for row in t["perms"]]
    (value * t["w"]).sum().backward()
    assert est.grad.shape == t["grad"].shape
    assert_close_rows(est.grad, t["grad"], 1e-12, c["name"])


def test_snr_golden_covers_the_degenerate_rows():
    """The all-silent item scores 0 for every permutation and has no gradient; the tie item is in the set."""
    for c, t in SNR:
        if c["name"] == "degenerate":
            assert float(t["value"][2]) == 0.0
            assert float(t["grad"][2].abs().max()) == 0.0
            assert torch.equal(t["est"][3, 1], t["est"][3, 0])
    assert {c["name"] for c, _ in SNR} >= {"flags", "degenerate", "crop"}
    assert any(t["est"].shape[-1] > t["tgt"].shape[-1] for _, t in SNR)
    assert any(t["est"].shape[-1] < t["tgt"].shape[-1] for _, t in SNR)


@pytest.mark.parametrize("mi", range(len(MC)), ids=[f"{c['kind']}-S{c['S']}" for c, _ in MC])
def test_mixture_consistency_oracle_gradients_match_reference_golden(mi):
    c, t = MC[mi]
    est = t["est"].clone().requires_grad_(True)
    mix = t["mix"].clone().requires_grad_(True)
    out = O.mixture_consistency(est, mix, c["kind"])
    assert torch.allclose(out.detach(), t["out"], atol=1e-12, rtol=0)
    (out * t["g"]).sum().backward()
    assert_close_rows(est.grad, t["grad_est"], 1e-12, "grad_est")
    assert_close_rows(mix.grad, t["grad_mix"], 1e-12, "grad_mix")


def test_new_symbols_bind():
    lib = N.lib()
    for name in SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS
        assert getattr(lib, name) is not None


def test_scratch_queries():
    lib = N.lib()
    assert lib.sdr_snr_zero_refs_scratch_bytes(3, 5, 1000) == 0
    assert lib.sdr_snr_zero_refs_scratch_bytes(3, 0, 1000) == 0
    for S in range(1, 5):
        n_gram = 2 * S + 2 * S * S + S
        assert lib.sdr_snr_zero_refs_scratch_bytes(3, S, 4096) == 8 * 3 * n_gram
        assert lib.sdr_snr_zero_refs_scratch_bytes(3, S, 4097) == 8 * 3 * 2 * n_gram
        assert lib.sdr_snr_zero_refs_scratch_bytes(2, S, 10 ** 7) == 8 * 2 * 64 * n_gram
        assert lib.sdr_snr_zero_refs_coef_bytes(7, S) == 8 * 7 * 4 * S
    assert lib.sdr_mixture_consistency_backward_scratch_bytes(2, 4, 1000, 0) == 0
    assert lib.sdr_mixture_consistency_backward_scratch_bytes(2, 4, 4097, 1) == 16 * 2 * 4 * 3


def test_entries_refuse_bad_arguments_without_launching():
    lib = N.lib()
    assert lib.sdr_snr_zero_refs(None, None, None, None, None, 2, 2, 100, 0, -40.0, 1e-9, None, None) == -2   # SDR_ERR_BAD_ARGUMENT
    assert lib.sdr_snr_zero_refs_backward(None, None, None, None, None, 2, 2, 100, 100, None) == -2
    assert lib.sdr_mixture_consistency_backward(None, None, None, None, None, 2, 2, 100, 0, None, None) == -2


def loss(**kw):
    d = dict(n_sources=4, zero_mean=False, backward_loss=True, inactivity_threshold=-40.)
    d.update(kw)
    return P.snr.PermInvariantSNRwithZeroRefs(**d)


def test_snr_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        loss()(torch.randn(2, 4, 100), torch.randn(2, 4, 100))


def test_snr_refuses_five_sources():
    with pytest.raises(N.NativeError, match="1..4 sources"):
        loss(n_sources=5)(torch.randn(2, 5, 100), torch.randn(2, 5, 100))


def test_snr_refuses_targets_that_require_grad():
    with pytest.raises(RuntimeError, match="t_batch"):
        loss()(torch.randn(2, 4, 100, requires_grad=True), torch.randn(2, 4, 100, requires_grad=True))


@pytest.mark.parametrize("pr,t", [((2, 4, 100), (3, 4, 100)), ((2, 3, 100), (2, 4, 100)), ((2, 4, 100), (2, 4)),
                                  ((2, 3, 100), (2, 3, 100))])
def test_snr_refuses_mismatched_shapes(pr, t):
    with pytest.raises(RuntimeError, match="shape"):
        loss()(torch.randn(*pr), torch.randn(*t))


def test_snr_keeps_the_reference_constructor():
    fn = loss(zero_mean=True, return_individual_results=True)
    assert fn.perform_zero_mean and fn.backward_loss and fn.return_individual_results
    assert fn.inactivity_threshold == -40. and fn.n_sources == 4
    assert fn.permutations_tensor.tolist() == [list(p) for p in itertools.permutations(range(4))]


def test_mixture_consistency_refusals_unchanged_under_grad():
    est = torch.randn(2, 3, 100, requires_grad=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.mixture_consistency.apply(est, torch.randn(2, 1, 100))
    with pytest.raises(ValueError, match="weight type"):
        P.mixture_consistency.apply(est, torch.randn(2, 1, 100), "bogus")
