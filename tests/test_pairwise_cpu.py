"""The improved model's training loss without a GPU: the fp64 oracle (``O.pairwise_neg_sdr``, ``O.pit_from_pairwise``)
against goldens from the unmodified reference (tests/golden/make_golden_pairwise.py) in values and autograd gradients,
the new C-ABI symbols and size queries, and the refusals that fire before any device work."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import sisdr as S
from oracle import sudormrf_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prepost_pairwise_grad.npz")
SYMBOLS = ("sdr_pairwise_neg_sdr_train", "sdr_pairwise_neg_sdr_backward", "sdr_pairwise_neg_sdr_train_scratch_bytes",
           "sdr_pairwise_neg_sdr_coef_bytes")
BAD_ARGUMENT, UNSUPPORTED = -2, -5


def load():
    z = np.load(GOLDEN)
    meta = json.loads(bytes(z["meta"]).decode())
    # the fp32 inputs are computed on in fp64, as the reference was
    pick = lambda prefix: {k[len(prefix):]: torch.from_numpy(z[k]).to(torch.float64)   # noqa: E731
                           for k in z.files if k.startswith(prefix)}
    return [(c, pick(f"c{i}/")) for i, c in enumerate(meta["cases"])]


CASES = load()


def assert_close_rows(got, ref, tol, label):
    """max |got - ref| per row (all but the last axis) within tol of that row's max |ref|."""
    d = (got - ref).abs().reshape(-1, ref.shape[-1]).amax(1)
    m = ref.abs().reshape(-1, ref.shape[-1]).amax(1)
    assert bool((d <= tol * m).all()), (label, (d / m.clamp_min(1e-300)).max().item())


@pytest.mark.parametrize("ci", range(len(CASES)), ids=[f"{i}-{c['name']}-{c['sdr_type']}-zm{int(c['zero_mean'])}-"
                                                        f"log{int(c['take_log'])}-S{c['S']}"
                                                        for i, (c, _) in enumerate(CASES)])
def test_pairwise_oracle_matches_reference_golden(ci):
    c, t = CASES[ci]
    est = t["est"].clone().requires_grad_(True)
    pw = O.pairwise_neg_sdr(est, t["tgt"], c["sdr_type"], c["zero_mean"], c["take_log"])
    assert torch.allclose(pw.detach(), t["pw"], atol=1e-12, rtol=1e-12), (pw, t["pw"])
    (pw * t["w"]).sum().backward()
    assert_close_rows(est.grad, t["grad"], 1e-12, "pairwise grad")
    est2 = t["est"].clone().requires_grad_(True)
    best, _ = O.pit_from_pairwise(O.pairwise_neg_sdr(est2, t["tgt"], c["sdr_type"], c["zero_mean"], c["take_log"]))
    loss = best.mean()
    assert torch.allclose(loss.detach(), t["pit_loss"], atol=1e-12, rtol=1e-12), (loss, t["pit_loss"])
    loss.backward()
    assert_close_rows(est2.grad, t["pit_grad"], 1e-12, "PIT grad")


def test_golden_covers_every_type_flag_source_count_and_the_degenerate_rows():
    seen = {(c["sdr_type"], c["zero_mean"], c["take_log"], c["S"]) for c, _ in CASES if c["name"] == "flags"}
    assert len(seen) == 3 * 4 * 4
    degenerate = [(c, t) for c, t in CASES if c["name"] == "degenerate"]
    assert len(degenerate) == 3 * 4
    for c, t in degenerate:
        assert float(t["tgt"][0, 0].abs().max()) == 0.0                         # a silent target
        assert bool((t["est"][1, 1] == t["est"][1, 1, 0]).all())                # a constant estimate row
        assert torch.equal(t["est"][2, 2], t["tgt"][2, 2])                      # an estimate equal to its target
    assert all(t["est"].shape[-1] % 2 == 1 for _, t in CASES)


def test_new_symbols_bind():
    lib = N.lib()
    for name in SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS
        assert getattr(lib, name) is not None


def test_scratch_and_coef_sizes():
    lib = N.lib()
    for bad in (0, 5):
        assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(3, bad, 1000) == 0
        assert lib.sdr_pairwise_neg_sdr_coef_bytes(3, bad) == 0
    assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(0, 2, 1000) == 0
    assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(2, 2, 0) == 0
    for s in range(1, 5):
        n_gram = 2 * s + 2 * s * s + s                       # sums of e and t, ET, EE, the full TT
        assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(3, s, 1) == 8 * 3 * n_gram
        assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(3, s, 4096) == 8 * 3 * n_gram
        assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(3, s, 4097) == 8 * 3 * 2 * n_gram
        assert lib.sdr_pairwise_neg_sdr_train_scratch_bytes(2, s, 10 ** 7) == 8 * 2 * 64 * n_gram
        assert lib.sdr_pairwise_neg_sdr_coef_bytes(7, s) == 8 * 7 * (3 * s * s + 2 * s)


def test_entries_refuse_bad_arguments_without_launching():
    lib = N.lib()
    fake = C.c_void_p(4096)                                   # never dereferenced: every call below refuses first
    assert lib.sdr_pairwise_neg_sdr_train(None, None, None, None, 2, 2, 100, 1, 1, 1, None, None) == BAD_ARGUMENT
    assert lib.sdr_pairwise_neg_sdr_backward(None, None, None, None, None, 2, 2, 100, None) == BAD_ARGUMENT
    for B, T, sdr_type in ((0, 100, 1), (2, 0, 1), (2, 100, 3), (2, 100, -1)):
        assert lib.sdr_pairwise_neg_sdr_train(fake, fake, fake, fake, B, 2, T, sdr_type, 1, 1, fake, None) == BAD_ARGUMENT
    for B, T in ((0, 100), (2, 0)):
        assert lib.sdr_pairwise_neg_sdr_backward(fake, fake, fake, fake, fake, B, 2, T, None) == BAD_ARGUMENT
    odd = C.c_void_p(4100)                                    # coef and scratch must be 8-byte aligned
    assert lib.sdr_pairwise_neg_sdr_train(fake, fake, fake, odd, 2, 2, 100, 1, 1, 1, fake, None) == BAD_ARGUMENT
    assert lib.sdr_pairwise_neg_sdr_train(fake, fake, fake, fake, 2, 2, 100, 1, 1, 1, odd, None) == BAD_ARGUMENT
    assert lib.sdr_pairwise_neg_sdr_backward(fake, fake, odd, fake, fake, 2, 2, 100, None) == BAD_ARGUMENT
    for s in (0, 5):
        assert lib.sdr_pairwise_neg_sdr_train(fake, fake, fake, fake, 2, s, 100, 1, 1, 1, fake, None) == UNSUPPORTED
        assert lib.sdr_pairwise_neg_sdr_backward(fake, fake, fake, fake, fake, 2, s, 100, None) == UNSUPPORTED


def test_refuses_targets_that_require_grad():
    fn = S.PairwiseNegSDR("sisdr")
    with pytest.raises(RuntimeError, match="targets that do not require grad"):
        fn(torch.randn(2, 2, 100, requires_grad=True), torch.randn(2, 2, 100, requires_grad=True))
    with pytest.raises(RuntimeError, match="targets that do not require grad"):
        fn(torch.randn(2, 2, 100), torch.randn(2, 2, 100, requires_grad=True))


@pytest.mark.parametrize("est_grad", [False, True])
def test_refuses_cpu_tensors(est_grad):
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        S.PairwiseNegSDR("sdsdr")(torch.randn(2, 3, 100, requires_grad=est_grad), torch.randn(2, 3, 100))


@pytest.mark.parametrize("est_grad", [False, True])
def test_refuses_five_sources(est_grad):
    with pytest.raises(N.NativeError, match="1..4 sources"):
        S.PairwiseNegSDR("snr")(torch.randn(2, 5, 100, requires_grad=est_grad), torch.randn(2, 5, 100))


@pytest.mark.parametrize("e,t", [((2, 2, 100), (3, 2, 100)), ((2, 3, 100), (2, 2, 100)), ((2, 2, 100), (2, 2, 99))])
def test_refuses_mismatched_shapes(e, t):
    with pytest.raises(AssertionError):                       # the reference's own assert (sisdr.py:417)
        S.PairwiseNegSDR("sisdr")(torch.randn(*e, requires_grad=True), torch.randn(*t))


def test_refuses_inputs_that_are_not_three_dimensional():
    with pytest.raises(RuntimeError, match="shape"):
        S.PairwiseNegSDR("sisdr")(torch.randn(2, 100, requires_grad=True), torch.randn(2, 100))


def test_wrapper_permutation_table_is_made_once_per_source_count_and_device():
    a = S._perms(3, torch.device("cpu"))
    assert a is S._perms(3, torch.device("cpu"))
    assert a.tolist() == [[0, 1, 2], [0, 2, 1], [1, 0, 2], [1, 2, 0], [2, 0, 1], [2, 1, 0]]
    assert a.dtype == torch.long


def test_wrapper_on_the_cpu_oracle_still_backpropagates():
    """find_best_perm and reorder_source on the cached table: the wrapper's loss, index and gradient as the oracle's."""
    g = torch.Generator().manual_seed(5)
    tgt = torch.randn(3, 3, 40, generator=g, dtype=torch.float64)
    est = (tgt[:, [2, 0, 1]] + 0.1 * torch.randn(3, 3, 40, generator=g, dtype=torch.float64)).requires_grad_(True)
    pw = lambda e, t: O.pairwise_neg_sdr(e, t, "sisdr")                                     # noqa: E731
    loss, reordered = S.PITLossWrapper(pw, pit_from="pw_mtx")(est, tgt, return_est=True)
    loss.backward()
    e2 = est.detach().clone().requires_grad_(True)
    best, idx = O.pit_from_pairwise(pw(e2, tgt))
    best.mean().backward()
    assert torch.allclose(loss, best.mean(), atol=1e-12, rtol=0)
    assert torch.allclose(est.grad, e2.grad, atol=1e-12, rtol=0)
    assert float((reordered.detach() - tgt).abs().max()) < 1.0
