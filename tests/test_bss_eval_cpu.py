"""BSS-eval without a GPU: the two fp64 oracle formulations agree, the C-ABI symbols bind, the scratch query refuses
unsupported arguments, and the Python entry refuses CPU tensors and inputs that require grad."""
import numpy as np
import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from bss_oracle import bss_eval, bss_eval_direct

SYMBOLS = ("sdr_bss_eval_scratch_bytes", "sdr_bss_eval", "sdr_bss_eval_mixture")


def agree(a, b, tol):
    """Equal where infinite or NaN, within tol elsewhere."""
    a, b = np.asarray(a), np.asarray(b)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    return bool(np.all(same | (np.abs(a - b) <= tol)))


@pytest.mark.parametrize("S,T,F,seed", [(1, 60, 8, 0), (2, 200, 16, 1), (3, 150, 24, 2), (4, 120, 12, 3),
                                        (2, 90, 30, 4)])
def test_oracle_formulations_agree(S, T, F, seed):
    rng = np.random.default_rng(seed)
    refs = rng.standard_normal((S, T))
    refs[-1] = np.convolve(refs[-1], [1.0, 0.9, 0.5])[:T]                    # one coloured reference
    ests = rng.standard_normal((S, S)) @ refs + 0.05 * rng.standard_normal((S, T))
    ests[0] = np.convolve(ests[0], [0.7, -0.2, 0.1])[:T]
    for perm in (True, False):
        a, b = bss_eval(refs, ests, perm, F), bss_eval_direct(refs, ests, perm, F)
        for x, y in zip(a[:3], b[:3]):
            assert agree(x, y, 1e-9), (x, y)
        assert np.array_equal(a[3], b[3])


def test_oracle_silent_rows():
    refs = np.ones((2, 50))
    ests = np.ones((2, 50))
    ests[1] = 0
    sdr, sir, sar, perm = bss_eval(refs, ests, True, 4)
    assert np.isnan(sdr).all() and np.isnan(sir).all() and np.isnan(sar).all() and (perm == -1).all()


def test_symbols_bind_and_scratch_limits():
    lib = N.lib()
    for name in SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 32000, 512) > 0
    assert lib.sdr_bss_eval_scratch_bytes(1, 4, 4, 1) > 0 and lib.sdr_bss_eval_scratch_bytes(1, 4, 3, 1) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 5, 1000, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 0, 1000, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 1000, 0) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 1000, 513) == 0
    assert lib.sdr_bss_eval_scratch_bytes(0, 2, 1000, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 2, 0, 512) == 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 1, 1, 512) > 0                    # one reference: any length
    assert lib.sdr_bss_eval_scratch_bytes(4, 3, 1025, 512) > 0
    assert lib.sdr_bss_eval_scratch_bytes(4, 3, 1024, 512) == 0                # 3 x 512 delays in R^1535
    # null buffers are refused before anything is enqueued
    assert lib.sdr_bss_eval(None, None, None, None, None, None, 1, 2, 100, 16, 1, None, None) == -2


def test_refusals():
    x = torch.zeros(2, 100)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.bss_eval_sources(x, x)
    with pytest.raises(RuntimeError, match="shape"):
        P.bss_eval_sources(x, torch.zeros(3, 100))
    g = torch.zeros(2, 100, requires_grad=True)
    with pytest.raises(RuntimeError, match="CUDA|no autograd"):
        P.bss_eval_sources(g, x)
    assert P.bss_eval_sources is P.bss_eval.bss_eval_sources
