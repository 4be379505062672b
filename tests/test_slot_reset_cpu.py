"""The refusals of the five slot-reset entries, without a GPU: every faulty argument and pair of them returns the code
it returned before the resets shared one helper.  Each call is refused before any CUDA call, so the state addresses
are never dereferenced."""
import ctypes as C
import os

import pytest

from sudo_rm_rf_b200 import _native as N

BAD_CONFIG, BAD_ARGUMENT, WORKSPACE, UNSUPPORTED = -1, -2, -3, -5
X = 1 << 20                  # a non-null address aligned to 256 bytes
MIS = X + 8                  # misaligned for every state (16 bytes for the causal one, 256 for the others)
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sudo_rm_rf_b200", "csrc")


def slots(*idx):
    return (C.c_int32 * max(1, len(idx)))(*idx)


def causal_cfg(variant=2, k=21):
    return N.SdrConfig(variant, 1, 16, 32, 1, 4, k, 16, 2, 1)


# (state, B, slots, n, cfg) -> code
CAUSAL = [
    ("B=0", dict(B=0), BAD_ARGUMENT),
    ("n<0", dict(sl=slots(0), n=-1), BAD_ARGUMENT),
    ("index -1", dict(sl=slots(0, -1), n=2), BAD_ARGUMENT),
    ("index B", dict(sl=slots(1, 2), n=2), BAD_ARGUMENT),
    ("null state", dict(state=None), BAD_ARGUMENT),
    ("misaligned", dict(state=MIS), BAD_ARGUMENT),
    ("bad config", dict(cfg=causal_cfg(k=20)), BAD_CONFIG),
    ("not causal", dict(cfg=causal_cfg(variant=0)), UNSUPPORTED),
    ("bad config, null state", dict(cfg=causal_cfg(k=20), state=None), BAD_CONFIG),
    ("not causal, B=0", dict(cfg=causal_cfg(variant=0), B=0), UNSUPPORTED),
    ("B=0, null state", dict(B=0, state=None), BAD_ARGUMENT),
    ("n<0, misaligned", dict(sl=slots(0), n=-1, state=MIS), BAD_ARGUMENT),
    ("index B, misaligned", dict(sl=slots(2), n=1, state=MIS), BAD_ARGUMENT),
]


@pytest.mark.parametrize("kw,want", [c[1:] for c in CAUSAL], ids=[c[0] for c in CAUSAL])
def test_causal_reset(kw, want):
    a = dict(state=X, B=2, sl=None, n=0, cfg=causal_cfg())
    a.update(kw)
    assert N.lib().sdr_stream_reset(C.byref(a["cfg"]), a["state"], a["B"], a["sl"], a["n"], None) == want


CAUSAL_MASKED = [
    ("B=0", dict(B=0), BAD_ARGUMENT),
    ("null mask", dict(mask=None), BAD_ARGUMENT),
    ("null state", dict(state=None), BAD_ARGUMENT),
    ("misaligned", dict(state=MIS), BAD_ARGUMENT),
    ("bad config", dict(cfg=causal_cfg(k=20)), BAD_CONFIG),
    ("not causal", dict(cfg=causal_cfg(variant=0)), UNSUPPORTED),
    ("bad config, null mask", dict(cfg=causal_cfg(k=20), mask=None), BAD_CONFIG),
    ("not causal, null state", dict(cfg=causal_cfg(variant=0), state=None), UNSUPPORTED),
    ("null mask, misaligned", dict(mask=None, state=MIS), BAD_ARGUMENT),
    ("B=0, null mask", dict(B=0, mask=None), BAD_ARGUMENT),
]


@pytest.mark.parametrize("kw,want", [c[1:] for c in CAUSAL_MASKED], ids=[c[0] for c in CAUSAL_MASKED])
def test_causal_reset_masked(kw, want):
    a = dict(state=X, B=2, mask=X, cfg=causal_cfg())
    a.update(kw)
    assert N.lib().sdr_stream_reset_masked(C.byref(a["cfg"]), a["state"], a["B"], a["mask"], None) == want


# windowed shape (B, S, A, W, H) = (2, 2, 1, 10, 5)
WINDOWED = [
    ("B=0", dict(B=0), BAD_ARGUMENT),
    ("n<0", dict(sl=slots(0), n=-1), BAD_ARGUMENT),
    ("index -1", dict(sl=slots(-1), n=1), BAD_ARGUMENT),
    ("index B", dict(sl=slots(0, 2), n=2), BAD_ARGUMENT),
    ("null state", dict(state=None), BAD_ARGUMENT),
    ("misaligned", dict(state=MIS), BAD_ARGUMENT),
    ("S=5", dict(S=5), UNSUPPORTED),
    ("H>=W", dict(H=10), BAD_ARGUMENT),
    ("H<W/2", dict(H=4), BAD_ARGUMENT),
    ("A=0", dict(A=0), BAD_ARGUMENT),
    ("S=5, B=0", dict(S=5, B=0), UNSUPPORTED),
    ("S=5, null state", dict(S=5, state=None), BAD_ARGUMENT),
    ("S=5, misaligned", dict(S=5, state=MIS), UNSUPPORTED),
    ("S=5, n<0", dict(S=5, sl=slots(0), n=-1), BAD_ARGUMENT),
    ("S=5, index B", dict(S=5, sl=slots(2), n=1), UNSUPPORTED),
    ("H>=W, misaligned", dict(H=10, state=MIS), BAD_ARGUMENT),
    ("index B, misaligned", dict(sl=slots(2), n=1, state=MIS), BAD_ARGUMENT),
]


@pytest.mark.parametrize("kw,want", [c[1:] for c in WINDOWED], ids=[c[0] for c in WINDOWED])
def test_windowed_reset(kw, want):
    a = dict(state=X, B=2, S=2, A=1, W=10, H=5, sl=None, n=0)
    a.update(kw)
    assert N.lib().sdr_window_stream_reset(a["state"], a["B"], a["S"], a["A"], a["W"], a["H"], a["sl"], a["n"],
                                           None) == want


WINDOWED_MASKED = [
    ("B=0", dict(B=0), BAD_ARGUMENT),
    ("null mask", dict(mask=None), BAD_ARGUMENT),
    ("null state", dict(state=None), BAD_ARGUMENT),
    ("misaligned", dict(state=MIS), BAD_ARGUMENT),
    ("S=5", dict(S=5), UNSUPPORTED),
    ("H>=W", dict(H=10), BAD_ARGUMENT),
    ("S=5, null mask", dict(S=5, mask=None), BAD_ARGUMENT),
    ("S=5, misaligned", dict(S=5, state=MIS), UNSUPPORTED),
    ("S=5, B=0", dict(S=5, B=0), UNSUPPORTED),
    ("H>=W, misaligned", dict(H=10, state=MIS), BAD_ARGUMENT),
]


@pytest.mark.parametrize("kw,want", [c[1:] for c in WINDOWED_MASKED], ids=[c[0] for c in WINDOWED_MASKED])
def test_windowed_reset_masked(kw, want):
    a = dict(state=X, B=2, S=2, A=1, W=10, H=5, mask=X)
    a.update(kw)
    assert N.lib().sdr_window_stream_reset_masked(a["state"], a["B"], a["S"], a["A"], a["W"], a["H"], a["mask"],
                                                  None) == want


# resampling plan (B, rows, C, up, down, delay, lead) = (2, 1, 441, 8000, 44100, 10, 0)
PLAN = dict(B=2, rows=1, C=441, up=8000, down=44100, delay=10, lead=0)
RESAMPLING = [
    ("B=0", dict(B=0), BAD_ARGUMENT),
    ("n<0", dict(sl=slots(0), n=-1), BAD_ARGUMENT),
    ("index -1", dict(sl=slots(1, -1), n=2), BAD_ARGUMENT),
    ("index B", dict(sl=slots(2), n=1), BAD_ARGUMENT),
    ("null state", dict(state=None), BAD_ARGUMENT),
    ("misaligned", dict(state=MIS), BAD_ARGUMENT),
    ("small state", dict(nb=-1), WORKSPACE),
    ("ratio past 4096", dict(up=1, down=4097, C=4097), UNSUPPORTED),
    ("delay below its least", dict(delay=9), BAD_ARGUMENT),
    ("n<0, small state", dict(sl=slots(0), n=-1, nb=-1), BAD_ARGUMENT),
    ("index B, small state", dict(sl=slots(2), n=1, nb=-1), WORKSPACE),
    ("index -1, misaligned", dict(sl=slots(-1), n=1, state=MIS), BAD_ARGUMENT),
    ("misaligned, small state", dict(state=MIS, nb=-1), WORKSPACE),
    ("null state, small state", dict(state=None, nb=-1), BAD_ARGUMENT),
    ("ratio past 4096, null state", dict(up=1, down=4097, C=4097, state=None), UNSUPPORTED),
    ("ratio past 4096, n<0", dict(up=1, down=4097, C=4097, sl=slots(0), n=-1), UNSUPPORTED),
    ("B=0, small state", dict(B=0, nb=-1), BAD_ARGUMENT),
    ("delay below its least, misaligned", dict(delay=9, state=MIS), BAD_ARGUMENT),
]


@pytest.mark.parametrize("kw,want", [c[1:] for c in RESAMPLING], ids=[c[0] for c in RESAMPLING])
def test_resampling_reset(kw, want):
    lib = N.lib()
    need = lib.sdr_resample_stream_state_bytes(*PLAN.values())
    assert need > 0
    a = dict(PLAN, state=X, nb=0, sl=None, n=0)
    a.update(kw)
    plan = [a[k] for k in PLAN]
    assert lib.sdr_resample_stream_reset(a["state"], need + a["nb"], *plan, a["sl"], a["n"], None) == want


def test_every_cuda_status_goes_through_cuda_status():
    """Only launch.cuh compares a runtime status with cudaSuccess: every other call goes through cuda_status, which
    clears the runtime's last error on the way out."""
    found = []
    for name in sorted(os.listdir(CSRC)):
        if name != "launch.cuh" and name.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                found += [f"{name}:{i}" for i, line in enumerate(f, 1) if "cudaSuccess" in line]
    assert not found, found
