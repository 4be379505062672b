"""Polyphase resampling without a GPU: the C-ABI symbols, the scratch query and the refusals before any launch, the
Python entry's refusals and the rate arguments of ``separate`` / ``separate_long``."""
import itertools
import math
import os
import re

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import resample

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("sdr_resample_poly_scratch_bytes", "sdr_resample_poly")
RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000)
ERR_BAD_ARGUMENT, ERR_WORKSPACE, ERR_UNSUPPORTED = -2, -3, -5


def test_symbols_bind_and_match_the_header():
    lib = N.lib()
    header = open(os.path.join(REPO, "include", "sudormrf_b200.h")).read()
    for name in SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\b" + name + r"\(", header), name
    assert P.resample_poly is resample.resample_poly


@pytest.mark.parametrize("up,down", [(1, 1), (3, 3), (1, 6), (6, 1), (80, 441), (441, 80), (147, 2560),
                                     (2560, 147), (1, 4096), (4096, 1), (4096, 4095), (6, 36)])
def test_scratch_is_the_filter(up, down):
    g = math.gcd(up, down)
    mx = max(up, down) // g
    assert N.lib().sdr_resample_poly_scratch_bytes(up, down) == 8 * (20 * mx + 1)


def test_scratch_refuses_ratios():
    lib = N.lib()
    for up, down in ((0, 1), (1, 0), (-1, 1), (1, -8), (0, 0), (1, 4097), (4097, 1), (4097, 4096), (4099, 2)):
        assert lib.sdr_resample_poly_scratch_bytes(up, down) == 0, (up, down)
    assert lib.sdr_resample_poly_scratch_bytes(8194, 2) == 0             # reduces to 4097 / 1
    assert lib.sdr_resample_poly_scratch_bytes(8192, 2) > 0              # reduces to 4096 / 1


def test_every_standard_pair_is_within_the_limit():
    worst = 0
    for a, b in itertools.permutations(RATES, 2):
        g = math.gcd(a, b)
        worst = max(worst, a // g, b // g)
        assert N.lib().sdr_resample_poly_scratch_bytes(a, b) > 0, (a, b)
    assert worst == 2560                                                  # 11.025 <-> 192 kHz: 147 / 2560


def test_abi_refusals_before_any_launch():
    lib = N.lib()
    x = 8                       # any non-null, 8-byte aligned address: these calls return before reading a buffer
    need = lib.sdr_resample_poly_scratch_bytes(1, 6)

    def call(xp, op, rows, T, up, down, sp, sb):
        return lib.sdr_resample_poly(xp, op, rows, T, up, down, sp, sb, None)
    assert call(None, x, 1, 100, 1, 6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, None, 1, 100, 1, 6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 1, 100, 1, 6, None, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 1, 100, 1, 6, 12, need) == ERR_BAD_ARGUMENT                # misaligned scratch
    assert call(x, x, 1, 100, 1, 6, x, need - 8) == ERR_WORKSPACE
    assert call(x, x, 0, 100, 1, 6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 1, 0, 1, 6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 1, 2 ** 40 + 1, 1, 6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 2 ** 40, 2 ** 40, 1, 6, x, need) == ERR_BAD_ARGUMENT           # rows x length past 2^62 / 4096
    assert call(x, x, 1, 100, 0, 6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 1, 100, 1, -6, x, need) == ERR_BAD_ARGUMENT
    assert call(x, x, 1, 100, 1, 4097, x, 1 << 30) == ERR_UNSUPPORTED


def test_python_refusals():
    x = torch.zeros(2, 100)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.resample_poly(x, 1, 6)
    for up, down in ((0, 1), (1, 0), (-2, 3), (1.5, 2), (True, 2), (2, None), (1, 4097), (4097 * 2, 2)):
        with pytest.raises(ValueError):
            P.resample_poly(x, up, down)


MODELS = {
    "improved": (P.SuDORMRF, dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=2,
                                  enc_kernel_size=5, enc_num_basis=16, num_sources=2)),
    "groupcomm": (P.GroupCommSudoRmRf, dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=2,
                                            enc_kernel_size=5, enc_num_basis=16, num_sources=2, group_size=4)),
    "causal": (P.CausalSuDORMRF, dict(in_audio_channels=1, out_channels=16, in_channels=32, num_blocks=1,
                                      upsampling_depth=2, enc_kernel_size=5, enc_num_basis=16, num_sources=2)),
    "original": (P.OriginalSuDORMRF, dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=2,
                                          enc_kernel_size=5, enc_num_basis=16, num_sources=2)),
}


@pytest.mark.parametrize("name", list(MODELS))
def test_rate_arguments(name):
    cls, kw = MODELS[name]
    m = cls(**kw).eval()
    x = torch.zeros(1, 1, 400)
    bad = [dict(sample_rate=44100), dict(model_rate=8000), dict(sample_rate=0, model_rate=8000),
           dict(sample_rate=44100, model_rate=-8000), dict(sample_rate=44100.0, model_rate=8000),
           dict(sample_rate=True, model_rate=8000), dict(sample_rate=8000, model_rate=8000 * 4097)]
    for rates in bad:
        with pytest.raises(ValueError):
            m.separate(x, **rates)
        with pytest.raises(ValueError):
            m.separate_long(x, 200, **rates)
    # equal rates (or none) are the existing call: on a CPU tensor, its own refusal
    for rates in (dict(), dict(sample_rate=16000, model_rate=16000)):
        with pytest.raises(RuntimeError) as plain:
            m.separate(x)
        with pytest.raises(RuntimeError) as same:
            m.separate(x, **rates)
        assert str(plain.value) == str(same.value)
    # different rates: the mixture must be on the GPU for the resampler
    with pytest.raises(RuntimeError, match="CUDA"):
        m.separate(x, sample_rate=44100, model_rate=8000)
