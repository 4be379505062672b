"""Oracle <-> unmodified original models.  The original's outputs on seeded weights and inputs are
stored in tests/golden/reference_live.npz (tests/golden/make_golden_live.py regenerates them from a
checkout of the original repository); the oracle must reproduce them."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import sudormrf_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.npz")
CASES = [
    ("improved", dict(out_channels=64, in_channels=128, num_blocks=4, upsampling_depth=5,
                      enc_kernel_size=21, enc_num_basis=128, num_sources=2), 3333),
    ("improved", dict(out_channels=32, in_channels=32, num_blocks=1, upsampling_depth=1,
                      enc_kernel_size=21, enc_num_basis=16, num_sources=1), 7),
    ("groupcomm", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                       enc_kernel_size=21, enc_num_basis=64, num_sources=2,
                       group_size=16), 2000),
    ("causal", dict(in_audio_channels=1, out_channels=32, in_channels=64, num_blocks=3, upsampling_depth=4,
                    enc_kernel_size=21, enc_num_basis=64, num_sources=2), 2000),
    ("original", dict(out_channels=64, in_channels=128, num_blocks=3, upsampling_depth=4,
                      enc_kernel_size=21, enc_num_basis=128, num_sources=2), 3333),
    ("original", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=5,
                      enc_kernel_size=21, enc_num_basis=32, num_sources=4), 1600),      # no reshape layer, T a multiple of the lcm
    # filter lengths 3 / 5 / 41 / 91, 1 / 4 / 5 / 16 sources, 4 and 16 audio channels, 3 and 12 groups
    ("improved", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
                      enc_kernel_size=41, enc_num_basis=64, num_sources=4), 341),
    ("improved", dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=3,
                      enc_kernel_size=3, enc_num_basis=32, num_sources=16), 151),
    ("improved", dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=3,
                      enc_kernel_size=5, enc_num_basis=32, num_sources=1), 333),
    ("groupcomm", dict(out_channels=64, in_channels=128, num_blocks=1, upsampling_depth=3,
                       enc_kernel_size=91, enc_num_basis=64, num_sources=4, group_size=16), 401),
    ("groupcomm", dict(in_audio_channels=4, out_channels=24, in_channels=48, num_blocks=1, upsampling_depth=3,
                       enc_kernel_size=5, enc_num_basis=16, num_sources=4, group_size=3), 101),
    ("groupcomm", dict(in_audio_channels=16, out_channels=48, in_channels=96, num_blocks=1, upsampling_depth=3,
                       enc_kernel_size=3, enc_num_basis=16, num_sources=1, group_size=12), 101),
    ("original", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
                      enc_kernel_size=11, enc_num_basis=48, num_sources=5), 401),       # hop 5: lcm 80
    ("original", dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3,
                      enc_kernel_size=5, enc_num_basis=32, num_sources=1), 400),        # one source: sigmoid
    ("original", dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=3,
                      enc_kernel_size=3, enc_num_basis=16, num_sources=16), 48),        # hop 1
    ("original", dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=4,
                      enc_kernel_size=41, enc_num_basis=32, num_sources=4), 401),       # hop 20: pads to 480, L = 24
]


def _stored_output(variant, kw, T):
    """The original model's output for this case, located by its constructor arguments in the golden file."""
    z = np.load(GOLDEN)
    meta = json.loads(bytes(z["meta"]).decode())
    for i, c in enumerate(meta["cases"]):
        if c["variant"] == variant and c["kw"] == kw and c["T"] == T:
            return meta, torch.from_numpy(z[f"c{i}/out"])
    raise AssertionError(f"no stored output for {variant} {kw} T={T}")


@pytest.mark.parametrize("variant,kw,T", CASES)
def test_live(variant, kw, T):
    meta, ref = _stored_output(variant, kw, T)
    cfg = O.Config(variant=variant, **kw)
    sd = O.make_state_dict(cfg, seed=meta["model_seed"])
    x = torch.randn(2, kw.get("in_audio_channels", 1), T, generator=torch.Generator().manual_seed(meta["input_seed"]))
    assert max(O.parity_errors(O.forward(cfg, sd, x), ref)) < 2e-5


def test_original_length_rule_is_the_reference_s():
    """The original model fails at K = 41, D = 4, T = 240 (the fixture records the reference's error): padding to a
    multiple of lcm(20, 16) = 80 leaves L = 12 frames, which its D - 1 = 3 stride-2 levels cannot halve exactly.  The
    C-ABI refuses that length before anything is enqueued (null buffers are never reached) and accepts T = 160 (L = 8),
    where only the null buffers are refused."""
    z = np.load(GOLDEN)
    refused = json.loads(bytes(z["meta"]).decode())["reference_refuses"]
    kw = dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=4, enc_kernel_size=41, enc_num_basis=32,
              num_sources=4)
    assert [(c["variant"], c["kw"], c["T"]) for c in refused] == [("original", kw, 240)]
    assert "must match" in refused[0]["error"]
    cfg = O.Config(variant="original", **kw)
    assert O.padded_length(cfg, 240) // cfg.hop == 12 and O.padded_length(cfg, 160) // cfg.hop == 8
    from sudo_rm_rf_b200 import _engine, _native
    import sudo_rm_rf_b200 as P
    lib = _native.lib()
    c = _engine.make_config(P.OriginalSuDORMRF(**kw))

    def fwd(T):
        return lib.sdr_forward(C.byref(c), None, None, None, 2, T, 0, None, 0, None)
    assert fwd(240) == -5                      # SDR_ERR_UNSUPPORTED
    assert fwd(160) == -2                      # SDR_ERR_BAD_ARGUMENT: past the length rule, stopped at the null buffers
