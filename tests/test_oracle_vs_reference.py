"""Oracle <-> unmodified original models.  The original's outputs on seeded weights and inputs are
stored in tests/golden/reference_live.npz (tests/golden/make_golden_live.py regenerates them from a
checkout of the original repository); the oracle must reproduce them."""
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
    x = torch.randn(2, 1, T, generator=torch.Generator().manual_seed(meta["input_seed"]))
    assert max(O.parity_errors(O.forward(cfg, sd, x), ref)) < 2e-5
