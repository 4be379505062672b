"""Golden fixture ``reference_live.npz``: outputs of the UNMODIFIED original models and of its
``PermInvariantSISDR`` on seeded inputs, for tests/test_oracle_vs_reference.py and
tests/test_prepost_oracle.py::test_pit_sisdr_live_against_reference.  Needs a checkout of the
original sudo_rm_rf repository, named by SUDO_RM_RF_REFERENCE:

    SUDO_RM_RF_REFERENCE=/path/to/sudo_rm_rf python tests/golden/make_golden_live.py

Only the reference outputs are stored: the weights (``O.make_state_dict``) and the inputs are
regenerated from their seeds by the tests.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.environ["SUDO_RM_RF_REFERENCE"])
sys.path.insert(0, REPO)
warnings.filterwarnings("ignore")

import sudo_rm_rf.dnn.models.improved_sudormrf as ri                      # noqa: E402
import sudo_rm_rf.dnn.models.groupcomm_sudormrf_v2 as rg                  # noqa: E402
import sudo_rm_rf.dnn.models.causal_improved_sudormrf_v3 as rc            # noqa: E402
import sudo_rm_rf.dnn.models.sudormrf as ro                               # noqa: E402
import sudo_rm_rf.dnn.losses.sisdr as ref_sisdr                           # noqa: E402
from oracle import sudormrf_oracle as O                                   # noqa: E402

MODEL_SEED, INPUT_SEED = 11, 5
CASES = [
    ("improved", dict(out_channels=64, in_channels=128, num_blocks=4, upsampling_depth=5,
                      enc_kernel_size=21, enc_num_basis=128, num_sources=2), 3333),
    ("improved", dict(out_channels=32, in_channels=32, num_blocks=1, upsampling_depth=1,
                      enc_kernel_size=21, enc_num_basis=16, num_sources=1), 7),
    ("groupcomm", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                       enc_kernel_size=21, enc_num_basis=64, num_sources=2, group_size=16), 2000),
    ("causal", dict(in_audio_channels=1, out_channels=32, in_channels=64, num_blocks=3, upsampling_depth=4,
                    enc_kernel_size=21, enc_num_basis=64, num_sources=2), 2000),
    ("original", dict(out_channels=64, in_channels=128, num_blocks=3, upsampling_depth=4,
                      enc_kernel_size=21, enc_num_basis=128, num_sources=2), 3333),
    ("original", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=5,
                      enc_kernel_size=21, enc_num_basis=32, num_sources=4), 1600),   # no reshape layer, T a multiple of the lcm
    # the geometry around the blocks: filter lengths 3 / 5 / 41 / 91 (hop 1, 2, 20, 45), 1 / 4 / 5 / 16 sources,
    # 4 and 16 audio channels, a group count that is not a power of two
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
                      enc_kernel_size=11, enc_num_basis=48, num_sources=5), 401),    # hop 5: lcm 80
    ("original", dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3,
                      enc_kernel_size=5, enc_num_basis=32, num_sources=1), 400),     # one source: sigmoid
    ("original", dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=3,
                      enc_kernel_size=3, enc_num_basis=16, num_sources=16), 48),     # hop 1
    ("original", dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=4,
                      enc_kernel_size=41, enc_num_basis=32, num_sources=4), 401),    # hop 20: pads to 480, L = 24
]
# Lengths the original model itself cannot run: padding to a multiple of lcm(hop, 2^D) leaves L = Tp / hop with
# L % 2^(D-1) != 0, and the up-sample + add of its U-ConvBlock (sudormrf.py:180-182) then meets mismatched lengths.
# The C-ABI refuses these lengths for the same reason.
REFUSED = [
    ("original", dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=4,
                      enc_kernel_size=41, enc_num_basis=32, num_sources=4), 240),    # L = 12
]
CLASSES = {"improved": ri.SuDORMRF, "groupcomm": rg.GroupCommSudoRmRf, "causal": rc.CausalSuDORMRF,
           "original": ro.SuDORMRF}


def pit_inputs():
    """Seeded PIT inputs: 6 mixtures of 3 sources, estimates permuted and noisy."""
    g = torch.Generator().manual_seed(5)
    tgt = torch.randn(6, 3, 3000, generator=g)
    est = tgt[:, [2, 0, 1]] + 0.3 * torch.randn(6, 3, 3000, generator=g)
    return est, tgt, tgt.sum(1, keepdim=True)


def main():
    arrays, meta = {}, {"model_seed": MODEL_SEED, "input_seed": INPUT_SEED, "cases": []}
    for i, (variant, kw, T) in enumerate(CASES):
        cfg = O.Config(variant=variant, **kw)
        sd = O.make_state_dict(cfg, seed=MODEL_SEED)
        m = CLASSES[variant](**kw).eval()
        assert list(m.state_dict().keys()) == list(sd.keys())
        m.load_state_dict(sd)
        x = torch.randn(2, kw.get("in_audio_channels", 1), T, generator=torch.Generator().manual_seed(INPUT_SEED))
        with torch.no_grad():
            arrays[f"c{i}/out"] = m(x).numpy().astype(np.float32)
        meta["cases"].append({"variant": variant, "kw": kw, "T": T})
    meta["reference_refuses"] = []
    for variant, kw, T in REFUSED:
        m = CLASSES[variant](**kw).eval()
        m.load_state_dict(O.make_state_dict(O.Config(variant=variant, **kw), seed=MODEL_SEED))
        try:
            with torch.no_grad():
                m(torch.randn(2, 1, T, generator=torch.Generator().manual_seed(INPUT_SEED)))
        except RuntimeError as e:
            meta["reference_refuses"].append({"variant": variant, "kw": kw, "T": T, "error": str(e).splitlines()[0]})
        else:
            raise AssertionError(f"the reference ran {variant} {kw} at T = {T}")
    est, tgt, mix = pit_inputs()
    fn = ref_sisdr.PermInvariantSISDR(batch_size=6, zero_mean=True, n_sources=3, backward_loss=False,
                                      improvement=True, return_individual_results=True)
    want, perms = fn(est, tgt, initial_mixtures=mix, return_best_permutation=True)
    arrays["pit/best"] = want.numpy()
    arrays["pit/perms"] = np.asarray([list(p) for p in perms], dtype=np.int64)
    arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "reference_live.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
