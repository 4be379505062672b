"""Generate the golden fixtures in this directory from the UNMODIFIED reference.

Needs a checkout of the original sudo_rm_rf repository, named by SUDO_RM_RF_REFERENCE:

    SUDO_RM_RF_REFERENCE=/path/to/sudo_rm_rf python tests/golden/make_golden.py

The reference (etzinis/sudo_rm_rf) ships no golden vectors for its forward path
(SURVEY.md §4), so these fixtures are outputs of the reference's own
``nn.Module``s (CPU, fp32) on seeded inputs and seeded, non-trivial weights.
Each ``case_*.npz`` holds: the ctor kwargs (json), the full ``state_dict``,
the input mixture, the model output, the mixture-consistency output and a few
intermediate activations captured with forward hooks on the reference's leaf
modules (SURVEY §8c) so single stages can be checked too.
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

import sudo_rm_rf.dnn.models.improved_sudormrf as ref_improved            # noqa: E402
import sudo_rm_rf.dnn.models.groupcomm_sudormrf_v2 as ref_gc              # noqa: E402
import sudo_rm_rf.dnn.models.causal_improved_sudormrf_v3 as ref_causal    # noqa: E402
import sudo_rm_rf.dnn.models.sudormrf as ref_original                      # noqa: E402
import sudo_rm_rf.dnn.experiments.utils.mixture_consistency as ref_mc     # noqa: E402
from oracle import sudormrf_oracle as O                                    # noqa: E402

CASES = [
    # name, variant, ctor kwargs, batch, T, input kind
    ("improved_small_odd", "improved",
     dict(out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=3,
          enc_kernel_size=21, enc_num_basis=24, num_sources=2), 2, 517, "randn"),
    ("improved_short", "improved",           # T < hop * 2^D  (improved_sudormrf.py:305-306)
     dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=5,
          enc_kernel_size=21, enc_num_basis=32, num_sources=2), 3, 100, "rand"),
    ("improved_exact_multiple", "improved",  # T already a multiple of hop * 2^D
     dict(out_channels=32, in_channels=64, num_blocks=3, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=40, num_sources=3), 1, 640, "randn"),
    ("improved_default_init", "improved",    # the reference ctor's own init
     dict(out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=32, num_sources=2), 2, 801, "randn"),
    ("groupcomm_small", "groupcomm",
     dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=48, num_sources=2, group_size=4),
     2, 1001, "randn"),
    ("groupcomm_g16", "groupcomm",           # production group geometry 16 x (16 -> 32)
     dict(out_channels=256, in_channels=512, num_blocks=1, upsampling_depth=3,
          enc_kernel_size=21, enc_num_basis=32, num_sources=2, group_size=16),
     1, 333, "rand"),
    ("groupcomm_stereo", "groupcomm",        # in_audio_channels=2, other kernel size
     dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3,
          enc_kernel_size=11, enc_num_basis=16, num_sources=2, group_size=8,
          in_audio_channels=2), 2, 333, "randn"),
    ("causal_small_odd", "causal",           # causal_improved_sudormrf_v3.py: masked 21-tap depthwise, no norms
     dict(in_audio_channels=1, out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=48, num_sources=2), 2, 1003, "randn"),
    ("causal_stereo", "causal",              # in_audio_channels=2, other kernel size, depth 5, short input (T < hop*2^D)
     dict(in_audio_channels=2, out_channels=16, in_channels=32, num_blocks=3, upsampling_depth=5,
          enc_kernel_size=11, enc_num_basis=24, num_sources=3), 2, 131, "rand"),
    ("causal_default_init", "causal",        # the reference ctor's own init (skipinit_gain = 0: every block the identity)
     dict(in_audio_channels=1, out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=3,
          enc_kernel_size=21, enc_num_basis=32, num_sources=2), 2, 801, "randn"),
    # the original SuDoRM-RF (sudormrf.py): GroupNorm, per-channel PReLU, Conv2d + softmax masks, grouped decoder
    ("original_small_odd", "original",       # out_channels != enc_num_basis: reshape_before_masks exists
     dict(out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=3,
          enc_kernel_size=21, enc_num_basis=24, num_sources=2), 2, 517, "randn"),
    ("original_three_src", "original",       # out_channels == enc_num_basis (no reshape layer), T a multiple of the lcm
     dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=32, num_sources=3), 2, 800, "rand"),
    ("original_sigmoid", "original",         # one source: sigmoid instead of softmax (:285-286); other kernel size
     dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=4,
          enc_kernel_size=11, enc_num_basis=16, num_sources=1), 1, 333, "randn"),
    ("original_default_init", "original",    # the reference ctor's own init
     dict(out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=32, num_sources=2), 2, 801, "randn"),
]

HOOKS = ["encoder", "bottleneck", "sm.0.proj_1x1.conv", "sm.0.spp_dw.0.conv",
         "sm.0.spp_dw.1.conv", "sm.0.final_norm.norm", "sm.0", "sm.1",
         "sm.0.UBlock.proj_1x1.conv", "sm.0.UBlock.spp_dw.1.conv", "sm.0.TAC",
         "mask_net.1", "decoder", "l1", "sm.0.conv_1x1_exp.conv", "m"]


def main():
    only = sys.argv[1:]                      # optional name prefixes: regenerate a subset, leave the other fixtures alone
    for idx, (name, variant, kw, B, T, kind) in enumerate(CASES):
        if only and not any(name.startswith(o) for o in only):
            continue
        torch.manual_seed(100 + idx)
        cls = {"improved": ref_improved.SuDORMRF, "groupcomm": ref_gc.GroupCommSudoRmRf,
               "causal": ref_causal.CausalSuDORMRF, "original": ref_original.SuDORMRF}[variant]
        model = cls(**kw).eval()
        cfg = O.Config(variant=variant, **kw)
        if not name.endswith("default_init"):
            model.load_state_dict(O.make_state_dict(cfg, seed=7 + idx, perturbed=True))
        sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
        A = kw.get("in_audio_channels", 1)
        g = torch.Generator().manual_seed(1000 + idx)
        x = torch.randn(B, A, T, generator=g) if kind == "randn" \
            else torch.rand(B, A, T, generator=g)
        if kind == "randn":      # README.md:101-103 per-utterance normalisation
            x = (x - x.mean(-1, keepdim=True)) / (x.std(-1, keepdim=True) + 1e-9)
        taps = {}
        handles = []
        mods = dict(model.named_modules())
        for h in HOOKS:
            if h in mods:
                handles.append(mods[h].register_forward_hook(
                    lambda m, i, o, h=h: taps.__setitem__(h, o.detach().clone())))
        with torch.no_grad():
            y = model(x)
            out = {"output": y}
            if A == 1:
                out["mc_uniform"] = ref_mc.apply(y, x)
                out["mc_magsq"] = ref_mc.apply(y, x, "magsq")
        for h in handles:
            h.remove()
        arrays = {"input": x.numpy()}
        arrays.update({"out/" + k: v.numpy() for k, v in out.items()})
        arrays.update({"sd/" + k: v.numpy() for k, v in sd.items()})
        arrays.update({"tap/" + k: v.numpy() for k, v in taps.items()})
        meta = dict(name=name, variant=variant, kwargs=kw, B=B, T=T,
                    torch=torch.__version__)
        arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        path = os.path.join(HERE, f"case_{name}.npz")
        np.savez_compressed(path, **arrays)
        print(f"{name}: out {tuple(y.shape)} |y|max={float(y.abs().max()):.4f} "
              f"-> {os.path.getsize(path)/1024:.0f} KiB")


if __name__ == "__main__":
    main()
