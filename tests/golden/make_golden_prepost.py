"""Golden fixtures for the steps either side of the forward (SURVEY.md 8f rows 1-2),
generated from the UNMODIFIED reference.  Needs a checkout of the original sudo_rm_rf repository,
named by SUDO_RM_RF_REFERENCE:

    SUDO_RM_RF_REFERENCE=/path/to/sudo_rm_rf python tests/golden/make_golden_prepost.py

* ``prepost_separate_*.npz``: the README inference recipe (README.md:100-114) executed with
  the reference's own modules on raw (un-normalised) mixtures: state_dict, wav, estimates
  without and with the mixture-consistency step.
* ``prepost_sisdr.npz``: ``PermInvariantSISDR`` (dnn/losses/sisdr.py:66-194) outputs for
  2, 3 and 4 sources, with/without zero-mean and improvement.
* ``prepost_degenerate.npz``: the three metrics on degenerate rows (a NaN sample, a constant target under
  zero-mean, a silent target, two identical estimates, a perfect estimate).
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
import sudo_rm_rf.dnn.experiments.utils.mixture_consistency as ref_mc     # noqa: E402
import sudo_rm_rf.dnn.losses.sisdr as ref_sisdr                            # noqa: E402
from oracle import sudormrf_oracle as O                                    # noqa: E402

SEPARATE_CASES = [
    ("improved", "improved",
     dict(out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=3,
          enc_kernel_size=21, enc_num_basis=24, num_sources=2), 3, 517),
    ("groupcomm", "groupcomm",
     dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
          enc_kernel_size=21, enc_num_basis=48, num_sources=2, group_size=4), 2, 1001),
]


def readme_recipe(model, wav, use_mc):
    """README.md:100-114, verbatim order of operations."""
    input_mix_std = wav.std(-1, keepdim=True)
    input_mix_mean = wav.mean(-1, keepdim=True)
    input_mix = (wav - input_mix_mean) / (input_mix_std + 1e-9)
    rec = model(input_mix.unsqueeze(1))
    rec = (rec * input_mix_std.unsqueeze(1)) + input_mix_mean.unsqueeze(1)
    if use_mc:
        rec = ref_mc.apply(rec, input_mix.unsqueeze(1))
    return rec


def make_separate():
    for idx, (name, variant, kw, B, T) in enumerate(SEPARATE_CASES):
        torch.manual_seed(300 + idx)
        cls = ref_improved.SuDORMRF if variant == "improved" else ref_gc.GroupCommSudoRmRf
        model = cls(**kw).eval()
        cfg = O.Config(variant=variant, **kw)
        model.load_state_dict(O.make_state_dict(cfg, seed=31 + idx, perturbed=True))
        g = torch.Generator().manual_seed(3000 + idx)
        scale = torch.tensor([0.05, 1.0, 7.0])[:B].view(B, 1) if B == 3 else torch.tensor([0.3, 4.0]).view(B, 1)
        offset = torch.linspace(-0.5, 0.8, B).view(B, 1)
        wav = torch.randn(B, T, generator=g) * scale + offset          # raw: per-utterance gain and DC offset
        with torch.no_grad():
            plain = readme_recipe(model, wav, False)
            with_mc = readme_recipe(model, wav, True)
        arrays = {"wav": wav.numpy(), "out/plain": plain.numpy(), "out/mc": with_mc.numpy()}
        arrays.update({"sd/" + k: v.detach().numpy() for k, v in model.state_dict().items()})
        meta = dict(name=name, variant=variant, kwargs=kw, B=B, T=T, torch=torch.__version__)
        arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        path = os.path.join(HERE, f"prepost_separate_{name}.npz")
        np.savez_compressed(path, **arrays)
        print(f"separate/{name}: {tuple(plain.shape)} -> {os.path.getsize(path)/1024:.0f} KiB")


def make_sisdr():
    arrays, cases = {}, []
    g = torch.Generator().manual_seed(4242)
    for ci, (S, B, T, zero_mean, improvement) in enumerate([
            (2, 5, 4000, True, True), (2, 3, 1234, False, False), (3, 4, 2000, True, True),
            (4, 3, 1500, True, False), (2, 2, 777, False, True), (1, 2, 500, True, False)]):
        tgt = torch.randn(B, S, T, generator=g) * (0.2 + torch.rand(B, S, 1, generator=g)) + 0.05
        perm = [torch.randperm(S, generator=g) for _ in range(B)]
        est = torch.stack([tgt[b, perm[b]] for b in range(B)])
        est = est * 0.8 + torch.randn(B, S, T, generator=g) * torch.logspace(-2.5, -0.3, B).view(B, 1, 1)
        mix = tgt.sum(1, keepdim=True)
        fn = ref_sisdr.PermInvariantSISDR(batch_size=B, zero_mean=zero_mean, n_sources=S,
                                          backward_loss=False, improvement=improvement,
                                          return_individual_results=True)
        with torch.no_grad():
            best, perms = fn(est, tgt, initial_mixtures=mix, return_best_permutation=True)
        loss = ref_sisdr.PermInvariantSISDR(batch_size=B, zero_mean=zero_mean, n_sources=S,
                                            backward_loss=True, improvement=improvement,
                                            return_individual_results=False)
        with torch.no_grad():
            scalar = loss(est, tgt, initial_mixtures=mix)
        k = f"c{ci}/"
        arrays.update({k + "est": est.numpy(), k + "tgt": tgt.numpy(), k + "mix": mix.numpy(),
                       k + "best": best.numpy(), k + "perms": perms.numpy(),
                       k + "loss": scalar.reshape(1).numpy()})
        cases.append(dict(S=S, B=B, T=T, zero_mean=zero_mean, improvement=improvement))
        print(f"sisdr/c{ci}: S={S} best={best.numpy().round(3)}")
    arrays["meta"] = np.frombuffer(json.dumps(dict(cases=cases, torch=torch.__version__)).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "prepost_sisdr.npz")
    np.savez_compressed(path, **arrays)
    print(f"sisdr -> {os.path.getsize(path)/1024:.0f} KiB")


def make_pairwise():
    """``prepost_pairwise.npz``: ``PairwiseNegSDR`` (dnn/losses/sisdr.py:372-457) for every sdr_type / zero_mean /
    take_log combination and ``PITLossWrapper(..., pit_from='pw_mtx')`` (sisdr.py:197-369) on top of it."""
    arrays = {}
    g = torch.Generator().manual_seed(11)
    ci = 0
    for si, (S, T, B) in enumerate(((2, 4001, 3), (3, 1777, 2), (1, 900, 2), (4, 640, 2))):
        tgt = torch.randn(B, S, T, generator=g) + 0.3
        est = tgt[:, torch.randperm(S, generator=g)] * 0.7 + 0.4 * torch.randn(B, S, T, generator=g) + 0.1
        arrays[f"s{si}/est"] = est.numpy()
        arrays[f"s{si}/tgt"] = tgt.numpy()
        for sdr_type in ("snr", "sisdr", "sdsdr"):
            for zero_mean, take_log in ((True, True), (False, True), (True, False)):
                fn = ref_sisdr.PairwiseNegSDR(sdr_type, zero_mean=zero_mean, take_log=take_log)
                pw = fn(est, tgt)
                loss = ref_sisdr.PITLossWrapper(fn, pit_from="pw_mtx")(est, tgt)
                key = f"c{ci}"
                arrays[key + "/meta"] = np.frombuffer(json.dumps(dict(S=S, T=T, B=B, signals=si, sdr_type=sdr_type,
                                                                       zero_mean=zero_mean, take_log=take_log)).encode(),
                                                      dtype=np.uint8)
                arrays[key + "/pw"] = pw.numpy()
                arrays[key + "/pit_loss"] = loss.numpy()
                ci += 1
    path = os.path.join(HERE, "prepost_pairwise.npz")
    np.savez_compressed(path, **arrays)
    print(f"pairwise: {ci} cases -> {os.path.getsize(path)/1024:.0f} KiB")


def make_stabilized():
    """``prepost_stabilized.npz``: ``StabilizedPermInvSISDRMetric`` (dnn/losses/sisdr.py:460-591), the validation
    metric of run_fuss_separation.py:111-131: more estimated than actual sources, one source, single_source (the
    estimates are summed first), with / without zero-mean and improvement, and the script's one-source set: a metric
    constructed for one estimated source and handed all four output rows, of which it scores the first."""
    arrays, cases = {}, []
    g = torch.Generator().manual_seed(777)
    for ci, (n_est, n_act, B, T, zero_mean, improvement, single, ctor_est) in enumerate([
            (4, 2, 4, 3000, True, True, False, 4), (4, 3, 3, 2000, True, True, False, 4),
            (4, 4, 2, 1500, True, True, False, 4), (3, 1, 3, 1234, False, False, False, 3),
            (2, 2, 3, 800, False, True, False, 2), (1, 1, 2, 600, True, False, False, 1),
            # single_source sums the estimates first (sisdr.py:576-577), so the constructor is given ONE estimated
            # source (its permutation table indexes the summed tensor, :490-492,527); the model still returned n_est
            (3, 1, 2, 900, True, False, True, 1), (4, 1, 2, 500, False, False, False, 4),
            # run_fuss_separation.py:111-116,296-307: n_estimated_sources=1 without single_source on four rows
            (4, 1, 3, 700, True, False, False, 1)]):
        tgt = torch.randn(B, n_act, T, generator=g) * (0.2 + torch.rand(B, n_act, 1, generator=g)) + 0.05
        est = torch.randn(B, n_est, T, generator=g) * 0.05                       # inactive outputs: low-level noise
        for b in range(B):
            slots = torch.randperm(n_est, generator=g)[:n_act]
            for j in range(n_act):
                est[b, slots[j]] += 0.8 * tgt[b, j] + torch.randn(T, generator=g) * float(10 ** (-2.0 + 1.5 * b / max(1, B - 1)))
        fn = ref_sisdr.StabilizedPermInvSISDRMetric(zero_mean=zero_mean, single_source=single, n_estimated_sources=ctor_est,
                                                    n_actual_sources=n_act, backward_loss=False, improvement=improvement,
                                                    return_individual_results=True)
        with torch.no_grad():
            best, perms = fn(est, tgt, return_best_permutation=True)
        loss = ref_sisdr.StabilizedPermInvSISDRMetric(zero_mean=zero_mean, single_source=single,
                                                      n_estimated_sources=ctor_est, n_actual_sources=n_act, backward_loss=True,
                                                      improvement=improvement, return_individual_results=False)
        with torch.no_grad():
            scalar = loss(est, tgt)
        k = f"c{ci}/"
        arrays.update({k + "est": est.numpy(), k + "tgt": tgt.numpy(), k + "best": best.numpy(),
                       k + "perms": perms.numpy(), k + "loss": scalar.reshape(1).numpy()})
        cases.append(dict(n_est=n_est, n_act=n_act, B=B, T=T, zero_mean=zero_mean, improvement=improvement,
                          single_source=single, ctor_est=ctor_est))
        print(f"stabilized/c{ci}: {n_est}->{n_act} best={best.numpy().round(3)} perms={perms.numpy().tolist()}")
    arrays["meta"] = np.frombuffer(json.dumps(dict(cases=cases, torch=torch.__version__)).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "prepost_stabilized.npz")
    np.savez_compressed(path, **arrays)
    print(f"stabilized -> {os.path.getsize(path)/1024:.0f} KiB")


DEGENERATE_CASES = ["nan_row", "constant_target", "silent_target", "tie", "perfect"]


def degenerate_signals(case, n_est, n_act, B, T, g):
    """Item 0 of the batch carries the case; the other items are ordinary."""
    tgt = torch.randn(B, n_act, T, generator=g) * (0.2 + torch.rand(B, n_act, 1, generator=g)) + 0.05
    est = torch.randn(B, n_est, T, generator=g) * 0.05
    est[:, :n_act] += 0.8 * tgt.flip(1) + 0.1 * torch.randn(B, n_act, T, generator=g)
    if case == "nan_row":
        est[0, n_est - 1, T // 3] = float("nan")
    elif case == "constant_target":
        tgt[0] = torch.tensor([0.37, -1.7, 3.3, 1000.0][:n_act]).view(n_act, 1).expand(n_act, T)
    elif case == "silent_target":
        tgt[0, 0] = 0.0
    elif case == "tie":
        est[0, 1] = est[0, 0]
    elif case == "perfect":
        est[0, :n_act] = tgt[0]
    return est, tgt


def make_degenerate():
    """``prepost_degenerate.npz``: ``PermInvariantSISDR`` (2 sources, SI-SDRi), ``StabilizedPermInvSISDRMetric``
    (4 estimated, 1 actual source for the NaN row as FUSS scores it, else 2) and ``PairwiseNegSDR`` (sisdr, 3 sources)
    on each degenerate case, zero-mean on (which the constant target needs)."""
    arrays, cases = {}, []
    g = torch.Generator().manual_seed(2024)
    B, T = 3, 500
    ci = 0
    for case in DEGENERATE_CASES:
        for metric in ("pit", "stabilized", "pairwise"):
            k = f"c{ci}/"
            meta = dict(name=f"{metric}/{case}", case=case, metric=metric, zero_mean=True, B=B, T=T)
            if metric == "pit":
                est, tgt = degenerate_signals(case, 2, 2, B, T, g)
                mix = tgt.sum(1, keepdim=True)
                improvement = case != "constant_target"      # SI-SDRi against a constant target is -inf - (-inf)
                fn = ref_sisdr.PermInvariantSISDR(batch_size=B, zero_mean=True, n_sources=2, backward_loss=False,
                                                  improvement=improvement, return_individual_results=True)
                with torch.no_grad():
                    best, perms = fn(est, tgt, initial_mixtures=mix, return_best_permutation=True)
                allp = fn.permutations_tensor.tolist()
                arrays[k + "mix"] = mix.numpy()
                meta["improvement"] = improvement
            elif metric == "stabilized":
                n_act = 1 if case == "nan_row" else 2
                est, tgt = degenerate_signals(case, 4, n_act, B, T, g)
                fn = ref_sisdr.StabilizedPermInvSISDRMetric(zero_mean=True, n_estimated_sources=4,
                                                            n_actual_sources=n_act, backward_loss=False,
                                                            improvement=False, return_individual_results=True)
                with torch.no_grad():
                    best, perms = fn(est, tgt, return_best_permutation=True)
                allp = fn.permutations_tensor.tolist()
                meta["improvement"] = False
            else:
                est, tgt = degenerate_signals(case, 3, 3, B, T, g)
                with torch.no_grad():
                    best = -ref_sisdr.PairwiseNegSDR("sisdr", zero_mean=True, take_log=True)(est, tgt)   # SDR in dB
                meta["sdr_type"] = "sisdr"
            if metric != "pairwise":
                idx = torch.tensor([allp.index(r) for r in perms.tolist()], dtype=torch.int64)
                arrays[k + "idx"] = idx.numpy()
            arrays.update({k + "est": est.numpy(), k + "tgt": tgt.numpy(), k + "score": best.numpy()})
            cases.append(meta)
            print(f"degenerate/c{ci} {meta['name']}: {best.flatten()[:6].numpy()}")
            ci += 1
    arrays["meta"] = np.frombuffer(json.dumps(dict(cases=cases, torch=torch.__version__)).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "prepost_degenerate.npz")
    np.savez_compressed(path, **arrays)
    print(f"degenerate: {ci} cases -> {os.path.getsize(path)/1024:.0f} KiB")


if __name__ == "__main__":
    todo = sys.argv[1:] or ["separate", "sisdr", "pairwise", "stabilized", "degenerate"]   # name a subset to leave the other fixtures alone
    for name in todo:
        {"separate": make_separate, "sisdr": make_sisdr, "pairwise": make_pairwise, "stabilized": make_stabilized,
         "degenerate": make_degenerate}[name]()
