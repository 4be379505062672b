"""GPU parity of the steps either side of the forward (SURVEY 8f rows 1-2), through the public
API (which calls the C-ABI): per-utterance statistics, `separate(..., normalize=True)` = the README
recipe, and the PIT SI-SDR metric.  Checked against the reference's golden vectors, the CPU oracle,
and size-independent properties at the benchmark shape."""
import ctypes as C
import itertools

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import sisdr as S
from oracle import sudormrf_oracle as O
from test_prepost_oracle import GOLDEN_DIR, SEPARATE, load_separate, load_sisdr

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-3


def build(variant, kw, sd):
    cls = {"improved": P.SuDORMRF, "groupcomm": P.GroupCommSudoRmRf, "causal": P.CausalSuDORMRF,
           "original": P.OriginalSuDORMRF}[variant]
    m = cls(**kw)
    m.load_state_dict(sd)
    return m.to(DEV).eval()


@pytest.mark.parametrize("rows,T,r", [pytest.param(rows, T, None, id=f"{rows}-{T}")
                                      for rows, T in [(1, 1000), (5, 517), (32, 32000), (3, 7), (2, 100003)]]
                         # 8192-sample chunks, 64 at most per row; r = |mean| / std up to 1e4
                         + [(3, 8191, 1e4), (3, 8192, 10.0), (3, 8193, 1e3), (2, 524288, 1e4), (2, 524289, 1e4)])
def test_utterance_stats(rows, T, r):
    g = torch.Generator().manual_seed(rows * 1000 + T)
    if r is None:
        wav = (torch.randn(rows, T, generator=g) * torch.logspace(-2, 1, rows).view(rows, 1)
               + torch.linspace(-3, 50, rows).view(rows, 1)).to(DEV)      # DC up to 50x the AC level
    else:
        ac = torch.logspace(-2, 1, rows).view(rows, 1)
        wav = ((torch.randn(rows, T, generator=g) + r * torch.linspace(-1, 1, rows).view(rows, 1)) * ac).to(DEV)
    ms = torch.full((rows, 2), float("nan"), device=DEV)
    scratch = torch.empty(rows * 2, dtype=torch.float64, device=DEV)
    N.check(N.lib().sdr_utterance_stats(C.c_void_p(wav.data_ptr()), C.c_void_p(ms.data_ptr()), rows, T,
                                        C.c_void_p(scratch.data_ptr()),
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    want_mean = wav.double().mean(-1)
    want_std = wav.double().std(-1)
    assert torch.allclose(ms[:, 0].double(), want_mean, rtol=2e-7, atol=0)
    assert torch.allclose(ms[:, 1].double(), want_std, rtol=2e-6, atol=0)


@pytest.mark.parametrize("path", SEPARATE, ids=lambda p: p.split("prepost_separate_")[1][:-4])
def test_separate_golden(path):
    """README.md:100-114 end to end against the reference's own outputs."""
    meta, sd, wav, plain, with_mc = load_separate(path)
    m = build(meta["variant"], meta["kwargs"], sd)
    with torch.no_grad():
        got = m.separate(wav.to(DEV), mixture_consistency=False, normalize=True)
        assert got.shape == plain.shape and got.dtype == torch.float32 and got.is_cuda
        e = O.parity_errors(got, plain)
        print("separate golden", meta["name"], "rel_max %.2e rel_l2 %.2e" % e)
        assert max(e) < TOL, e
        got = m.separate(wav.to(DEV).unsqueeze(1), mixture_consistency=True, normalize=True)   # [B,1,T] also accepted
        e = O.parity_errors(got, with_mc)
        assert max(e) < TOL, e
        # and it really is the composition of the public pieces
        x = wav.to(DEV)
        xn = (x - x.mean(-1, keepdim=True)) / (x.std(-1, keepdim=True) + 1e-9)
        ref = m(xn.unsqueeze(1)) * x.std(-1, keepdim=True).unsqueeze(1) + x.mean(-1, keepdim=True).unsqueeze(1)
        assert max(O.parity_errors(m.separate(x, normalize=True, mixture_consistency=False), ref)) < TOL


def test_separate_vs_oracle_mid_size():
    kw = dict(out_channels=128, in_channels=256, num_blocks=2, upsampling_depth=4,
              enc_kernel_size=21, enc_num_basis=256, num_sources=2)
    cfg = O.Config(variant="improved", **kw)
    sd = O.make_state_dict(cfg, seed=3, perturbed=True)
    g = torch.Generator().manual_seed(9)
    scale = torch.tensor([0.01, 1.0, 30.0]).view(3, 1)
    wav = torch.randn(3, 8013, generator=g) * scale + 0.2 * scale
    want = O.separate(cfg, sd, wav, apply_mixture_consistency=True)
    m = build("improved", kw, sd)
    with torch.no_grad():
        got = m.separate(wav.to(DEV), mixture_consistency=True, normalize=True)
    e = O.parity_errors(got, want)
    assert max(e) < TOL, e


def test_separate_gain_and_offset_equivariance_full_size():
    """separate(a * wav + c) == a * separate(wav) + c for a > 0 (benchmark shape: 32 x 4 s)."""
    kw = dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5,
              enc_kernel_size=21, enc_num_basis=512, num_sources=2)
    cfg = O.Config(variant="improved", **kw)
    m = build("improved", kw, O.make_state_dict(cfg, seed=1, perturbed=True))
    g = torch.Generator().manual_seed(2)
    wav = torch.randn(32, 32000, generator=g).to(DEV)
    a = torch.logspace(-1, 1, 32, device=DEV).view(32, 1)
    c = torch.linspace(-0.2, 0.2, 32, device=DEV).view(32, 1)
    with torch.no_grad():
        y0 = m.separate(wav, normalize=True)
        y1 = m.separate(a * wav + c, normalize=True)
    want = a.unsqueeze(1) * y0 + c.unsqueeze(1)
    e = O.parity_errors(y1, want)
    print("separate equivariance rel_max %.2e rel_l2 %.2e" % e)
    assert max(e) < TOL, e
    assert torch.isfinite(y1).all()


def test_separate_refuses_multichannel():
    kw = dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3, enc_kernel_size=11,
              enc_num_basis=16, num_sources=2, group_size=8, in_audio_channels=2)
    m = P.GroupCommSudoRmRf(**kw).to(DEV).eval()
    with torch.no_grad(), pytest.raises(RuntimeError):
        m.separate(torch.randn(2, 2, 333, device=DEV), normalize=True)


@pytest.mark.parametrize("ci", range(6))
def test_pit_sisdr_golden(ci):
    c, t = load_sisdr()[ci]
    fn = S.PermInvariantSISDR(batch_size=c["B"], zero_mean=c["zero_mean"], n_sources=c["S"],
                              backward_loss=False, improvement=c["improvement"],
                              return_individual_results=True)
    with torch.no_grad():
        best, perms = fn(t["est"].to(DEV), t["tgt"].to(DEV), initial_mixtures=t["mix"].to(DEV),
                         return_best_permutation=True)
    assert best.shape == t["best"].shape and best.is_cuda
    assert torch.allclose(best.cpu(), t["best"], atol=1e-3, rtol=0), (best.cpu() - t["best"]).abs().max()
    assert torch.equal(perms.cpu(), t["perms"])
    loss = S.PermInvariantSISDR(batch_size=c["B"], zero_mean=c["zero_mean"], n_sources=c["S"],
                                backward_loss=True, improvement=c["improvement"],
                                return_individual_results=False)
    with torch.no_grad():
        scalar = loss(t["est"].to(DEV), t["tgt"].to(DEV), initial_mixtures=t["mix"].to(DEV))
    assert abs(float(scalar) - float(t["loss"][0])) < 1e-3


def _stabilized_cases():
    import json
    import os
    import numpy as np
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prepost_stabilized.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    return [(c, {n: torch.from_numpy(z[f"c{ci}/" + n]) for n in ("est", "tgt", "best", "perms", "loss")})
            for ci, c in enumerate(meta["cases"])]


@pytest.mark.parametrize("ci", range(9))
def test_stabilized_sisdr_golden(ci):
    """sisdr.StabilizedPermInvSISDRMetric (same constructor / forward as dnn/losses/sisdr.py:460-591) against outputs of
    the reference class: 4 -> 2 / 3 / 4 and 3 / 4 -> 1 sources, single_source, zero-mean and improvement on and off,
    and a metric constructed for one estimated source given four rows (it scores the first)."""
    c, t = _stabilized_cases()[ci]
    n_est = c["ctor_est"]
    fn = S.StabilizedPermInvSISDRMetric(zero_mean=c["zero_mean"], single_source=c["single_source"],
                                        n_estimated_sources=n_est, n_actual_sources=c["n_act"], backward_loss=False,
                                        improvement=c["improvement"], return_individual_results=True)
    with torch.no_grad():
        best, perms = fn(t["est"].to(DEV), t["tgt"].to(DEV), return_best_permutation=True)
    assert best.shape == t["best"].shape and best.is_cuda
    assert torch.allclose(best.cpu(), t["best"], atol=2e-3, rtol=0), (best.cpu() - t["best"]).abs().max()
    assert torch.equal(perms.cpu(), t["perms"])
    loss = S.StabilizedPermInvSISDRMetric(zero_mean=c["zero_mean"], single_source=c["single_source"],
                                          n_estimated_sources=n_est, n_actual_sources=c["n_act"], backward_loss=True,
                                          improvement=c["improvement"], return_individual_results=False)
    with torch.no_grad():
        scalar = loss(t["est"].to(DEV), t["tgt"].to(DEV))
    assert abs(float(scalar) - float(t["loss"][0])) < 2e-3


def test_stabilized_sisdr_fuss_validation_shape_vs_oracle():
    """run_fuss_separation.py:111-131,280-310: 4 estimated sources against 1..4 actual ones, 10 s @ 16 kHz, zero-mean,
    SI-SDRi for more than one actual source; against the CPU oracle, plus argument errors."""
    g = torch.Generator().manual_seed(5)
    B, T = 6, 160000
    for n_act in (1, 2, 3, 4):
        tgt = torch.randn(B, n_act, T, generator=g) * (0.3 + torch.rand(B, n_act, 1, generator=g))
        est = 0.03 * torch.randn(B, 4, T, generator=g)
        for b in range(B):
            slots = torch.randperm(4, generator=g)[:n_act]
            for j in range(n_act):
                est[b, slots[j]] += tgt[b, j] + torch.randn(T, generator=g) * float(10 ** (-1.5 + 0.3 * b))
        fn = S.StabilizedPermInvSISDRMetric(zero_mean=True, single_source=False, n_estimated_sources=4,
                                            n_actual_sources=n_act, backward_loss=False, improvement=n_act > 1,
                                            return_individual_results=True)
        with torch.no_grad():
            best, perms = fn(est.to(DEV), tgt.to(DEV), return_best_permutation=True)
        want, idx = O.stabilized_pit_sisdr(est.double(), tgt.double(), zero_mean=True, improvement=n_act > 1)
        assert torch.allclose(best.cpu().double(), want, atol=2e-3, rtol=0), (n_act, best.cpu(), want)
        assert torch.equal(perms.cpu(), fn.permutations_tensor[idx])
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(est, tgt)
    with pytest.raises(RuntimeError, match="actual"):
        fn(est.to(DEV), tgt[:, :2].to(DEV))
    with pytest.raises(AssertionError):
        S.StabilizedPermInvSISDRMetric(n_estimated_sources=2, n_actual_sources=3)
    five = S.StabilizedPermInvSISDRMetric(n_estimated_sources=5, n_actual_sources=2)
    with torch.no_grad(), pytest.raises(N.NativeError):
        five(torch.zeros(1, 5, 50, device=DEV), torch.zeros(1, 2, 50, device=DEV))


def test_pit_sisdr_full_size_vs_oracle_and_permutation_property():
    """Validation-loop shape (32 x 2 x 4 s): against the CPU oracle, and permuting the estimates'
    source order must permute the reported assignment and leave the score unchanged."""
    g = torch.Generator().manual_seed(11)
    B, Sn, T = 32, 2, 32000
    tgt = torch.randn(B, Sn, T, generator=g)
    est = tgt + torch.randn(B, Sn, T, generator=g) * torch.logspace(-2, 0.5, B).view(B, 1, 1)
    swap = torch.rand(B, generator=g) < 0.5
    est[swap] = est[swap][:, [1, 0]]
    mix = tgt.sum(1, keepdim=True)
    want, widx = O.pit_sisdr(est, tgt, mix, zero_mean=True, improvement=True)
    fn = S.PermInvariantSISDR(batch_size=B, zero_mean=True, n_sources=Sn, backward_loss=False,
                              improvement=True, return_individual_results=True)
    with torch.no_grad():
        best, perms = fn(est.to(DEV), tgt.to(DEV), initial_mixtures=mix.to(DEV), return_best_permutation=True)
        best2, perms2 = fn(est[:, [1, 0]].to(DEV), tgt.to(DEV), initial_mixtures=mix.to(DEV),
                           return_best_permutation=True)
    assert torch.allclose(best.cpu(), want, atol=1e-3, rtol=0), (best.cpu() - want).abs().max()
    allp = list(itertools.permutations(range(Sn)))
    assert [tuple(int(v) for v in r) for r in perms.cpu()] == [allp[int(i)] for i in widx]
    assert torch.allclose(best, best2, atol=1e-5, rtol=0)
    assert torch.equal(perms2.cpu(), 1 - perms.cpu())
    assert torch.equal(perms.cpu()[:, 0] == 1, swap)


def test_pit_sisdr_argument_errors():
    fn = S.PermInvariantSISDR(n_sources=2, improvement=True)
    with pytest.raises(RuntimeError):
        fn(torch.zeros(2, 2, 100), torch.zeros(2, 2, 100))                       # CPU tensors: no CPU path
    with torch.no_grad(), pytest.raises(RuntimeError):
        fn(torch.zeros(2, 2, 100, device=DEV), torch.zeros(2, 2, 100, device=DEV))   # SI-SDRi without the mixture
    with pytest.raises(RuntimeError):
        fn(torch.zeros(2, 2, 100, device=DEV, requires_grad=True), torch.zeros(2, 2, 100, device=DEV),
           initial_mixtures=torch.zeros(2, 1, 100, device=DEV))                  # metric only: no autograd
    five = S.PermInvariantSISDR(n_sources=5)
    with torch.no_grad(), pytest.raises(N.NativeError):
        five(torch.zeros(1, 5, 50, device=DEV), torch.zeros(1, 5, 50, device=DEV))


CORPUS_MODELS = [
    ("improved", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=3,
                      enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    ("groupcomm", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
                       enc_kernel_size=21, enc_num_basis=48, num_sources=3, group_size=4)),
    ("causal", dict(in_audio_channels=1, out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
                    enc_kernel_size=21, enc_num_basis=48, num_sources=2)),
    ("original", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,      # buckets by ITS padding rule:
                      enc_kernel_size=21, enc_num_basis=48, num_sources=2)),                   # multiples of lcm(10, 16) = 80
]


@pytest.mark.parametrize("variant,kw", CORPUS_MODELS, ids=[c[0] for c in CORPUS_MODELS])
@pytest.mark.parametrize("mc", [False, True])
def test_separate_corpus_equals_one_at_a_time(variant, kw, mc):
    """Bucketed ragged batches reproduce the reference's one-utterance-at-a-time loop
    (simple_whamr_evaluation.py:138-148 / README.md:100-114)."""
    from sudo_rm_rf_b200.corpus import separate_corpus
    cfg = O.Config(variant=variant, **kw)
    sd = O.make_state_dict(cfg, seed=5, perturbed=True)
    m = build(variant, kw, sd)
    q = O.padded_length(cfg, 1)                # the model's padding quantum (hop * 2^D; lcm(hop, 2^D) for the original model)
    g = torch.Generator().manual_seed(17)
    lengths = [q, q - 1, 1500, 1501, 1502, 37, 2 * q, 2 * q + 1, 5000, 4999, 1499, q + 3, 4990]
    wavs = [torch.randn(T, generator=g) * (0.1 + 3 * torch.rand(1, generator=g)) + 0.1 * torch.randn(1, generator=g)
            for T in lengths]
    with torch.no_grad():
        got = separate_corpus(m, wavs, max_batch=3, mixture_consistency=mc)
        assert len(got) == len(wavs)
        for w, y in zip(wavs, got):
            assert y.shape == (cfg.num_sources, w.shape[0]) and y.is_cuda
            alone = m.separate(w.to(DEV)[None], mixture_consistency=mc, normalize=True)[0]
            e = O.parity_errors(y[None], alone[None])
            assert max(e) < 1e-5, (w.shape[0], e)
        # against the CPU oracle for a few of them
        for i in (0, 3, 5, 8):
            want = O.separate(cfg, sd, wavs[i][None], apply_mixture_consistency=mc)[0]
            assert max(O.parity_errors(got[i][None], want[None])) < TOL
        # rescale=False: estimates of the normalised mixture (what the evaluation script scores)
        raw = separate_corpus(m, wavs[:5], max_batch=4, mixture_consistency=mc, rescale=False)
        for w, y in zip(wavs[:5], raw):
            x = w.to(DEV)
            xn = ((x - x.mean()) / (x.std() + 1e-9))[None, None]
            want = m.separate(xn, mixture_consistency=mc)[0]
            assert max(O.parity_errors(y[None], want[None])) < 1e-4


def _pairwise_cases():
    import json
    import os
    import numpy as np
    z = np.load(os.path.join(GOLDEN_DIR, "prepost_pairwise.npz"))
    out, ci = [], 0
    while f"c{ci}/meta" in z.files:
        meta = json.loads(bytes(z[f"c{ci}/meta"]).decode())
        si = meta["signals"]
        out.append((meta, torch.from_numpy(z[f"s{si}/est"]), torch.from_numpy(z[f"s{si}/tgt"]),
                    torch.from_numpy(z[f"c{ci}/pw"]), torch.from_numpy(z[f"c{ci}/pit_loss"])))
        ci += 1
    return out


def test_pairwise_neg_sdr_and_pit_wrapper_golden():
    """`sisdr.PairwiseNegSDR` / `PITLossWrapper` (same constructors as dnn/losses/sisdr.py:197-457) against the
    reference's own outputs: 36 cases (snr / sisdr / sdsdr x zero_mean x take_log, 1-4 sources)."""
    from sudo_rm_rf_b200 import sisdr as S
    for meta, est, tgt, pw, loss in _pairwise_cases():
        fn = S.PairwiseNegSDR(meta["sdr_type"], zero_mean=meta["zero_mean"], take_log=meta["take_log"])
        with torch.no_grad():
            got = fn(est.to(DEV), tgt.to(DEV))
            got_loss = S.PITLossWrapper(fn, pit_from="pw_mtx")(est.to(DEV), tgt.to(DEV))
        assert got.shape == pw.shape
        if meta["take_log"]:
            assert torch.allclose(got.cpu(), pw, atol=2e-3, rtol=0), (meta, (got.cpu() - pw).abs().max())     # dB
        else:
            assert torch.allclose(got.cpu(), pw, rtol=2e-4, atol=1e-6), meta
        assert torch.allclose(got_loss.cpu(), loss, atol=2e-3, rtol=2e-4), meta


def test_pit_wrapper_modes_and_reordering():
    """pw_pt / perm_avg modes and return_est follow the asteroid semantics the reference file was copied from."""
    from sudo_rm_rf_b200 import sisdr as S
    g = torch.Generator().manual_seed(3)
    tgt = torch.randn(5, 3, 2000, generator=g)
    perm = [2, 0, 1]
    est = (tgt[:, perm] + 0.05 * torch.randn(5, 3, 2000, generator=g)).to(DEV)
    tgt = tgt.to(DEV)
    pw = S.PairwiseNegSDR("sisdr")
    with torch.no_grad():
        loss, reordered = S.PITLossWrapper(pw, pit_from="pw_mtx")(est, tgt, return_est=True)
        want = O.pairwise_neg_sdr(est.cpu(), tgt.cpu(), "sisdr")
        assert torch.allclose(loss.cpu(), O.pit_from_pairwise(want)[0].mean(), atol=2e-3)
        # the reordered estimates line up with the targets again
        assert float((reordered - tgt).abs().mean()) < 0.1
        single = lambda e, t: pw(e.unsqueeze(1), t.unsqueeze(1))[:, 0, 0]
        loss_pt = S.PITLossWrapper(single, pit_from="pw_pt")(est, tgt)
        assert torch.allclose(loss_pt, loss, atol=1e-3)
        avg = lambda e, t: torch.stack([single(e[:, i], t[:, i]) for i in range(3)], 1).mean(1)
        loss_avg = S.PITLossWrapper(avg, pit_from="perm_avg")(est, tgt)
        assert torch.allclose(loss_avg, loss, atol=1e-3)
    with pytest.raises(RuntimeError):
        pw(est.cpu(), tgt.cpu())
    with pytest.raises(ValueError):
        S.PITLossWrapper(pw, pit_from="nope")


def test_corpus_separator_pipeline_equals_bucketed_loop(tmp_path):
    """CorpusSeparator (pinned staging, copy streams, CUDA graph per bucket) == separate_corpus, bit for bit, on a second
    and third pass too (graph capture, then replay); wav files in, wav files out (simple_whamr_evaluation.py:138-148)."""
    from sudo_rm_rf_b200 import corpus as Cp
    kw = dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4,
              enc_kernel_size=21, enc_num_basis=48, num_sources=2)
    cfg = O.Config(variant="improved", **kw)
    m = build("improved", kw, O.make_state_dict(cfg, seed=3))
    g = torch.Generator().manual_seed(8)
    lengths = [4000, 3999, 3850, 4160, 4001, 2000, 2100, 4000, 3900, 160, 90, 4100, 3841]
    wavs = [torch.randn(n, generator=g) * (0.2 + 0.1 * i) + 0.05 * i for i, n in enumerate(lengths)]
    want = Cp.separate_corpus(m, wavs, max_batch=4)
    sep = Cp.CorpusSeparator(m, max_batch=4)
    for _ in range(3):
        got = sep.run(wavs)
        assert len(got) == len(want)
        for a, b in zip(got, want):
            assert not a.is_cuda and torch.equal(a, b.cpu())
    assert sep.launches["captured"] > 0 and sep.launches["replayed"] > 0
    # wav files
    paths = []
    for i, w in enumerate(wavs[:5]):
        p = str(tmp_path / f"mix{i}.wav")
        Cp.save_wav(p, w, 8000)
        paths.append(p)
    written = Cp.separate_wav_files(m, paths, str(tmp_path / "out"), max_samples=4000, max_batch=4)
    assert len(written) == 5 and all(len(w) == 2 for w in written)
    ref = Cp.separate_corpus(m, [w[:4000] for w in wavs[:5]], max_batch=4)
    for outs, r in zip(written, ref):
        for k, path in enumerate(outs):
            y, sr = Cp.load_wav(path)
            assert sr == 8000 and torch.equal(y[0], r[k].cpu())
