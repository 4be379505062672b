"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports
every symbol include/sudormrf_b200.h declares, and its layout functions agree
with the reference's state_dict inventory.  No compute calls (no GPU here)."""
import ctypes as C
import os
import re

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine, _native
from oracle import sudormrf_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASSES = {"improved": P.SuDORMRF, "groupcomm": P.GroupCommSudoRmRf, "causal": P.CausalSuDORMRF,
           "original": P.OriginalSuDORMRF}


def _param_name(lib, cfg, i):
    """sdr_param_name of entry i: a size query, then the name into a buffer one byte longer."""
    n = lib.sdr_param_name(C.byref(cfg), i, None, 0)
    assert n > 0, n
    buf = C.create_string_buffer(n + 1)
    assert lib.sdr_param_name(C.byref(cfg), i, buf, n + 1) == n
    return buf.value.decode()


def test_header_symbols_are_exported():
    hdr = open(os.path.join(REPO, "include", "sudormrf_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(sdr_[a-z_0-9]+)\s*\(", hdr))
    assert len(declared) >= 24
    lib = _native.lib()
    for name in declared:
        assert hasattr(lib, name), name
    assert declared == set(_native.EXPORTED_SYMBOLS)
    assert lib.sdr_abi_version() == _native.ABI_VERSION == 2
    assert lib.sdr_error_string(0) == b"ok"
    assert b"unknown" not in lib.sdr_error_string(-5)


@pytest.mark.parametrize("variant,kw", [
    ("improved", dict(out_channels=256, in_channels=512, num_blocks=16, upsampling_depth=5,
                      enc_kernel_size=21, enc_num_basis=512, num_sources=2)),
    ("improved", dict(out_channels=512, in_channels=512, num_blocks=36, upsampling_depth=6,
                      enc_kernel_size=21, enc_num_basis=2048, num_sources=2)),
    ("groupcomm", dict(out_channels=256, in_channels=512, num_blocks=8, upsampling_depth=5,
                       enc_kernel_size=21, enc_num_basis=512, num_sources=2, group_size=16)),
    ("groupcomm", dict(out_channels=32, in_channels=64, num_blocks=1, upsampling_depth=3,
                       enc_kernel_size=11, enc_num_basis=16, num_sources=2, group_size=8,
                       in_audio_channels=2)),
    ("causal", dict(in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=4,
                    enc_kernel_size=21, enc_num_basis=512, num_sources=2)),
    ("causal", dict(in_audio_channels=2, out_channels=16, in_channels=32, num_blocks=3, upsampling_depth=5,
                    enc_kernel_size=11, enc_num_basis=24, num_sources=3)),
    ("original", dict(out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=4,
                      enc_kernel_size=21, enc_num_basis=512, num_sources=2)),
    ("original", dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=5,
                      enc_kernel_size=11, enc_num_basis=32, num_sources=3)),      # out_channels == enc_num_basis: no reshape layer
])
def test_layout_matches_state_dict(variant, kw):
    m = CLASSES[variant](**kw)
    cfg_o = O.Config(variant=variant, **kw)
    sd = m.state_dict()
    shapes = O.param_shapes(cfg_o)
    assert list(sd.keys()) == list(shapes.keys())
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(shapes[k]), k
    cfg = _engine.make_config(m)
    if variant == "original":          # ln_mask_in is registered last and never read by forward (sudormrf.py:253): not packed
        assert list(sd.keys())[-2:] == ["ln_mask_in.weight", "ln_mask_in.bias"]
        sd = {k: v for k, v in list(sd.items())[:-2]}
    assert _engine.state_dict_names(cfg) == list(sd.keys())
    lib = _native.lib()
    assert lib.sdr_num_params(C.byref(cfg)) == len(sd)
    total = 0
    for i, (k, v) in enumerate(sd.items()):
        assert _param_name(lib, cfg, i) == k
        assert lib.sdr_param_numel(C.byref(cfg), i) == v.numel()
        total += v.numel()
    assert lib.sdr_packed_weight_bytes(C.byref(cfg)) >= 4 * total
    for T in (1, 100, 160, 320, 321, 32000, 32079):
        assert lib.sdr_padded_length(C.byref(cfg), T) == O.padded_length(cfg_o, T)
    assert lib.sdr_workspace_bytes(C.byref(cfg), 2, 32000) > 0


def _name_grid():
    small = dict(out_channels=16, in_channels=32, enc_kernel_size=11, enc_num_basis=16, num_sources=2)
    for U in (0, 1, 3):
        for D in range(1, 9):          # 8: the deepest level the layout takes (test_param_name_refusals: 9 is refused)
            kw = dict(small, num_blocks=U, upsampling_depth=D)
            at = f"U{U}-D{D}"
            yield pytest.param("improved", kw, id=f"improved-{at}")
            yield pytest.param("causal", kw, id=f"causal-{at}")
            for G in (2, 4):
                yield pytest.param("groupcomm", dict(kw, group_size=G), id=f"groupcomm-{at}-G{G}")
            for Co in (16, 8):         # out_channels == enc_num_basis: no reshape_before_masks
                yield pytest.param("original", dict(kw, out_channels=Co), id=f"original-{at}-Co{Co}")
    stereo = dict(small, num_blocks=2, upsampling_depth=3, in_audio_channels=2)
    yield pytest.param("groupcomm", dict(stereo, group_size=4), id="groupcomm-stereo")
    yield pytest.param("causal", stereo, id="causal-stereo")


@pytest.mark.parametrize("variant,kw", list(_name_grid()))
def test_param_names_are_the_state_dict_keys(variant, kw):
    """The library names every entry it packs with the module's state_dict key, in the module's order."""
    m = CLASSES[variant](**kw)
    keys = list(m.state_dict().keys())
    if variant == "original":          # not packed: see test_layout_matches_state_dict
        assert keys[-2:] == ["ln_mask_in.weight", "ln_mask_in.bias"]
        keys = keys[:-2]
    cfg = _engine.make_config(m)
    lib = _native.lib()
    assert lib.sdr_num_params(C.byref(cfg)) == len(keys)
    assert [_param_name(lib, cfg, i) for i in range(len(keys))] == keys


def test_param_name_refusals():
    """Each refusal of sdr_param_name returns its code and writes nothing; a fitting buffer gets the name and its NUL."""
    lib = _native.lib()
    cfg = _engine.make_config(P.GroupCommSudoRmRf(1, 16, 32, 2, 3, 11, 16, 2, 4))
    deep = _engine.make_config(P.SuDORMRF(16, 32, 1, 9, 11, 16, 2))      # one level deeper than the layout takes
    n = lib.sdr_num_params(C.byref(cfg))
    name = b"decoder.weight"
    L = len(name)
    assert lib.sdr_num_params(C.byref(deep)) == -1 and _param_name(lib, cfg, n - 1) == name.decode()
    size = 64
    for what, c, i, has_buf, nbytes, want in [
        ("bad config", deep, 0, True, size, -1),
        ("bad config, size query", deep, 0, False, 0, -1),
        ("bad config before a bad index", deep, -1, True, size, -1),
        ("index -1", cfg, -1, True, size, -2),
        ("index n", cfg, n, True, size, -2),
        ("index n, size query", cfg, n, False, 0, -2),
        ("NULL buffer with a size", cfg, n - 1, False, size, -2),
        ("NULL buffer of one byte", cfg, 0, False, 1, -2),
        ("buffer as long as the name", cfg, n - 1, True, L, -3),
        ("buffer of zero bytes", cfg, n - 1, True, 0, -3),
        ("size query", cfg, n - 1, False, 0, L),
        ("buffer one byte longer than the name", cfg, n - 1, True, L + 1, L),
    ]:
        buf = C.create_string_buffer(b"\xa5" * size, size)
        got = lib.sdr_param_name(C.byref(c), i, buf if has_buf else None, nbytes)
        assert got == want, what
        written = name + b"\0" if has_buf and want >= 0 else b""
        assert buf.raw == written + b"\xa5" * (size - len(written)), what


def test_published_parameter_counts():
    # README.md:122-124 of the reference: 5.02 M / 23.24 M / 0.51 M parameters
    n = lambda m: sum(p.numel() for p in m.parameters())
    assert n(P.SuDORMRF(256, 512, 16, 5, 21, 512, 2)) == 5016353
    assert n(P.GroupCommSudoRmRf(1, 256, 512, 8, 5, 21, 512, 2, 16)) == 507177


def test_bad_configs_rejected():
    lib = _native.lib()
    bad = _native.SdrConfig(0, 1, 16, 32, 1, 3, 20, 16, 2, 1)      # even kernel
    assert lib.sdr_num_params(C.byref(bad)) == -1
    assert lib.sdr_workspace_bytes(C.byref(bad), 1, 100) == 0
    bad = _native.SdrConfig(1, 1, 30, 64, 1, 3, 21, 16, 2, 4)      # Co % G != 0
    assert lib.sdr_num_params(C.byref(bad)) == -1
    bad = _native.SdrConfig(3, 1, 16, 32, 1, 3, 21, 25, 2, 1)      # original model, odd basis count: its mask Conv2d returns N + 1 rows
    assert lib.sdr_num_params(C.byref(bad)) == -1
    bad = _native.SdrConfig(4, 1, 16, 32, 1, 3, 21, 24, 2, 1)      # no such variant
    assert lib.sdr_num_params(C.byref(bad)) == -1
    with pytest.raises(AssertionError):
        P.GroupCommSudoRmRf(enc_kernel_size=20)


def test_no_cpu_fallback_and_error_conventions():
    m = P.SuDORMRF(16, 32, 1, 2, 21, 16, 2).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 1, 100))
    with pytest.raises(RuntimeError, match="3D"):
        m(torch.zeros(1, 100))
    with pytest.raises(NotImplementedError):
        m.sm[0](torch.zeros(1, 16, 10))
    with pytest.raises(ValueError):
        P.mixture_consistency.apply(torch.zeros(1, 2, 4), torch.zeros(1, 1, 4), "nope")
    with pytest.raises(RuntimeError):
        P.mixture_consistency.apply(torch.zeros(1, 2, 4), torch.zeros(1, 1, 4))


def test_state_dict_roundtrip_and_module_prefix():
    m = P.SuDORMRF(16, 32, 2, 3, 21, 24, 2)
    cfg = O.Config("improved", 16, 32, 2, 3, 21, 24, 2)
    sd = O.make_state_dict(cfg, seed=1)
    m.load_state_dict(sd)
    # DataParallel-saved checkpoints carry a "module." prefix (run_improved_sudormrf.py:221-227)
    dp = {"module." + k: v for k, v in sd.items()}
    m.load_state_dict({k[len("module."):]: v for k, v in dp.items()})
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k])


def test_prepost_entry_points_have_no_cpu_path():
    """separate(normalize=True), separate_corpus and the SI-SDR metric raise on CPU tensors / models
    (no fallback), and reject what the reference's recipe does not cover."""
    from sudo_rm_rf_b200 import sisdr
    from sudo_rm_rf_b200.corpus import separate_corpus
    m = P.SuDORMRF(16, 32, 1, 2, 21, 16, 2).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.separate(torch.zeros(2, 100), normalize=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        separate_corpus(m, [torch.zeros(50), torch.zeros(70)])
    with pytest.raises(RuntimeError, match="1-D"):
        separate_corpus(m, [torch.zeros(1, 50)])
    assert separate_corpus(m, []) == []
    metric = sisdr.PermInvariantSISDR(n_sources=2)
    with pytest.raises(RuntimeError, match="CUDA"):
        metric(torch.zeros(1, 2, 10), torch.zeros(1, 2, 10))
    with pytest.raises(RuntimeError, match="n_sources"):
        metric(torch.zeros(1, 3, 10), torch.zeros(1, 3, 10))
    assert metric.permutations == [(0, 1), (1, 0)] or [tuple(int(i) for i in p) for p in metric.permutations] == [(0, 1), (1, 0)]
    lib = _native.lib()
    assert lib.sdr_pit_sisdr_scratch_bytes(4, 2) > 0 and lib.sdr_pit_sisdr_scratch_bytes(4, 5) == 0
    cfg = _native.SdrConfig(0, 1, 16, 32, 1, 2, 21, 16, 2, 1)
    assert lib.sdr_separate_workspace_bytes(C.byref(cfg), 2, 100) > lib.sdr_workspace_bytes(C.byref(cfg), 2, 100)


def test_sibling_variants_host_conventions():
    """The original and the causal model mirrors on the CPU side: constructor defaults and attributes of the reference
    (sudormrf.py:186-209, causal_improved_sudormrf_v3.py:121-140), state_dict round trip incl. the unused ln_mask_in,
    whole-module pickle, no CPU path, parameter containers are not callable on their own."""
    import io
    m = P.OriginalSuDORMRF()
    assert (m.out_channels, m.in_channels, m.num_blocks, m.upsampling_depth, m.enc_kernel_size, m.enc_num_basis,
            m.num_sources) == (128, 512, 16, 4, 21, 512, 2)
    assert m.lcm == 80 and P.OriginalSuDORMRF(upsampling_depth=5, enc_kernel_size=11).lcm == 160
    small = dict(out_channels=16, in_channels=32, num_blocks=2, upsampling_depth=3, enc_kernel_size=21,
                 enc_num_basis=24, num_sources=2)
    m = P.OriginalSuDORMRF(**small)
    cfg = O.Config(variant="original", **small)
    sd = O.make_state_dict(cfg, seed=2)
    m.load_state_dict(sd)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert hasattr(m, "reshape_before_masks") and not hasattr(P.OriginalSuDORMRF(32, 64, 1, 3, 21, 32, 2), "reshape_before_masks")
    x = torch.zeros(2, 1, 517)
    assert m.pad_to_appropriate_length(x).shape[-1] == 520 and m.pad_to_appropriate_length(x[..., :480]) is not None
    assert m.pad_to_appropriate_length(x[..., :480]).shape[-1] == 480          # a multiple of the lcm is left alone (:284-285)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(x)
    with pytest.raises(NotImplementedError):
        m.sm[0](torch.zeros(1, 16, 10))
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    m2 = torch.load(buf, weights_only=False)
    assert type(m2) is P.OriginalSuDORMRF and list(m2.state_dict().keys()) == list(sd.keys())
    c = P.CausalSuDORMRF()
    assert (c.in_audio_channels, c.out_channels, c.in_channels, c.num_blocks, c.upsampling_depth) == (1, 128, 512, 16, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        c.eval()(torch.zeros(1, 1, 400))
    # odd basis count: the reference's mask Conv2d then returns N + 1 rows and its forward fails; here the library refuses
    odd = P.OriginalSuDORMRF(16, 32, 1, 3, 21, 25, 2)
    assert _native.lib().sdr_num_params(C.byref(_engine.make_config(odd))) == -1


def test_stabilized_metric_host_conventions():
    from sudo_rm_rf_b200 import sisdr
    fn = sisdr.StabilizedPermInvSISDRMetric(zero_mean=True, n_estimated_sources=4, n_actual_sources=2, backward_loss=False,
                                            improvement=True, return_individual_results=True)
    assert len(fn.permutations) == 12 and tuple(int(i) for i in fn.permutations[1]) == (0, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(torch.zeros(1, 4, 10), torch.zeros(1, 2, 10))
    with pytest.raises(RuntimeError, match="actual"):
        fn(torch.zeros(1, 4, 10), torch.zeros(1, 3, 10))
    with pytest.raises(RuntimeError, match="estimated"):       # fewer rows than estimated sources: the reference fails too
        fn(torch.zeros(1, 3, 10), torch.zeros(1, 2, 10))
    one = sisdr.StabilizedPermInvSISDRMetric(zero_mean=True, n_estimated_sources=1, n_actual_sources=1)
    with pytest.raises(RuntimeError, match="CUDA"):             # four rows pass the row check: the first one is scored
        one(torch.zeros(1, 4, 10), torch.zeros(1, 1, 10))
    with pytest.raises(AssertionError):
        sisdr.StabilizedPermInvSISDRMetric(n_estimated_sources=1, n_actual_sources=2)
    with pytest.raises(AssertionError):
        sisdr.StabilizedPermInvSISDRMetric(single_source=True, n_estimated_sources=2, n_actual_sources=2)
    lib = _native.lib()
    assert lib.sdr_stabilized_sisdr_scratch_bytes(3, 4, 2) == 8 * 3 * (4 + 2 + 8 + 4 + 4)
    assert lib.sdr_stabilized_sisdr_scratch_bytes(3, 2, 3) == 0 and lib.sdr_stabilized_sisdr_scratch_bytes(3, 5, 2) == 0


def test_ffma_encoder_limit_refused_before_launch():
    """Below 32 basis functions the encoder is the FFMA kernel, whose CTA holds A channels x K taps of weights and
    waveform in at most 200 KB of shared memory: A = 4 takes K = 99 and not 101, A = 16 takes K = 25 and not 27.
    sdr_forward refuses the larger filters with its other argument checks, before it reads a buffer or enqueues a
    kernel (null buffers then return SDR_ERR_BAD_ARGUMENT instead); the tensor-core encoder (N = 32) has no such limit."""
    lib = _native.lib()

    def fwd(A, K, N_, S):
        m = P.GroupCommSudoRmRf(in_audio_channels=A, out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=3,
                                enc_kernel_size=K, enc_num_basis=N_, num_sources=S, group_size=4)
        c = _engine.make_config(m)
        assert lib.sdr_workspace_bytes(C.byref(c), 2, 1001) > 0
        return lib.sdr_forward(C.byref(c), None, None, None, 2, 1001, 0, None, 0, None)
    assert (fwd(4, 99, 16, 4), fwd(4, 101, 16, 4)) == (-2, -5)
    assert (fwd(16, 25, 16, 1), fwd(16, 27, 16, 1)) == (-2, -5)
    assert lib.sdr_encoder_mma_packed_bytes(32, 4, 101) > 0 and fwd(4, 101, 32, 4) == -2
