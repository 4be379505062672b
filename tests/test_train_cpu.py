"""Training interface checks that need no GPU: the new C-ABI symbols, the saved-activation size, the refusals of the
variants without a backward, and the ``native_training`` flag's life cycle."""
import copy
import ctypes as C
import io
import pickle

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N

TRAIN_SYMBOLS = ("sdr_train_saved_bytes", "sdr_backward_workspace_bytes", "sdr_forward_train", "sdr_backward",
                 "sdr_backward_launch_count", "sdr_pointwise_wgrad", "sdr_norm_act_backward",
                 "sdr_depthwise_backward", "sdr_mask_backward", "sdr_overlap_add_backward", "sdr_encoder_wgrad")

SMALL = dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=3, enc_kernel_size=21,
             enc_num_basis=128, num_sources=2)


def test_train_symbols_bind():
    lib = N.lib()
    for name in TRAIN_SYMBOLS:
        assert name in N.EXPORTED_SYMBOLS
        assert getattr(lib, name) is not None


def cfg_of(variant=0, **kw):
    d = dict(variant=variant, in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=16,
             upsampling_depth=4, enc_kernel_size=21, enc_num_basis=512, num_sources=2, group_size=16)
    d.update(kw)
    return N.SdrConfig(**d)


def r256(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("kw,B,T", [
    (dict(), 32, 32000),
    (dict(out_channels=256, upsampling_depth=5), 2, 32079),
    (dict(out_channels=48, in_channels=96, num_blocks=3, upsampling_depth=1, enc_kernel_size=3, enc_num_basis=64,
          num_sources=1), 3, 1001),
    (dict(out_channels=512, num_blocks=36, upsampling_depth=6, enc_num_basis=2048), 1, 32000),
])
def test_saved_bytes_formula(kw, B, T):
    lib = N.lib()
    cfg = cfg_of(**kw)
    L = lib.sdr_padded_length(C.byref(cfg), T) // (cfg.enc_kernel_size // 2)
    U, D, Co, Nb = cfg.num_blocks, cfg.upsampling_depth, cfg.out_channels, cfg.enc_num_basis
    stats = (1 + U * (D + 2)) * B * 2 * 8
    want = r256(stats) + r256(4 * B * L * Nb) + (U + 1) * r256(4 * B * L * Co)
    assert lib.sdr_train_saved_bytes(C.byref(cfg), B, T) == want
    assert lib.sdr_backward_workspace_bytes(C.byref(cfg), B, T) > 0
    assert lib.sdr_backward_launch_count(C.byref(cfg), B, T) == 22 + U * (14 + 5 * D + (1 if D > 1 else 0))


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_other_variants_unsupported(variant):
    lib = N.lib()
    cfg = cfg_of(variant, out_channels=64, in_channels=128, enc_num_basis=64, group_size=4)
    assert lib.sdr_train_saved_bytes(C.byref(cfg), 1, 8000) == 0
    assert lib.sdr_backward_workspace_bytes(C.byref(cfg), 1, 8000) == 0
    assert lib.sdr_backward_launch_count(C.byref(cfg), 1, 8000) == -5      # SDR_ERR_UNSUPPORTED
    assert lib.sdr_forward_train(C.byref(cfg), None, None, None, 1, 8000, None, 0, None, 0, None) == -5
    assert lib.sdr_backward(C.byref(cfg), None, None, None, None, None, 1, 8000, None, 0, None) == -5


@pytest.mark.parametrize("cls,kw,word", [
    (P.GroupCommSudoRmRf, dict(out_channels=64, in_channels=128, num_blocks=1, enc_num_basis=64, group_size=4),
     "GroupComm"),
    (P.CausalSuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=1, enc_num_basis=64), "Causal"),
    (P.OriginalSuDORMRF, dict(out_channels=64, in_channels=128, num_blocks=1, enc_num_basis=64), "original"),
])
def test_enable_training_refused_on_other_variants(cls, kw, word):
    with pytest.raises(NotImplementedError, match=word):
        cls(**kw).enable_training()


def test_flag_default_off_and_returns_self():
    m = P.SuDORMRF(**SMALL)
    assert m.native_training is False
    assert m.enable_training() is m and m.native_training is True
    assert m.enable_training(False) is m and m.native_training is False


def test_flag_travels_and_stays_out_of_state_dict():
    m = P.SuDORMRF(**SMALL)
    keys = list(m.state_dict().keys())
    m.enable_training()
    assert list(m.state_dict().keys()) == keys
    assert "native_training" not in m.state_dict()
    assert copy.deepcopy(m).native_training
    assert pickle.loads(pickle.dumps(m)).native_training
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    assert torch.load(buf, weights_only=False).native_training
    assert m._replicate_for_data_parallel().native_training
    names = _engine.state_dict_names(_engine.make_config(m))
    assert names == keys


def test_flag_through_the_overlay_import_path():
    import importlib
    import sys
    from sudo_rm_rf_b200 import dropin
    sys.path.insert(0, dropin.__path__[0])
    try:
        mod = importlib.import_module("sudo_rm_rf.dnn.models.improved_sudormrf")
        m = mod.SuDORMRF(**SMALL).enable_training()
        assert isinstance(m, P.SuDORMRF) and m.native_training
        assert pickle.loads(pickle.dumps(m)).native_training
    finally:
        sys.path.remove(dropin.__path__[0])


def test_mixture_requiring_grad_raises():
    m = P.SuDORMRF(**SMALL).enable_training()
    with pytest.raises(RuntimeError, match="mixture"):
        m(torch.randn(1, 1, 8000, requires_grad=True))


def test_cpu_tensors_raise():
    m = P.SuDORMRF(**SMALL).enable_training()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 1, 8000))
