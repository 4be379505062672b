"""Streaming of the causal model on the CPU: the chunked restatement (tests/stream_oracle.py) against the whole-clip
oracle in fp64, and the C-ABI's stream arithmetic and refusals (no compute calls)."""
import ctypes as C

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine, _native
from oracle import sudormrf_oracle as O
from stream_oracle import causal_stream_forward, granule


def small_causal(A, D, k):
    return O.Config(variant="causal", in_audio_channels=A, out_channels=8, in_channels=12, num_blocks=2,
                    upsampling_depth=D, enc_kernel_size=k, enc_num_basis=16, num_sources=2)


CASES = [(A, D, k, g, aligned) for A in (1, 2) for D in (1, 4, 5) for k in (11, 21) for g in (1, 3)
         for aligned in (True, False)]


@pytest.mark.parametrize("A,D,k,g,aligned", CASES)
def test_restatement_matches_whole_clip(A, D, k, g, aligned):
    cfg = small_causal(A, D, k)
    C_ = g * granule(cfg)
    q = cfg.n_least_samples_req
    ns = [n for n in range(1, 9) if ((n * C_) % q == 0) == aligned]
    if not ns:
        pytest.skip("every chunk count is a multiple of the padding quantum here")
    n = ns[0] if aligned else ns[min(1, len(ns) - 1)]
    sd = O.make_state_dict(cfg, seed=7)
    x = torch.randn(2, A, n * C_, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    ref = O.causal_forward(cfg, sd, x, dtype=torch.float64)
    out, tail = causal_stream_forward(cfg, sd, x, C_)
    hop, T = cfg.hop, n * C_
    assert torch.equal(out[..., :hop], torch.zeros_like(out[..., :hop]))
    scale = ref.abs().max()
    assert float((out[..., hop:] - ref[..., :T - hop]).abs().max() / scale) <= 1e-12
    if aligned:
        assert float((tail - ref[..., T - hop:]).abs().max() / scale) <= 1e-12


def cfg_of(variant=2, A=1, Co=128, Ci=512, U=16, D=4, k=21, N=512, S=2):
    return _native.SdrConfig(variant, A, Co, Ci, U, D, k, N, S, 1)


@pytest.mark.parametrize("D,k", [(1, 21), (3, 21), (4, 21), (5, 21), (5, 11), (6, 11), (8, 21)])
def test_granule_state_and_launch_count(D, k):
    lib = _native.lib()
    cfg = cfg_of(D=D, k=k, U=3, A=2, S=3, Ci=40)
    hop = k // 2
    G = hop * max(4, 2 ** (D - 1))
    assert lib.sdr_stream_granule(C.byref(cfg)) == G
    state_floats = 2 * 2 * hop + 3 * 2 * (hop + 1) + 1 + 3 * D * 10 * 40     # context, carry, started flag, histories
    for B in (1, 3, 256):
        sb = lib.sdr_stream_state_bytes(C.byref(cfg), B)
        assert sb >= 4 * B * state_floats and sb % (256 * B) == 0 and sb - 4 * B * state_floats < B * 512
        assert lib.sdr_stream_launch_count(C.byref(cfg), B, G) == 3 * 3 + 6
        assert lib.sdr_stream_workspace_bytes(C.byref(cfg), B, 2 * G) > lib.sdr_stream_workspace_bytes(C.byref(cfg), B, G) > 0
    assert lib.sdr_stream_workspace_bytes(C.byref(cfg), 2, G + hop) == 0
    assert lib.sdr_stream_launch_count(C.byref(cfg), 2, G + hop) == -5
    F_max = 4096
    assert lib.sdr_stream_workspace_bytes(C.byref(cfg), 1, F_max * hop) > 0
    assert lib.sdr_stream_workspace_bytes(C.byref(cfg), 1, F_max * hop + G) == 0


def test_default_model_numbers():
    lib = _native.lib()
    cfg = cfg_of()
    assert lib.sdr_stream_granule(C.byref(cfg)) == 80
    assert lib.sdr_stream_launch_count(C.byref(cfg), 256, 80) == 54
    assert abs(lib.sdr_stream_state_bytes(C.byref(cfg), 1) - 16 * 4 * 512 * 10 * 4) < 1024   # ~1.3 MB per slot


@pytest.mark.parametrize("variant", [0, 1, 3])
def test_other_variants_refused(variant):
    lib = _native.lib()
    cfg = cfg_of(variant=variant, Co=16, Ci=32, U=1, D=3, N=16)
    assert lib.sdr_stream_granule(C.byref(cfg)) == -5
    assert lib.sdr_stream_state_bytes(C.byref(cfg), 2) == 0
    assert lib.sdr_stream_workspace_bytes(C.byref(cfg), 2, 80) == 0
    assert lib.sdr_stream_launch_count(C.byref(cfg), 2, 80) == -5
    buf = (C.c_char * 64)()
    assert lib.sdr_stream_reset(C.byref(cfg), buf, 2, None, 0, None) == -5
    assert lib.sdr_stream_step(C.byref(cfg), buf, buf, buf, buf, 2, 80, 0, buf, 64, None) == -5
    assert lib.sdr_stream_flush(C.byref(cfg), buf, buf, 2, 0, None) == -5


def test_step_argument_errors_before_any_launch():
    lib = _native.lib()
    cfg = cfg_of(U=1, Co=16, Ci=32, N=16)
    buf = (C.c_char * 64)()
    assert lib.sdr_stream_step(C.byref(cfg), buf, buf, buf, buf, 2, 88, 0, buf, 64, None) == -5      # not a granule multiple
    assert lib.sdr_stream_step(C.byref(cfg), buf, buf, buf, buf, 0, 80, 0, buf, 64, None) == -2
    assert lib.sdr_stream_step(C.byref(cfg), buf, buf, buf, buf, 2, 80, 0, buf, 64, None) == -3      # workspace too small
    assert lib.sdr_stream_step(C.byref(cfg_of(A=2, U=1, Co=16, Ci=32, N=16)), buf, buf, buf, buf, 2, 80, 1, buf,
                               1 << 30, None) == -5                                                  # stereo mixture consistency
    bad = cfg_of(k=20)
    assert lib.sdr_stream_granule(C.byref(bad)) == -1
    slots = (C.c_int32 * 1)(5)
    assert lib.sdr_stream_reset(C.byref(cfg), buf, 2, slots, 1, None) == -2
    assert lib.sdr_causal_stream_stage(None, None, None, None, None, None, None, 4, 1, 32, 8, None) == -2
    ptrs = (C.c_void_p * 8)(*([C.cast(buf, C.c_void_p)] * 8))
    p = C.cast(buf, C.c_void_p)
    assert lib.sdr_causal_stream_stage(p, p, ptrs, ptrs, ptrs, p, p, 4, 1, 32, 12, None) == -5      # F % 2^(D-1)
    assert lib.sdr_causal_stream_stage(p, p, ptrs, ptrs, ptrs, p, p, 4, 1, 32, 4096 + 8, None) == -5


def test_stream_needs_a_causal_cuda_model():
    m = P.CausalSuDORMRF(1, 16, 32, 1, 3, 21, 16, 2).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.stream(2, 40)
    with pytest.raises(RuntimeError, match="CausalSuDORMRF"):
        from sudo_rm_rf_b200.streaming import CausalStream
        CausalStream(P.SuDORMRF(16, 32, 1, 2, 21, 16, 2), 2, 40)
    cfg = _engine.make_config(m)
    assert _native.lib().sdr_stream_granule(C.byref(cfg)) == 40
