"""Streaming of the causal model on the CPU: the chunked restatement (tests/stream_oracle.py) against the whole-clip
oracle in fp64, and the C-ABI's stream arithmetic and refusals (no compute calls)."""
import ctypes as C

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine, _native
from oracle import sudormrf_oracle as O
from stream_oracle import causal_stream_forward, granule


def small_causal(A, D, k, S=2):
    return O.Config(variant="causal", in_audio_channels=A, out_channels=8, in_channels=12, num_blocks=2,
                    upsampling_depth=D, enc_kernel_size=k, enc_num_basis=16, num_sources=S)


CASES = [(A, D, k, g, aligned, 2) for A in (1, 2) for D in (1, 4, 5) for k in (11, 21) for g in (1, 3)
         for aligned in (True, False)]
# every other depth, the shortest filters (hop 1 and 2) and the longest the stream takes (hop 127), one and three
# sources: the GPU weight-swap test steps this restatement, so it has to hold wherever the stream does
CASES += [(1, D, 21, 1, aligned, 2) for D in (2, 3, 6, 7, 8) for aligned in (True, False)]
CASES += [(1, 4, k, 1, aligned, 2) for k in (3, 5, 255) for aligned in (True, False)]
CASES += [(A, 4, 11, 1, aligned, S) for A, S in ((1, 1), (1, 3), (2, 3)) for aligned in (True, False)]


def case_id(c):
    return "-".join(str(v) for v in c[:5]) + ("" if c[5] == 2 else f"-S{c[5]}")


@pytest.mark.parametrize("A,D,k,g,aligned,S", CASES, ids=[case_id(c) for c in CASES])
def test_restatement_matches_whole_clip(A, D, k, g, aligned, S):
    cfg = small_causal(A, D, k, S)
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


@pytest.mark.parametrize("D,k", [(1, 21), (3, 21), (4, 21), (5, 21), (5, 11), (6, 11), (8, 21), (2, 21), (6, 21),
                                 (7, 21)])
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


def test_refusal_boundaries():
    """The largest filter, source count, slot count and chunk the stream takes, and one past each; no launch."""
    lib = _native.lib()
    ok = cfg_of(k=255, U=1, Co=16, Ci=32, N=16)                       # hop 127: 2*hop + 2 == 256 overlap-add threads
    assert lib.sdr_stream_granule(C.byref(ok)) == 127 * 8
    assert lib.sdr_stream_workspace_bytes(C.byref(ok), 2, 127 * 4096) > 0
    too_long = cfg_of(k=257, U=1, Co=16, Ci=32, N=16)
    assert lib.sdr_stream_granule(C.byref(too_long)) == -5
    assert lib.sdr_stream_state_bytes(C.byref(too_long), 2) == 0
    assert lib.sdr_stream_workspace_bytes(C.byref(too_long), 2, 128 * 8) == 0
    for S, A in ((16, 1), (8, 2)):                                    # S*A == 16, the overlap-add's per-source array
        c = cfg_of(S=S, A=A, U=1, Co=16, Ci=32, N=16)
        assert lib.sdr_stream_granule(C.byref(c)) == 80
        assert lib.sdr_stream_state_bytes(C.byref(c), 2) > 0
        assert lib.sdr_stream_launch_count(C.byref(c), 2, 80) == 9
    for S, A in ((17, 1), (9, 2)):                                    # S*A == 17, 18: not a valid configuration
        c = cfg_of(S=S, A=A, U=1, Co=16, Ci=32, N=16)
        assert lib.sdr_stream_granule(C.byref(c)) == -1
        assert lib.sdr_stream_state_bytes(C.byref(c), 2) == 0
        assert lib.sdr_stream_workspace_bytes(C.byref(c), 2, 80) == 0
    c = cfg_of(U=1, Co=16, Ci=32, N=16)
    assert lib.sdr_stream_workspace_bytes(C.byref(c), 65535, 80) > 0
    assert lib.sdr_stream_launch_count(C.byref(c), 65535, 80) == 9
    assert lib.sdr_stream_workspace_bytes(C.byref(c), 65536, 80) == 0
    assert lib.sdr_stream_launch_count(C.byref(c), 65536, 80) == -2
    for D in range(1, 9):
        c = cfg_of(D=D, U=1, Co=16, Ci=32, N=16)
        G = 10 * max(4, 2 ** (D - 1))
        assert lib.sdr_stream_workspace_bytes(C.byref(c), 3, 4096 * 10) > 0, D
        assert lib.sdr_stream_launch_count(C.byref(c), 3, 4096 * 10 + G) == -5, D


def test_stream_names_the_limit_it_hit():
    """CausalStream's argument errors come before the device check, so a CPU model shows them."""
    m = P.CausalSuDORMRF(1, 16, 32, 1, 3, 21, 16, 2).eval()           # granule 40, at most 40960 samples per step
    with pytest.raises(ValueError, match="batch_size=65536 is outside the slots"):
        m.stream(65536, 40)
    with pytest.raises(ValueError, match="batch_size=0 is outside the slots"):
        m.stream(0, 40)
    with pytest.raises(ValueError, match="granule"):
        m.stream(2, 50)
    with pytest.raises(ValueError, match="chunk_samples=41000 is longer than a step takes .at most 40960"):
        m.stream(2, 41000)
    with pytest.raises(RuntimeError, match="CUDA"):                  # the largest of each is accepted
        m.stream(65535, 40960)
    st = P.CausalSuDORMRF(2, 16, 32, 1, 3, 21, 16, 2).eval()
    with pytest.raises(RuntimeError, match="mono"):
        st.stream(2, 40, mixture_consistency=True)
