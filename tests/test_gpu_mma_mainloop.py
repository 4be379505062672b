"""The wgmma GEMM's main loop: the consumer warpgroups transform the raw activation k-blocks into register A fragments,
the weight stages rotate through a 3-deep ring, and each warpgroup's two epilogue slots load the next tile's residual /
gate quarters while the current tile is still being computed.  Shapes at the edges of those rings."""
import pytest

import test_gpu_stages as S

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("samples,M,K,L,mode", [
    (40, 256, 64, 1280, "res"),           # one k-block, 800 tiles: the slots wrap across tiles with loads in flight
    (40, 512, 64, 1280, "mask"),          # the same with the gate, 1600 tiles
    (6, 256, 192, 1280, "norm"),          # 3 k-blocks against the 3-stage weight ring
    (5, 512, 192, 640, "res_out"),        # the same with an out-of-place residual
    (2, 256, 4096, 640, "norm"),          # the cfg-5 bottleneck's K: per-channel affines over 64 k-blocks
    (40, 512, 128, 640, "pc"),            # per-channel slopes, 800 tiles
])
def test_pointwise_tensor_core_mainloop(samples, M, K, L, mode):
    S.test_pointwise_tensor_core(samples, M, K, L, mode)


@pytest.mark.parametrize("B,A,T,N_,K,D", [
    (2, 1, 64000, 4096, 21, 5),           # 32 channel tiles per position tile, 8 s at 8 kHz
])
def test_encoder_tensor_core_mainloop(B, A, T, N_, K, D):
    S.test_encoder_tensor_core(B, A, T, N_, K, D)
