"""The wgmma GEMM's epilogue: residual / gate quarters loaded into a shared-memory slot by TMA and the output stored
from it by TMA.  Shapes where the slot passes through many quarters per CTA, where the boxes are clipped at L and at
M, and the 16 B alignment the tensor maps need of y, residual and gate."""
import ctypes as C

import pytest
import torch

import test_gpu_stages as S
from sudo_rm_rf_b200 import _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("samples,M,K,L,mode", [
    (40, 256, 512, 384, "res"),           # 240 tiles: the one slot serves 8 quarters and more per CTA
    (40, 256, 64, 640, "mask"),           # a single k-block per tile, 400 tiles
    (3, 300, 128, 200, "res_out"),        # ragged last position tile (72 of 128) and 300 rows padded to 384
])
def test_pointwise_tensor_core_epilogue(samples, M, K, L, mode):
    S.test_pointwise_tensor_core(samples, M, K, L, mode)


@pytest.mark.parametrize("which", ["y", "residual", "gate"])
def test_pointwise_tensor_core_refuses_unaligned_epilogue(which):
    """y, residual and gate are moved by TMA: a pointer that is not 16 B aligned is refused (SDR_ERR_UNSUPPORTED)."""
    lib = N.lib()
    samples, M, K, L = 1, 256, 64, 128
    x = torch.zeros(samples, K, L, device=DEV)
    W = torch.zeros(M, K, device=DEV)
    wpk = torch.empty(lib.sdr_pointwise_mma_packed_bytes(M, K), dtype=torch.uint8, device=DEV)
    N.check(lib.sdr_pointwise_mma_pack(S.p(W), M, K, S.p(wpk), S.stream()))

    def buf(C_, shifted):
        t = torch.zeros(samples * C_ * L + 4, device=DEV)
        return t[1:1 + samples * C_ * L] if shifted else t[:samples * C_ * L]

    y = buf(M, which == "y")
    residual = buf(M, which == "residual") if which != "gate" else None
    gate = buf(M // 2, which == "gate") if which == "gate" else None
    nin = S.norm_in()
    rc = lib.sdr_pointwise_mma(S.p(x), C.byref(nin), S.p(wpk), S.p(None), S.p(residual), S.p(gate),
                               M // 2 if gate is not None else 0, S.p(y), S.p(None), samples, M, K, L,
                               1 if gate is not None else 0, S.stream())
    assert rc == -5
    # the same call with every pointer aligned runs
    aligned = lib.sdr_pointwise_mma(S.p(x), C.byref(nin), S.p(wpk), S.p(None),
                                    S.p(buf(M, False)) if which == "residual" else S.p(None),
                                    S.p(buf(M // 2, False)) if which == "gate" else S.p(None),
                                    M // 2 if which == "gate" else 0, S.p(buf(M, False)), S.p(None),
                                    samples, M, K, L, 1 if which == "gate" else 0, S.stream())
    torch.cuda.synchronize()
    assert aligned == 0
