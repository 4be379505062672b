"""The wgmma GEMM's store warp: it stores every quarter the consumer warpgroups combine and refills the slot with the
CTA's next residual / gate quarter.  Tile counts at the edges of the persistent schedule (one tile, fewer tiles than
SMs, one CTA with a second tile), many tiles per CTA with a single k-block, and the bias-only mode with statistics."""
import pytest

import test_gpu_stages as S

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("samples,M,K,L,mode", [
    (1, 128, 128, 128, "res"),            # exactly one tile: one CTA, no refill
    (2, 256, 256, 1280, "mask"),          # 40 tiles: fewer than the SMs, one tile per CTA
    (7, 128, 192, 2432, "res_out"),       # 133 tiles on an H100 SXM's 132 SMs: CTA 0 runs a second tile
    (64, 256, 64, 1280, "res"),           # in place, 1280 tiles of a single k-block: ~10 refills per slot and CTA
    (20, 512, 128, 600, "plain_stats"),   # bias only with statistics, 400 tiles, ragged last position tile
])
def test_pointwise_tensor_core_store_warp(samples, M, K, L, mode):
    S.test_pointwise_tensor_core(samples, M, K, L, mode)
