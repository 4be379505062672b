"""``sudo_rm_rf.dnn.models.groupcomm_sudormrf_v2`` -> H100-native implementation."""
from sudo_rm_rf_b200.groupcomm_sudormrf_v2 import (GroupCommSudoRmRf, TAC, GC_UConvBlock, UConvBlock,  # noqa: F401
                                                   GlobLN, ConvNormAct, NormAct, DilatedConvNorm, _LayerNorm)
