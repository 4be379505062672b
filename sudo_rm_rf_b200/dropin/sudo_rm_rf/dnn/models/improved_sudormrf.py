"""``sudo_rm_rf.dnn.models.improved_sudormrf`` -> H100-native implementation."""
from sudo_rm_rf_b200.improved_sudormrf import (SuDORMRF, UConvBlock, GlobLN, ConvNormAct, NormAct,  # noqa: F401
                                               DilatedConvNorm, _LayerNorm)
