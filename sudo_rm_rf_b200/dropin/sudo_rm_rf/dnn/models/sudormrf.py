"""``sudo_rm_rf.dnn.models.sudormrf`` (the original SuDoRM-RF) -> H100-native implementation."""
from sudo_rm_rf_b200.sudormrf import (SuDORMRF, UBlock, ConvNormAct, ConvNorm, NormAct,  # noqa: F401
                                      DilatedConv, DilatedConvNorm)
