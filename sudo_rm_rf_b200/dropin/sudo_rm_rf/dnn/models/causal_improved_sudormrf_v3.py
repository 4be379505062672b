"""``sudo_rm_rf.dnn.models.causal_improved_sudormrf_v3`` -> H100-native implementation."""
from sudo_rm_rf_b200.causal_improved_sudormrf_v3 import (CausalSuDORMRF, UConvBlock, ConvAct,  # noqa: F401
                                                         ScaledWSConv1d)
