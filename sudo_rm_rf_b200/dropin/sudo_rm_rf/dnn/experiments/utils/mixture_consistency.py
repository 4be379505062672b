"""``sudo_rm_rf.dnn.experiments.utils.mixture_consistency`` -> H100-native implementation."""
from sudo_rm_rf_b200.mixture_consistency import apply  # noqa: F401
