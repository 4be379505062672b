"""sudo_rm_rf_b200: H100-native (sm_90a) forward inference path of SuDoRM-RF.

Mirrors ``sudo_rm_rf.dnn.models.improved_sudormrf`` /
``sudo_rm_rf.dnn.models.groupcomm_sudormrf_v2`` /
``sudo_rm_rf.dnn.models.causal_improved_sudormrf_v3`` /
``sudo_rm_rf.dnn.models.sudormrf`` (the original model; its class is also called ``SuDORMRF``, so it is
exported here as ``OriginalSuDORMRF``) /
``sudo_rm_rf.dnn.experiments.utils.mixture_consistency`` of etzinis/sudo_rm_rf, and the FUSS training loss
``PermInvariantSNRwithZeroRefs`` of ``sudo_rm_rf.dnn.losses.snr`` (module ``snr``), and the BSS-eval
source criteria of the evaluation scripts (``bss_eval_sources``, mir_eval's definition) and their STOI (``stoi``,
pystoi's definition; module ``stoi_metric``), and scipy's ``resample_poly`` (module ``resample``).
"""
from . import improved_sudormrf, groupcomm_sudormrf_v2, causal_improved_sudormrf_v3, sudormrf, mixture_consistency   # noqa: F401
from . import snr                                                             # noqa: F401
from .bss_eval import bss_eval_sources                                         # noqa: F401
from .stoi_metric import stoi                                                 # noqa: F401
from .resample import resample_poly                                           # noqa: F401
from .improved_sudormrf import SuDORMRF                                       # noqa: F401
from .groupcomm_sudormrf_v2 import GroupCommSudoRmRf                          # noqa: F401
from .causal_improved_sudormrf_v3 import CausalSuDORMRF                       # noqa: F401
from .sudormrf import SuDORMRF as OriginalSuDORMRF                            # noqa: F401
from ._engine import refresh_weights                                          # noqa: F401
from .window_stream import WindowedStream                                     # noqa: F401
from .resample_stream import ResampleStream, ResampledStream                   # noqa: F401

__all__ = ["SuDORMRF", "GroupCommSudoRmRf", "CausalSuDORMRF", "OriginalSuDORMRF", "improved_sudormrf",
           "groupcomm_sudormrf_v2", "causal_improved_sudormrf_v3", "sudormrf", "mixture_consistency", "snr",
           "bss_eval_sources", "stoi", "resample_poly", "refresh_weights", "WindowedStream",
           "ResampleStream", "ResampledStream"]
