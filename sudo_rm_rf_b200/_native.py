"""ctypes binding of the C-ABI in ``include/sudormrf_b200.h``.

The shared library is built in-tree (``sudo_rm_rf_b200/libsudormrf_b200.so``)
by ``build()`` / ``__graft_entry__.build()``.  There is NO fallback: if the
library is missing or a call fails this module raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SDR_B200_LIB") or os.path.join(_HERE, "libsudormrf_b200.so")   # env override: A/B-testing kernel builds
CSRC = os.path.join(_HERE, "csrc")

ABI_VERSION = 2


class SdrConfig(C.Structure):
    """``sdr_config`` (include/sudormrf_b200.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "variant", "in_audio_channels", "out_channels", "in_channels", "num_blocks",
        "upsampling_depth", "enc_kernel_size", "enc_num_basis", "num_sources", "group_size")]

    def key(self):
        return tuple(getattr(self, n) for n, _ in self._fields_)


class SdrNormIn(C.Structure):
    """``sdr_norm_in``."""
    _fields_ = [("stats", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("prelu", C.c_void_p), ("count", C.c_double), ("prelu_per_channel", C.c_int32)]


class NativeError(RuntimeError):
    pass


_lib = None
_lock = threading.Lock()

_SIGNATURES = {
    "sdr_abi_version": (C.c_int, []),
    "sdr_error_string": (C.c_char_p, [C.c_int]),
    "sdr_num_params": (C.c_int, [C.POINTER(SdrConfig)]),
    "sdr_param_numel": (C.c_int64, [C.POINTER(SdrConfig), C.c_int]),
    "sdr_param_name": (C.c_int64, [C.POINTER(SdrConfig), C.c_int, C.c_char_p, C.c_size_t]),
    "sdr_padded_length": (C.c_int64, [C.POINTER(SdrConfig), C.c_int64]),
    "sdr_packed_weight_bytes": (C.c_size_t, [C.POINTER(SdrConfig)]),
    "sdr_pack_weights": (C.c_int, [C.POINTER(SdrConfig), C.POINTER(C.c_void_p), C.c_int,
                                   C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_workspace_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_forward": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                              C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_forward_launch_count": (C.c_int, [C.POINTER(SdrConfig)]),
    "sdr_forward_launch_count_at": (C.c_int, [C.POINTER(SdrConfig), C.c_int64]),
    "sdr_forward_launch_count_for": (C.c_int, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_host_staging_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_forward_host": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_size_t,
                                   C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_stream_granule": (C.c_int64, [C.POINTER(SdrConfig)]),
    "sdr_stream_state_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int]),
    "sdr_stream_workspace_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_stream_launch_count": (C.c_int, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_stream_reset": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "sdr_stream_reset_masked": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_stream_step": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_stream_flush": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "sdr_causal_stream_stage": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                          C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_void_p]),
    "sdr_mixture_consistency": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                          C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_mixture_consistency_backward_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.c_int]),
    "sdr_mixture_consistency_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_int, C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_encoder": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                              C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_encoder_mma_packed_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "sdr_encoder_mma_pack": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_encoder_mma": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                  C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_encoder_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_encoder_mma_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_pointwise": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_pointwise_mma_packed_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_pointwise_mma_pack": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_pointwise_mma": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_depthwise": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                C.c_void_p]),
    "sdr_pyramid_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "sdr_depthwise_pyramid": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p,
                                        C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_merge_pyramid": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_depthwise_pyramid_fused": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.POINTER(C.c_void_p),
                                              C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_void_p]),
    "sdr_causal_pyramid": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                     C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_merge": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(SdrNormIn), C.c_int, C.c_void_p,
                            C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_tac": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_int,
                          C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_tac_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                C.c_void_p]),
    "sdr_pointwise_preadd": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p]),
    "sdr_residual_norm": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p,
                                    C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_softmax_gate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_overlap_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_int64, C.c_void_p]),
    "sdr_utterance_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]),
    "sdr_separate_workspace_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_separate": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                               C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_separate_ragged": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_pairwise_neg_sdr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int,
                                       C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_pairwise_neg_sdr_train_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64]),
    "sdr_pairwise_neg_sdr_coef_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_pairwise_neg_sdr_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                             C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_pairwise_neg_sdr_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                C.c_int, C.c_int64, C.c_void_p]),
    "sdr_pit_sisdr_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_pit_sisdr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                C.c_int, C.c_int64, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]),
    "sdr_stabilized_sisdr_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "sdr_stabilized_sisdr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int64, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]),
    "sdr_snr_zero_refs_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64]),
    "sdr_snr_zero_refs_coef_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_snr_zero_refs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                    C.c_int64, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "sdr_snr_zero_refs_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                             C.c_int, C.c_int64, C.c_int64, C.c_void_p]),
    "sdr_bss_eval_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.c_int]),
    "sdr_bss_eval": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                               C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_bss_eval_mixture": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64,
                                       C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_stoi_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.c_int]),
    "sdr_stoi": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                           C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_resample_poly_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_resample_poly": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                    C.c_size_t, C.c_void_p]),
    "sdr_resample_stream_state_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int64,
                                                     C.c_int64]),
    "sdr_resample_stream_reset": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int,
                                            C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    "sdr_resample_stream_step": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_void_p]),
    "sdr_resample_stream_flush": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                            C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                            C.c_void_p]),
    "sdr_window_count": (C.c_int64, [C.c_int64, C.c_int64, C.c_int64]),
    "sdr_window_carry_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int64]),
    "sdr_window_merge_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "sdr_window_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64,
                                    C.c_int64, C.c_int, C.c_void_p]),
    "sdr_window_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                   C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_window_ragged_carry_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64]),
    "sdr_window_ragged_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_window_gather_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64,
                                           C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_window_merge_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                          C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "sdr_window_stream_state_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64]),
    "sdr_window_stream_reset": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_void_p,
                                          C.c_int, C.c_void_p]),
    "sdr_window_stream_reset_masked": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                                 C.c_void_p, C.c_void_p]),
    "sdr_window_stream_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64,
                                           C.c_int64, C.c_int64, C.c_void_p]),
    "sdr_window_stream_merge_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.c_int64]),
    "sdr_window_stream_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64,
                                          C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "sdr_window_stream_flush_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_window_stream_flush": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                          C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "sdr_window_stream_launch_count": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64]),
    "sdr_train_saved_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_backward_workspace_bytes": (C.c_size_t, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_forward_train": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                    C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_backward": (C.c_int, [C.POINTER(SdrConfig), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_int, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdr_backward_launch_count": (C.c_int, [C.POINTER(SdrConfig), C.c_int, C.c_int64]),
    "sdr_pointwise_wgrad_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "sdr_pointwise_wgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sdr_norm_act_backward_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_norm_act_backward": (C.c_int, [C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p]),
    "sdr_depthwise_backward_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "sdr_depthwise_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(SdrNormIn), C.c_void_p, C.c_void_p,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_void_p]),
    "sdr_mask_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_void_p]),
    "sdr_overlap_add_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64,
                                           C.c_void_p]),
    "sdr_encoder_wgrad_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "sdr_encoder_wgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int64, C.c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources for sm_90a into the in-tree shared library."""
    proc = subprocess.run(["make", "-C", CSRC, "-j8"], capture_output=True, text=True)
    if proc.returncode != 0:
        raise NativeError("building libsudormrf_b200.so failed:\n" + proc.stdout + proc.stderr)
    if verbose:
        print(proc.stdout)
    return LIB_PATH


def lib():
    """The loaded library (loads on first use; raises if it was never built)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise NativeError(
                    f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                    "g.build()'` (there is no CPU / eager fallback).")
            handle = C.CDLL(LIB_PATH)
            for name, (res, args) in _SIGNATURES.items():
                fn = getattr(handle, name)
                fn.restype, fn.argtypes = res, args
            if handle.sdr_abi_version() != ABI_VERSION:
                raise NativeError("libsudormrf_b200.so ABI version mismatch; rebuild")
            _lib = handle
    return _lib


def stream(device) -> C.c_void_p:
    """The current CUDA stream of `device`, as the ``cudaStream_t`` argument every entry takes.  Every handle the
    package passes to the library is spelled this way, inside the function that makes the call, so that
    ``tests/test_gpu_concurrency.py`` finds every entry that enqueues work."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t) -> C.c_void_p:
    """The address of tensor ``t`` as a pointer argument; NULL for None."""
    return C.c_void_p(t.data_ptr() if t is not None else None)


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib().sdr_error_string(code).decode()
        raise NativeError(f"{what or 'native call'} failed: {msg} (code {code})")
