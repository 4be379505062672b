"""H100-native mirror of ``sudo_rm_rf/dnn/models/groupcomm_sudormrf_v2.py``.

Same constructor, attributes, sub-module / parameter names (``state_dict()``
keys such as ``sm.3.TAC.TAC_input.0.weight`` / ``sm.3.UBlock.proj_1x1.conv.weight``)
and ``forward(input_wav)`` as the reference's ``GroupCommSudoRmRf``
(groupcomm_sudormrf_v2.py:231-339); the arithmetic runs in the sm_90a
kernels behind ``include/sudormrf_b200.h``.
"""
import torch.nn as nn

from . import _engine
from ._surface import NativeSeparator, _not_standalone
from .improved_sudormrf import (GlobLN, ConvNormAct, NormAct, DilatedConvNorm, UConvBlock,
                                _LayerNorm, _xavier_uniform_)

__all__ = ["GroupCommSudoRmRf", "TAC", "GC_UConvBlock", "GlobLN", "ConvNormAct", "NormAct",
           "DilatedConvNorm", "UConvBlock"]


class TAC(nn.Module):
    """Transform-average-concatenate parameters (reference :343-384)."""

    def __init__(self, input_size, hidden_size):
        super().__init__()
        self.TAC_input = nn.Sequential(nn.Linear(input_size, hidden_size), nn.PReLU())
        self.TAC_mean = nn.Sequential(nn.Linear(hidden_size, hidden_size), nn.PReLU())
        self.TAC_output = nn.Sequential(nn.Linear(hidden_size * 2, input_size), nn.PReLU())
        self.TAC_norm = GlobLN(input_size)

    forward = _not_standalone


class GC_UConvBlock(nn.Module):
    """TAC across groups + one U-ConvBlock shared by all groups (reference :388-418)."""

    def __init__(self, out_channels=128, in_channels=512, upsampling_depth=4, num_group=16):
        super().__init__()
        self.num_group = num_group
        self.TAC = TAC(out_channels // num_group, out_channels * 3 // num_group)
        self.UBlock = UConvBlock(out_channels // num_group, in_channels // num_group,
                                 upsampling_depth=upsampling_depth)

    forward = _not_standalone


class GroupCommSudoRmRf(NativeSeparator, nn.Module):
    """Group-communication SuDoRM-RF (reference :231-339) on the H100 native path."""

    def __init__(self, in_audio_channels=1, out_channels=256, in_channels=512, num_blocks=16,
                 upsampling_depth=5, enc_kernel_size=21, enc_num_basis=512, num_sources=2,
                 group_size=16):
        super().__init__()
        self.in_audio_channels = in_audio_channels
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.num_blocks = num_blocks
        self.upsampling_depth = upsampling_depth
        self.enc_kernel_size = enc_kernel_size
        self.enc_num_basis = enc_num_basis
        self.num_sources = num_sources
        assert self.enc_kernel_size % 2, (
            "enc_kernel_size must be odd: the hop size is enc_kernel_size // 2 and the "
            "padding arithmetic assumes an odd analysis filter.")
        self.n_least_samples_req = self.enc_kernel_size // 2 * 2 ** self.upsampling_depth

        hop = enc_kernel_size // 2
        self.encoder = nn.Conv1d(in_audio_channels, enc_num_basis, enc_kernel_size, stride=hop,
                                 padding=hop, bias=False)
        _xavier_uniform_(self.encoder.weight)
        self.ln = GlobLN(enc_num_basis)
        self.bottleneck = nn.Conv1d(enc_num_basis, out_channels, 1)
        self.sm = nn.Sequential(*[
            GC_UConvBlock(out_channels=out_channels, in_channels=in_channels,
                          upsampling_depth=upsampling_depth, num_group=group_size)
            for _ in range(num_blocks)])
        self.mask_net = nn.Sequential(
            nn.PReLU(), nn.Conv1d(out_channels, num_sources * enc_num_basis * in_audio_channels, 1))
        self.decoder = nn.ConvTranspose1d(enc_num_basis * num_sources * in_audio_channels,
                                          num_sources * in_audio_channels,
                                          kernel_size=enc_kernel_size, stride=hop, padding=hop,
                                          output_padding=hop - 1, groups=1, bias=False)
        _xavier_uniform_(self.decoder.weight)
        self.mask_nl_class = nn.ReLU()

    def enable_training(self, enabled: bool = True):
        """Native training covers the improved SuDORMRF only."""
        raise NotImplementedError("GroupCommSudoRmRf: native training (enable_training) covers the improved SuDORMRF "
                                  "only; the GroupComm model (TAC backward) has no backward kernels")

    def forward(self, input_wav):
        """[B, in_audio_channels, T] -> [B, num_sources*in_audio_channels, T]."""
        return _engine.forward(self, input_wav, mixture_consistency=False)

    # The reference applies the uniform mixture consistency to this model family (README.md:113-114): on by default.
    def separate(self, input_wav, mixture_consistency=True, normalize=False, sample_rate=None, model_rate=None):
        return super().separate(input_wav, mixture_consistency, normalize, sample_rate, model_rate)

    def separate_long(self, input_wav, window, hop=None, normalize=True, mixture_consistency=True,
                      max_windows=32, sample_rate=None, model_rate=None):
        return super().separate_long(input_wav, window, hop, normalize, mixture_consistency, max_windows,
                                     sample_rate, model_rate)

    def separate_long_corpus(self, wavs, window, hop=None, normalize=True, mixture_consistency=True, max_windows=32,
                             return_permutations=False):
        return super().separate_long_corpus(wavs, window, hop, normalize, mixture_consistency, max_windows,
                                            return_permutations)

    def stream_windows(self, batch_size, chunk_samples, window, hop=None, normalize=True,
                       mixture_consistency=True, sample_rate=None, model_rate=None):
        return super().stream_windows(batch_size, chunk_samples, window, hop, normalize, mixture_consistency,
                                      sample_rate, model_rate)
