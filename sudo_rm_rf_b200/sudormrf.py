"""H100-native mirror of ``sudo_rm_rf/dnn/models/sudormrf.py`` (the ORIGINAL SuDoRM-RF).

Same public surface as the reference module (class names, constructor arguments and defaults, public
attributes, sub-module / parameter names and therefore ``state_dict()`` keys, ``forward(input_wav)``), so
``run_fuss_separation.py:134-170``-style model selection, ``load_state_dict`` of checkpoints and whole-module
pickles keep working.  The arithmetic of ``SuDORMRF.forward`` (reference :266-292) is done by the sm_90a kernels
behind ``include/sudormrf_b200.h`` (variant 3): ``GroupNorm(1, C, eps=1e-8)`` is the same normalisation as the
improved model's GlobLN and is deferred to the consumers' operand loads in the same way, the per-channel PReLUs
ride on those loads, the ``(N + 1) x 1`` mask ``Conv2d`` runs as one more GEMM on the wgmma kernel (a Toeplitz
matrix expanded at pack time), the grouped decoder as block-diagonal weights of the frames GEMM
(``csrc/original.cu``).  The sub-modules below only own the parameters.  Inference only; no CPU path.
"""
import math

import torch
import torch.nn as nn

from . import _engine
from ._surface import NativeSeparator, _not_standalone


class ConvNormAct(nn.Module):
    """conv -> GroupNorm(1, C) -> PReLU(C) parameters (reference :13-38)."""

    def __init__(self, nIn, nOut, kSize, stride=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(nIn, nOut, kSize, stride=stride, padding=int((kSize - 1) / 2), bias=True, groups=groups)
        self.norm = nn.GroupNorm(1, nOut, eps=1e-08)
        self.act = nn.PReLU(nOut)

    forward = _not_standalone


class ConvNorm(nn.Module):
    """conv -> GroupNorm(1, C) parameters (reference :41-61)."""

    def __init__(self, nIn, nOut, kSize, stride=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(nIn, nOut, kSize, stride=stride, padding=int((kSize - 1) / 2), bias=True, groups=groups)
        self.norm = nn.GroupNorm(1, nOut, eps=1e-08)

    forward = _not_standalone


class NormAct(nn.Module):
    """GroupNorm(1, C) -> PReLU(C) parameters (reference :64-77)."""

    def __init__(self, nOut):
        super().__init__()
        self.norm = nn.GroupNorm(1, nOut, eps=1e-08)
        self.act = nn.PReLU(nOut)

    forward = _not_standalone


class DilatedConv(nn.Module):
    """Reference :80-98 (defined there, not used by the model)."""

    def __init__(self, nIn, nOut, kSize, stride=1, d=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(nIn, nOut, kSize, stride=stride, dilation=d, padding=((kSize - 1) // 2) * d, groups=groups)

    forward = _not_standalone


class DilatedConvNorm(nn.Module):
    """depthwise conv -> GroupNorm(1, C) parameters (reference :101-122)."""

    def __init__(self, nIn, nOut, kSize, stride=1, d=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(nIn, nOut, kSize, stride=stride, dilation=d, padding=((kSize - 1) // 2) * d, groups=groups)
        self.norm = nn.GroupNorm(1, nOut, eps=1e-08)

    forward = _not_standalone


class UBlock(nn.Module):
    """Parameters of one U-block (reference :125-186): ``proj_1x1``, ``spp_dw[0..depth)``, ``conv_1x1_exp``,
    ``final_norm``, ``module_act`` (registered in this order: it is the ``state_dict`` order)."""

    def __init__(self, out_channels=128, in_channels=512, upsampling_depth=4):
        super().__init__()
        self.proj_1x1 = ConvNormAct(out_channels, in_channels, 1, stride=1, groups=1)
        self.depth = upsampling_depth
        self.spp_dw = nn.ModuleList()
        self.spp_dw.append(DilatedConvNorm(in_channels, in_channels, kSize=5, stride=1, groups=in_channels, d=1))
        for i in range(1, upsampling_depth):
            self.spp_dw.append(DilatedConvNorm(in_channels, in_channels, kSize=5, stride=2, groups=in_channels, d=1))
        if upsampling_depth > 1:
            self.upsampler = nn.Upsample(scale_factor=2)
        self.conv_1x1_exp = ConvNorm(in_channels, out_channels, 1, 1, groups=1)
        self.final_norm = NormAct(in_channels)
        self.module_act = NormAct(out_channels)

    forward = _not_standalone


class SuDORMRF(NativeSeparator, nn.Module):
    """The original SuDoRM-RF separator (reference :185-297) on the H100 native path."""

    _b200_variant = 3

    def __init__(self, out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=4,
                 enc_kernel_size=21, enc_num_basis=512, num_sources=2):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.num_blocks = num_blocks
        self.upsampling_depth = upsampling_depth
        self.enc_kernel_size = enc_kernel_size
        self.enc_num_basis = enc_num_basis
        self.num_sources = num_sources
        hop = enc_kernel_size // 2
        # appropriate padding for arbitrary lengths (reference :206-209)
        self.lcm = abs(hop * 2 ** upsampling_depth) // math.gcd(hop, 2 ** upsampling_depth)

        self.encoder = nn.Sequential(
            nn.Conv1d(in_channels=1, out_channels=enc_num_basis, kernel_size=enc_kernel_size, stride=hop, padding=hop),
            nn.ReLU())
        self.ln = nn.GroupNorm(1, enc_num_basis, eps=1e-08)
        self.l1 = nn.Conv1d(in_channels=enc_num_basis, out_channels=out_channels, kernel_size=1)
        self.sm = nn.Sequential(*[
            UBlock(out_channels=out_channels, in_channels=in_channels, upsampling_depth=upsampling_depth)
            for _ in range(num_blocks)])
        if out_channels != enc_num_basis:
            self.reshape_before_masks = nn.Conv1d(in_channels=out_channels, out_channels=enc_num_basis, kernel_size=1)
        self.m = nn.Conv2d(in_channels=1, out_channels=num_sources, kernel_size=(enc_num_basis + 1, 1),
                           padding=(enc_num_basis - enc_num_basis // 2, 0))
        self.decoder = nn.ConvTranspose1d(in_channels=enc_num_basis * num_sources, out_channels=num_sources,
                                          output_padding=hop - 1, kernel_size=enc_kernel_size, stride=hop,
                                          padding=hop, groups=num_sources)
        self.ln_mask_in = nn.GroupNorm(1, enc_num_basis, eps=1e-08)      # registered by the reference (:253), never used

    def enable_training(self, enabled: bool = True):
        """Native training covers the improved SuDORMRF only."""
        raise NotImplementedError("SuDORMRF (original, sudormrf.py): native training (enable_training) covers the improved SuDORMRF "
                                  "only; the original model has no backward kernels")

    def forward(self, input_wav):
        """[B, 1, T] mixture -> [B, num_sources, T] estimates (fp32, same device)."""
        return _engine.forward(self, input_wav, mixture_consistency=False)

    def pad_to_appropriate_length(self, x):
        """Reference :283-293 (device-side; the native encoder pads implicitly)."""
        rem = int(x.shape[-1]) % self.lcm
        if rem:
            out = torch.zeros(list(x.shape[:-1]) + [x.shape[-1] + self.lcm - rem], dtype=torch.float32, device=x.device)
            out[..., :x.shape[-1]] = x
            return out
        return x
