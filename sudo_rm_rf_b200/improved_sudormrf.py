"""H100-native mirror of ``sudo_rm_rf/dnn/models/improved_sudormrf.py``.

Same public surface as the reference module (class names, constructor
arguments and defaults, public attributes, sub-module / parameter names and
therefore ``state_dict()`` keys, ``forward(input_wav)`` signature), so the
reference's notebooks, ``dnn/experiments`` runners, ``load_state_dict`` of
published checkpoints and ``torch.load`` of whole-module pickles keep working.
The arithmetic of ``SuDORMRF.forward`` (improved_sudormrf.py:283-301) is done
by hand-written sm_90a kernels behind ``include/sudormrf_b200.h``; the
sub-modules below only own the parameters.  Inference only: there is no
autograd through the native path and no CPU path.
"""
import math

import torch
import torch.nn as nn

from . import _engine


def _not_standalone(self, *_, **__):
    raise NotImplementedError(
        f"{type(self).__name__} is a parameter container of the H100 forward path; "
        "call the parent SuDORMRF / GroupCommSudoRmRf module instead.")


class _LayerNorm(nn.Module):
    """Holds gamma/beta of a global layer norm (reference :13-27)."""

    def __init__(self, channel_size):
        super().__init__()
        self.channel_size = channel_size
        self.gamma = nn.Parameter(torch.ones(channel_size))
        self.beta = nn.Parameter(torch.zeros(channel_size))

    forward = _not_standalone


class GlobLN(_LayerNorm):
    """Global layer norm over (channel, time) (reference :30-47).  Fused into the
    consumers' operand loads by the native kernels (deferred normalisation)."""


class ConvNormAct(nn.Module):
    """conv -> GlobLN -> PReLU parameters (reference :50-73)."""

    def __init__(self, nIn, nOut, kSize, stride=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(nIn, nOut, kSize, stride=stride, padding=(kSize - 1) // 2,
                              bias=True, groups=groups)
        self.norm = GlobLN(nOut)
        self.act = nn.PReLU()

    forward = _not_standalone


class NormAct(nn.Module):
    """GlobLN -> PReLU parameters (reference :99-114)."""

    def __init__(self, nOut):
        super().__init__()
        self.norm = GlobLN(nOut)
        self.act = nn.PReLU()

    forward = _not_standalone


class DilatedConvNorm(nn.Module):
    """depthwise conv -> GlobLN parameters (reference :138-159)."""

    def __init__(self, nIn, nOut, kSize, stride=1, d=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(nIn, nOut, kSize, stride=stride, dilation=d,
                              padding=((kSize - 1) // 2) * d, groups=groups)
        self.norm = GlobLN(nOut)

    forward = _not_standalone


class UConvBlock(nn.Module):
    """Parameters of one U-ConvBlock (reference :162-220): ``proj_1x1``,
    ``spp_dw[0..depth)``, ``final_norm``, ``res_conv``."""

    def __init__(self, out_channels=128, in_channels=512, upsampling_depth=4):
        super().__init__()
        self.proj_1x1 = ConvNormAct(out_channels, in_channels, 1, stride=1, groups=1)
        self.depth = upsampling_depth
        self.spp_dw = nn.ModuleList(
            DilatedConvNorm(in_channels, in_channels, kSize=5, stride=1 if i == 0 else 2,
                            groups=in_channels, d=1)
            for i in range(upsampling_depth))
        if upsampling_depth > 1:
            self.upsampler = nn.Upsample(scale_factor=2)
        self.final_norm = NormAct(in_channels)
        self.res_conv = nn.Conv1d(in_channels, out_channels, 1)

    forward = _not_standalone


def _xavier_uniform_(w):
    # same distribution as torch.nn.init.xavier_uniform on a Conv weight (reference :252,280)
    fan_in = w.shape[1] * w[0][0].numel()
    fan_out = w.shape[0] * w[0][0].numel()
    bound = math.sqrt(6.0 / (fan_in + fan_out))
    with torch.no_grad():
        w.uniform_(-bound, bound)


class SuDORMRF(_engine.NativeModuleMixin, nn.Module):
    """Improved SuDoRM-RF separator (reference :223-318) on the H100 native path."""

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
        self.n_least_samples_req = self.enc_kernel_size // 2 * 2 ** self.upsampling_depth

        hop = enc_kernel_size // 2
        self.encoder = nn.Conv1d(1, enc_num_basis, enc_kernel_size, stride=hop, padding=hop,
                                 bias=False)
        _xavier_uniform_(self.encoder.weight)
        self.ln = GlobLN(enc_num_basis)
        self.bottleneck = nn.Conv1d(enc_num_basis, out_channels, 1)
        self.sm = nn.Sequential(*[
            UConvBlock(out_channels=out_channels, in_channels=in_channels,
                       upsampling_depth=upsampling_depth) for _ in range(num_blocks)])
        self.mask_net = nn.Sequential(nn.PReLU(),
                                      nn.Conv1d(out_channels, num_sources * enc_num_basis, 1))
        self.decoder = nn.ConvTranspose1d(enc_num_basis * num_sources, num_sources,
                                          kernel_size=enc_kernel_size, stride=hop, padding=hop,
                                          output_padding=hop - 1, groups=1, bias=False)
        _xavier_uniform_(self.decoder.weight)
        self.mask_nl_class = nn.ReLU()

    def forward(self, input_wav):
        """[B, 1, T] mixture -> [B, num_sources, T] estimates (fp32, same device)."""
        return _engine.forward(self, input_wav, mixture_consistency=False)

    def separate(self, input_wav, mixture_consistency=False, normalize=False):
        """forward() with the uniform mixture-consistency projection
        (mixture_consistency.py:14-36) fused into the decoder epilogue.

        ``normalize=True`` runs the whole README recipe (reference README.md:100-114) on the
        device: ``input_wav`` is the raw mixture ``[B, T]`` or ``[B, 1, T]``; it is normalised per
        utterance (mean, unbiased std), separated, and the estimates are rescaled with the
        mixture's std and mean (then, optionally, projected onto the normalised mixture)."""
        if normalize:
            return _engine.separate(self, input_wav, mixture_consistency=mixture_consistency)
        return _engine.forward(self, input_wav, mixture_consistency=mixture_consistency)

    def forward_host(self, host_wav, host_out=None, mixture_consistency=False):
        """End-to-end call on pinned HOST tensors (H2D, forward, D2H on the current stream)."""
        return _engine.forward_host(self, host_wav, host_out, mixture_consistency)

    def pad_to_appropriate_length(self, x):
        """Reference :303-314.  The native encoder pads implicitly; this helper is
        kept for callers that use it directly (device-side, no host round trip)."""
        T = x.shape[-1]
        q = self.n_least_samples_req
        Tp = q if T < q else ((T + q - 1) // q) * q
        out = torch.zeros(list(x.shape[:-1]) + [Tp], dtype=torch.float32, device=x.device)
        out[..., :T] = x
        return out

    @staticmethod
    def remove_trailing_zeros(padded_x, initial_x):
        return padded_x[..., :initial_x.shape[-1]]
