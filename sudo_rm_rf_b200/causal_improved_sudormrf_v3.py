"""H100-native mirror of ``sudo_rm_rf/dnn/models/causal_improved_sudormrf_v3.py``.

Same public surface as the reference module (class names, constructor arguments and defaults, public
attributes, sub-module / parameter names and therefore ``state_dict()`` keys, ``forward(input_wav)``), so
``run_fuss_separation.py:134-170``-style model selection, ``load_state_dict`` of checkpoints and whole-module
pickles keep working.  The arithmetic of ``CausalSuDORMRF.forward`` (reference :191-211) is done by the sm_90a
kernels behind ``include/sudormrf_b200.h`` (variant 2): the wgmma GEMM for every 1x1 convolution, the encoder
and the decoder, and one pass per block for the whole causal depthwise pyramid (``csrc/causal.cu``).  The
sub-modules below only own the parameters.  Inference only; no CPU path.
"""
import torch
import torch.nn as nn

from . import _engine
from .improved_sudormrf import _not_standalone, _xavier_uniform_


class ScaledWSConv1d(nn.Conv1d):
    """Conv1d whose last ``kernel_size // 2`` taps are masked out (reference :12-32); the native kernels simply
    never read those taps.  ``causal_mask`` / ``get_weight`` are kept for callers that inspect them."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, gain=False, eps=1e-8):
        nn.Conv1d.__init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        self.causal_mask = torch.ones_like(self.weight)
        if kernel_size >= 3:
            self.causal_mask[..., -(kernel_size // 2):] = 0.

    def get_weight(self):
        return self.weight * self.causal_mask.to(self.weight.device)

    forward = _not_standalone


class ConvAct(nn.Module):
    """masked conv -> PReLU parameters (reference :34-54)."""

    def __init__(self, nIn, nOut, kSize, stride=1, groups=1):
        super().__init__()
        self.conv = ScaledWSConv1d(nIn, nOut, kSize, stride=stride, padding=((kSize - 1) // 2), groups=groups)
        self.act = nn.PReLU()

    forward = _not_standalone


class UConvBlock(nn.Module):
    """Parameters of one causal U-ConvBlock (reference :57-118): ``skipinit_gain``, ``proj_1x1``,
    ``spp_dw[0..depth)`` (21-tap depthwise, causally masked), ``res_conv``."""

    def __init__(self, out_channels=128, in_channels=512, upsampling_depth=4, alpha=1., beta=1.):
        super().__init__()
        self.beta, self.alpha = beta, alpha
        self.skipinit_gain = nn.Parameter(torch.zeros(()))
        self.proj_1x1 = ConvAct(out_channels, in_channels, 1, stride=1, groups=1)
        self.depth = upsampling_depth
        self.spp_dw = nn.ModuleList(
            ConvAct(in_channels, in_channels, kSize=21, stride=1 if i == 0 else 2, groups=in_channels)
            for i in range(upsampling_depth))
        if upsampling_depth > 1:
            self.upsampler = nn.Upsample(scale_factor=2)
        self.res_conv = ScaledWSConv1d(in_channels, out_channels, 1)

    forward = _not_standalone


class CausalSuDORMRF(_engine.NativeModuleMixin, nn.Module):
    """Causal SuDoRM-RF separator (reference :120-231) on the H100 native path."""

    _b200_variant = 2

    def __init__(self, in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=4,
                 enc_kernel_size=21, enc_num_basis=512, num_sources=2):
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
            'Be mindful to signal processing and choose an odd number for '
            'your filter size, since the hop size is going to be an even '
            'number.')
        self.n_least_samples_req = self.enc_kernel_size // 2 * 2 ** self.upsampling_depth

        hop = enc_kernel_size // 2
        self.encoder = ScaledWSConv1d(in_audio_channels, enc_num_basis, enc_kernel_size * 2 - 1, stride=hop,
                                      padding=(enc_kernel_size * 2 - 1) // 2, bias=False)
        _xavier_uniform_(self.encoder.weight)
        self.bottleneck = ScaledWSConv1d(enc_num_basis, out_channels, 1)
        # the reference keeps expected_var at 1.0 (its update is commented out, :173), so alpha = beta = 1
        self.sm = nn.Sequential(*[
            UConvBlock(out_channels=out_channels, in_channels=in_channels, upsampling_depth=upsampling_depth,
                       alpha=1., beta=1.) for _ in range(num_blocks)])
        self.mask_net = nn.Sequential(
            nn.PReLU(), ScaledWSConv1d(out_channels, num_sources * enc_num_basis * in_audio_channels, 1))
        self.decoder = nn.ConvTranspose1d(enc_num_basis * num_sources * in_audio_channels,
                                          num_sources * in_audio_channels, kernel_size=enc_kernel_size, stride=hop,
                                          padding=hop, output_padding=hop - 1, groups=1, bias=False)
        _xavier_uniform_(self.decoder.weight)
        self.mask_nl_class = nn.PReLU()

    def _b200_param_transform(self, name, tensor):
        """skipinit_gain * alpha and proj_1x1 weight / beta (reference :105,118) are folded at pack time."""
        if name.endswith("skipinit_gain") or name.endswith("proj_1x1.conv.weight"):
            blk = self.sm[int(name.split(".")[1])]
            if name.endswith("skipinit_gain"):
                return tensor * float(blk.alpha) if float(blk.alpha) != 1.0 else tensor
            return tensor / float(blk.beta) if float(blk.beta) != 1.0 else tensor
        return tensor

    def forward(self, input_wav):
        """[B, in_audio_channels, T] mixture -> [B, num_sources * in_audio_channels, T] estimates (fp32)."""
        return _engine.forward(self, input_wav, mixture_consistency=False)

    def separate(self, input_wav, mixture_consistency=False, normalize=False):
        """forward() with the uniform mixture-consistency projection fused into the decoder epilogue (mono models);
        ``normalize=True`` runs the README recipe (README.md:100-114) on the device, see ``SuDORMRF.separate``."""
        if normalize:
            return _engine.separate(self, input_wav, mixture_consistency=mixture_consistency)
        return _engine.forward(self, input_wav, mixture_consistency=mixture_consistency)

    def forward_host(self, host_wav, host_out=None, mixture_consistency=False):
        """End-to-end call on pinned HOST tensors (H2D, forward, D2H on the current stream)."""
        return _engine.forward_host(self, host_wav, host_out, mixture_consistency)

    def pad_to_appropriate_length(self, x):
        """Reference :213-224 (device-side; the native encoder pads implicitly)."""
        T = x.shape[-1]
        q = self.n_least_samples_req
        Tp = q if T < q else ((T + q - 1) // q) * q
        out = torch.zeros(list(x.shape[:-1]) + [Tp], dtype=torch.float32, device=x.device)
        out[..., :T] = x
        return out

    @staticmethod
    def remove_trailing_zeros(padded_x, initial_x):
        return padded_x[..., :initial_x.shape[-1]]
