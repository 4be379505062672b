"""The causal oracle's two readings of the masked taps (no device needed).

The reference zeroes the future taps of every causal convolution by multiplying them by zero; the native kernels and
the stream read only the surviving taps.  On finite input the two agree; a NaN or inf at t0 reaches outputs far before
t0 under "zeroed" (0 * NaN = NaN) and none before t0 - hop under "dropped"."""
import pytest
import torch

from oracle import sudormrf_oracle as O

CFG = O.Config(variant="causal", in_audio_channels=1, out_channels=64, in_channels=64, num_blocks=2,
               upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64, num_sources=2)
T = 4000


def mixture(dtype):
    return torch.randn(2, 1, T, generator=torch.Generator().manual_seed(0)).to(dtype)


def footprint(y):
    """Sample indices of mixture 0 where any source is non-finite."""
    return (~torch.isfinite(y[0])).any(0).nonzero().flatten()


def test_dropped_taps_agree_on_finite_input():
    sd = O.make_state_dict(CFG, seed=3)
    x = mixture(torch.float32)
    a = O.causal_forward(CFG, sd, x)
    b = O.causal_forward(CFG, sd, x, masked_taps="dropped")
    assert a.shape == b.shape
    assert float((a - b).abs().max() / a.abs().max()) < 1e-5
    with pytest.raises(ValueError):
        O.causal_forward(CFG, sd, x, masked_taps="masked")


@pytest.mark.parametrize("value", [float("nan"), float("inf"), -float("inf")], ids=["nan", "+inf", "-inf"])
@pytest.mark.parametrize("t0", [0, 2000, 3001])
def test_dropped_taps_footprint(value, t0):
    sd = O.make_state_dict(CFG, seed=3)
    x = mixture(torch.float64)
    clean = O.causal_forward(CFG, sd, x, dtype=torch.float64, masked_taps="dropped")
    x[0, 0, t0] = value
    zeroed = O.causal_forward(CFG, sd, x, dtype=torch.float64)
    dropped = O.causal_forward(CFG, sd, x, dtype=torch.float64, masked_taps="dropped")
    hop = CFG.hop
    fd, fz = footprint(dropped), footprint(zeroed)
    # one contiguous range from one hop before the first frame that reads t0 (the decoder's overlap): t0 - hop when
    # t0 is a multiple of the hop
    first_frame = -(-t0 // hop)
    assert fd.numel() > 0 and int(fd[0]) == max(hop * first_frame - hop, 0)
    assert int(fd[-1]) - int(fd[0]) + 1 == fd.numel()
    # the zero-weighted future taps of the reference reach further back
    if t0 > hop:
        assert int(fz[0]) < int(fd[0]) and set(fd.tolist()) <= set(fz.tolist())
    # outside the footprint and in the other mixture nothing changes
    keep = torch.ones(T, dtype=torch.bool)
    keep[fd] = False
    assert torch.equal(dropped[0][:, keep], clean[0][:, keep])
    assert torch.equal(dropped[1], clean[1])
    assert torch.isfinite(zeroed[1]).all()
