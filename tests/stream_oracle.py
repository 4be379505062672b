"""CPU restatement of chunk-by-chunk streaming of the causal model, carrying exactly the state the native stream keeps.

Per slot:
  - waveform context: the last 2*hop input samples (encoder frame f reads samples hop*f - 2*hop .. hop*f);
  - level histories: per block and level, the last 10 values of the level's input (after its PReLU), at its rate;
  - decoder carry: the hop + 1 partial overlap-add sums that the next chunk's frames still add to;
  - whether the slot has stepped since its reset (the first step's first hop samples precede the stream: zeros).
Every function is the oracle's (oracle/sudormrf_oracle.py) formula for the same layer, applied to history + chunk
without padding, so agreement with ``causal_forward`` on the whole clip pins the streaming contract independently of
the GPU."""
import torch
import torch.nn.functional as F

from oracle import sudormrf_oracle as O


def granule(cfg: O.Config) -> int:
    return cfg.hop * max(4, 2 ** (cfg.upsampling_depth - 1))


class CausalStreamOracle:
    def __init__(self, cfg: O.Config, sd, batch: int, dtype=torch.float64):
        self.cfg, self.dtype = cfg, dtype
        self.sd = {k: v.to(dtype) for k, v in sd.items()}
        hop, A, D = cfg.hop, cfg.in_audio_channels, cfg.upsampling_depth
        SA = cfg.num_sources * A
        self.ctx = torch.zeros(batch, A, 2 * hop, dtype=dtype)
        self.hist = [[torch.zeros(batch, cfg.in_channels, 10, dtype=dtype) for _ in range(D)]
                     for _ in range(cfg.num_blocks)]
        self.carry = torch.zeros(batch, SA, hop + 1, dtype=dtype)
        self.started = False

    def set_weights(self, sd):
        """New weights from the next step on (the state is kept), as a stream picks up a model's changed weights."""
        self.sd = {k: v.to(self.dtype) for k, v in sd.items()}

    def _block(self, x, i):
        sd, p, D = self.sd, f"sm.{i}.", self.cfg.upsampling_depth
        Ci = sd[p + "proj_1x1.conv.weight"].shape[0]
        o = O.prelu1(F.conv1d(x, sd[p + "proj_1x1.conv.weight"], sd[p + "proj_1x1.conv.bias"]),
                     sd[p + "proj_1x1.act.weight"])
        outs = []
        for d in range(D):
            inp = torch.cat([self.hist[i][d], o], -1)
            self.hist[i][d] = inp[..., -10:].clone()
            w = O.causal_weight(sd[p + f"spp_dw.{d}.conv.weight"])[..., :11]      # the taps the causal mask keeps
            o = F.conv1d(inp, w, sd[p + f"spp_dw.{d}.conv.bias"], stride=1 if d == 0 else 2, groups=Ci)
            o = O.prelu1(o, sd[p + f"spp_dw.{d}.act.weight"])
            outs.append(o)
        for _ in range(D - 1):
            up = F.interpolate(outs.pop(-1), scale_factor=2, mode="nearest")
            outs[-1] = outs[-1] + up
        y = F.conv1d(outs[-1], sd[p + "res_conv.weight"], sd[p + "res_conv.bias"])
        return y * sd[p + "skipinit_gain"] + x

    def step(self, chunk):
        """chunk [B, A, C] -> [B, S*A, C]: the model's output samples c*C - hop .. (c+1)*C - hop - 1."""
        cfg, sd = self.cfg, self.sd
        k, hop = cfg.enc_kernel_size, cfg.hop
        C = chunk.shape[-1]
        assert C % granule(cfg) == 0
        ext = torch.cat([self.ctx, chunk.to(self.dtype)], -1)
        self.ctx = ext[..., -2 * hop:].clone()
        enc_w = O.causal_weight(sd["encoder.weight"])[..., :k]
        x = F.conv1d(ext, enc_w, None, stride=hop)                            # C / hop frames
        x = F.conv1d(x, sd["bottleneck.weight"], sd["bottleneck.bias"])
        for i in range(cfg.num_blocks):
            x = self._block(x, i)
        x = O.prelu1(x, sd["mask_net.0.weight"])
        x = F.conv1d(x, sd["mask_net.1.weight"], sd["mask_net.1.bias"])
        x = O.prelu1(x, sd["mask_nl_class.weight"])
        full = F.conv_transpose1d(x, sd["decoder.weight"], None, stride=hop)  # C + hop + 1 samples from c*C - hop on
        full[..., :hop + 1] += self.carry
        self.carry = full[..., C:].clone()
        if not self.started:                   # samples before the start of the stream: the reference crops them
            full[..., :hop] = 0
            self.started = True
        return full[..., :C]

    def flush(self):
        return self.carry[..., :self.cfg.hop].clone()


def causal_stream_forward(cfg: O.Config, sd, wav, chunk: int, dtype=torch.float64):
    """wav [B, A, n*chunk] streamed chunk by chunk -> (concatenated steps [B, S*A, n*chunk], flush tail)."""
    assert wav.shape[-1] % chunk == 0
    s = CausalStreamOracle(cfg, sd, wav.shape[0], dtype)
    outs = [s.step(wav[..., c:c + chunk]) for c in range(0, wav.shape[-1], chunk)]
    return torch.cat(outs, -1), s.flush()
