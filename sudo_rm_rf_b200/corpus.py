"""Bucketed inference over a corpus of variable-length mixtures (SURVEY.md 8f row 4).

The reference evaluates a corpus one utterance at a time
(``sudo_rm_rf/utils/simple_whamr_evaluation.py:138-148``: normalise, ``model(x.unsqueeze(1))``,
mixture consistency).  Utterances cannot simply be stacked: the model pads every input to a
multiple of ``hop * 2**upsampling_depth`` samples (improved_sudormrf.py:303-314) and its global
layer norms see that padded length, so the estimate of an utterance depends on ITS padded length.
Utterances that share a padded length, however, are computed identically alone or side by side
(every reduction of the forward is per sample).  ``separate_corpus`` therefore buckets the corpus
by padded length, runs each bucket as zero-padded batches through ``sdr_separate_ragged``
(per-utterance statistics over the true length) and crops: every result equals what the
one-at-a-time loop of the reference produces for that utterance.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Sequence, Tuple

import torch

from . import _engine
from . import _native as N


def padded_length(T: int, quantum: int) -> int:
    """improved_sudormrf.py:303-310 with quantum = hop * 2**upsampling_depth (= n_least_samples_req)."""
    if T <= 0:
        raise ValueError("empty utterance")
    return quantum if T < quantum else -(-T // quantum) * quantum


def plan_buckets(lengths: Sequence[int], quantum, max_batch: int) -> List[Tuple[int, List[int]]]:
    """Groups utterance indices into batches that share a padded length.

    ``quantum``: ``hop * 2**upsampling_depth`` (the improved / GroupComm / causal rule above), or a callable
    ``T -> padded length`` (the model's own rule, e.g. the original model's lcm padding, sudormrf.py:283-293).
    Returns ``[(padded_length, [indices...]), ...]``: buckets in increasing padded length, inside a
    bucket the corpus order is kept and batches hold at most ``max_batch`` utterances.  Pure host
    logic (deterministic, no torch)."""
    if max_batch < 1:
        raise ValueError("max_batch must be >= 1")
    pad = quantum if callable(quantum) else (lambda T: padded_length(T, quantum))
    buckets = {}
    for i, T in enumerate(lengths):
        if int(T) <= 0:
            raise ValueError("empty utterance")
        buckets.setdefault(int(pad(int(T))), []).append(i)
    plan = []
    for Tp in sorted(buckets):
        idx = buckets[Tp]
        for k in range(0, len(idx), max_batch):
            plan.append((Tp, idx[k:k + max_batch]))
    return plan


def model_padding_rule(cfg):
    """``T -> padded length`` of the model behind ``cfg`` (the library's ``sdr_padded_length``: one rule for all variants)."""
    lib = N.lib()

    def pad(T: int) -> int:
        Tp = lib.sdr_padded_length(C.byref(cfg), int(T))
        if Tp <= 0:
            raise N.NativeError("sdr_padded_length failed (bad model configuration or empty utterance)")
        return int(Tp)
    return pad


def separate_corpus(model, wavs: Iterable[torch.Tensor], max_batch: int = 32,
                    mixture_consistency: bool = False, rescale: bool = True) -> List[torch.Tensor]:
    """Separates a corpus of mono mixtures of different lengths.

    ``wavs``: 1-D tensors (CPU or CUDA, any float dtype).  Returns, in corpus order, one ``[S, T_i]``
    fp32 CUDA tensor per utterance = ``model.separate(w[None], normalize=True, ...)[0]``.
    ``rescale=False`` returns the estimates of the normalised mixture, as the reference's evaluation
    script scores them (simple_whamr_evaluation.py:141-148); ``mixture_consistency`` as in
    README.md:113-114."""
    wavs = list(wavs)
    if not wavs:
        return []
    for w in wavs:
        if w.dim() != 1:
            raise RuntimeError("separate_corpus expects 1-D waveforms")
    lib = N.lib()
    cfg = _engine.make_config(model)
    if cfg.in_audio_channels != 1:
        raise RuntimeError("separate_corpus follows the README recipe, which is written for mono mixtures")
    device = _engine._model_device(model, "sudo_rm_rf_b200 runs on CUDA (sm_90a) only: move the model to an H100")
    if torch.is_grad_enabled() and model.training:
        raise RuntimeError("sudo_rm_rf_b200 implements the inference forward only: call model.eval()")
    plan = plan_buckets([int(w.shape[0]) for w in wavs], model_padding_rule(cfg), max_batch)
    results: List[torch.Tensor] = [None] * len(wavs)
    S = cfg.num_sources
    with torch.cuda.device(device), torch.no_grad():
        for Tp, idx in plan:
            B = len(idx)
            batch = torch.zeros((B, 1, Tp), dtype=torch.float32, device=device)
            for r, i in enumerate(idx):
                batch[r, 0, :wavs[i].shape[0]] = wavs[i].detach().to(device=device, dtype=torch.float32)
            lengths = torch.tensor([int(wavs[i].shape[0]) for i in idx], dtype=torch.int64, device=device)
            out = torch.empty((B, S, Tp), dtype=torch.float32, device=device)

            def enqueue(packed, ws):
                N.check(lib.sdr_separate_ragged(
                    C.byref(cfg), N.ptr(packed), N.ptr(batch), N.ptr(lengths), N.ptr(out), B, Tp,
                    1 if mixture_consistency else 0, 1 if rescale else 0,
                    N.ptr(ws), ws.numel(), N.stream(device)), "sdr_separate_ragged")
            _engine._call_shared(model, cfg, device, lib.sdr_separate_workspace_bytes(C.byref(cfg), B, Tp),
                                 "bad model configuration (sdr_separate_workspace_bytes returned 0)", enqueue)
            for r, i in enumerate(idx):
                results[i] = out[r, :, :wavs[i].shape[0]].clone()
    return results


# ---------------------------------------------------------------------------------------------------------------
# wav I/O + pipelined corpus inference (SURVEY.md 8f row 4; simple_whamr_evaluation.py:55-66,125-148)
# ---------------------------------------------------------------------------------------------------------------
def load_wav(path: str) -> Tuple[torch.Tensor, int]:
    """``torchaudio.load(path)`` semantics (simple_whamr_evaluation.py:56): ``([channels, T] float32 in [-1, 1],
    sample_rate)`` for PCM 8 / 16 / 32-bit and IEEE-float RIFF/WAVE files (torchaudio is not a dependency)."""
    import numpy as np
    from scipy.io import wavfile
    rate, data = wavfile.read(path)
    if data.ndim == 1:
        data = data[:, None]
    if data.dtype == np.int16:
        x = data.astype(np.float32) / 32768.0
    elif data.dtype == np.int32:
        x = data.astype(np.float32) / 2147483648.0
    elif data.dtype == np.uint8:
        x = (data.astype(np.float32) - 128.0) / 128.0
    elif data.dtype in (np.float32, np.float64):
        x = data.astype(np.float32)
    else:
        raise RuntimeError(f"unsupported wav sample type {data.dtype} in {path}")
    return torch.from_numpy(np.ascontiguousarray(x.T)), int(rate)


def save_wav(path: str, wav: torch.Tensor, sample_rate: int) -> None:
    """Writes ``[channels, T]`` (or ``[T]``) float32 samples as an IEEE-float WAV."""
    import numpy as np
    from scipy.io import wavfile
    w = wav.detach().to("cpu", torch.float32)
    if w.dim() == 1:
        w = w.unsqueeze(0)
    wavfile.write(path, int(sample_rate), np.ascontiguousarray(w.numpy().T))


class CorpusSeparator:
    """Pipelined version of ``separate_corpus`` for corpora that live on the host.

    Per batch of a bucket: the utterances are packed into a PINNED staging buffer, copied to the device on a copy
    stream, separated by a CUDA graph of ``sdr_separate_ragged`` captured once per (batch size, padded length, slot)
    and copied back into pinned memory on a second copy stream, with two slots in flight so the host packs batch
    k + 1 while the GPU works on batch k.  Results are ``[S, T_i]`` fp32 CPU tensors in corpus order and equal
    ``separate_corpus`` (hence the reference's one-utterance-at-a-time loop) to the last bit."""

    def __init__(self, model, max_batch: int = 32, mixture_consistency: bool = False, rescale: bool = True,
                 use_graphs: bool = True, max_graphs: int = 16):
        self.model = model
        self.max_batch = int(max_batch)
        self.mc = 1 if mixture_consistency else 0
        self.rescale = 1 if rescale else 0
        self.use_graphs = use_graphs
        self.max_graphs = max_graphs
        self.cfg = _engine.make_config(model)
        if self.cfg.in_audio_channels != 1:
            raise RuntimeError("CorpusSeparator follows the README recipe, which is written for mono mixtures")
        self.device = _engine._model_device(model,
                                            "sudo_rm_rf_b200 runs on CUDA (sm_90a) only: move the model to an H100")
        self.quantum = model_padding_rule(self.cfg)      # T -> padded length (the model's own rule)
        self.graphs = {}           # (B, Tp, slot) -> "warm" | CUDAGraph
        self._s_in, self._s_cmp, self._s_out = (torch.cuda.Stream(device=self.device) for _ in range(3))
        self.launches = {"eager": 0, "captured": 0, "replayed": 0}

    def run(self, wavs: Iterable[torch.Tensor]) -> List[torch.Tensor]:
        wavs = [w.detach().to("cpu", torch.float32).contiguous() for w in wavs]
        if not wavs:
            return []
        for w in wavs:
            if w.dim() != 1:
                raise RuntimeError("CorpusSeparator expects 1-D waveforms")
        if torch.is_grad_enabled() and self.model.training:
            raise RuntimeError("sudo_rm_rf_b200 implements the inference forward only: call model.eval()")
        lib, cfg, dev, S = N.lib(), self.cfg, self.device, self.cfg.num_sources
        plan = plan_buckets([int(w.shape[0]) for w in wavs], self.quantum, self.max_batch)
        max_in = max(len(idx) * Tp for Tp, idx in plan)
        ws_bytes = max(lib.sdr_separate_workspace_bytes(C.byref(cfg), len(idx), Tp) for Tp, idx in plan)
        if ws_bytes == 0:
            raise N.NativeError("bad model configuration (sdr_separate_workspace_bytes returned 0)")
        results: List[torch.Tensor] = [None] * len(wavs)
        with torch.cuda.device(dev), torch.no_grad():
            packed = _engine.packed_for(self.model, cfg, dev, self._s_cmp)
            key_buf = (max_in, ws_bytes, packed.data_ptr())
            if getattr(self, "_buf_key", None) != key_buf:      # (re)allocate staging once per corpus shape: graphs hold addresses
                self.graphs.clear()
                self._buf_key = key_buf
                self._ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                self._h_in = [torch.zeros(max_in, dtype=torch.float32).pin_memory() for _ in range(2)]
                self._h_len = [torch.zeros(self.max_batch, dtype=torch.int64).pin_memory() for _ in range(2)]
                self._h_out = [torch.empty(max_in * S, dtype=torch.float32).pin_memory() for _ in range(2)]
                self._d_in = [torch.empty(max_in, dtype=torch.float32, device=dev) for _ in range(2)]
                self._d_len = [torch.empty(self.max_batch, dtype=torch.int64, device=dev) for _ in range(2)]
                self._d_out = [torch.empty(max_in * S, dtype=torch.float32, device=dev) for _ in range(2)]
            cur = torch.cuda.current_stream(dev)
            for s in (self._s_in, self._s_cmp, self._s_out):
                s.wait_stream(cur)
            done = [None, None]          # per slot: (event of the D2H copy, batch indices, Tp) still to be unpacked
            free_in = [None, None]       # per slot: event after which the device input buffer may be overwritten

            def unpack(slot):
                if done[slot] is None:
                    return
                ev, idx, Tp = done[slot]
                ev.synchronize()
                out = self._h_out[slot][:len(idx) * S * Tp].view(len(idx), S, Tp)
                for r, i in enumerate(idx):
                    results[i] = out[r, :, :wavs[i].shape[0]].clone()
                done[slot] = None

            for k, (Tp, idx) in enumerate(plan):
                slot = k & 1
                unpack(slot)                                     # the slot's pinned buffers are free again
                B = len(idx)
                h_in = self._h_in[slot][:B * Tp].view(B, Tp)
                h_in.zero_()
                for r, i in enumerate(idx):
                    h_in[r, :wavs[i].shape[0]] = wavs[i]
                    self._h_len[slot][r] = int(wavs[i].shape[0])
                with torch.cuda.stream(self._s_in):
                    if free_in[slot] is not None:
                        self._s_in.wait_event(free_in[slot])
                    self._d_in[slot][:B * Tp].copy_(self._h_in[slot][:B * Tp], non_blocking=True)
                    self._d_len[slot][:B].copy_(self._h_len[slot][:B], non_blocking=True)
                    ev_in = torch.cuda.Event()
                    ev_in.record(self._s_in)

                def enqueue():
                    N.check(lib.sdr_separate_ragged(
                        C.byref(cfg), N.ptr(packed), N.ptr(self._d_in[slot]), N.ptr(self._d_len[slot]),
                        N.ptr(self._d_out[slot]), B, Tp, self.mc, self.rescale, N.ptr(self._ws), self._ws.numel(),
                        N.stream(dev)),
                        "sdr_separate_ragged")

                with torch.cuda.stream(self._s_cmp):
                    self._s_cmp.wait_event(ev_in)
                    if self.use_graphs:
                        how = _engine._graphed(self.graphs, (B, Tp, slot), self.max_graphs, dev, enqueue)
                    else:
                        enqueue()
                        how = "eager"
                    self.launches[how] += 1
                    ev_cmp = torch.cuda.Event()
                    ev_cmp.record(self._s_cmp)
                free_in[slot] = ev_cmp
                with torch.cuda.stream(self._s_out):
                    self._s_out.wait_event(ev_cmp)
                    self._h_out[slot][:B * S * Tp].copy_(self._d_out[slot][:B * S * Tp], non_blocking=True)
                    ev_out = torch.cuda.Event()
                    ev_out.record(self._s_out)
                done[slot] = (ev_out, idx, Tp)
            unpack(0)
            unpack(1)
            cur.wait_stream(self._s_cmp)
        return results


def separate_wav_files(model, paths: Sequence[str], out_dir: str, max_samples: int = 56000, max_batch: int = 32,
                       mixture_consistency: bool = False, rescale: bool = True) -> List[List[str]]:
    """The file loop of ``simple_whamr_evaluation.py:138-148`` as one pipelined call: loads every mixture (first
    channel, cropped to ``max_samples`` as the script does, :66), separates the corpus and writes
    ``<out_dir>/<name>_s<k>.wav`` per source.  Returns the written paths per input file."""
    import os
    os.makedirs(out_dir, exist_ok=True)
    wavs, rates = [], []
    for p in paths:
        w, sr = load_wav(p)
        wavs.append(w[0, :max_samples] if max_samples else w[0])
        rates.append(sr)
    est = CorpusSeparator(model, max_batch=max_batch, mixture_consistency=mixture_consistency, rescale=rescale).run(wavs)
    written = []
    for p, e, sr in zip(paths, est, rates):
        stem = os.path.splitext(os.path.basename(p))[0]
        outs = []
        for k in range(e.shape[0]):
            o = os.path.join(out_dir, f"{stem}_s{k + 1}.wav")
            save_wav(o, e[k], sr)
            outs.append(o)
        written.append(outs)
    return written
