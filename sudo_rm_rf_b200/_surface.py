"""The inference methods every model class shares: ``separate``, ``separate_long``, ``stream_windows`` and
``forward_host``, stated once on top of the engine, the windowed path and the resamplers."""
import torch

from . import _engine
from . import resample, resample_stream, windowed


def _not_standalone(self, *_, **__):
    raise NotImplementedError(
        f"{type(self).__name__} is a parameter container of the H100 forward path; "
        "call the parent SuDORMRF / GroupCommSudoRmRf module instead.")


class NativeSeparator(_engine.NativeModuleMixin):
    """The inference surface of the four model classes.  A class that needs other defaults overrides a method with
    its own signature and delegates here."""

    def separate(self, input_wav, mixture_consistency=False, normalize=False, sample_rate=None, model_rate=None):
        """forward() with the uniform mixture-consistency projection
        (mixture_consistency.py:14-36) fused into the decoder epilogue.

        ``normalize=True`` runs the whole README recipe (reference README.md:100-114) on the
        device: ``input_wav`` is the raw mixture ``[B, T]`` or ``[B, 1, T]``; it is normalised per
        utterance (mean, unbiased std), separated, and the estimates are rescaled with the
        mixture's std and mean (then, optionally, projected onto the normalised mixture).

        ``sample_rate`` and ``model_rate`` (both or neither): the mixture's rate and the rate the model was trained
        at.  When they differ the mixture is resampled to ``model_rate`` (``resample.resample_poly``), separated there,
        and every source is resampled back and cropped to the input's length, so the sources sum to the band-limited
        mixture rather than to the mixture itself (``resample.at_model_rate``)."""
        run = _engine.separate if normalize else _engine.forward
        return resample.at_model_rate(lambda wav: run(self, wav, mixture_consistency=mixture_consistency),
                                      input_wav, sample_rate, model_rate)

    def separate_long(self, input_wav, window, hop=None, normalize=True, mixture_consistency=False,
                      max_windows=32, sample_rate=None, model_rate=None):
        """``separate`` for recordings of any length: overlapping windows of ``window`` samples every ``hop``,
        separated in batches of ``max_windows`` per recording, aligned and cross-faded on the device (see
        ``windowed.separate_long``).  ``window`` and ``hop`` count samples at ``model_rate``; ``sample_rate`` and
        ``model_rate`` as for ``separate``."""
        return resample.at_model_rate(
            lambda wav: windowed.separate_long(self, wav, window, hop, normalize=normalize,
                                               mixture_consistency=mixture_consistency, max_windows=max_windows),
            input_wav, sample_rate, model_rate)

    def separate_long_corpus(self, wavs, window, hop=None, normalize=True, mixture_consistency=False,
                             max_windows=32, return_permutations=False):
        """``separate_long`` for a corpus of recordings of different lengths (a sequence of CUDA tensors [A, T_r] or
        [T_r] on one device): their windows share batches of ``max_windows``, and recording r's [S A, T_r] result is
        ``separate_long`` on it alone (see ``windowed.separate_long_corpus``).  Returns a list, and with
        ``return_permutations`` also the list of each recording's [K_r, S] window orders (None for one window)."""
        return windowed.separate_long_corpus(self, wavs, window, hop, normalize=normalize,
                                             mixture_consistency=mixture_consistency, max_windows=max_windows,
                                             return_permutations=return_permutations)

    def stream_windows(self, batch_size, chunk_samples, window, hop=None, normalize=True,
                       mixture_consistency=False, sample_rate=None, model_rate=None):
        """A ``window_stream.WindowedStream``: ``separate_long``'s windows taken step by step for ``batch_size``
        slots of ``chunk_samples`` samples per step (a multiple of the hop), one hop late.

        ``sample_rate`` and ``model_rate`` (both or neither, as for ``separate``): with different rates, a
        ``resample_stream.ResampledStream`` whose output is ``separate_long``'s with those rates, ``latency``
        samples late; ``chunk_samples`` then counts input-rate samples and ``window`` / ``hop`` model-rate ones."""
        return resample_stream.windowed_stream(self, batch_size, chunk_samples, window, hop, normalize,
                                               mixture_consistency, sample_rate, model_rate)

    def forward_host(self, host_wav, host_out=None, mixture_consistency=False):
        """End-to-end call on pinned HOST tensors (H2D, forward, D2H on the current stream)."""
        return _engine.forward_host(self, host_wav, host_out, mixture_consistency)

    def pad_to_appropriate_length(self, x):
        """The reference's padding to a multiple of ``n_least_samples_req`` (improved_sudormrf.py:303-314,
        causal_improved_sudormrf_v3.py:213-224).  The native encoder pads implicitly; this helper is kept for callers
        that use it directly (device-side, no host round trip)."""
        T = x.shape[-1]
        q = self.n_least_samples_req
        Tp = q if T < q else ((T + q - 1) // q) * q
        out = torch.zeros(list(x.shape[:-1]) + [Tp], dtype=torch.float32, device=x.device)
        out[..., :T] = x
        return out

    @staticmethod
    def remove_trailing_zeros(padded_x, initial_x):
        return padded_x[..., :initial_x.shape[-1]]
