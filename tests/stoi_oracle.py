"""fp64 numpy / scipy restatement of pystoi 0.3.3's ``stoi(x, y, fs_sig, extended=False)`` (Taal et al., "An Algorithm
for Intelligibility Prediction of Time-Frequency Weighted Noisy Speech", IEEE TASLP 2011), the STOI that asteroid's
``get_metrics`` reports.  One function per pystoi function; each names the one it restates.  No dependency on pystoi.

Two cases where pystoi raises are given values here, as on the GPU: a signal of at most N_FRAME samples after
resampling has no frame (pystoi fails in ``np.max`` of an empty array) and scores 1e-5 like any other signal with fewer
than N spectral frames."""
import math

import numpy as np
from scipy.signal import resample_poly

FS = 10000                      # pystoi/stoi.py: sampling rate the algorithm runs at
N_FRAME = 256                   # window length
NFFT = 512                      # FFT length
NUMBAND = 15                    # third-octave bands
MINFREQ = 150                   # centre of the first band
N = 30                          # frames per segment (384 ms)
BETA = -15.                     # lower signal-to-distortion bound of the clip, dB
DYN_RANGE = 40                  # silent-frame range, dB
EPS = np.finfo(float).eps


def thirdoct(fs, nfft, num_bands, min_freq):
    """pystoi/utils.py ``thirdoct``: the [num_bands, nfft / 2 + 1] 0/1 band matrix and the centre frequencies.  Each
    band edge snaps to the nearest FFT bin; a band covers the half-open bin range [low, high)."""
    f = np.linspace(0, fs, nfft + 1)
    f = f[:int(nfft / 2) + 1]
    k = np.array(range(num_bands)).astype(float)
    cf = np.power(2. ** (1. / 3), k) * min_freq
    freq_low = min_freq * np.power(2., (2 * k - 1) / 6)
    freq_high = min_freq * np.power(2., (2 * k + 1) / 6)
    obm = np.zeros((num_bands, len(f)))
    for i in range(len(cf)):
        fl_ii = int(np.argmin(np.square(f - freq_low[i])))
        fh_ii = int(np.argmin(np.square(f - freq_high[i])))
        obm[i, fl_ii:fh_ii] = 1
    return obm, cf


OBM, CF = thirdoct(FS, NFFT, NUMBAND, MINFREQ)


def band_edges():
    """(low, high) bin range of each band of OBM."""
    return [(int(np.flatnonzero(r)[0]), int(np.flatnonzero(r)[-1]) + 1) for r in OBM]


def resample_window_oct(p, q):
    """pystoi/utils.py ``_resample_window_oct``, the port of Octave's ``resample`` filter design: a Kaiser-windowed
    ideal low-pass at 1 / (2 max(p, q)) of the upsampled rate, 60 dB rejection, roll-off a tenth of the cutoff."""
    gcd = np.gcd(p, q)
    if gcd > 1:
        p /= gcd
        q /= gcd
    log10_rejection = -3.0
    stopband_cutoff_f = 1. / (2 * max(p, q))
    roll_off_width = stopband_cutoff_f / 10
    rejection_db = -20 * log10_rejection
    L = np.ceil((rejection_db - 8) / (28.714 * roll_off_width))
    t = np.arange(-L, L + 1)
    ideal_filter = 2 * p * stopband_cutoff_f * np.sinc(2 * stopband_cutoff_f * t)
    if 21 <= rejection_db <= 50:
        beta = 0.5842 * (rejection_db - 21) ** 0.4 + 0.07886 * (rejection_db - 21)
    elif rejection_db > 50:
        beta = 0.1102 * (rejection_db - 8.7)
    else:
        beta = 0.0
    return np.kaiser(2 * L + 1, beta) * ideal_filter


def resample_oct(x, p, q):
    """pystoi/utils.py ``resample_oct``: the window normalised to sum 1, then scipy's ``resample_poly`` (its zero
    padding, alignment and output length ceil(n p / q))."""
    h = resample_window_oct(p, q)
    window = h / np.sum(h)
    return resample_poly(x, p, q, window=window)


def hann():
    """pystoi/utils.py: ``np.hanning(framelen + 2)[1:-1]``, MATLAB's ``hanning(framelen)``."""
    return np.hanning(N_FRAME + 2)[1:-1]


def stft(x, win_size, fft_size, overlap=4):
    """pystoi/utils.py ``stft``: Hann-windowed frames at hop win_size / overlap, starting at 0 and strictly before
    len(x) - win_size (so the last full frame is dropped when len(x) - win_size is a multiple of the hop), rfft(n)."""
    hop = int(win_size / overlap)
    w = np.hanning(win_size + 2)[1:-1]
    return np.array([np.fft.rfft(w * x[i:i + win_size], n=fft_size) for i in range(0, len(x) - win_size, hop)])


def overlap_and_add(x_frames, hop):
    """pystoi/utils.py ``_overlap_and_add``: frame k added at k hop; length (K - 1) hop + framelen."""
    num_frames, framelen = x_frames.shape
    out = np.zeros((num_frames - 1) * hop + framelen)
    for k in range(num_frames):
        out[k * hop:k * hop + framelen] += x_frames[k]
    return out


def remove_silent_frames(x, y, dyn_range, framelen, hop):
    """pystoi/utils.py ``remove_silent_frames``: the frames of x whose energy lies within dyn_range dB of the loudest
    frame of x, the same frames of y, each overlap-added back.  None when x has no frame."""
    w = np.hanning(framelen + 2)[1:-1]
    x_frames = np.array([w * x[i:i + framelen] for i in range(0, len(x) - framelen, hop)])
    y_frames = np.array([w * y[i:i + framelen] for i in range(0, len(x) - framelen, hop)])
    if len(x_frames) == 0:
        return None
    x_energies = 20 * np.log10(np.linalg.norm(x_frames, axis=1) + EPS)
    mask = (np.max(x_energies) - dyn_range - x_energies) < 0
    return overlap_and_add(x_frames[mask], hop), overlap_and_add(y_frames[mask], hop), mask


def stoi(x, y, fs_sig):
    """pystoi/stoi.py ``stoi(x, y, fs_sig, extended=False)``, x the clean reference, y the processed signal."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    if x.shape != y.shape:
        raise ValueError("x and y should have the same length")
    if fs_sig != FS:
        x = resample_oct(x, FS, fs_sig)
        y = resample_oct(y, FS, fs_sig)
    return stoi_at_fs(x, y)


def stoi_at_fs(x, y):
    """The rest of ``stoi`` once x and y are at FS."""
    kept = remove_silent_frames(x, y, DYN_RANGE, N_FRAME, int(N_FRAME / 2))
    if kept is None:
        return 1e-5
    x, y, _ = kept
    x_spec = stft(x, N_FRAME, NFFT, overlap=2).transpose()
    y_spec = stft(y, N_FRAME, NFFT, overlap=2).transpose()
    if x_spec.shape[-1] < N:                        # pystoi warns here
        return 1e-5
    x_tob = np.sqrt(np.matmul(OBM, np.square(np.abs(x_spec))))
    y_tob = np.sqrt(np.matmul(OBM, np.square(np.abs(y_spec))))
    x_segments = np.array([x_tob[:, m - N:m] for m in range(N, x_tob.shape[1] + 1)])
    y_segments = np.array([y_tob[:, m - N:m] for m in range(N, x_tob.shape[1] + 1)])
    norm_const = np.linalg.norm(x_segments, axis=2, keepdims=True) / (
        np.linalg.norm(y_segments, axis=2, keepdims=True) + EPS)
    y_segments_normalized = y_segments * norm_const
    clip_value = 10 ** (-BETA / 20)
    y_primes = np.minimum(y_segments_normalized, x_segments * (1 + clip_value))
    y_primes = y_primes - np.mean(y_primes, axis=2, keepdims=True)
    x_segments = x_segments - np.mean(x_segments, axis=2, keepdims=True)
    y_primes /= (np.linalg.norm(y_primes, axis=2, keepdims=True) + EPS)
    x_segments /= (np.linalg.norm(x_segments, axis=2, keepdims=True) + EPS)
    correlations_components = y_primes * x_segments
    J = x_segments.shape[0]
    M = x_segments.shape[1]
    return float(np.sum(correlations_components) / (J * M))


def resampled_length(n, fs_sig):
    """Length of a signal of n samples at fs_sig after resample_oct to FS: ceil(n p / q), p / q = FS / fs_sig reduced."""
    g = math.gcd(FS, fs_sig)
    p, q = FS // g, fs_sig // g
    return n if p == q else -(-n * p // q)


def at_fs(x, fs_sig):
    """x as fp64 at FS, as ``stoi`` resamples it."""
    x = np.asarray(x, np.float64)
    return x if fs_sig == FS else resample_oct(x, FS, fs_sig)


def frame_energies(x, fs_sig=FS):
    """The energies in dB that ``remove_silent_frames`` gives the frames of clean signal x."""
    x = at_fs(x, fs_sig)
    w = hann()
    frames = np.array([w * x[i:i + N_FRAME] for i in range(0, len(x) - N_FRAME, N_FRAME // 2)])
    return 20 * np.log10(np.linalg.norm(frames, axis=1) + EPS) if len(frames) else np.zeros(0)


def mask_margin(x, fs_sig=FS):
    """(indices of the frames of clean signal x that ``remove_silent_frames`` keeps, and the smallest distance in dB of
    any frame energy from the threshold max - DYN_RANGE).  A computation that rounds a frame energy differently keeps
    the same frames as long as its error stays below the margin.  ([], inf) when x has no frame."""
    e = frame_energies(x, fs_sig)
    if len(e) == 0:
        return np.zeros(0, np.int64), math.inf
    d = np.max(e) - DYN_RANGE - e
    return np.flatnonzero(d < 0), float(np.min(np.abs(d)))


def score(x, ys, fs_sig):
    """(``stoi(x, y, fs_sig)`` for every y of ys, kept frame indices, mask margin) with x resampled once."""
    x10 = at_fs(x, fs_sig)
    kept, margin = mask_margin(x10)
    return [stoi_at_fs(x10, at_fs(y, fs_sig)) for y in ys], kept, margin


def spectral_frames(x, fs_sig):
    """Number of spectral frames stoi() analyses for clean signal x (before the N-frame check)."""
    x = np.asarray(x, np.float64)
    if fs_sig != FS:
        x = resample_oct(x, FS, fs_sig)
    kept = remove_silent_frames(x, x, DYN_RANGE, N_FRAME, N_FRAME // 2)
    return 0 if kept is None else max(int(kept[2].sum()) - 1, 0)
