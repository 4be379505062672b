"""Slot resets of the three stream states on the GPU, byte by byte.

A guarded state is filled with a byte pattern, then reset through the host-listed entry, the masked entry where one
exists, and the whole-state entry.  The result is compared with an image built on the host from the documented
layout: exactly the named slots' bytes of every per-slot region are zero, every other byte and both guard bands are
unchanged, and the host-listed and masked resets agree bitwise."""
import ctypes as C

import numpy as np
import pytest
import torch

from guards import check_bands, poisoned, repoison
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.resample_stream import min_delay

pytestmark = pytest.mark.gpu
PATTERN = 0x5AC3E196
B = 4
CHOSEN = (B - 1, 0)          # the first and last slot, listed out of order; slots 1 and 2 stay


def r256(n):
    return (n + 255) // 256 * 256


def cur():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def listed(slots):
    return (C.c_int32 * len(slots))(*slots), len(slots)


def device_mask(slots):
    m = torch.zeros(B, dtype=torch.uint8, device="cuda")
    m[list(slots)] = 1
    return m


def zeroed(image, regions, slots):
    """`image` with bytes [off + b * size, off + (b + 1) * size) of every region (off, size) zeroed for b in slots."""
    out = image.copy()
    for off, size in regions:
        for b in slots:
            out[off + b * size:off + (b + 1) * size] = 0
    return out


def run(nbytes, regions, reset_listed, reset_masked, reset_all, whole):
    """Each reset on a freshly patterned state; `whole(image)` is the image reset_all leaves."""
    state = poisoned(nbytes, PATTERN)
    image = state.cpu().numpy().copy()
    want = zeroed(image, regions, CHOSEN)
    N.check(reset_listed(state, *listed(CHOSEN)), "host-listed reset")
    check_bands(state, "state")
    got = state.cpu().numpy()
    assert np.array_equal(got, want)
    if reset_masked is not None:
        repoison(state, PATTERN)
        N.check(reset_masked(state, device_mask(CHOSEN)), "masked reset")
        check_bands(state, "state")
        assert np.array_equal(state.cpu().numpy(), got)
    repoison(state, PATTERN)
    N.check(reset_all(state), "whole reset")
    check_bands(state, "state")
    assert np.array_equal(state.cpu().numpy(), whole(image))


@pytest.mark.parametrize("A,U,D,k,S", [(1, 1, 4, 21, 2), (2, 3, 3, 11, 3)])
def test_causal_state(A, U, D, k, S):
    lib = N.lib()
    cfg = N.SdrConfig(2, A, 16, 40, U, D, k, 16, S, 1)
    nbytes = lib.sdr_stream_state_bytes(C.byref(cfg), B)
    assert nbytes > 0 and nbytes % B == 0
    run(nbytes, [(0, nbytes // B)],
        lambda t, arr, n: lib.sdr_stream_reset(C.byref(cfg), N.ptr(t), B, arr, n, cur()),
        lambda t, m: lib.sdr_stream_reset_masked(C.byref(cfg), N.ptr(t), B, N.ptr(m), cur()),
        lambda t: lib.sdr_stream_reset(C.byref(cfg), N.ptr(t), B, None, 0, cur()),
        np.zeros_like)


@pytest.mark.parametrize("S", [1, 2, 3, 4])
def test_windowed_state(S):
    lib = N.lib()
    A, W, H = 2, 16, 10
    # the carry's pi [B][S] int32, its estimate [B][S A][W], the history [B][A][H], the counters [B] int64
    pi_bytes = r256(B * S * 4)
    hist_off = r256(pi_bytes + B * S * A * W * 4)
    count_off = hist_off + r256(B * A * H * 4)
    nbytes = lib.sdr_window_stream_state_bytes(B, S, A, W, H)
    assert nbytes == count_off + 8 * B
    run(nbytes, [(0, S * 4), (pi_bytes, S * A * W * 4), (hist_off, A * H * 4), (count_off, 8)],
        lambda t, arr, n: lib.sdr_window_stream_reset(N.ptr(t), B, S, A, W, H, arr, n, cur()),
        lambda t, m: lib.sdr_window_stream_reset_masked(N.ptr(t), B, S, A, W, H, N.ptr(m), cur()),
        lambda t: lib.sdr_window_stream_reset(N.ptr(t), B, S, A, W, H, None, 0, cur()),
        np.zeros_like)


@pytest.mark.parametrize("up,down,C_,lead,p,q", [(8000, 44100, 441, 0, 80, 441), (16000, 48000, 300, 5, 1, 3)])
def test_resampling_state(up, down, C_, lead, p, q):
    lib = N.lib()
    rows = 2
    args = (B, rows, C_, up, down, min_delay(up, down, lead), lead)
    # the filter [2 L + 1] fp64, the counters [B] int64, then two histories [B][rows][Hs] fp32
    L = 10 * max(p, q)
    Hs = lead + (args[5] * q + L) // p + 1
    taps_bytes = (2 * L + 1) * 8
    count_off = r256(taps_bytes)
    hist_off = count_off + r256(8 * B)
    slot = rows * Hs * 4
    nbytes = lib.sdr_resample_stream_state_bytes(*args)
    assert nbytes == hist_off + 2 * B * slot

    def reset(t, arr, n):
        return lib.sdr_resample_stream_reset(N.ptr(t), t.numel(), *args, arr, n, cur())

    fresh = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    N.check(reset(fresh, None, 0), "sdr_resample_stream_reset")
    taps = fresh[:taps_bytes].cpu().numpy()
    assert np.abs(taps.view(np.float64)).sum() > 0

    def whole(image):               # the filter designed again, the padding after it kept, the rest zeroed
        out = image.copy()
        out[:taps_bytes] = taps
        out[count_off:] = 0
        return out

    run(nbytes, [(count_off, 8), (hist_off, slot), (hist_off + B * slot, slot)], reset, None,
        lambda t: reset(t, None, 0), whole)
