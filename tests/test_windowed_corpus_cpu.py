"""Windowed separation of a corpus without a GPU: the packing of recordings of different lengths into shared window
batches, the argument checks of ``separate_long_corpus``, and the ragged C-ABI entries' bindings, size queries and
refusals next to those of ``sdr_window_merge``."""
import pytest
import torch

import sudo_rm_rf_b200 as P
import windowed_oracle as WO
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200 import windowed

W, H = 10, 6
X = 1 << 20                       # a non-null device address aligned to 256 bytes (never dereferenced)
Y = 1 << 30
BAD_ARGUMENT, UNSUPPORTED = -2, -5


def edge_lengths():
    """1, W - 1, W, W + 1, W + H, exact window multiples (the last window ends at T) and one-sample tails, mixed."""
    return [W + 3 * H, 1, W + 1, W - 1, W + H, W, W + 5 * H + 1, W + H + 1, 2, W + 7 * H, W + 1, W + 2 * H + 1]


def check_plan(lengths, max_windows):
    plan = windowed.corpus_plan(lengths, W, H, max_windows)
    assert plan.long == [i for i, T in enumerate(lengths) if T > W]
    assert plan.short == [i for i, T in enumerate(lengths) if T <= W]
    off = g = 0
    for j, i in enumerate(plan.long):
        assert plan.counts[j] == WO.plan(lengths[i], W, H)[0] > 1
        assert (plan.offsets[j], plan.firsts[j]) == (off, g)
        off += lengths[i]
        g += plan.counts[j]
    assert plan.windows == g and plan.samples == off
    # contiguous batches of M = min(max_windows, G) windows, the last one possibly shorter
    M = min(max_windows, g)
    assert [b for b in plan.batches] == [(g0, min(M, g - g0)) for g0 in range(0, g, M)] if g else plan.batches == []
    # every global window is window k of its recording, in recording-major order
    want = [(j, k) for j in range(len(plan.long)) for k in range(plan.counts[j])]
    assert [plan.locate(x) for x in range(g)] == want
    for g0, m in plan.batches:
        recs = [plan.locate(x)[0] for x in range(g0, g0 + m)]
        assert recs == sorted(recs) and set(recs) == set(range(recs[0], recs[-1] + 1))
        # a batch boundary splits at most one recording: the one that holds both g0 - 1 and g0
        split = [j for j in range(len(plan.long)) if plan.firsts[j] < g0 < plan.firsts[j] + plan.counts[j]]
        assert len(split) <= 1
    return plan


@pytest.mark.parametrize("max_windows", [1, 2, 3, 7, 32])
def test_packing_of_the_edge_lengths(max_windows):
    check_plan(edge_lengths(), max_windows)


def test_one_recording_spans_three_batches():
    T = W + 7 * H                               # 8 windows
    plan = check_plan([W + H, T, 5], 3)
    j = plan.long.index(1)
    batches = {g0 for g0, m in plan.batches
               for x in range(g0, g0 + m) if plan.locate(x)[0] == j}
    assert len(batches) >= 3


def test_one_batch_holds_three_recordings():
    plan = check_plan([W + 1, 3, W + H, W + 2, W - 1, W + 2 * H], 8)
    g0, m = plan.batches[0]
    assert len({plan.locate(x)[0] for x in range(g0, g0 + m)}) >= 3


def test_all_short_all_long_and_one_window_batches():
    short = check_plan([1, W, W - 1, 3], 4)
    assert short.long == [] and short.windows == 0 and short.batches == []
    long_ = check_plan([W + 1, W + H, W + 9 * H + 1], 4)
    assert long_.short == []
    one = check_plan(edge_lengths(), 1)
    assert all(m == 1 for _, m in one.batches) and len(one.batches) == one.windows


def test_offsets_are_exact_past_2_31():
    T = 3 * (1 << 30) + 7                      # past 2^31 samples in one recording, then more behind it
    plan = windowed.corpus_plan([T, T, 5, T], 32000, 16000, 32)
    assert plan.offsets == [0, T, 2 * T] and plan.samples == 3 * T
    K = WO.plan(T, 32000, 16000)[0]
    assert plan.firsts == [0, K, 2 * K] and plan.locate(2 * K + 5) == (2, 5)


def test_packing_refusals():
    with pytest.raises(ValueError, match="at least one"):
        windowed.corpus_plan([], W, H, 4)
    with pytest.raises(ValueError):
        windowed.corpus_plan([W + 1, 0], W, H, 4)
    with pytest.raises(ValueError):
        windowed.corpus_plan([W + 1], W, H, 0)


def test_separate_long_corpus_checks_before_any_work():
    m = P.SuDORMRF(16, 32, 1, 2, 21, 16, 2).eval()
    x = [torch.zeros(100), torch.zeros(1, 50)]
    with pytest.raises(ValueError, match="at least one"):
        windowed.separate_long_corpus(m, [], 20)
    with pytest.raises(ValueError, match="window"):
        windowed.separate_long_corpus(m, x, 1)
    with pytest.raises(ValueError, match="hop"):
        windowed.separate_long_corpus(m, x, 20, 9)
    with pytest.raises(ValueError, match="max_windows"):
        windowed.separate_long_corpus(m, x, 20, max_windows=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        windowed.separate_long_corpus(m, x, 20)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.separate_long_corpus(x, 20, normalize=False)
    # the same messages as separate_long's
    for kw in (dict(window=1), dict(window=20, hop=9), dict(window=20, max_windows=True)):
        with pytest.raises(ValueError) as a:
            windowed.separate_long(m, torch.zeros(1, 100), **kw)
        with pytest.raises(ValueError) as b:
            windowed.separate_long_corpus(m, [torch.zeros(100)], **kw)
        assert str(a.value) == str(b.value)


def test_ragged_entries_bind():
    lib = N.lib()
    for name in ("sdr_window_ragged_carry_bytes", "sdr_window_ragged_scratch_bytes", "sdr_window_gather_ragged",
                 "sdr_window_merge_ragged"):
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name), name


def test_ragged_size_queries_are_the_single_recording_ones():
    lib = N.lib()
    for S in (0, 1, 2, 4, 5):
        for A in (0, 1, 2):
            for Wq in (1, 2, 10, 32000, 1 << 24, (1 << 24) + 1):
                assert lib.sdr_window_ragged_carry_bytes(S, A, Wq) == lib.sdr_window_carry_bytes(1, S, A, Wq)
        for M in (0, 1, 7, 32, 1 << 20):
            assert lib.sdr_window_ragged_scratch_bytes(S, M) == lib.sdr_window_merge_scratch_bytes(1, S, M)
    assert lib.sdr_window_ragged_carry_bytes(2, 1, 100) == 256 + 2 * 100 * 4
    assert lib.sdr_window_ragged_scratch_bytes(3, 4) == (4 * 3 + 5 * 3) * 4


GATHER = dict(x=X, desc=X, R=3, A=1, W=10, H=5, g0=0, M=4, batch=Y, stream=None)
MERGE = dict(est=X, desc=X, R=3, carry=X, perm=None, out=Y, S=2, A=1, W=10, H=5, g0=0, M=4, scratch=X, stream=None)
# the same faults given to sdr_window_merge (est carry perm out B S A T W H k0 M scratch stream)
MERGE_ONE = dict(est=X, carry=X, perm=None, out=Y, B=1, S=2, A=1, T=100, W=10, H=5, k0=0, M=4, scratch=X, stream=None)
MERGE_FAULTS = [
    ("null estimates", dict(est=None), BAD_ARGUMENT),
    ("null carry", dict(carry=None), BAD_ARGUMENT),
    ("null output", dict(out=None), BAD_ARGUMENT),
    ("null scratch", dict(scratch=None), BAD_ARGUMENT),
    ("misaligned carry", dict(carry=X + 8), BAD_ARGUMENT),
    ("misaligned scratch", dict(scratch=X + 4), BAD_ARGUMENT),
    ("S=5", dict(S=5), UNSUPPORTED),
    ("S=0", dict(S=0), BAD_ARGUMENT),
    ("A=0", dict(A=0), BAD_ARGUMENT),
    ("M=0", dict(M=0), BAD_ARGUMENT),
    ("H < W/2", dict(H=4), BAD_ARGUMENT),
    ("H = W", dict(H=10), BAD_ARGUMENT),
    ("W past 2^24", dict(W=(1 << 24) + 2, H=(1 << 23) + 1), BAD_ARGUMENT),
    ("misaligned carry, S=5", dict(carry=X + 8, S=5), BAD_ARGUMENT),
    ("misaligned scratch, S=5", dict(scratch=X + 4, S=5), BAD_ARGUMENT),
    ("null output, S=5", dict(out=None, S=5), BAD_ARGUMENT),
    ("S=5, M=0", dict(S=5, M=0), UNSUPPORTED),
]


@pytest.mark.parametrize("case,kw,want", MERGE_FAULTS, ids=[c[0] for c in MERGE_FAULTS])
def test_ragged_merge_refuses_as_the_merge_does(case, kw, want):
    lib = N.lib()
    names = "est desc R carry perm out S A W H g0 M scratch stream".split()
    one = "est carry perm out B S A T W H k0 M scratch stream".split()
    a, b = dict(MERGE, **kw), dict(MERGE_ONE, **kw)
    assert lib.sdr_window_merge_ragged(*[a[n] for n in names]) == want
    assert lib.sdr_window_merge(*[b[n] for n in one]) == want


@pytest.mark.parametrize("kw,want", [
    (dict(desc=None), BAD_ARGUMENT), (dict(desc=X + 4), BAD_ARGUMENT), (dict(R=0), BAD_ARGUMENT),
    (dict(g0=-1), BAD_ARGUMENT), (dict(desc=X + 4, S=5), BAD_ARGUMENT), (dict(R=0, S=5), UNSUPPORTED)])
def test_ragged_merge_refuses_bad_descriptors(kw, want):
    names = "est desc R carry perm out S A W H g0 M scratch stream".split()
    a = dict(MERGE, **kw)
    assert N.lib().sdr_window_merge_ragged(*[a[n] for n in names]) == want


@pytest.mark.parametrize("kw", [dict(x=None), dict(desc=None), dict(batch=None), dict(desc=X + 4), dict(R=0),
                                dict(A=0), dict(M=0), dict(g0=-1), dict(H=10), dict(H=4), dict(W=1, H=1)])
def test_ragged_gather_refusals(kw):
    names = "x desc R A W H g0 M batch stream".split()
    a = dict(GATHER, **kw)
    assert N.lib().sdr_window_gather_ragged(*[a[n] for n in names]) == BAD_ARGUMENT
