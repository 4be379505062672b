"""Native calls across CUDA streams and host threads: buffer lifetimes, stream hand-over and re-entrancy.

Each case makes one hazard deterministic and runs once.  The call's stream is held by a sleep (about 0.5 s) and the
call is enqueued behind it.  The host then releases or replaces a buffer the call reads, and at once allocates
sentinels of exactly the released sizes on the other streams whose pool the buffer could return to, filled with 3.0f
words on a stream nothing holds.  Free blocks of those sizes are cached beforehand, so that no sentinel needs new
device memory (``cudaMalloc`` can synchronise the device), and each case asserts that the held call was still queued
when the sentinels were written.  If the caching allocator hands the buffer out while the call is still queued, the
call reads 3.0 where its weights, state or scratch were.  Every buffer touched here holds floats only: the packed
weights, the workspaces and staging buffers, and the stream state (histories, carries and a float "started" flag).  So
a clobbered buffer gives wrong numbers, never a fault.  The held call's result is compared with the same call run
undisturbed (bitwise for the causal model, the stream and the backward; within 1e-5 of max |ref| where fp64 atomics
sum the GlobLN statistics) and with the fp64 oracle at the usual 1e-3 bar.

Host threads are ordered by ``threading.Event`` hooks, never by repetition.
"""
import ast
import gc
import glob
import json
import os
import subprocess
import sys
import threading

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200.corpus import CorpusSeparator
from oracle import sudormrf_oracle as O
from stream_oracle import CausalStreamOracle, granule

gpu = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
SLEEP = 1_000_000_000   # cycles: about 0.5 s, longer than any call here and than a gc.collect() in pytest
KW = dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64,
          num_sources=2)
CLS = {"improved": P.SuDORMRF, "causal": P.CausalSuDORMRF}


def build(variant, seed=5):
    cfg = O.Config(variant=variant, **KW)
    sd = O.make_state_dict(cfg, seed=seed)
    m = CLS[variant](**KW)
    m.load_state_dict(sd)
    return cfg, sd, m.to(DEV).eval()


def mixture(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def hold():
    # first launches of the kernels the host runs while the stream is held, done here: loading a module can
    # synchronise the device, which would let the held call finish before the buffer is released
    torch.empty(1024, device=DEV).fill_(3.0).mul_(1.0)
    torch.cuda._sleep(SLEEP)


def reserve(sizes, streams):
    """Caches two free blocks of each size on each stream, so that ``sentinels`` needs no new device memory: a
    ``cudaMalloc`` may synchronise the device and let the held call finish first."""
    for s in streams:
        with torch.cuda.stream(s):
            [torch.empty(int(n), dtype=torch.uint8, device=DEV) for n in sizes for _ in range(2)]


def sentinels(sizes, streams, held):
    """Two tensors of exactly each size on each stream (the released block, if the allocator hands it out, and a
    reserved one), filled with 3.0f on a fresh stream while ``held`` is still busy.  The caller keeps them until it has
    synchronised."""
    keep = []
    for s in streams:
        with torch.cuda.stream(s):
            keep += [torch.empty(int(n), dtype=torch.uint8, device=DEV) for n in sizes for _ in range(2)]
    free = torch.cuda.Stream()
    with torch.cuda.stream(free):
        for t in keep:
            t[:t.numel() // 4 * 4].view(torch.float32).fill_(3.0)
    assert not held.query(), "the held call ran before the sentinels were written: the case proves nothing"
    return keep


def buffer_bytes(m):
    st = _engine._state(m, torch.device(DEV, torch.cuda.current_device()))
    return [b.numel() for b in (st.packed, st.workspace, st.staging) if b is not None]


def same(got, ref, exact):
    got, ref = got.cpu(), ref.cpu()
    if exact:
        assert torch.equal(got, ref), f"max |d| = {(got - ref).abs().max().item():.3e}"
    else:
        d = (got - ref).abs().max().item()
        assert d <= 1e-5 * ref.abs().max().item(), f"max |d| = {d:.3e}, max |ref| = {ref.abs().max().item():.3e}"


def fp64(got, ref):
    e = O.parity_errors(got.cpu(), ref)
    assert max(e) < 1e-3, e


# ---------------------------------------------------------------------------------------------------------------------
# 1. Weights repacked while a call that reads them is in flight
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_stream_step_survives_a_repack():
    """``model(x)`` packs on the default stream, a step reads that buffer on a held side stream, and a weight change
    makes the next ``model(x)`` repack and free it into the default stream's pool."""
    cfg, sd, m = build("causal")
    Cs = 4 * granule(cfg)
    x = mixture(2, 1, Cs, seed=1)
    xd = x.to(DEV)
    with torch.no_grad():
        want = m.stream(2, Cs).step(xd)
        m(xd)
        s = m.stream(2, Cs)
        torch.cuda.synchronize()
        old = buffer_bytes(m)[0]
        reserve([old], [torch.cuda.current_stream()])
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            hold()
            got = s.step(xd)
        m.encoder.weight.mul_(1.0)          # a version bump: same values, new packed buffer
        m(xd)
        keep = sentinels([old], [torch.cuda.current_stream()], side)
        torch.cuda.synchronize()
    del keep
    same(got, want, exact=True)
    fp64(got, CausalStreamOracle(cfg, sd, 2).step(x))


@gpu
def test_forward_reads_weights_a_step_packed():
    """The packed buffer comes from a step on the default stream (no model call has run yet), ``model(x)`` reads it on
    a held stream, and the next step repacks."""
    cfg, sd, m = build("causal")
    _, _, twin = build("causal")
    Cs = 4 * granule(cfg)
    x = mixture(2, 1, 2 * Cs, seed=2)
    xd = x.to(DEV)
    with torch.no_grad():
        want = twin(xd)
        s = m.stream(2, Cs)
        s.step(xd[..., :Cs])
        torch.cuda.synchronize()
        old = buffer_bytes(m)[0]
        reserve([old], [torch.cuda.current_stream()])
        a = torch.cuda.Stream()
        with torch.cuda.stream(a):
            hold()
            got = m(xd)
        m.encoder.weight.mul_(1.0)
        s.step(xd[..., Cs:])
        keep = sentinels([old], [torch.cuda.current_stream()], a)
        torch.cuda.synchronize()
    del keep
    same(got, want, exact=True)
    fp64(got, O.causal_forward(cfg, sd, x, dtype=torch.float64))


@gpu
def test_corpus_run_while_another_thread_repacks(monkeypatch):
    """``CorpusSeparator.run`` in one thread; once it has packed, the main thread halves a weight and calls
    ``model(x)``.  The corpus gives what the weights packed at its start give, the forward what the new ones give."""
    cfg, sd, m = build("improved")
    wavs = [mixture(T, seed=T) * 2.0 + 0.1 for T in (1500, 2300, 977, 3100)]
    want = CorpusSeparator(m).run(wavs)
    sep = CorpusSeparator(m)
    packed_ev, ev_packed = threading.Event(), torch.cuda.Event()
    orig = _engine.packed_weights
    worker = {}

    def packed_weights(*a, **k):
        r = orig(*a, **k)
        if threading.current_thread() is worker.get("t"):
            ev_packed.record()
            hold()                          # the corpus kernels queue behind this
            packed_ev.set()
        return r
    monkeypatch.setattr(_engine, "packed_weights", packed_weights)
    out = {}
    held = torch.cuda.Stream()

    def run():
        with torch.cuda.stream(held):
            out["res"] = sep.run(wavs)
    reserve([buffer_bytes(m)[0]], [torch.cuda.current_stream()])
    t = worker["t"] = threading.Thread(target=run)
    t.start()
    assert packed_ev.wait(60), "the corpus thread never packed"
    x = mixture(2, 1, 1600, seed=7)
    with torch.no_grad():
        old = buffer_bytes(m)[0]
        torch.cuda.current_stream().wait_event(ev_packed)
        m.bottleneck.weight.mul_(0.5)
        y = m(x.to(DEV))
        keep = sentinels([old], [torch.cuda.current_stream()], held)
    t.join(60)
    assert not t.is_alive()
    torch.cuda.synchronize()
    del keep
    for got, ref in zip(out["res"], want):
        same(got, ref, exact=False)
    fp64(torch.cat(out["res"], -1).unsqueeze(0),
         torch.cat([O.separate(cfg, sd, w[None].double(), dtype=torch.float64)[0] for w in wavs], -1).unsqueeze(0))
    sd_new = dict(sd, **{"bottleneck.weight": sd["bottleneck.weight"] * 0.5})
    fp64(y, O.forward(cfg, sd_new, x, dtype=torch.float64))


def grads(m):
    return torch.cat([p.grad.reshape(-1) for p in m.parameters()])


@gpu
def test_training_on_a_side_stream_survives_a_repack():
    """Forward and backward on a held stream; the graph is freed and the next forward (on the default stream) repacks."""
    cfg, sd, m = build("improved")
    m.train().enable_training()
    x = mixture(2, 1, 1600, seed=3).to(DEV)
    g = mixture(2, 2, 1600, seed=4).to(DEV)
    (m(x) * g).sum().backward()
    want = grads(m).clone()
    m.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    old = buffer_bytes(m)
    reserve(old, [torch.cuda.current_stream()])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        hold()
        loss = (m(x) * g).sum()
        loss.backward()
        got = grads(m)
    del loss
    with torch.no_grad():
        m.encoder.weight.mul_(1.0)
    m(x)
    keep = sentinels(old, [torch.cuda.current_stream()], side)
    torch.cuda.synchronize()
    del keep
    same(got, want, exact=True)


# ---------------------------------------------------------------------------------------------------------------------
# 2. Buffers released while a call that reads them is in flight
# ---------------------------------------------------------------------------------------------------------------------
def entry_call(name, m, seed):
    """Inputs go to the device here: a copy from pageable memory on a held stream would block the host until the
    stream is free."""
    x = mixture(2, 1, 1600, seed=seed)
    xd = x.to(DEV)
    if name == "forward":
        def call():
            with torch.no_grad():
                return m(xd)
    elif name == "separate":
        def call():
            with torch.no_grad():
                return m.separate(xd[:, 0], normalize=True)
    elif name == "forward_host":
        h_in = x.pin_memory()

        def call():
            return _engine.forward_host(m, h_in)
    else:
        m.train().enable_training()

        def call():
            return m(xd).detach()
    return x, call


@gpu
@pytest.mark.parametrize("how", ["drop_cache", "del_model"])
@pytest.mark.parametrize("name", ["forward", "separate", "forward_host", "train_forward"])
def test_buffers_released_during_a_call(name, how):
    cfg, sd, m = build("improved")
    x, call = entry_call(name, m, seed=11)
    call()
    want = call()                  # forward_host: eager, then captured; the held call below replays
    torch.cuda.synchronize()
    want = want.clone()
    sizes = buffer_bytes(m)
    reserve(sizes, [torch.cuda.current_stream()])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        hold()
        got = call()
    if how == "drop_cache":
        _engine.drop_cache(m)
    else:
        del m, call
        gc.collect()
    keep = sentinels(sizes, [torch.cuda.current_stream()], side)
    torch.cuda.synchronize()
    del keep
    same(got, want, exact=False)
    ref = O.separate(cfg, sd, x[:, 0].double(), dtype=torch.float64) if name == "separate" else \
        O.forward(cfg, sd, x, dtype=torch.float64)
    fp64(got, ref)


@gpu
@pytest.mark.parametrize("name", ["forward", "forward_host"])
def test_workspace_growth_on_a_second_stream(name):
    """A larger call on stream B replaces the workspace (and staging buffer) a held call on stream A reads."""
    cfg, sd, m = build("improved")
    _, _, twin = build("improved")
    small, large = mixture(2, 1, 1600, seed=12), mixture(4, 1, 4000, seed=13)

    staged = {id(x): (x.pin_memory(), x.to(DEV)) for x in (small, large)}

    def call(model, x):
        h, d = staged[id(x)]
        if name == "forward_host":
            return _engine.forward_host(model, h, use_graph=False)
        with torch.no_grad():
            return model(d)
    want_small, want_large = call(m, small), call(twin, large)
    torch.cuda.synchronize()
    want_small, want_large = want_small.clone(), want_large.clone()
    sizes = buffer_bytes(m)[1:]
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    reserve(sizes, [torch.cuda.current_stream(), b])
    with torch.cuda.stream(a):
        hold()
        got_small = call(m, small)
    with torch.cuda.stream(b):
        got_large = call(m, large)
    assert buffer_bytes(m)[1] > sizes[0]
    keep = sentinels(sizes, [torch.cuda.current_stream(), b], a)
    torch.cuda.synchronize()
    del keep
    same(got_small, want_small, exact=False)
    same(got_large, want_large, exact=False)
    fp64(got_small, O.forward(cfg, sd, small, dtype=torch.float64))
    fp64(got_large, O.forward(cfg, sd, large, dtype=torch.float64))


@gpu
def test_stream_deleted_while_a_step_is_in_flight():
    cfg, sd, m = build("causal")
    Cs = 4 * granule(cfg)
    x = mixture(2, 1, Cs, seed=14)
    xd = x.to(DEV)
    with torch.no_grad():
        want = m.stream(2, Cs).step(xd)
        s = m.stream(2, Cs)
        torch.cuda.synchronize()
        sizes = [s._state.numel(), s._ws.numel()]
        reserve(sizes, [torch.cuda.current_stream()])
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            hold()
            got = s.step(xd)
        del s
        gc.collect()
        keep = sentinels(sizes, [torch.cuda.current_stream()], side)
        torch.cuda.synchronize()
    del keep
    same(got, want, exact=True)
    fp64(got, CausalStreamOracle(cfg, sd, 2).step(x))


@gpu
def test_forward_host_graph_evicted_while_its_replay_is_queued():
    """A replay of a captured ``forward_host`` graph is queued on a held stream; eight more keys clear the cache."""
    cfg, sd, m = build("improved")
    h_in = [mixture(2, 1, 1600, seed=20 + k).pin_memory() for k in range(9)]
    h_out = [torch.empty(2, 2, 1600).pin_memory() for _ in range(9)]
    _engine.forward_host(m, h_in[0], h_out[0])
    _engine.forward_host(m, h_in[0], h_out[0])          # captured
    torch.cuda.synchronize()
    want = h_out[0].clone()
    h_out[0].fill_(float("nan"))
    graphs = _engine._state(m, torch.device(DEV, torch.cuda.current_device())).graphs
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        hold()
        _engine.forward_host(m, h_in[0], h_out[0])      # replayed
    for k in range(1, 9):
        _engine.forward_host(m, h_in[k], h_out[k])
    assert len(graphs) == 1, "the cache was not cleared"
    torch.cuda.synchronize()
    same(h_out[0], want, exact=False)
    for k in range(9):
        fp64(h_out[k], O.forward(cfg, sd, h_in[k], dtype=torch.float64))


@gpu
def test_corpus_graphs_evicted_while_replays_are_queued():
    """``max_graphs=2``: two passes capture the two slots of one bucket; a third pass replays both behind a held
    stream, and its next bucket clears the cache while those replays are still queued."""
    cfg, sd, m = build("improved")
    short = [mixture(T, seed=T) + 0.2 for T in (1500, 1510, 1520, 1530)]       # one bucket, two batches of two
    wavs = short + [mixture(2300, seed=2300) + 0.2]                               # a second bucket, one batch of one
    want = CorpusSeparator(m, max_batch=2, use_graphs=False).run(wavs)
    sep = CorpusSeparator(m, max_batch=2, max_graphs=2)
    sep.run(short)
    sep.run(short)
    assert sep.launches["captured"] == 2, sep.launches
    held = torch.cuda.Stream()
    with torch.cuda.stream(held):
        hold()
        got = sep.run(wavs)
    assert sep.launches["replayed"] == 2 and len(sep.graphs) == 1, (sep.launches, sep.graphs)
    for g, w in zip(got, want):
        same(g, w, exact=False)
    fp64(torch.cat(got, -1).unsqueeze(0),
         torch.cat([O.separate(cfg, sd, w[None].double(), dtype=torch.float64)[0] for w in wavs], -1).unsqueeze(0))


# ---------------------------------------------------------------------------------------------------------------------
# 3. One CausalStream across streams
# ---------------------------------------------------------------------------------------------------------------------
def alternated(s, chunks, streams, hold_on):
    """Steps, a reset of slot 1 and the flush, the i-th on ``streams[i % len(streams)]``; those in ``hold_on`` sleep
    first."""
    ops = [("step", 0), ("step", 1), ("reset", None), ("step", 2), ("step", 3), ("flush", None)]
    outs = []
    for i, (op, k) in enumerate(ops):
        st = streams[i % len(streams)]
        with torch.cuda.stream(st):
            if st in hold_on:
                hold()
            if op == "step":
                outs.append(s.step(chunks[k]))
            elif op == "reset":
                s.reset([1])
            else:
                outs.append(s.flush())
    return outs


@gpu
def test_causal_stream_alternating_streams():
    cfg, sd, m = build("causal")
    Cs = 4 * granule(cfg)
    x = mixture(3, 1, 4 * Cs, seed=30)
    chunks = [x[..., k * Cs:(k + 1) * Cs].to(DEV) for k in range(4)]
    with torch.no_grad():
        cur = torch.cuda.current_stream()
        want = alternated(m.stream(3, Cs), chunks, [cur], [])
        torch.cuda.synchronize()
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        s = m.stream(3, Cs)
        got = alternated(s, chunks, [a, b], [a])
        torch.cuda.synchronize()
    for k, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"output {k}: max |d| = {(g - w).abs().max().item():.3e}"
    # slots 0 and 2 stream all four chunks; slot 1 starts over at chunk 2
    whole = CausalStreamOracle(cfg, sd, 3)
    ref = [whole.step(x[..., k * Cs:(k + 1) * Cs]) for k in range(4)] + [whole.flush()]
    fresh = CausalStreamOracle(cfg, sd, 1)
    ref1 = [ref[0][1:2], ref[1][1:2]] + [fresh.step(x[1:2, :, k * Cs:(k + 1) * Cs]) for k in (2, 3)] + [fresh.flush()]
    for k in range(5):
        for row, r in ((0, ref[k][0:1]), (1, ref1[k]), (2, ref[k][2:3])):
            fp64(got[k][row:row + 1], r)


@gpu
@pytest.mark.parametrize("inner", ["causal", "windowed"])
def test_resampled_stream_alternating_streams(inner):
    """A ``ResampledStream`` at 44.1 kHz around the model at 8 kHz: its two resamplers, the inner stream (a
    ``CausalStream`` or a ``WindowedStream``) and the inner stream's masked reset.  The steps alternate between two
    side streams, the first of them held; ``reset([1])`` runs on the other stream than the step before it and the flush
    on a third.  Bitwise the same calls on one stream."""
    cfg, sd, m = build("causal")
    Cs = 4 * 441                    # 320 samples at 8 kHz: four granules of the causal stream, one hop of the windows
    x = mixture(3, 1, 4 * Cs, seed=31)
    chunks = [x[..., k * Cs:(k + 1) * Cs].to(DEV) for k in range(4)]

    def make():
        if inner == "causal":
            return m.stream(3, Cs, sample_rate=44100, model_rate=8000)
        return m.stream_windows(3, Cs, 480, 320, sample_rate=44100, model_rate=8000)
    with torch.no_grad():
        want = alternated(make(), chunks, [torch.cuda.current_stream()], [])
        torch.cuda.synchronize()
        a, b, c = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
        s = make()
        assert isinstance(s, P.ResampledStream)
        got = alternated(s, chunks, [a, b, a, b, a, c], [a])
        torch.cuda.synchronize()
    for k, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"output {k}: max |d| = {(g - w).abs().max().item():.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# 4. Host threads in a fresh process: first launches race through the opt-in table and the SM-count cache
# ---------------------------------------------------------------------------------------------------------------------
THREADS = r'''
import json, sys, threading
import torch
import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200.bss_eval import bss_eval_sources
from sudo_rm_rf_b200.sisdr import PermInvariantSISDR
from oracle import sudormrf_oracle as O
from stream_oracle import CausalStreamOracle, granule
import bss_oracle

DEV = "cuda"
G = lambda *s, seed: torch.randn(*s, generator=torch.Generator().manual_seed(seed))


def model(variant, kw, seed):
    cfg = O.Config(variant=variant, **kw)
    sd = O.make_state_dict(cfg, seed=seed)
    m = {"improved": P.SuDORMRF, "groupcomm": P.GroupCommSudoRmRf, "causal": P.CausalSuDORMRF,
         "original": P.OriginalSuDORMRF}[variant](**kw)
    m.load_state_dict(sd)
    return cfg, sd, m.to(DEV).eval()


def forward_case(variant, kw, A=1):
    cfg, sd, m = model(variant, kw, seed=3)
    x = G(2, A, 1600, seed=4)

    def run():
        with torch.no_grad():
            return m(x.to(DEV))
    return run, lambda: O.forward(cfg, sd, x, dtype=torch.float64), variant == "causal"


def stream_case():
    kw = dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
              enc_num_basis=64, num_sources=2)
    cfg, sd, m = model("causal", kw, seed=5)
    Cs = 4 * granule(cfg)
    x = G(2, 1, 2 * Cs, seed=6)

    def run():
        s = m.stream(2, Cs)
        with torch.no_grad():
            return torch.cat([s.step(x[..., :Cs].to(DEV)), s.step(x[..., Cs:].to(DEV))], -1)
    o = CausalStreamOracle(cfg, sd, 2)
    return run, lambda: torch.cat([o.step(x[..., :Cs]), o.step(x[..., Cs:])], -1), True


def bss_case():
    ref, est = G(2, 3, 4000, seed=7).double(), None
    est = torch.einsum("ij,bjt->bit", torch.tensor([[1.0, 0.3, 0.1], [0.2, 1.0, 0.3], [0.1, 0.2, 1.0]],
                                                    dtype=torch.float64), ref) + 0.1 * G(2, 3, 4000, seed=8).double()
    ref, est = ref.float(), est.float()

    def run():
        return torch.cat([t.double() for t in bss_eval_sources(ref.to(DEV), est.to(DEV), filter_length=32)], -1)

    def oracle():
        rows = []
        for b in range(2):
            sdr, sir, sar, perm = bss_oracle.bss_eval(ref[b].double().numpy(), est[b].double().numpy(), True, 32)
            rows.append(torch.cat([torch.as_tensor(v, dtype=torch.float64) for v in (sdr, sir, sar, perm)]))
        return torch.stack(rows)
    return run, oracle, True


def pit_case():
    tgt = G(4, 3, 3000, seed=9)
    pr = tgt[:, [2, 0, 1]] + 0.3 * G(4, 3, 3000, seed=10)
    metric = PermInvariantSISDR(batch_size=4, n_sources=3, backward_loss=False, return_individual_results=True)

    def run():
        with torch.no_grad():
            return metric(pr.to(DEV), tgt.to(DEV)).reshape(-1).double()
    return run, lambda: O.pit_sisdr(pr.double(), tgt.double())[0].reshape(-1), False


def backward_case():
    kw = dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
              enc_num_basis=64, num_sources=2)
    cfg, sd, m = model("improved", kw, seed=11)
    m.train().enable_training()
    x, g = G(2, 1, 1600, seed=12), G(2, 2, 1600, seed=13)

    def run():
        m.zero_grad(set_to_none=True)
        (m(x.to(DEV)) * g.to(DEV)).sum().backward()
        return torch.cat([p.grad.reshape(-1) for p in m.parameters()])

    def oracle():
        sd64 = {k: v.double().requires_grad_() for k, v in sd.items()}
        (O.forward(cfg, sd64, x, dtype=torch.float64) * g.double()).sum().backward()
        names = [n for n, _ in m.named_parameters()]
        return torch.cat([sd64[n].grad.reshape(-1) for n in names])
    return run, oracle, True


CASES = {
    # every 1x1 on wgmma
    "improved_wgmma": forward_case("improved", dict(out_channels=128, in_channels=128, num_blocks=2, upsampling_depth=4,
                                                    enc_kernel_size=21, enc_num_basis=256, num_sources=2)),
    # 16 channels per group: tac_mma16_kernel
    "groupcomm_tac_mma16": forward_case("groupcomm", dict(in_audio_channels=2, out_channels=32, in_channels=64,
                                                          num_blocks=2, upsampling_depth=4, enc_kernel_size=21,
                                                          enc_num_basis=64, num_sources=2, group_size=2), A=2),
    "causal": forward_case("causal", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                          enc_kernel_size=21, enc_num_basis=128, num_sources=2)),
    "original": forward_case("original", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                              enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    "stream_step": stream_case(),
    "bss_eval_sources": bss_case(),
    "pit_sisdr": pit_case(),
    "train_backward": backward_case(),
}
names = list(CASES)
barrier = threading.Barrier(len(names))
first, errors = {}, {}


def worker(name):
    run = CASES[name][0]
    s = torch.cuda.Stream()
    try:
        barrier.wait(60)
        with torch.cuda.stream(s):
            out = run()
        s.synchronize()
        first[name] = out.cpu()
    except BaseException as e:
        errors[name] = repr(e)


threads = [threading.Thread(target=worker, args=(n,)) for n in names]
for t in threads:
    t.start()
for t in threads:
    t.join(300)
report = {"errors": errors, "alive": [n for n, t in zip(names, threads) if t.is_alive()], "cases": {}}
for name in names:
    if name not in first:
        continue
    run, oracle, exact = CASES[name]
    again = run().cpu()
    got = first[name]
    ref = oracle()
    scale = again.abs().max().item()
    fin = torch.isfinite(ref)
    report["cases"][name] = {
        "exact": exact, "bitwise": bool(torch.equal(got, again)),
        "repeat": (got - again).abs().max().item() / max(scale, 1e-30),
        "fp64": ((got.double() - ref)[fin].abs().max().item() / max(ref[fin].abs().max().item(), 1e-30)),
        "fp64_l2": ((got.double() - ref)[fin].norm().item() / max(ref[fin].norm().item(), 1e-30)),
        "shape_ok": tuple(got.shape) == tuple(ref.shape),
    }
print("RESULT " + json.dumps(report))
'''


@gpu
def test_first_launches_from_racing_threads():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([REPO, os.path.join(REPO, "tests")]))
    flags = ["-s"] if sys.flags.no_user_site else []
    p = subprocess.run([sys.executable, *flags, "-c", THREADS], cwd=REPO, env=env, capture_output=True, text=True,
                       timeout=600)
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
    assert p.returncode == 0 and line, (p.returncode, p.stdout[-2000:], p.stderr[-4000:])
    report = json.loads(line[-1][len("RESULT "):])
    assert not report["errors"] and not report["alive"], report
    assert len(report["cases"]) == 8, report
    for name, r in report["cases"].items():
        print(name, r)
        assert r["shape_ok"], (name, r)
        if r["exact"]:
            assert r["bitwise"], (name, r)
        else:
            assert r["repeat"] <= 1e-5, (name, r)
        if name == "train_backward":       # the whole-model gradient bar of test_gpu_train.py
            assert r["fp64_l2"] <= 1e-2, (name, r)
        else:
            assert r["fp64"] < 1e-3, (name, r)


# ---------------------------------------------------------------------------------------------------------------------
# 5. One model shared by host threads
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_one_model_two_threads(monkeypatch):
    """Two threads run ``model(x)``, ``separate`` and ``forward_host`` on one model, each on its own stream.  Thread 1
    holds its stream and, inside its first enqueue, waits until thread 2 has entered ``_call_shared`` and (for at
    most 0.5 s) until thread 2 reaches its own enqueue.  Thread 2's first call must still run after thread 1's."""
    cfg, sd, m = build("improved")
    xs = [mixture(2, 1, 1600, seed=40), mixture(3, 1, 2400, seed=41)]
    hosts = [x.pin_memory() for x in xs]
    xds = [x.to(DEV) for x in xs]

    def work(i):
        with torch.no_grad():
            y = m(xds[i])
            z = m.separate(xds[i][:, 0], normalize=True)
        h = _engine.forward_host(m, hosts[i], use_graph=False)
        return [y, z, h]
    want = [work(0), work(1)]
    torch.cuda.synchronize()
    want = [[t.clone() for t in w] for w in want]

    entered, reached, inside = threading.Event(), threading.Event(), threading.Event()
    ev1, ev1_recorded, order = torch.cuda.Event(), threading.Event(), {}
    who = {}
    orig = _engine._call_shared

    def call_shared(model, cfg_, device, ws_bytes, refusal, enqueue):
        me = who.get(threading.current_thread())
        first = me is not None and not who.get(("done", me))
        if first and me == 2:
            entered.set()

        def hooked(packed, ws):
            if first and me == 1:
                inside.set()
                assert entered.wait(30), "thread 2 never entered _call_shared"
                reached.wait(0.5)
            if first and me == 2:
                reached.set()
            enqueue(packed, ws)
            if first and me == 1:
                ev1.record()
                ev1_recorded.set()
        r = orig(model, cfg_, device, ws_bytes, refusal, hooked)
        if me is not None:
            who[("done", me)] = True
        return r
    monkeypatch.setattr(_engine, "_call_shared", call_shared)
    got, errs = {}, []
    streams = {1: torch.cuda.Stream(), 2: torch.cuda.Stream()}

    def thread(i):
        try:
            s = streams[i]
            with torch.cuda.stream(s):
                if i == 1:
                    hold()
                else:
                    assert inside.wait(30)
                with torch.no_grad():
                    y = m(xds[i - 1])
                if i == 2:
                    ev2 = torch.cuda.Event()
                    ev2.record(s)
                    ev2.synchronize()
                    order["waited"] = ev1_recorded.is_set() and ev1.query()
                with torch.no_grad():
                    z = m.separate(xds[i - 1][:, 0], normalize=True)
                h = _engine.forward_host(m, hosts[i - 1], use_graph=False)
                s.synchronize()
            got[i] = [y, z, h]
        except BaseException as e:
            errs.append(e)
            entered.set()
            inside.set()
    ts = {i: threading.Thread(target=thread, args=(i,)) for i in (1, 2)}
    for i, t in ts.items():
        who[t] = i
    for t in ts.values():
        t.start()
    for t in ts.values():
        t.join(60)
    assert not errs, errs
    assert all(not t.is_alive() for t in ts.values())
    torch.cuda.synchronize()
    assert order["waited"], "thread 2's first call did not wait for thread 1's, which sat behind the sleep"
    for i in (1, 2):
        for g, w in zip(got[i], want[i - 1]):
            same(g, w, exact=False)
        fp64(got[i][0], O.forward(cfg, sd, xs[i - 1], dtype=torch.float64))
        fp64(got[i][1], O.separate(cfg, sd, xs[i - 1][:, 0].double(), dtype=torch.float64))


# ---------------------------------------------------------------------------------------------------------------------
# 6. CPU: every Python entry that enqueues device work is exercised above
# ---------------------------------------------------------------------------------------------------------------------
COVERED = {
    "_engine.forward": ["test_stream_step_survives_a_repack", "test_buffers_released_during_a_call",
                        "test_workspace_growth_on_a_second_stream", "test_one_model_two_threads",
                        "test_first_launches_from_racing_threads"],
    "_engine.separate": ["test_buffers_released_during_a_call", "test_one_model_two_threads"],
    "_engine.forward_host": ["test_buffers_released_during_a_call", "test_workspace_growth_on_a_second_stream",
                             "test_forward_host_graph_evicted_while_its_replay_is_queued", "test_one_model_two_threads"],
    "corpus.separate_corpus": ["test_second_stream_waits_for_the_first (test_gpu_engine_streams.py)"],
    "corpus.CorpusSeparator.run": ["test_corpus_run_while_another_thread_repacks",
                                   "test_corpus_graphs_evicted_while_replays_are_queued"],
    "streaming.CausalStream.step": ["test_stream_step_survives_a_repack", "test_forward_reads_weights_a_step_packed",
                                    "test_stream_deleted_while_a_step_is_in_flight",
                                    "test_causal_stream_alternating_streams", "test_first_launches_from_racing_threads"],
    "streaming.CausalStream.reset": ["test_causal_stream_alternating_streams"],
    "streaming.CausalStream.flush": ["test_causal_stream_alternating_streams"],
    "streaming.CausalStream._reset_masked": ["test_resampled_stream_alternating_streams"],
    "window_stream.WindowedStream.step": ["test_steps_alternating_between_cuda_streams (test_gpu_window_stream.py)",
                                         "test_resampled_stream_alternating_streams"],
    "window_stream.WindowedStream.reset": ["test_steps_alternating_between_cuda_streams (test_gpu_window_stream.py)"],
    "window_stream.WindowedStream.flush": ["test_steps_alternating_between_cuda_streams (test_gpu_window_stream.py)",
                                          "test_resampled_stream_alternating_streams"],
    "window_stream.WindowedStream._reset_masked": ["test_resampled_stream_alternating_streams"],
    "resample_stream.ResampleStream._step": [
        "test_alternating_cuda_streams_and_host_threads (test_gpu_resample_stream.py)",
        "test_resampled_stream_alternating_streams"],
    "resample_stream.ResampleStream._flush": [
        "test_alternating_cuda_streams_and_host_threads (test_gpu_resample_stream.py)",
        "test_resampled_stream_alternating_streams"],
    "resample_stream.ResampleStream.reset": ["test_resampled_stream_alternating_streams"],
    "resample_stream.ResampledStream.step": ["test_resampled_stream_alternating_streams"],
    "resample_stream.ResampledStream.reset": ["test_resampled_stream_alternating_streams"],
    "resample_stream.ResampledStream.flush": ["test_resampled_stream_alternating_streams"],
    "training._NativeTrain.forward": ["test_training_on_a_side_stream_survives_a_repack",
                                      "test_buffers_released_during_a_call"],
    "training._NativeTrain.backward": ["test_training_on_a_side_stream_survives_a_repack",
                                       "test_first_launches_from_racing_threads"],
    "bss_eval.bss_eval_sources": ["test_first_launches_from_racing_threads"],
    "sisdr.PermInvariantSISDR.forward": ["test_first_launches_from_racing_threads"],
}
# Entries whose buffers are all allocated, read and released on the caller's stream within the call (per-call scratch
# and outputs): the caching allocator orders their reuse by itself, and no state outlives the call.
PER_CALL = {"sisdr.StabilizedPermInvSISDRMetric.forward", "sisdr._PairwiseNegSDR.forward",
            "sisdr._PairwiseNegSDR.backward", "sisdr.PairwiseNegSDR.forward", "snr._forward",
            "snr._SNRZeroRefs.backward", "mixture_consistency._project", "mixture_consistency._Consistency.backward",
            "windowed.gather", "windowed.merge", "resample.resample_poly", "stoi_metric.stoi"}
# The shared machinery every entry above goes through.
MACHINERY = {"_engine._call_shared", "_engine.packed_weights", "streaming.SlotStream._ordered"}


def enqueuing_functions():
    """``module.Class.method`` of every function in the package that hands a stream to the library (``N.stream``), runs
    a call on the model's shared state (``_call_shared``) or orders a stream's calls (``_ordered``)."""
    found = set()
    for path in glob.glob(os.path.join(REPO, "sudo_rm_rf_b200", "*.py")):
        mod = os.path.basename(path)[:-3]

        def walk(node, prefix):
            for ch in ast.iter_child_nodes(node):
                if isinstance(ch, ast.ClassDef):
                    walk(ch, prefix + ch.name + ".")
                elif isinstance(ch, ast.FunctionDef):
                    src = ast.unparse(ch)
                    if "N.stream(" in src or "_call_shared(" in src or "_ordered(" in src:
                        found.add(mod + "." + prefix + ch.name)
        walk(ast.parse(open(path).read()), "")
    return found


def test_every_enqueuing_or_ordered_entry_is_covered():
    found = enqueuing_functions()
    assert len(found) >= 20
    listed = set(COVERED) | PER_CALL | MACHINERY
    assert found == listed, (sorted(found - listed), sorted(listed - found))
    here = set(globals())
    for entry, tests in COVERED.items():
        for t in tests:
            assert t.split(" ")[0] in here or "(" in t, (entry, t)
