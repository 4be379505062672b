"""Calls on one model from two CUDA streams hand the model's shared workspace over.

A model keeps one workspace (and one staging buffer) per device, shared by every native call that runs on its cached
state.  A call that arrives on a different stream than the previous one must wait for it.  Here each such entry, and
the plain forward it shares the workspace with, run across two streams A and B in both orders: A sleeps, the first
call is enqueued on A, the second on B.  Once B's work is done A's must be too, so B waited for A; and both results
equal the same two calls run one after the other on one stream.
"""
import itertools

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200.corpus import separate_corpus
from oracle import sudormrf_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLEEP = 200_000_000     # cycles: about 0.1 s, far longer than any call here
KW = dict(out_channels=32, in_channels=64, num_blocks=2, upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64,
          num_sources=2)


def model(variant):
    m = {"improved": P.SuDORMRF, "causal": P.CausalSuDORMRF}[variant](**KW)
    m.load_state_dict(O.make_state_dict(O.Config(variant=variant, **KW), seed=5))
    return m.to(DEV).eval()


def mixture(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def inference(m, x):
    def run():
        with torch.no_grad():
            return m(x)
    return run


def e_forward(variant):
    m = model(variant)
    return m, inference(m, mixture(2, 1, 4000, seed=1).to(DEV))


def e_separate():
    m = model("improved")
    wav = (mixture(2, 4000, seed=2) * 3.0 + 0.5).to(DEV)

    def run():
        with torch.no_grad():
            return m.separate(wav, normalize=True)
    return m, run


def e_forward_host():
    m = model("improved")
    h_in = mixture(2, 1, 4000, seed=3).pin_memory()
    h_out = itertools.cycle([torch.empty(2, 2, 4000).pin_memory() for _ in range(2)])    # one per run of the pair
    return m, lambda: _engine.forward_host(m, h_in, next(h_out), use_graph=False)


def e_train():
    m = model("improved").enable_training()
    x = mixture(2, 1, 4000, seed=4).to(DEV)

    def run():
        y = m(x)
        assert y.grad_fn is not None
        return y.detach()
    return m, run


def e_separate_corpus():
    m = model("improved")
    wavs = [(mixture(T, seed=T) * 2.0 + 0.1).to(DEV) for T in (1500, 2300, 977)]     # three buckets
    return m, lambda: torch.cat(separate_corpus(m, wavs), -1)


ENTRIES = {"forward_improved": lambda: e_forward("improved"), "forward_causal": lambda: e_forward("causal"),
           "separate": e_separate, "forward_host": e_forward_host, "train_forward": e_train,
           "separate_corpus": e_separate_corpus}


@pytest.mark.parametrize("entry_first", [True, False], ids=["entry_on_A", "entry_on_B"])
@pytest.mark.parametrize("name", list(ENTRIES))
def test_second_stream_waits_for_the_first(name, entry_first):
    m, entry = ENTRIES[name]()
    forward = inference(m, mixture(3, 1, 1600, seed=6).to(DEV))
    first, second = (entry, forward) if entry_first else (forward, entry)
    want = (first(), second())                  # one stream; also sizes the workspace and packs the weights
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    ev_a, ev_b = torch.cuda.Event(), torch.cuda.Event()
    with torch.cuda.stream(a):
        torch.cuda._sleep(SLEEP)
        got_first = first()
        ev_a.record(a)
    with torch.cuda.stream(b):
        got_second = second()
        ev_b.record(b)
    ev_b.synchronize()
    assert ev_a.query(), f"{name}: the call on B did not wait for the call on A"
    torch.cuda.synchronize()
    for got, ref, what in ((got_first, want[0], "first"), (got_second, want[1], "second")):
        assert torch.equal(got, ref), f"{name}: the {what} result differs from the one-stream run"
