"""Every native path runs the weights the module holds now, and a captured forward keeps the memory it addresses.

Each native call reads the weights from a cached packed buffer, re-packed when the weight signature changes
(sudo_rm_rf_b200/_engine.py).  Here every entry point (model(x) of the four models, one with its 1x1 convolutions and
encoder on wgmma, separate(), forward_host eager and through its internal graph, separate_corpus, CorpusSeparator.run
with graphs, CausalStream.step, and the enable_training() forward and backward) meets every way a user changes weights:
load_state_dict, in-place writes under no_grad, through detach() and through state_dict() tensors, nn.init, SGD, Adam
and AdamW steps (foreach and fused), p.data = t at an address the cache has seen, and a replaced Parameter.  After
the change the output is held to the fp64 oracle on the new state_dict, and must differ from the old output, so an
update that changes nothing cannot pass.  Writes that bypass the version counter (p.data ops, DLPack,
dist.broadcast(p.data)) are held to the new weights after refresh_weights().  The runner loop of test_gpu_train runs
with fused optimizers.

Then graphs captured as bench.py captures them (eager warm-up, capture on a side stream) for model(x), separate() and
CausalStream.step, against workspace growth, a repack, and both: sentinels of exactly the sizes of the buffers the cache
held at capture take whatever the allocator frees, and one replay must leave them intact and give the pre-change
output.  torch.cuda.empty_cache() is never called here, so every block a stale replay could touch belongs to a sentinel.
"""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
from torch.utils import dlpack

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N
from sudo_rm_rf_b200.corpus import CorpusSeparator, separate_corpus
from oracle import sudormrf_oracle as O
from stream_oracle import granule
from test_gpu_long import normalised_input
from test_gpu_model_space import TOL, build, paths
from test_gpu_stream import TOL as STREAM_TOL
from test_gpu_train import RUNNER, _oracle_step_params, _runner_loop, nn_prelu_oracle, oracle_grads

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHANGED = 1e-3          # an update must move the output by more than this, relative to max|old output|
GRAD_TOL = 1e-2         # whole-model gradient, rel-L2 against fp64 (test_gpu_train.assert_grads_match)

MODELS = {
    # the 1x1 convolutions (256 x 128 and 128 x 256), encoder, mask and decoder all on wgmma: bf16 hi/lo images
    "improved_wgmma": ("improved", dict(out_channels=128, in_channels=256, num_blocks=2, upsampling_depth=4,
                                        enc_kernel_size=21, enc_num_basis=256, num_sources=2)),
    "groupcomm": ("groupcomm", dict(in_audio_channels=1, out_channels=64, in_channels=128, num_blocks=2,
                                    upsampling_depth=4, enc_kernel_size=21, enc_num_basis=64, num_sources=2,
                                    group_size=4)),
    "causal": ("causal", dict(in_audio_channels=1, out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                              enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
    "original": ("original", dict(out_channels=64, in_channels=128, num_blocks=2, upsampling_depth=4,
                                  enc_kernel_size=21, enc_num_basis=64, num_sources=2)),
}


def new_sd(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def rel_change(a, b):
    return ((a.double().cpu() - b.double().cpu()).abs().max() / b.double().abs().max().cpu()).item()


def perturbed(t, seed):
    """t * (1 + 0.05 r), r standard normal: every weight moves, none far."""
    r = torch.randn(t.shape, generator=torch.Generator().manual_seed(seed)).to(t.device)
    return (t.detach() * (1 + 0.05 * r)).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# entry points: each returns (run, oracle); run() gives the outputs, oracle(sd) the fp64 oracle's on weights sd
# ---------------------------------------------------------------------------------------------------------------------
class Entry:
    def __init__(self, model, run, oracle, training=False):
        self.cfg, self.m = model
        self.run, self.oracle, self.training = run, oracle, training
        self.tol = tol_of(self.cfg)


def tol_of(cfg):
    """test_gpu_model_space's bar; the causal model's is test_gpu_stream's."""
    return STREAM_TOL if cfg.variant == "causal" else TOL


def make_model(key):
    variant, kw = MODELS[key]
    cfg, _, m = build(variant, kw, seed=31)
    return cfg, m


def e_forward(key):
    def make():
        cfg, m = make_model(key)
        A = cfg.in_audio_channels if cfg.variant == "groupcomm" else 1
        x = normalised_input(2, A, 2001, seed=41).to(DEV)

        def run():
            with torch.no_grad():
                return m(x)
        return Entry((cfg, m), run, lambda sd: O.forward(cfg, sd, x, dtype=torch.float64))
    return make


def e_separate():
    cfg, m = make_model("improved_wgmma")
    g = torch.Generator().manual_seed(43)
    wav = (torch.randn(2, 2001, generator=g) * torch.tensor([[0.05], [4.0]]) + torch.tensor([[0.3], [-1.0]])).to(DEV)

    def run():
        with torch.no_grad():
            return m.separate(wav, normalize=True)
    return Entry((cfg, m), run, lambda sd: O.separate(cfg, sd, wav, dtype=torch.float64))


def e_forward_host(graph):
    def make():
        cfg, m = make_model("improved_wgmma")
        x = normalised_input(2, 1, 2001, seed=47)
        h_in = x.pin_memory() if graph else x.clone()
        h_out = torch.empty(2, 2, 2001).pin_memory() if graph else None

        def run():
            st = _engine._state(m, torch.device(DEV, torch.cuda.current_device()))
            with torch.no_grad():
                for _ in range(3 if graph else 1):      # warm-up, capture, replay
                    out = m.forward_host(h_in, h_out)
            torch.cuda.synchronize()
            if graph:
                assert any(isinstance(v, torch.cuda.CUDAGraph) for v in st.graphs.values())
            return out.clone()
        return Entry((cfg, m), run, lambda sd: O.forward(cfg, sd, x.to(DEV), dtype=torch.float64))
    return make


CORPUS_T = (1500, 2300, 977)


def corpus_oracle(cfg, wavs):
    return lambda sd: torch.cat([O.separate(cfg, sd, w.to(DEV)[None], dtype=torch.float64)[0] for w in wavs], -1)


def e_separate_corpus():
    cfg, m = make_model("improved_wgmma")
    wavs = [normalised_input(1, 1, T, seed=T)[0, 0] * 2.0 + 0.1 for T in CORPUS_T]

    def run():
        return torch.cat(separate_corpus(m, [w.to(DEV) for w in wavs]), -1)
    return Entry((cfg, m), run, corpus_oracle(cfg, wavs))


def e_corpus_separator():
    cfg, m = make_model("improved_wgmma")
    wavs = [normalised_input(1, 1, T, seed=T + 1)[0, 0] * 2.0 + 0.1 for T in CORPUS_T]
    cs = CorpusSeparator(m, max_batch=2, use_graphs=True)

    def run():
        for _ in range(3):                  # eager, capture, replay
            replayed = cs.launches["replayed"]
            res = cs.run(wavs)
        assert cs.launches["replayed"] > replayed
        return torch.cat(res, -1)
    return Entry((cfg, m), run, corpus_oracle(cfg, wavs))


def e_stream_step():
    cfg, m = make_model("causal")
    C_ = 2 * granule(cfg)
    x = normalised_input(2, 1, 3 * C_, seed=53).to(DEV)
    s = m.stream(2, C_)
    hop = cfg.hop

    def run():
        s.reset()
        with torch.no_grad():
            out = torch.cat([s.step(x[..., i:i + C_]) for i in range(0, x.shape[-1], C_)], -1)
        return out[..., hop:]
    return Entry((cfg, m), run, lambda sd: O.forward(cfg, sd, x, dtype=torch.float64)[..., :x.shape[-1] - hop])


def e_training():
    cfg, m = make_model("improved_wgmma")
    m.enable_training().train()
    x = normalised_input(2, 1, 2001, seed=59)
    G = torch.randn(2, 2, 2001, generator=torch.Generator().manual_seed(61)).to(DEV)

    def loss_fn(y):
        return (y * G.to(y.dtype)).sum()

    def run():
        m.zero_grad(set_to_none=True)
        y = m(x.to(DEV))
        assert y.grad_fn is not None
        loss_fn(y).backward()
        return y.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters()}

    def oracle(sd):
        with nn_prelu_oracle():
            y = O.forward(cfg, sd, x.to(DEV), dtype=torch.float64)
        return y, oracle_grads(cfg, sd, x, loss_fn)[0]
    return Entry((cfg, m), run, oracle, training=True)


ENTRIES = {
    "forward_improved_wgmma": e_forward("improved_wgmma"),
    "forward_groupcomm": e_forward("groupcomm"),
    "forward_causal": e_forward("causal"),
    "forward_original": e_forward("original"),
    "separate": e_separate,
    "forward_host_eager": e_forward_host(False),
    "forward_host_graph": e_forward_host(True),
    "separate_corpus": e_separate_corpus,
    "corpus_separator": e_corpus_separator,
    "stream_step": e_stream_step,
    "training": e_training,
}


# ---------------------------------------------------------------------------------------------------------------------
# update idioms
# ---------------------------------------------------------------------------------------------------------------------
def u_load_state_dict(m):
    m.load_state_dict({k: perturbed(v, i) for i, (k, v) in enumerate(m.state_dict().items())})


def u_no_grad_inplace(m):
    with torch.no_grad():
        for i, p in enumerate(m.parameters()):
            p.mul_(perturbed(torch.ones_like(p), i))


def u_detach_write(m):
    for i, p in enumerate(m.parameters()):
        p.detach().copy_(perturbed(p, i))


def u_state_dict_write(m):
    for i, v in enumerate(m.state_dict().values()):
        v.copy_(perturbed(v, i))


def u_nn_init(m):
    g = torch.Generator(device=DEV).manual_seed(5)
    nn.init.xavier_uniform_(m.decoder.weight, generator=g)


def u_optimizer(name, fused):
    def update(m):
        params = list(m.parameters())
        targets = [perturbed(p, i) for i, p in enumerate(params)]
        for p, t in zip(params, targets):
            p.grad = p.detach() - t
        lr = 1.0 if name == "SGD" else 2e-3          # SGD(lr=1) lands on the targets; Adam moves each weight by ~lr
        opt = getattr(torch.optim, name)(params, lr=lr, **({"fused": True} if fused else {"foreach": True}))
        opt.step()
        for p in params:
            p.grad = None
    return update


def u_data_at_seen_address(m):
    """p.data = t with t at the address the cache's signature holds for p, as two vector_to_parameters calls without
    a forward between them can produce.  The old storage is dropped, then same-size blocks are taken from the
    allocator until one lands on that address.  The cache keeps the storages of its signature, so with it the address
    stays taken; either the address came back or the cache holds it."""
    p = m.decoder.weight
    seen = p.data_ptr()
    new = perturbed(p, 7)
    p.data = torch.empty(0, device=DEV)
    hold, t = [], None
    for _ in range(2048):
        c = torch.empty_like(new)
        if c.data_ptr() == seen:
            t = c
            break
        hold.append(c)
    reused = t is not None
    if t is None:
        t = hold.pop()
    del hold
    t.copy_(new)
    p.data = t
    st = _engine._state(m, p.device)
    kept = [s.data_ptr() for s in (getattr(st, "storages", None) or [])]
    print(f"p.data = t: address {'reused' if reused else 'not reused'}; kept by the cache: {seen in kept}")
    assert reused or seen in kept


def u_replaced_parameter(m):
    m.decoder.weight = nn.Parameter(perturbed(m.decoder.weight, 9))


IDIOMS = {
    "load_state_dict": u_load_state_dict,
    "no_grad_inplace": u_no_grad_inplace,
    "detach_write": u_detach_write,
    "state_dict_write": u_state_dict_write,
    "nn_init": u_nn_init,
    "sgd_foreach": u_optimizer("SGD", False),
    "sgd_fused": u_optimizer("SGD", True),
    "adam_foreach": u_optimizer("Adam", False),
    "adam_fused": u_optimizer("Adam", True),
    "adamw_foreach": u_optimizer("AdamW", False),
    "adamw_fused": u_optimizer("AdamW", True),
    "data_at_seen_address": u_data_at_seen_address,
    "replaced_parameter": u_replaced_parameter,
}


def check_fresh(e, before, label):
    """The entry's outputs now against the oracle on the current state_dict, and moved away from `before`."""
    got = e.run()
    want = e.oracle(new_sd(e.m))
    if e.training:
        (y, grads), (y_ref, g_ref) = got, want
        num = sum(((grads[k].double() - g_ref[k]) ** 2).sum().item() for k in g_ref)
        den = sum((g_ref[k] ** 2).sum().item() for k in g_ref)
        g_err = (num / den) ** 0.5
        print(f"{label}: whole gradient rel_l2 {g_err:.2e}")
        assert g_err <= GRAD_TOL, g_err
        got, want, before = y, y_ref, (before[0] if before is not None else None)
    e_ = O.parity_errors(got, want)
    moved = rel_change(got, before) if before is not None else float("nan")
    print(f"{label}: rel_max {e_[0]:.3e} rel_l2 {e_[1]:.3e}; moved {moved:.2e} from the old output")
    assert max(e_) < e.tol, e_
    if before is not None:
        assert moved > CHANGED, moved
    return got


@pytest.mark.parametrize("idiom", list(IDIOMS))
@pytest.mark.parametrize("entry", list(ENTRIES))
def test_entry_point_runs_the_current_weights(entry, idiom):
    e = ENTRIES[entry]()
    before = e.run()
    check_fresh(e, None, f"{entry} before")
    IDIOMS[idiom](e.m)
    check_fresh(e, before, f"{entry} after {idiom}")


def test_improved_wgmma_model_runs_its_convolutions_on_tensor_cores():
    """The premise of improved_wgmma: the bf16 hi/lo images of every GEMM are part of what is re-packed."""
    variant, kw = MODELS["improved_wgmma"]
    cfg = O.Config(variant=variant, **kw)
    lib = N.lib()
    assert paths(cfg) == (True, True, True)
    assert lib.sdr_pointwise_mma_packed_bytes(kw["in_channels"], kw["out_channels"]) > 0       # proj_1x1
    assert lib.sdr_pointwise_mma_packed_bytes(kw["out_channels"], kw["in_channels"]) > 0       # res_conv


# ---------------------------------------------------------------------------------------------------------------------
# writes the version counter cannot see: refresh_weights()
# ---------------------------------------------------------------------------------------------------------------------
def w_data_mul(m):
    for i, p in enumerate(m.parameters()):
        p.data.mul_(perturbed(torch.ones_like(p), i))


def w_data_copy(m):
    for i, p in enumerate(m.parameters()):
        p.data.copy_(perturbed(p, i))


def w_dlpack(m):
    for i, p in enumerate(m.parameters()):
        dlpack.from_dlpack(dlpack.to_dlpack(p.data)).copy_(perturbed(p, i))


UNTRACKED = {"data_mul": w_data_mul, "data_copy": w_data_copy, "dlpack": w_dlpack}


@pytest.mark.parametrize("write", list(UNTRACKED))
@pytest.mark.parametrize("wrap", [False, True], ids=["module", "dataparallel"])
def test_untracked_writes_after_refresh_weights(write, wrap):
    e = e_forward("improved_wgmma")()
    before = e.run()
    versions = [p._version for p in e.m.parameters()]
    UNTRACKED[write](e.m)
    assert [p._version for p in e.m.parameters()] == versions         # invisible to the counter
    stale = e.run()
    print(f"{write} without refresh_weights: moved {rel_change(stale, before):.2e} from the old output")
    P.refresh_weights(nn.DataParallel(e.m, device_ids=[0]) if wrap else e.m)
    check_fresh(e, before, f"{write} + refresh_weights")


BROADCAST = r"""
import json, os, sys, torch
import torch.distributed as dist
sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
sys.path.insert(0, sys.argv[1])
rank = int(sys.argv[2])
dist.init_process_group("gloo", init_method="file://" + sys.argv[3], rank=rank, world_size=2)
import sudo_rm_rf_b200 as P
from oracle import sudormrf_oracle as O
from test_gpu_weight_cache import e_forward, new_sd, perturbed, rel_change
from test_gpu_model_space import TOL
e = e_forward("improved_wgmma")()
before = e.run()
if rank == 1:
    with torch.no_grad():
        for i, p in enumerate(e.m.parameters()):
            p.copy_(perturbed(p, i))
for p in e.m.parameters():
    dist.broadcast(p.data, src=1)
torch.cuda.synchronize()
stale = e.run()
P.refresh_weights(e.m)
y = e.run()
err = O.parity_errors(y, e.oracle(new_sd(e.m)))
print(json.dumps({"rank": rank, "err": max(err), "moved": rel_change(y, before), "stale": rel_change(stale, before)}))
dist.destroy_process_group()
"""


def test_dist_broadcast_of_data_after_refresh_weights(tmp_path):
    """dist.broadcast(p.data) from a rank with other weights (gloo, two processes on this GPU) writes past the version
    counter; after refresh_weights the receiving rank runs the broadcast weights."""
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    store = str(tmp_path / "store")
    procs = [subprocess.Popen([sys.executable, "-c", BROADCAST, repo, str(r), store], stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in (0, 1)]
    outs = [p.communicate(timeout=600) for p in procs]
    for p, (o, err) in zip(procs, outs):
        assert p.returncode == 0, err[-3000:]
    r0 = json.loads(outs[0][0].strip().splitlines()[-1])
    print(f"broadcast receiver: moved {r0['moved']:.2e} (without refresh_weights {r0['stale']:.2e}), "
          f"vs fp64 {r0['err']:.2e}")
    assert r0["err"] < TOL
    assert r0["moved"] > CHANGED


# ---------------------------------------------------------------------------------------------------------------------
# training with fused optimizers
# ---------------------------------------------------------------------------------------------------------------------
OPTS = {
    "Adam": lambda ps, **kw: torch.optim.Adam(ps, lr=1e-3, **kw),
    "AdamW": lambda ps, **kw: torch.optim.AdamW(ps, lr=1e-3, **kw),
    "SGD": lambda ps, **kw: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, **kw),
}


@pytest.mark.parametrize("opt", list(OPTS))
def test_runner_loop_fused_optimizer_tracks_oracle(opt):
    """test_gpu_train.test_runner_loop_adam_clip_tracks_oracle with a fused optimizer on the native side (the fp64
    trajectory uses the foreach one): the losses track fp64 step by step, and model(x) after the loop runs the final
    parameters."""
    cfg = O.Config(variant="improved", **RUNNER)
    sd = O.make_state_dict(cfg, seed=10)
    m = P.SuDORMRF(**RUNNER)
    m.load_state_dict(sd)
    m = m.to(DEV).enable_training().train()
    ln = _runner_loop(m, list(m.parameters()), lambda x: m(x.to(DEV)),
                      make_opt=lambda ps: OPTS[opt](ps, fused=True))
    p64 = _oracle_step_params(sd)

    def fwd(x):
        with nn_prelu_oracle():
            return O.forward(cfg, p64, x.to(DEV, torch.float64), dtype=torch.float64)
    lo = _runner_loop(None, list(p64.values()), fwd, make_opt=lambda ps: OPTS[opt](ps, foreach=True))
    print(f"{opt}(fused=True) native loss", [f"{v:.4f}" for v in ln])
    print(f"{opt}(foreach) fp64 loss     ", [f"{v:.4f}" for v in lo])
    for a, b in zip(ln, lo):
        assert abs(a - b) <= 1e-2 * abs(b)
    x = normalised_input(2, 1, 4000, seed=67).to(DEV)
    with torch.no_grad():
        y = m.eval()(x)
    e = O.parity_errors(y, O.forward(cfg, new_sd(m), x, dtype=torch.float64))
    moved = max(O.parity_errors(y, O.forward(cfg, sd, x, dtype=torch.float64)))
    print(f"model(x) after the loop: vs fp64 at the final parameters {max(e):.2e}, at the initial ones {moved:.2e}")
    assert max(e) < TOL, e
    assert moved > 10 * TOL


# ---------------------------------------------------------------------------------------------------------------------
# captured graphs against workspace growth and repacks
# ---------------------------------------------------------------------------------------------------------------------
def capture(m, call, pre=None):
    """bench.py's recipe: an eager warm-up, then a capture, both on one side stream.  -> (side stream, replay())."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        if pre is not None:
            pre()
        call()
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            y = call()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()

    def replay():
        with torch.cuda.stream(side):
            if pre is not None:
                pre()
            graph.replay()
        torch.cuda.synchronize()
        return y.clone()
    return side, replay


def capture_case(kind):
    """-> (cfg, model, call, pre, grow(), oracle(sd))."""
    if kind == "stream_step":
        cfg, m = make_model("causal")
        C_ = 2 * granule(cfg)
        inp = normalised_input(2, 1, C_, seed=71).to(DEV)
        out = torch.empty(2, 2, C_, device=DEV)
        s = m.stream(2, C_)
        big = normalised_input(2, 1, 6001, seed=73).to(DEV)
        hop = cfg.hop

        def call():
            return s.step(inp, out=out)

        def grow():
            with torch.no_grad():
                m(big)

        def oracle_cmp(y, sd):       # the first step after reset(): samples -hop .. C - hop - 1 of model(inp)
            return O.parity_errors(y[..., hop:], O.forward(cfg, sd, inp, dtype=torch.float64)[..., :C_ - hop])
        return cfg, m, call, s.reset, grow, oracle_cmp
    # workspaces above 10 MB: the allocator gives each its own segment, so a freed one is not merged into the next
    cfg, m = make_model("improved_wgmma")
    if kind == "forward":
        x = normalised_input(2, 1, 10001, seed=79).to(DEV)
        big = normalised_input(2, 1, 20001, seed=83).to(DEV)

        def call():
            return m(x)

        def grow():
            with torch.no_grad():
                m(big)
        return cfg, m, call, None, grow, lambda y, sd: O.parity_errors(y, O.forward(cfg, sd, x, dtype=torch.float64))
    g = torch.Generator().manual_seed(89)
    wav = (torch.randn(2, 10001, generator=g) * 3.0 + 0.5).to(DEV)
    big = (torch.randn(2, 20001, generator=g) * 3.0 + 0.5).to(DEV)

    def call():
        return m.separate(wav, normalize=True)

    def grow():
        with torch.no_grad():
            m.separate(big, normalize=True)
    return cfg, m, call, None, grow, lambda y, sd: O.parity_errors(y, O.separate(cfg, sd, wav, dtype=torch.float64))


@pytest.mark.parametrize("change", ["grow", "repack", "grow_and_repack"])
@pytest.mark.parametrize("kind", ["forward", "separate", "stream_step"])
def test_captured_graph_survives_the_cache(kind, change):
    cfg, m, call, pre, grow, oracle_cmp = capture_case(kind)
    side, replay = capture(m, call, pre)
    ref = replay()
    st = _engine._state(m, torch.device(DEV, torch.cuda.current_device()))
    held = [(name, b.numel(), b.data_ptr()) for name, b in (("workspace", st.workspace), ("packed", st.packed))
            if b is not None]
    # the calls and the sentinels stay on the stream the buffers were allocated on: its pool gets the freed blocks
    with torch.cuda.stream(side):
        if change != "grow":
            u_no_grad_inplace(m)
            with torch.no_grad():
                call()                   # an eager call: repack
        if change != "repack":
            grow()                       # an eager call with a larger T: workspace growth
        torch.cuda.synchronize()
        if change != "repack" and kind != "stream_step":
            assert st.workspace.numel() > held[0][1]
        if change != "grow":
            assert st.packed.data_ptr() != held[-1][2]
        sentinels = [torch.full((n,), 0xA5, dtype=torch.uint8, device=DEV) for _, n, _ in held]
    print(f"{kind} / {change}: sentinel took the freed block: "
          + ", ".join(f"{name} {s.data_ptr() == ptr}" for (name, _, ptr), s in zip(held, sentinels)))
    got = replay()
    for (name, _, _), s in zip(held, sentinels):
        assert bool((s == 0xA5).all()), f"the replay wrote into the block of the {name} it captured"
    d = (got - ref).abs().max().item()
    print(f"{kind} / {change}: replay vs pre-change replay max|d| {d:.2e} (max|ref| {ref.abs().max().item():.2e})")
    assert d <= 1e-6 * ref.abs().max().item()
    # a new capture after refresh_weights runs the new weights
    P.refresh_weights(m)
    _, replay2 = capture(m, call, pre)
    y2 = replay2()
    e = oracle_cmp(y2, new_sd(m))
    print(f"{kind} / {change}: re-captured graph vs fp64 on the current weights {max(e):.2e}")
    assert max(e) < tol_of(cfg), e
    if change != "grow":
        assert rel_change(y2, ref) > CHANGED
