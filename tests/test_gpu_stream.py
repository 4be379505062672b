"""Streaming of CausalSuDORMRF on the GPU: the concatenated steps against the fp64 oracle and the native offline
forward, the stream stage kernel against the one-pass causal pyramid and an fp64 chain at every depth and at each
channels-per-CTA width it picks, slot independence, reset, CUDA-graph replay,
mixture consistency, the launch count and argument errors.

Contract (model output delayed by hop samples):
    cat(step(x_0) .. step(x_{n-1}))[..., hop:] == model(x)[..., :n*C - hop]
    flush() == model(x)[..., n*C - hop:n*C]          when n*C % (hop * 2^D) == 0
Tolerance as everywhere else: <= 1e-3 max|ref| per sample and rel-L2 <= 1e-3 against the fp64 oracle; <= 1e-5 against
the native offline forward on the same weights (the same kernels in the same product order: usually bitwise)."""
import collections
import ctypes as C

import pytest
import torch

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine
from sudo_rm_rf_b200 import _native as N
from oracle import sudormrf_oracle as O
from guards import Guards
from stream_oracle import granule

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-3

DEFAULT = dict(in_audio_channels=1, out_channels=128, in_channels=512, num_blocks=16, upsampling_depth=4,
               enc_kernel_size=21, enc_num_basis=512, num_sources=2)
STEREO = dict(in_audio_channels=2, out_channels=256, in_channels=512, num_blocks=4, upsampling_depth=5,
              enc_kernel_size=21, enc_num_basis=512, num_sources=2)
SMALL = dict(in_audio_channels=1, out_channels=16, in_channels=24, num_blocks=2, upsampling_depth=3,
             enc_kernel_size=11, enc_num_basis=16, num_sources=2)          # every GEMM on the FFMA kernels, N < 32
MID = dict(in_audio_channels=1, out_channels=128, in_channels=256, num_blocks=2, upsampling_depth=4,
           enc_kernel_size=21, enc_num_basis=128, num_sources=2)


def build(kw, seed=11):
    cfg = O.Config(variant="causal", **kw)
    sd = O.make_state_dict(cfg, seed=seed)
    m = P.CausalSuDORMRF(**kw)
    m.load_state_dict(sd)
    return cfg, sd, m.to(DEV).eval()


def mixture(B, A, T, seed=1):
    x = torch.randn(B, A, T, generator=torch.Generator().manual_seed(seed))
    return (x - x.mean(-1, keepdim=True)) / (x.std(-1, keepdim=True) + 1e-9)


def streamed(m, x, chunk, mc=False):
    s = m.stream(x.shape[0], chunk, mixture_consistency=mc)
    with torch.no_grad():
        outs = [s.step(x[..., c:c + chunk]) for c in range(0, x.shape[-1], chunk)]
        tail = s.flush()
    return torch.cat(outs, -1), tail


def check_against_forward(cfg, sd, m, x, chunk, oracle=True):
    hop, T = cfg.hop, x.shape[-1]
    xd = x.to(DEV)
    out, tail = streamed(m, xd, chunk)
    with torch.no_grad():
        ref_native = m(xd)
    assert torch.equal(out[..., :hop], torch.zeros_like(out[..., :hop]))
    got = torch.cat([out[..., hop:], tail], -1)
    aligned = T % cfg.n_least_samples_req == 0
    n_cmp = T if aligned else T - hop
    e_nat = O.parity_errors(got[..., :n_cmp], ref_native[..., :n_cmp])
    print(f"chunk {chunk}: vs native offline rel_max {e_nat[0]:.2e} rel_l2 {e_nat[1]:.2e} "
          f"bitwise {torch.equal(got[..., :n_cmp], ref_native[..., :n_cmp])}")
    assert max(e_nat) <= 1e-5, e_nat
    if oracle:
        ref = O.causal_forward(cfg, sd, x, dtype=torch.float64)
        e = O.parity_errors(got[..., :n_cmp], ref[..., :n_cmp])
        print(f"chunk {chunk}: vs fp64 oracle rel_max {e[0]:.2e} rel_l2 {e[1]:.2e}")
        assert max(e) < TOL, e


def test_default_model_chunks():
    cfg, sd, m = build(DEFAULT)
    x = mixture(4, 1, 16000)
    G = granule(cfg)
    assert G == 80 and m.stream(4, G).latency == 10
    for g in (1, 4, 25):
        check_against_forward(cfg, sd, m, x, g * G, oracle=(g == 4))


def test_stereo_depth5_chunks():
    cfg, sd, m = build(STEREO)
    x = mixture(2, 2, 4800)
    G = granule(cfg)
    assert G == 160
    for g in (1, 3):
        check_against_forward(cfg, sd, m, x, g * G)


def test_small_model_on_ffma_kernels():
    cfg, sd, m = build(SMALL)
    x = mixture(3, 1, 400)
    lib = N.lib()
    assert lib.sdr_encoder_mma_packed_bytes(16, 1, 11) == 0
    for g in (1, 2):
        check_against_forward(cfg, sd, m, x, g * granule(cfg))


# ---- the stream stage alone against the one-pass causal pyramid and an fp64 chain ----
def stage_rows(D, F):
    """(R, dynamic shared memory) that launch_causal_stream (stream.cu) picks: every level's buffer holds 10 history
    values and its new inputs, pos = sum_d (10 + nin_d) + (F >> (D-1)) floats per channel, and R = 32 channels per CTA
    halve while R * pos floats exceed 48 KB (down to R = 1, which asks for more than 48 KB at D = 7 and 8, F = 4096)."""
    pos = sum(10 + (F if d == 0 else F >> (d - 1)) for d in range(D)) + (F >> (D - 1))
    R = 32
    while R > 1 and R * pos * 4 > 48 * 1024:
        R //= 2
    return R, R * pos * 4


def first_chunk_with_rows(D, R):
    """The shortest chunk (frames) at which the stage runs R channels per CTA, None if no chunk does."""
    gran = max(4, 2 ** (D - 1))
    return next((F for F in range(gran, 4097, gran) if stage_rows(D, F)[0] == R), None)


def stage_reference(y, slope_in, w, bias, sl):
    """fp64 PReLU -> D x (causally masked 21-tap depthwise conv + PReLU) -> nearest up-sampling and skip adds."""
    Cc = y.shape[1]
    cur = O.prelu1(y.double(), slope_in.double())
    levels = []
    for d in range(len(w)):
        cur = O.prelu1(torch.nn.functional.conv1d(cur, O.causal_weight(w[d].double()), bias[d].double(),
                                                  stride=1 if d == 0 else 2, padding=10, groups=Cc), sl[d].double())
        levels.append(cur)
    for _ in range(len(w) - 1):
        top = levels.pop()
        levels[-1] = levels[-1] + torch.nn.functional.interpolate(top, scale_factor=2, mode="nearest")
    return levels[0]


def _stage_case(D, F, B, Cc=40, n=6):
    """n chunks of F frames: six turn the deepest level's history over completely at the granule (2 new inputs per
    chunk, 4 at D = 1), and an even count keeps the concatenation a multiple of 2^D for sdr_causal_pyramid."""
    g = torch.Generator().manual_seed(D * 1000 + F + B)
    L = n * F
    y = torch.randn(B, Cc, L, generator=g).to(DEV)
    w = [(torch.randn(Cc, 1, 21, generator=g) / 3).to(DEV) for _ in range(D)]
    bias = [(0.1 * torch.randn(Cc, generator=g)).to(DEV) for _ in range(D)]
    sl = [torch.tensor([0.1 + 0.3 * d], device=DEV) for d in range(D)]
    if D > 1:
        sl[1] = torch.tensor([1.3], device=DEV)        # both branches of the two-instruction PReLU
    slope_in = torch.tensor([0.25], device=DEV)
    ptrs = lambda ts: (C.c_void_p * len(ts))(*[C.c_void_p(t.data_ptr()) for t in ts])
    lib = N.lib()
    ref = torch.empty_like(y)
    N.check(lib.sdr_causal_pyramid(C.c_void_p(y.data_ptr()), C.c_void_p(slope_in.data_ptr()), ptrs(w), ptrs(bias),
                                   ptrs(sl), C.c_void_p(ref.data_ptr()), D, B, Cc, L, None), "sdr_causal_pyramid")
    ref64 = stage_reference(y, slope_in, w, bias, sl)
    gd = Guards()
    hist = gd.output("history", torch.zeros(B, D, 10, Cc, device=DEV))
    wg = [gd.input(f"w{d}", w[d]) for d in range(D)]
    bg = [gd.input(f"b{d}", bias[d]) for d in range(D)]
    sg = [gd.input(f"slope{d}", sl[d]) for d in range(D)]
    sin = gd.input("slope_in", slope_in)
    err = 0.0
    for c in range(n):
        yc = gd.input(f"y{c}", y[..., c * F:(c + 1) * F].permute(1, 0, 2).reshape(Cc, B * F))
        mc = gd.output(f"m{c}", torch.full((Cc, B * F), float("nan"), device=DEV))
        N.check(lib.sdr_causal_stream_stage(C.c_void_p(yc.data_ptr()), C.c_void_p(sin.data_ptr()), ptrs(wg),
                                            ptrs(bg), ptrs(sg), C.c_void_p(hist.data_ptr()), C.c_void_p(mc.data_ptr()),
                                            D, B, Cc, F, None), "sdr_causal_stream_stage")
        gd.check()
        got = mc.reshape(Cc, B, F).permute(1, 0, 2)
        want = ref[..., c * F:(c + 1) * F]
        assert torch.equal(got, want), (D, F, B, c, float((got - want).abs().max()))
        e = O.parity_errors(got, ref64[..., c * F:(c + 1) * F])
        err = max(err, *e)
        assert max(e) < 2e-5, (D, F, B, c, e)
    R, smem = stage_rows(D, F)
    print(f"stage D={D} F={F} B={B} C={Cc}: R={R} smem={smem} B, {n} chunks bitwise == sdr_causal_pyramid, "
          f"vs fp64 chain {err:.2e}")
    return lib


STAGE_CHANNELS = {1: 40, 3: 37, 130: 5}     # 37: a partial CTA at every R >= 2; 5: fewer channels than one CTA's R


def stage_cases():
    """(D, chunk kind, F, B): the granule, twice, thrice it and 4096 frames at 1, 3 and 130 slots; at 3 slots, the
    shortest chunk at which the host picks each R that is not the granule's."""
    cases = []
    for B in (1, 3, 130):
        for kind in ("granule", "twice", "max", "thrice", "R32", "R16", "R8", "R4", "R2", "R1"):
            for D in (1, 4, 5, 6, 2, 3, 7, 8):
                gran = max(4, 2 ** (D - 1))
                if kind.startswith("R"):
                    F = first_chunk_with_rows(D, int(kind[1:]))
                    if B != 3 or F is None or F == gran:
                        continue
                else:
                    F = {"granule": gran, "twice": 2 * gran, "thrice": 3 * gran, "max": 4096}[kind]
                cases.append(pytest.param(D, kind, F, B, id=f"{B}-{kind}-{D}"))
    return cases


@pytest.mark.parametrize("D,F_kind,F,B", stage_cases())
def test_stream_stage_bitwise_vs_pyramid(D, F_kind, F, B):
    gran = max(4, 2 ** (D - 1))
    if F_kind.startswith("R"):
        assert stage_rows(D, F)[0] == int(F_kind[1:]) and stage_rows(D, F - gran)[0] != int(F_kind[1:])
    lib = _stage_case(D, F, B, Cc=STAGE_CHANNELS[B])
    if F_kind == "max":
        assert stage_rows(D, 4096)[1] > 48 * 1024 if D >= 7 else stage_rows(D, 4096)[1] <= 48 * 1024
        z = torch.zeros(16, device=DEV)
        ptrs = (C.c_void_p * D)(*([C.c_void_p(z.data_ptr())] * D))
        p = C.c_void_p(z.data_ptr())
        assert lib.sdr_causal_stream_stage(p, p, ptrs, ptrs, ptrs, p, p, D, B, 40, 4096 + gran, None) == -5


def test_stream_stage_65535_slots():
    """grid.y = 65535 CTAs, one per slot, at the granule; 65536 slots are refused."""
    _stage_case(3, 4, 65535, Cc=3)
    z = torch.zeros(16, device=DEV)
    ptrs = (C.c_void_p * 3)(*([C.c_void_p(z.data_ptr())] * 3))
    p = C.c_void_p(z.data_ptr())
    assert N.lib().sdr_causal_stream_stage(p, p, ptrs, ptrs, ptrs, p, p, 3, 65536, 3, 4, None) == -5


# ---- slots, reset, graphs ----
def test_slots_are_independent():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    x = mixture(4, 1, 6 * G, seed=5).to(DEV)
    a, ta = streamed(m, x, G)
    x2 = x.clone()
    x2[1] = 3.0 * torch.randn_like(x2[1])
    b, tb = streamed(m, x2, G)
    for j in (0, 2, 3):
        assert torch.equal(a[j], b[j]) and torch.equal(ta[j], tb[j]), j
    assert not torch.equal(a[1], b[1])


def test_reset_some_slots_mid_stream():
    cfg, sd, m = build(MID)
    G = 2 * granule(cfg)
    x1 = mixture(4, 1, 3 * G, seed=6).to(DEV)
    x2 = mixture(4, 1, 3 * G, seed=7).to(DEV)
    chunks = lambda x: [x[..., c:c + G] for c in range(0, x.shape[-1], G)]
    with torch.no_grad():
        s, keep, fresh = m.stream(4, G), m.stream(4, G), m.stream(4, G)
        for c in chunks(x1):
            s.step(c); keep.step(c)
        s.reset([0, 2])
        got = torch.cat([s.step(c) for c in chunks(x2)], -1)
        want_kept = torch.cat([keep.step(c) for c in chunks(x2)], -1)
        want_fresh = torch.cat([fresh.step(c) for c in chunks(x2)], -1)
    for j in (0, 2):
        assert torch.equal(got[j], want_fresh[j]), j
    for j in (1, 3):
        assert torch.equal(got[j], want_kept[j]), j


def test_cuda_graph_replay_matches_eager_and_holds_for_20s():
    cfg, sd, m = build(DEFAULT, seed=13)
    Cn = 320                                   # 40 ms at 8 kHz
    T = 160000                                 # 20 s
    x = mixture(1, 1, T, seed=8)
    xd = x.to(DEV)
    s_eager = m.stream(1, Cn)
    s_graph = m.stream(1, Cn)
    inp = torch.zeros(1, 1, Cn, device=DEV)
    out = torch.empty(1, 2, Cn, device=DEV)
    with torch.no_grad():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):           # warm-up outside capture, then start the graph stream over
            s_graph.step(inp, out=out)
        torch.cuda.current_stream().wait_stream(side)
        s_graph.reset()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            s_graph.step(inp, out=out)
        s_graph.reset()
        torch.cuda.synchronize()
        got, want = [], []
        for c in range(0, T, Cn):
            inp.copy_(xd[..., c:c + Cn])
            g.replay()
            got.append(out.clone())
            want.append(s_eager.step(xd[..., c:c + Cn]))
        tail = s_graph.flush()
    got = torch.cat(got, -1)
    assert torch.equal(got, torch.cat(want, -1))
    ref = O.causal_forward(O.Config(variant="causal", **DEFAULT), sd, x, dtype=torch.float64)
    hop = cfg.hop
    full = torch.cat([got[..., hop:], tail], -1)
    e = O.parity_errors(full[..., -8000:], ref[..., -8000:])          # the last second of the stream
    print("20 s graph-replayed stream, last second vs fp64 oracle: rel_max %.2e rel_l2 %.2e" % e)
    assert max(e) < TOL, e


def test_mixture_consistency_matches_separate():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    x = mixture(2, 1, 10 * G, seed=9).to(DEV)
    out, tail = streamed(m, x, G, mc=True)
    with torch.no_grad():
        ref = m.separate(x, mixture_consistency=True)
    hop = cfg.hop
    got = torch.cat([out[..., hop:], tail], -1)
    e = O.parity_errors(got, ref)
    print("mixture consistency vs separate: rel_max %.2e rel_l2 %.2e bitwise %s" % (e + (torch.equal(got, ref),)))
    assert max(e) <= 1e-5, e
    _, _, st = build(dict(STEREO, num_blocks=1))
    with pytest.raises(RuntimeError, match="mono"):
        st.stream(2, 160, mixture_consistency=True)


def test_launch_count_matches_captured_graph():
    """The kernels two consecutive steps enqueue, counted as the kernel nodes of a CUDA graph captured from them
    (memsets are nodes of another type), against sdr_stream_launch_count.  torch.profiler's device records are not
    used: in a process that has profiled many times they can miss a kernel or a whole step."""
    cfg, sd, m = build(MID)
    G = granule(cfg)
    s = m.stream(3, 2 * G)
    x = mixture(3, 1, 2 * G, seed=10).to(DEV)
    out = torch.empty(3, 2, 2 * G, device=DEV)
    want = N.lib().sdr_stream_launch_count(C.byref(_engine.make_config(m)), 3, 2 * G)
    assert want == 3 * MID["num_blocks"] + 6
    with torch.no_grad():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):           # warm-up outside capture: weights packed, shared memory opted in
            s.step(x, out=out)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(graph):
            s.step(x, out=out)
            s.step(x, out=out)
    cu = C.CDLL("libcuda.so.1")
    g = C.c_void_p(graph.raw_cuda_graph())
    n = C.c_size_t(0)
    assert cu.cuGraphGetNodes(g, None, C.byref(n)) == 0
    nodes = (C.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(g, nodes, C.byref(n)) == 0
    types = []
    for node in nodes:
        t = C.c_int(-1)
        assert cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(t)) == 0
        types.append(t.value)
    print("graph nodes of two steps by type:", collections.Counter(types))
    assert types.count(0) == 2 * want, (want, collections.Counter(types))      # 0: CU_GRAPH_NODE_TYPE_KERNEL


def test_argument_errors():
    cfg, sd, m = build(MID)
    G = granule(cfg)
    s = m.stream(2, G)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="shape"):
            s.step(torch.zeros(3, 1, G, device=DEV))
        with pytest.raises(RuntimeError, match="audio channel"):
            s.step(torch.zeros(2, 2, G, device=DEV))
        with pytest.raises(RuntimeError, match="shape"):
            s.step(torch.zeros(2, 1, 2 * G, device=DEV))
        with pytest.raises(RuntimeError, match="CUDA"):
            s.step(torch.zeros(2, 1, G))
        with pytest.raises(RuntimeError, match="out must be"):
            s.step(torch.zeros(2, 1, G, device=DEV), out=torch.empty(2, 2, G + 1, device=DEV))
    with pytest.raises(ValueError, match="granule"):
        m.stream(2, G + cfg.hop)
    with pytest.raises(IndexError):
        s.reset([2])
    lib = N.lib()
    c = _engine.make_config(m)
    packed = _engine.packed_weights(m, c, torch.device(DEV, torch.cuda.current_device()))
    state = torch.zeros(lib.sdr_stream_state_bytes(C.byref(c), 2), dtype=torch.uint8, device=DEV)
    need = lib.sdr_stream_workspace_bytes(C.byref(c), 2, G)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    x = torch.zeros(2, 1, G, device=DEV)
    out = torch.empty(2, 2, G, device=DEV)
    rc = lib.sdr_stream_step(C.byref(c), C.c_void_p(packed.data_ptr()), C.c_void_p(state.data_ptr()),
                             C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), 2, G, 0,
                             C.c_void_p(ws.data_ptr()), need - 256, None)
    assert rc == -3
    imp = P.SuDORMRF(16, 32, 1, 2, 21, 16, 2).to(DEV).eval()
    from sudo_rm_rf_b200.streaming import CausalStream
    with pytest.raises(RuntimeError, match="CausalSuDORMRF"):
        CausalStream(imp, 2, 80)
