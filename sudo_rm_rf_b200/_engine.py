"""Host-side glue between the ``nn.Module`` mirrors and the C-ABI.

PyTorch is used here only as plumbing: it owns device memory (parameters,
packed weights, workspace, outputs come from its caching allocator) and names
the CUDA stream the kernels are enqueued on.  All arithmetic happens in
``libsudormrf_b200.so``.
"""
from __future__ import annotations

import ctypes as C
import threading
import warnings
from typing import List

import torch
from torch.optim.optimizer import register_optimizer_step_post_hook

from . import _native as N

_tls_lock = threading.Lock()
_warned_detached = False

# Bumped after every optimizer step, of any optimizer.  Fused optimizers (``fused=True``) write the parameters
# without bumping their version counters, so the weight signature also carries this generation: any step forces a
# repack on the next call, as the foreach and single-tensor optimizers already do through the counters.
_generation = 0


def _bump_generation(*_):
    global _generation
    _generation += 1


register_optimizer_step_post_hook(_bump_generation)


def make_config(model) -> N.SdrConfig:
    """Constructor arguments -> ``sdr_config``; reads the public attributes the
    reference stores (improved_sudormrf.py:235-241, groupcomm_sudormrf_v2.py:245-252)."""
    variant = getattr(model, "_b200_variant", None)
    if variant is None:
        variant = 1 if hasattr(model, "in_audio_channels") else 0
    gc = variant == 1
    group = 1
    if gc:
        group = int(getattr(model, "group_size", 0) or
                    (model.sm[0].num_group if len(model.sm) else 16))
    return N.SdrConfig(
        variant=int(variant),
        in_audio_channels=int(getattr(model, "in_audio_channels", 1)),
        out_channels=int(model.out_channels), in_channels=int(model.in_channels),
        num_blocks=int(model.num_blocks), upsampling_depth=int(model.upsampling_depth),
        enc_kernel_size=int(model.enc_kernel_size), enc_num_basis=int(model.enc_num_basis),
        num_sources=int(model.num_sources), group_size=group)


_names = {}     # cfg.key() -> state_dict_names(cfg)


def state_dict_names(cfg: N.SdrConfig) -> List[str]:
    """The state_dict keys the library packs, in its order (``sdr_param_name``): every entry of the reference's
    ``state_dict()`` but the original model's unused ``ln_mask_in``."""
    names = _names.get(cfg.key())
    if names is None:
        lib, buf, names = N.lib(), C.create_string_buffer(256), []
        n = lib.sdr_num_params(C.byref(cfg))
        if n < 0:
            N.check(n, "sdr_num_params")
        for i in range(n):
            r = lib.sdr_param_name(C.byref(cfg), i, buf, len(buf))
            if r < 0:
                N.check(r, "sdr_param_name")
            names.append(buf.value.decode())
        names = _names[cfg.key()] = tuple(names)
    return list(names)


def _probe_names(model):
    """The first parameter and the decoder's weight, which every variant has (device / requires_grad probes)."""
    return (state_dict_names(make_config(model))[0], "decoder.weight")


def _fetch(model, dotted: str) -> torch.Tensor:
    # attribute walk (not named_parameters): nn.DataParallel replicas hold plain
    # tensors in _parameters and report no parameters()
    obj = model
    for part in dotted.split("."):
        obj = obj[int(part)] if part.isdigit() else getattr(obj, part)
    return obj


class _DeviceState:
    """Per (model, device) cache: packed weights + workspace."""
    __slots__ = ("sig", "storages", "packed", "workspace", "staging", "captured", "retired", "tensors", "pslots",
                 "mslots", "graphs", "stream", "event", "lock")

    def __init__(self):
        self.sig = None
        self.storages = None     # the storages `sig` describes, kept alive so that no other tensor takes their addresses
        self.captured = set()    # buffer slots ("packed", "workspace", "staging") a CUDA-graph capture has addressed
        self.retired = []        # replaced buffers a captured graph may still address: never handed back to the allocator
        self.packed = None
        self.workspace = None
        self.staging = None
        self.tensors = None      # cached parameter tensors in state_dict order (never for DataParallel replicas)
        self.pslots = None       # (leaf._parameters, key) per tensor: identity check without the attribute walk
        self.mslots = None       # (parent._modules, name, child) per module on the way: catches replaced sub-modules
        self.graphs = {}         # forward_host: CUDA graphs keyed by (host buffers, shape, weights signature)
        self.stream = None       # stream of the last enqueue on this workspace
        self.event = None        # recorded after the last enqueue (cross-stream serialisation)
        self.lock = threading.Lock()     # held over a call's host section: pack, size, hand-over, enqueue, event


def _state(model, device) -> _DeviceState:
    cache = model.__dict__.get("_b200_cache")
    if cache is None:
        with _tls_lock:
            cache = model.__dict__.setdefault("_b200_cache", {})
    st = cache.get(device.index)
    if st is None:
        st = cache.setdefault(device.index, _DeviceState())
    return st


def drop_cache(model) -> None:
    """Forget packed weights, workspaces and captured graphs (they are rebuilt on the next call).  This frees every
    buffer a CUDA graph captured from this model addresses: such graphs must not be replayed afterwards."""
    model.__dict__.pop("_b200_cache", None)


def refresh_weights(model) -> None:
    """Make the next native call re-pack ``model``'s weights.

    Writes through autograd-visible tensors (``load_state_dict``, in-place ops under ``no_grad``, ``detach()``,
    ``state_dict()`` tensors, ``nn.init``), optimizer steps of any kind and replaced Parameters or sub-modules are
    noticed without it.  Writes that bypass the version counter are not: ``p.data.<op>_()``, ``p.data.copy_()``,
    DLPack and other foreign writers, ``dist.broadcast(p.data)``.  Call this after them.  Graphs captured earlier keep
    the weights they were captured with; capture again after the next call."""
    if isinstance(model, torch.nn.DataParallel):
        model = model.module
    for st in model.__dict__.get("_b200_cache", {}).values():
        st.sig = None


class NativeModuleMixin:
    """Keeps the device-side cache (packed weights, a multi-GB workspace, CUDA graphs) out of pickles and
    deep copies: ``torch.save(model)`` / ``copy.deepcopy(model)`` after a forward behave as for the reference."""

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_b200_cache", None)
        return state


class _Order:
    """The stream and event of the last enqueue on buffers that several streams take turns on."""
    __slots__ = ("stream", "event")

    def __init__(self):
        self.stream = None
        self.event = None


def _enter_stream(order, device, buffers):
    """A call arriving on a different stream than the previous one (recorded in ``order``: a ``_DeviceState`` or an
    ``_Order``) waits for it.  Every buffer the call reads is recorded on its stream, whichever stream allocated it,
    so that the caching allocator does not hand it out again while the call is in flight."""
    cur = torch.cuda.current_stream(device)
    if torch.cuda.is_current_stream_capturing():     # the capturing caller owns the ordering
        return cur
    if order.stream is not None and order.stream != cur and order.event is not None:
        cur.wait_event(order.event)
    for buf in buffers:
        if buf is not None:
            buf.record_stream(cur)
    return cur


def _leave_stream(order, cur) -> None:
    if torch.cuda.is_current_stream_capturing():
        return
    if order.event is None:
        order.event = torch.cuda.Event()
    order.event.record(cur)
    order.stream = cur


def packed_for(model, cfg: N.SdrConfig, device, stream) -> torch.Tensor:
    """``packed_weights`` for a call that reads them on ``stream`` outside ``_call_shared`` (a stream step, a corpus
    pass), recorded on that stream: a repack by another call then cannot hand the buffer out early."""
    st = _state(model, device)
    with st.lock:
        packed = packed_weights(model, cfg, device)
    if not torch.cuda.is_current_stream_capturing():
        packed.record_stream(stream)
    return packed


def _hand_out(st: _DeviceState, slot: str) -> None:
    """Called when the buffer in ``slot`` is given to a kernel: under stream capture the graph keeps its address."""
    if torch.cuda.is_current_stream_capturing():
        st.captured.add(slot)


def _replace(st: _DeviceState, slot: str, buf) -> None:
    """Puts ``buf`` in ``slot``.  The old buffer is freed, unless a captured graph addresses it: a user's graph
    outlives the cache's view of it, and its replay would write into (or read weights from) whatever tensor the
    allocator handed that memory to next.  Such buffers are retired instead, and live as long as the cache."""
    old = getattr(st, slot)
    if old is not None and slot in st.captured:
        st.retired.append(old)
    st.captured.discard(slot)
    setattr(st, slot, buf)


def _ensure(st: _DeviceState, slot: str, nbytes: int, device) -> torch.Tensor:
    """The buffer in ``slot`` ("workspace" or "staging"), replaced by one of ``nbytes`` if it is smaller."""
    buf = getattr(st, slot)
    if buf is None or buf.numel() < nbytes:
        _replace(st, slot, None)        # recorded on every stream that read it: the allocator waits for those
        st.graphs.clear()               # captured graphs point into the old buffer
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        setattr(st, slot, buf)
    _hand_out(st, slot)
    return buf


def _call_shared(model, cfg: N.SdrConfig, device, ws_bytes: int, refusal: str, enqueue) -> torch.Tensor:
    """Every call that runs on the model's cached state goes through here: packs (or reuses) the weights, sizes the
    shared workspace, hands it over from the previous call's stream and runs ``enqueue(packed, workspace)``, which
    enqueues on the current stream.  ``ws_bytes`` is the caller's size query; 0 raises ``refusal``.  Returns the
    packed weights the call ran with.  One call at a time per (model, device): host threads sharing a model queue
    here, so each one's call waits on the stream for the previous one's."""
    st = _state(model, device)
    with torch.cuda.device(device), st.lock:         # host work only: nothing in here waits for the GPU
        packed = packed_weights(model, cfg, device)
        if ws_bytes == 0:
            raise N.NativeError(refusal)
        ws = _ensure(st, "workspace", ws_bytes, device)
        cur = _enter_stream(st, device, (st.workspace, st.staging, st.packed))
        enqueue(packed, ws)
        _leave_stream(st, cur)
    return packed


def _graphed(graphs: dict, key, bound: int, device, enqueue) -> str:
    """Runs ``enqueue`` (which enqueues on the current stream) eagerly on the first call with ``key``, which also warms
    every kernel; captures it into a CUDA graph on a side stream on the second, and replays that graph from then on.
    ``graphs`` is cleared when it holds ``bound`` keys.  Returns "eager", "captured" or "replayed"."""
    entry = graphs.get(key)
    if entry is None:
        if len(graphs) >= bound:
            graphs.clear()
        graphs[key] = "warm"
        enqueue()
        return "eager"
    if entry == "warm":
        cur = torch.cuda.current_stream(device)
        side = torch.cuda.Stream(device=device)
        side.wait_stream(cur)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            enqueue()
        cur.wait_stream(side)
        graphs[key] = graph
        graph.replay()
        return "captured"
    entry.replay()
    return "replayed"


def _cuda_device(device, refusal: str) -> torch.device:
    """``device`` with a missing index resolved to the current device.  Raises ``refusal`` when it is not a CUDA
    device, or when there is none."""
    device = torch.device(device)
    if device.type != "cuda" or not torch.cuda.is_available():
        raise RuntimeError(refusal)
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def _model_device(model, refusal: str, device=None) -> torch.device:
    """``_cuda_device`` of ``device``, or of the device of the model's parameters."""
    return _cuda_device(device if device is not None else _fetch(model, _probe_names(model)[0]).device, refusal)


def _walk(model, names):
    """Attribute walk recording, besides the tensors, where each one hangs (for the cheap identity check)."""
    tensors, pslots, mslots, seen = [], [], [], set()
    for dotted in names:
        obj = model
        parts = dotted.split(".")
        for part in parts[:-1]:
            child = obj._modules[part]
            key = (id(obj), part)
            if key not in seen:
                seen.add(key)
                mslots.append((obj._modules, part, child))
            obj = child
        t = obj._parameters[parts[-1]]
        tensors.append(t)
        pslots.append((obj._parameters, parts[-1]))
    return tensors, pslots, mslots


def _cached_tensors(st: _DeviceState):
    """The cached parameter list if every module and Parameter object on the way is still the same object."""
    if st.tensors is None:
        return None
    try:
        for d, k, child in st.mslots:
            if d[k] is not child:
                return None
        for (d, k), t in zip(st.pslots, st.tensors):
            if d[k] is not t:
                return None
    except KeyError:
        return None
    return st.tensors


def weight_signature(tensors) -> tuple:
    """What the packed weights were made from: the optimizer-step generation and each tensor's address and version
    counter.  Host only.  An address names the data only while its storage is alive; the cache keeps the storages
    of the signature it holds (``weight_storages``), so a tensor swapped in through ``p.data = t`` cannot land on the
    address of the one it replaced."""
    return (_generation, tuple([(t.data_ptr(), t._version) for t in tensors]))


def weight_storages(tensors) -> list:
    return [t.untyped_storage() for t in tensors]


def packed_weights(model, cfg: N.SdrConfig, device) -> torch.Tensor:
    """Flat packed-weight buffer for ``model`` on ``device``.

    Master modules: re-packed whenever a parameter's storage or version counter changes, an optimizer steps, or a
    Parameter / sub-module object was replaced (identity of every object on the path is checked, ~50 us), or after
    ``refresh_weights``.
    ``nn.DataParallel`` replicas: packed on EVERY forward.  Their parameters are fresh broadcast copies whose
    ``_version`` is always 0 and whose addresses the caching allocator reuses, so no signature can tell a new
    set of weights from the previous one; the replica shares ``_b200_cache`` with its master."""
    lib = N.lib()
    st = _state(model, device)
    replica = bool(getattr(model, "_is_replica", False))
    names = None
    if replica:
        names = state_dict_names(cfg)
        tensors = [_fetch(model, n) for n in names]
        sig = None
    else:
        tensors = _cached_tensors(st)
        if tensors is None:
            names = state_dict_names(cfg)
            try:
                tensors, st.pslots, st.mslots = _walk(model, names)
                st.tensors = tensors
            except KeyError:           # parameters held as plain attributes: no caching
                tensors = [_fetch(model, n) for n in names]
                st.tensors = st.pslots = st.mslots = None
        sig = weight_signature(tensors)
        if st.sig == sig and st.packed is not None:
            _hand_out(st, "packed")
            return st.packed
    if names is None:
        names = state_dict_names(cfg)
    n = lib.sdr_num_params(C.byref(cfg))
    if n < 0:
        N.check(n, "sdr_num_params")
    if n != len(tensors):
        raise N.NativeError(f"parameter inventory mismatch: library expects {n}, module has {len(tensors)}")
    flat = []
    transform = getattr(model, "_b200_param_transform", None)     # constants the reference applies around a parameter
    for i, (name, t) in enumerate(zip(names, tensors)):
        if t.device != device:
            raise RuntimeError(f"parameter {name} is on {t.device}, input is on {device}")
        want = lib.sdr_param_numel(C.byref(cfg), i)
        if t.numel() != want:
            raise RuntimeError(f"parameter {name} has {t.numel()} elements, expected {want}")
        t = t.detach().to(torch.float32)
        if transform is not None:
            t = transform(name, t)
        flat.append(t.contiguous())
    nbytes = lib.sdr_packed_weight_bytes(C.byref(cfg))
    # the master (and a replica on the master's device, which shares this state) may have graphs / in-flight
    # kernels on the old buffer: always pack into a fresh one, the allocator recycles it stream-safely
    packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
    ptrs = (C.c_void_p * n)(*[N.ptr(t) for t in flat])
    N.check(lib.sdr_pack_weights(C.byref(cfg), ptrs, n, N.ptr(packed), nbytes,
                                 N.stream(device)), "sdr_pack_weights")
    st.sig, st.storages = sig, (weight_storages(tensors) if sig is not None else None)
    _replace(st, "packed", packed)
    _hand_out(st, "packed")
    st.graphs.clear()          # captured graphs hold the old packed buffer
    return packed


def _check_mixture(cfg, wav: torch.Tensor) -> None:
    """A [B, A, T] CUDA mixture with the model's channel count and no empty dimension."""
    if wav.dim() != 3:
        raise RuntimeError(
            f"Expected 3D input [batch, channels, time] to the encoder, got {list(wav.shape)}")
    if wav.shape[1] != cfg.in_audio_channels:
        raise RuntimeError(f"expected {cfg.in_audio_channels} audio channel(s), got {wav.shape[1]}")
    if not wav.is_cuda:
        raise RuntimeError(
            "sudo_rm_rf_b200 runs on CUDA (sm_90a) only and has no CPU path: move the model "
            "and the mixture to an H100 (`model.cuda()`, `mixture.cuda()`).")
    if wav.shape[0] == 0 or wav.shape[-1] == 0:
        raise RuntimeError("empty batch or zero-length mixture")


def _check_input(model, cfg, wav: torch.Tensor) -> torch.Tensor:
    _check_mixture(cfg, wav)
    if torch.is_grad_enabled() and model.training and \
            any(_fetch(model, n).requires_grad for n in _probe_names(model)):
        raise RuntimeError(
            "sudo_rm_rf_b200 implements the inference forward only (no autograd): call "
            "model.eval() and/or wrap the call in torch.no_grad().")
    global _warned_detached
    if torch.is_grad_enabled() and not _warned_detached and \
            any(_fetch(model, n).requires_grad for n in _probe_names(model)):
        _warned_detached = True
        warnings.warn("sudo_rm_rf_b200: the native forward is inference-only; the returned estimates are detached "
                      "from autograd (wrap the call in torch.no_grad() to silence this).", stacklevel=3)
    # the reference casts to fp32 while padding (improved_sudormrf.py:312)
    return wav.detach().to(torch.float32).contiguous()


def forward(model, wav: torch.Tensor, mixture_consistency: bool = False) -> torch.Tensor:
    """``model(wav)`` on the native path.  [B, A, T] -> [B, S*A, T] fp32, same device."""
    lib = N.lib()
    cfg = make_config(model)
    x = _check_input(model, cfg, wav)
    if mixture_consistency and cfg.in_audio_channels != 1:
        raise RuntimeError("mixture consistency (mixture_consistency.py:14-36) is defined for mono mixtures only; "
                           f"this model has in_audio_channels={cfg.in_audio_channels}")
    device = x.device
    B, _, T = x.shape
    out = torch.empty((B, cfg.num_sources * cfg.in_audio_channels, T), dtype=torch.float32, device=device)

    def enqueue(packed, ws):
        N.check(lib.sdr_forward(C.byref(cfg), N.ptr(packed), N.ptr(x), N.ptr(out), B, T,
                                1 if mixture_consistency else 0, N.ptr(ws), ws.numel(), N.stream(device)),
                "sdr_forward")
    _call_shared(model, cfg, device, lib.sdr_workspace_bytes(C.byref(cfg), B, T),
                 "bad model configuration (sdr_workspace_bytes returned 0)", enqueue)
    return out


def separate(model, wav: torch.Tensor, mixture_consistency: bool = False) -> torch.Tensor:
    """The README inference recipe (reference README.md:100-114) as one native call:
    per-utterance normalisation, forward, rescale with the mixture's std / mean and, optionally, the
    uniform mixture-consistency projection against the normalised mixture (as the README applies it to
    the GroupComm checkpoints).  ``wav`` is ``[B, T]`` (as in the README) or ``[B, 1, T]``; returns
    ``[B, S, T]`` fp32 on the same device."""
    lib = N.lib()
    cfg = make_config(model)
    if wav.dim() == 2:
        wav = wav.unsqueeze(1)
    x = _check_input(model, cfg, wav)
    if cfg.in_audio_channels != 1:
        raise RuntimeError("separate() follows the README recipe, which is written for mono mixtures")
    device = x.device
    B, _, T = x.shape
    out = torch.empty((B, cfg.num_sources, T), dtype=torch.float32, device=device)

    def enqueue(packed, ws):
        N.check(lib.sdr_separate(C.byref(cfg), N.ptr(packed), N.ptr(x), N.ptr(out), B, T,
                                 1 if mixture_consistency else 0, N.ptr(ws), ws.numel(), N.stream(device)),
                "sdr_separate")
    _call_shared(model, cfg, device, lib.sdr_separate_workspace_bytes(C.byref(cfg), B, T),
                 "bad model configuration (sdr_separate_workspace_bytes returned 0)", enqueue)
    return out


def forward_host(model, host_wav: torch.Tensor, host_out: torch.Tensor = None,
                 mixture_consistency: bool = False, device=None, use_graph: bool = True) -> torch.Tensor:
    """End-to-end call with HOST buffers: H2D copy, forward, D2H copy, all enqueued on the current
    stream of the model's device.  The caller synchronises the stream before reading ``host_out``.

    With pinned buffers the whole sequence (2 copies + every kernel) is captured ONCE per
    (buffers, shape, weights) into a CUDA graph and replayed afterwards, so a call costs one graph
    launch instead of ~135 launches; pageable buffers (or ``use_graph=False``) take the eager path."""
    lib = N.lib()
    cfg = make_config(model)
    if host_wav.dim() != 3 or host_wav.is_cuda or host_wav.dtype != torch.float32 \
            or not host_wav.is_contiguous():
        raise RuntimeError("forward_host expects a contiguous fp32 CPU tensor [B, A, T]")
    device = _model_device(model, "the model must live on a CUDA device", device)
    B, A, T = host_wav.shape
    if A != cfg.in_audio_channels:
        raise RuntimeError(f"expected {cfg.in_audio_channels} audio channel(s), got {A}")
    if host_out is None:
        host_out = torch.empty((B, cfg.num_sources * A, T), dtype=torch.float32).pin_memory()
    if tuple(host_out.shape) != (B, cfg.num_sources * A, T) or host_out.dtype != torch.float32 \
            or host_out.is_cuda or not host_out.is_contiguous():
        raise RuntimeError("host_out must be a contiguous fp32 CPU tensor [B, S*A, T]")
    mc = 1 if mixture_consistency else 0
    io_bytes = lib.sdr_host_staging_bytes(C.byref(cfg), B, T)
    if io_bytes == 0:
        raise N.NativeError("bad model configuration")
    st = _state(model, device)

    def enqueue(packed, ws):
        staging = _ensure(st, "staging", io_bytes, device)

        def call():
            N.check(lib.sdr_forward_host(C.byref(cfg), N.ptr(packed), N.ptr(host_wav), N.ptr(host_out), B, T, mc,
                                         N.ptr(staging), staging.numel(), N.ptr(ws), ws.numel(), N.stream(device)),
                    "sdr_forward_host")

        if use_graph and host_wav.is_pinned() and host_out.is_pinned() \
                and not torch.cuda.is_current_stream_capturing():
            key = (host_wav.data_ptr(), host_out.data_ptr(), B, T, mc, ws.data_ptr(), staging.data_ptr(),
                   packed.data_ptr())
            _graphed(st.graphs, key, 8, device, call)
        else:
            call()
    _call_shared(model, cfg, device, lib.sdr_workspace_bytes(C.byref(cfg), B, T), "bad model configuration",
                 enqueue)
    return host_out
