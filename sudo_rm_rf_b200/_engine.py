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

from . import _native as N

_tls_lock = threading.Lock()
_warned_detached = False


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


def state_dict_names(cfg: N.SdrConfig) -> List[str]:
    """Parameter names in the reference's ``state_dict()`` order
    (improved_sudormrf.py:247-281,170-196; groupcomm_sudormrf_v2.py:347-354,401-403)."""
    if cfg.variant == 2:       # causal_improved_sudormrf_v3.py:146-189, block :71-96
        names = ["encoder.weight", "bottleneck.weight", "bottleneck.bias"]
        for i in range(cfg.num_blocks):
            p = f"sm.{i}."
            names += [p + "skipinit_gain", p + "proj_1x1.conv.weight", p + "proj_1x1.conv.bias", p + "proj_1x1.act.weight"]
            for d in range(cfg.upsampling_depth):
                names += [p + f"spp_dw.{d}.conv.weight", p + f"spp_dw.{d}.conv.bias", p + f"spp_dw.{d}.act.weight"]
            names += [p + "res_conv.weight", p + "res_conv.bias"]
        names += ["mask_net.0.weight", "mask_net.1.weight", "mask_net.1.bias", "decoder.weight", "mask_nl_class.weight"]
        return names
    if cfg.variant == 3:       # the original model, sudormrf.py:211-252 (block :134-162); ln_mask_in (:253) is never read
        names = ["encoder.0.weight", "encoder.0.bias", "ln.weight", "ln.bias", "l1.weight", "l1.bias"]
        for i in range(cfg.num_blocks):
            p = f"sm.{i}."
            names += [p + "proj_1x1.conv.weight", p + "proj_1x1.conv.bias", p + "proj_1x1.norm.weight",
                      p + "proj_1x1.norm.bias", p + "proj_1x1.act.weight"]
            for d in range(cfg.upsampling_depth):
                names += [p + f"spp_dw.{d}.conv.weight", p + f"spp_dw.{d}.conv.bias",
                          p + f"spp_dw.{d}.norm.weight", p + f"spp_dw.{d}.norm.bias"]
            names += [p + "conv_1x1_exp.conv.weight", p + "conv_1x1_exp.conv.bias", p + "conv_1x1_exp.norm.weight",
                      p + "conv_1x1_exp.norm.bias", p + "final_norm.norm.weight", p + "final_norm.norm.bias",
                      p + "final_norm.act.weight", p + "module_act.norm.weight", p + "module_act.norm.bias",
                      p + "module_act.act.weight"]
        if cfg.out_channels != cfg.enc_num_basis:
            names += ["reshape_before_masks.weight", "reshape_before_masks.bias"]
        names += ["m.weight", "m.bias", "decoder.weight", "decoder.bias"]
        return names
    names = ["encoder.weight", "ln.gamma", "ln.beta", "bottleneck.weight", "bottleneck.bias"]

    def ublock(p):
        out = [p + "proj_1x1.conv.weight", p + "proj_1x1.conv.bias", p + "proj_1x1.norm.gamma",
               p + "proj_1x1.norm.beta", p + "proj_1x1.act.weight"]
        for d in range(cfg.upsampling_depth):
            out += [p + f"spp_dw.{d}.conv.weight", p + f"spp_dw.{d}.conv.bias",
                    p + f"spp_dw.{d}.norm.gamma", p + f"spp_dw.{d}.norm.beta"]
        out += [p + "final_norm.norm.gamma", p + "final_norm.norm.beta",
                p + "final_norm.act.weight", p + "res_conv.weight", p + "res_conv.bias"]
        return out

    for i in range(cfg.num_blocks):
        if cfg.variant == 0:
            names += ublock(f"sm.{i}.")
        else:
            t = f"sm.{i}.TAC."
            names += [t + "TAC_input.0.weight", t + "TAC_input.0.bias", t + "TAC_input.1.weight",
                      t + "TAC_mean.0.weight", t + "TAC_mean.0.bias", t + "TAC_mean.1.weight",
                      t + "TAC_output.0.weight", t + "TAC_output.0.bias", t + "TAC_output.1.weight",
                      t + "TAC_norm.gamma", t + "TAC_norm.beta"]
            names += ublock(f"sm.{i}.UBlock.")
    names += ["mask_net.0.weight", "mask_net.1.weight", "mask_net.1.bias", "decoder.weight"]
    return names


def _probe_names(model):
    """First and last parameter of the model (device / requires_grad probes)."""
    if getattr(model, "_b200_variant", None) == 3:
        return ("encoder.0.weight", "decoder.weight")
    return ("encoder.weight", "decoder.weight")


def _fetch(model, dotted: str) -> torch.Tensor:
    # attribute walk (not named_parameters): nn.DataParallel replicas hold plain
    # tensors in _parameters and report no parameters()
    obj = model
    for part in dotted.split("."):
        obj = obj[int(part)] if part.isdigit() else getattr(obj, part)
    return obj


class _DeviceState:
    """Per (model, device) cache: packed weights + workspace."""
    __slots__ = ("sig", "packed", "workspace", "staging", "tensors", "pslots", "mslots", "graphs",
                 "stream", "event")

    def __init__(self):
        self.sig = None
        self.packed = None
        self.workspace = None
        self.staging = None
        self.tensors = None      # cached parameter tensors in state_dict order (never for DataParallel replicas)
        self.pslots = None       # (leaf._parameters, key) per tensor: identity check without the attribute walk
        self.mslots = None       # (parent._modules, name, child) per module on the way: catches replaced sub-modules
        self.graphs = {}         # forward_host: CUDA graphs keyed by (host buffers, shape, weights signature)
        self.stream = None       # stream of the last enqueue on this workspace
        self.event = None        # recorded after the last enqueue (cross-stream serialisation)


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
    """Forget packed weights, workspaces and captured graphs (they are rebuilt on the next call)."""
    model.__dict__.pop("_b200_cache", None)


class NativeModuleMixin:
    """Keeps the device-side cache (packed weights, a multi-GB workspace, CUDA graphs) out of pickles and
    deep copies: ``torch.save(model)`` / ``copy.deepcopy(model)`` after a forward behave as for the reference."""

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_b200_cache", None)
        return state


def _stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _enter_stream(st: _DeviceState, device):
    """One workspace per (model, device): a call arriving on a different stream than the previous one waits
    for it (the scratch buffers are shared), and tells the caching allocator about the second stream."""
    cur = torch.cuda.current_stream(device)
    if torch.cuda.is_current_stream_capturing():     # the capturing caller owns the ordering
        return cur
    if st.stream is not None and st.stream != cur and st.event is not None:
        cur.wait_event(st.event)
        for buf in (st.workspace, st.staging, st.packed):
            if buf is not None:
                buf.record_stream(cur)
    return cur


def _leave_stream(st: _DeviceState, cur) -> None:
    if torch.cuda.is_current_stream_capturing():
        return
    if st.event is None:
        st.event = torch.cuda.Event()
    st.event.record(cur)
    st.stream = cur


def _ensure_workspace(st: _DeviceState, nbytes: int, device) -> None:
    if st.workspace is None or st.workspace.numel() < nbytes:
        if st.event is not None:
            st.event.synchronize()      # kernels of an earlier call (possibly on another stream) still use it
        st.workspace = None
        st.graphs.clear()               # captured graphs point into the old workspace
        st.workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)


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


def packed_weights(model, cfg: N.SdrConfig, device) -> torch.Tensor:
    """Flat packed-weight buffer for ``model`` on ``device``.

    Master modules: re-packed whenever a parameter's storage or version counter changes, or a Parameter /
    sub-module object was replaced (identity of every object on the path is checked, ~50 us).
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
        sig = tuple([(t.data_ptr(), t._version) for t in tensors])
        if st.sig == sig and st.packed is not None:
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
    ptrs = (C.c_void_p * n)(*[C.c_void_p(t.data_ptr()) for t in flat])
    N.check(lib.sdr_pack_weights(C.byref(cfg), ptrs, n, C.c_void_p(packed.data_ptr()), nbytes,
                                 _stream_ptr(device)), "sdr_pack_weights")
    st.sig, st.packed = sig, packed
    st.graphs.clear()          # captured graphs hold the old packed buffer
    return packed


def _check_input(model, cfg, wav: torch.Tensor) -> torch.Tensor:
    if wav.dim() != 3:
        raise RuntimeError(
            f"Expected 3D input [batch, channels, time] to the encoder, got {list(wav.shape)}")
    if wav.shape[1] != cfg.in_audio_channels:
        raise RuntimeError(f"expected {cfg.in_audio_channels} audio channel(s), got {wav.shape[1]}")
    if not wav.is_cuda:
        raise RuntimeError(
            "sudo_rm_rf_b200 runs on CUDA (sm_90a) only and has no CPU path: move the model "
            "and the mixture to an H100 (`model.cuda()`, `mixture.cuda()`).")
    if torch.is_grad_enabled() and model.training and \
            any(_fetch(model, n).requires_grad for n in _probe_names(model)):
        raise RuntimeError(
            "sudo_rm_rf_b200 implements the inference forward only (no autograd): call "
            "model.eval() and/or wrap the call in torch.no_grad().")
    if wav.shape[0] == 0 or wav.shape[-1] == 0:
        raise RuntimeError("empty batch or zero-length mixture")
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
    with torch.cuda.device(device):
        packed = packed_weights(model, cfg, device)
        st = _state(model, device)
        ws_bytes = lib.sdr_workspace_bytes(C.byref(cfg), B, T)
        if ws_bytes == 0:
            raise N.NativeError("bad model configuration (sdr_workspace_bytes returned 0)")
        _ensure_workspace(st, ws_bytes, device)
        out = torch.empty((B, cfg.num_sources * cfg.in_audio_channels, T),
                          dtype=torch.float32, device=device)
        cur = _enter_stream(st, device)
        N.check(lib.sdr_forward(C.byref(cfg), C.c_void_p(packed.data_ptr()),
                                C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()),
                                B, T, 1 if mixture_consistency else 0,
                                C.c_void_p(st.workspace.data_ptr()), st.workspace.numel(),
                                C.c_void_p(cur.cuda_stream)), "sdr_forward")
        _leave_stream(st, cur)
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
    with torch.cuda.device(device):
        packed = packed_weights(model, cfg, device)
        st = _state(model, device)
        ws_bytes = lib.sdr_separate_workspace_bytes(C.byref(cfg), B, T)
        if ws_bytes == 0:
            raise N.NativeError("bad model configuration (sdr_separate_workspace_bytes returned 0)")
        _ensure_workspace(st, ws_bytes, device)
        out = torch.empty((B, cfg.num_sources, T), dtype=torch.float32, device=device)
        cur = _enter_stream(st, device)
        N.check(lib.sdr_separate(C.byref(cfg), C.c_void_p(packed.data_ptr()),
                                 C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()),
                                 B, T, 1 if mixture_consistency else 0,
                                 C.c_void_p(st.workspace.data_ptr()), st.workspace.numel(),
                                 C.c_void_p(cur.cuda_stream)), "sdr_separate")
        _leave_stream(st, cur)
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
    device = torch.device(device) if device is not None else _fetch(model, _probe_names(model)[0]).device
    if device.type != "cuda":
        raise RuntimeError("the model must live on a CUDA device")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    B, A, T = host_wav.shape
    if A != cfg.in_audio_channels:
        raise RuntimeError(f"expected {cfg.in_audio_channels} audio channel(s), got {A}")
    if host_out is None:
        host_out = torch.empty((B, cfg.num_sources * A, T), dtype=torch.float32).pin_memory()
    if tuple(host_out.shape) != (B, cfg.num_sources * A, T) or host_out.dtype != torch.float32 \
            or host_out.is_cuda or not host_out.is_contiguous():
        raise RuntimeError("host_out must be a contiguous fp32 CPU tensor [B, S*A, T]")
    mc = 1 if mixture_consistency else 0
    with torch.cuda.device(device):
        packed = packed_weights(model, cfg, device)
        st = _state(model, device)
        ws_bytes = lib.sdr_workspace_bytes(C.byref(cfg), B, T)
        io_bytes = lib.sdr_host_staging_bytes(C.byref(cfg), B, T)
        if ws_bytes == 0 or io_bytes == 0:
            raise N.NativeError("bad model configuration")
        _ensure_workspace(st, ws_bytes, device)
        if st.staging is None or st.staging.numel() < io_bytes:
            if st.event is not None:
                st.event.synchronize()
            st.graphs.clear()
            st.staging = torch.empty(io_bytes, dtype=torch.uint8, device=device)
        cur0 = _enter_stream(st, device)

        def enqueue():
            N.check(lib.sdr_forward_host(C.byref(cfg), C.c_void_p(packed.data_ptr()),
                                         C.c_void_p(host_wav.data_ptr()), C.c_void_p(host_out.data_ptr()),
                                         B, T, mc,
                                         C.c_void_p(st.staging.data_ptr()), st.staging.numel(),
                                         C.c_void_p(st.workspace.data_ptr()), st.workspace.numel(),
                                         _stream_ptr(device)), "sdr_forward_host")

        graphable = use_graph and host_wav.is_pinned() and host_out.is_pinned() \
            and not torch.cuda.is_current_stream_capturing()
        if not graphable:
            enqueue()
            _leave_stream(st, cur0)
            return host_out
        key = (host_wav.data_ptr(), host_out.data_ptr(), B, T, mc, st.workspace.data_ptr(),
               st.staging.data_ptr(), packed.data_ptr())
        entry = st.graphs.get(key)
        if entry is None:
            if len(st.graphs) >= 8:
                st.graphs.clear()
            st.graphs[key] = "warm"          # first call with this key: eager (also warms every kernel)
            enqueue()
        elif entry == "warm":
            cur = torch.cuda.current_stream(device)
            side = torch.cuda.Stream(device=device)
            side.wait_stream(cur)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                enqueue()
            cur.wait_stream(side)
            st.graphs[key] = graph
            graph.replay()
        else:
            entry.replay()
        _leave_stream(st, cur0)
    return host_out
