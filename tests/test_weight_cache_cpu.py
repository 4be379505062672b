"""Host logic of the packed-weight cache (sudo_rm_rf_b200/_engine.py), on CPU tensors.

The cache re-packs when the weight signature changes: each parameter's address and version counter, plus a generation
that every optimizer step bumps.  Which writes move a version counter is torch's behaviour, not ours, so it is pinned
here idiom by idiom: an upgrade that changes it is noticed.  Then the signature itself, the storages it keeps alive,
``refresh_weights`` and the retirement of buffers a captured graph may still address."""
import os
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.nn as nn
from torch.optim.swa_utils import AveragedModel
from torch.utils import dlpack

import sudo_rm_rf_b200 as P
from sudo_rm_rf_b200 import _engine as E

SMALL = dict(out_channels=16, in_channels=32, num_blocks=1, upsampling_depth=2, enc_kernel_size=21,
             enc_num_basis=24, num_sources=2)


def _param():
    p = nn.Parameter(torch.randn(4, 3, generator=torch.Generator().manual_seed(0)))
    p.grad = torch.randn(4, 3, generator=torch.Generator().manual_seed(1))
    return p


def _optimizer(name, mode):
    cls = getattr(torch.optim, name)

    def step(p):
        kw = {"foreach": True} if mode == "foreach" else {"fused": True} if mode == "fused" else {"foreach": False}
        cls([p], lr=0.1, **kw).step()
    return step


def _broadcast(p):
    store = tempfile.mktemp()
    dist.init_process_group("gloo", init_method="file://" + store, rank=0, world_size=1)
    try:
        dist.broadcast(p.data, 0)
    finally:
        dist.destroy_process_group()
        if os.path.exists(store):
            os.remove(store)


def _averaged(p):
    avg = AveragedModel(nn.Linear(3, 4))
    q = next(avg.module.parameters())
    v0 = q._version
    avg.update_parameters(nn.Linear(3, 4))
    avg.update_parameters(nn.Linear(3, 4))       # the first call copies, the second averages in place
    assert q._version > v0
    with torch.no_grad():
        p.add_(1.0)


def _no_grad(fn):
    def run(p):
        with torch.no_grad():
            fn(p)
    return run


# (idiom, writes p, bumps p._version on this torch)
IDIOMS = [
    ("load_state_dict", lambda p: _load_state_dict(p), True),
    ("no_grad_inplace", _no_grad(lambda p: p.mul_(2.0)), True),
    ("no_grad_copy", _no_grad(lambda p: p.copy_(torch.ones(4, 3))), True),
    ("detach_write", lambda p: p.detach().mul_(2.0), True),
    ("nn_init", lambda p: nn.init.normal_(p), True),
    ("averaged_model", _averaged, True),
    ("data_mul", lambda p: p.data.mul_(2.0), False),
    ("data_copy", lambda p: p.data.copy_(torch.ones(4, 3)), False),
    ("dlpack_write", lambda p: dlpack.from_dlpack(dlpack.to_dlpack(p.data)).mul_(2.0), False),
    ("dist_broadcast_data", _broadcast, False),
] + [(f"{o}_{mode}", _optimizer(o, mode), mode != "fused")
     for o in ("SGD", "Adam", "AdamW", "Adagrad") for mode in ("single", "foreach", "fused")]


def _load_state_dict(p):
    lin = nn.Linear(3, 4)
    lin.weight = p
    lin.load_state_dict({"weight": torch.zeros(4, 3), "bias": torch.zeros(4)})


@pytest.mark.parametrize("name,fn,bumps", IDIOMS, ids=[i[0] for i in IDIOMS])
def test_which_idioms_bump_the_version_counter(name, fn, bumps):
    p = _param()
    v0, ptr = p._version, p.data_ptr()
    fn(p)
    assert p.data_ptr() == ptr
    assert (p._version != v0) == bumps, (name, v0, p._version)


@pytest.mark.parametrize("name", ["SGD", "Adam", "AdamW", "Adagrad"])
@pytest.mark.parametrize("mode", ["single", "foreach", "fused"])
def test_every_optimizer_step_changes_the_signature(name, mode):
    """The fused steps leave the version counter alone (above); the generation moves for every kind."""
    p = _param()
    g0 = E._generation
    sig = E.weight_signature([p])
    _optimizer(name, mode)(p)
    assert E._generation == g0 + 1
    assert E.weight_signature([p]) != sig


def test_signature_of_untracked_writes_is_unchanged():
    """p.data writes are invisible to the signature: refresh_weights() is their remedy."""
    p = _param()
    sig = E.weight_signature([p])
    p.data.mul_(3.0)
    p.data.copy_(torch.zeros(4, 3))
    assert E.weight_signature([p]) == sig


def test_swapped_storage_cannot_come_back_under_the_kept_address():
    """p.data = t keeps p's version counter, so only the address tells the swap apart.  The cache keeps the storages
    its signature describes: the old address stays taken, and the new tensor's signature differs."""
    p = _param()
    q = nn.Parameter(torch.randn(7))
    sig = E.weight_signature([p, q])
    kept = E.weight_storages([p, q])
    old_ptr, old_val = p.data_ptr(), p.detach().clone()
    v0 = p._version
    p.data = torch.full((4, 3), 5.0)
    assert p._version == v0
    assert kept[0].data_ptr() == old_ptr
    assert torch.equal(torch.empty(0).set_(kept[0]).view(4, 3), old_val)     # still alive, untouched
    assert p.data_ptr() != old_ptr
    assert E.weight_signature([p, q]) != sig
    assert E.weight_signature([p, q])[1][1] == sig[1][1]                      # q unchanged


def test_replaced_parameter_changes_the_signature_tensors():
    m = P.SuDORMRF(**SMALL)
    names = E.state_dict_names(E.make_config(m))
    st = E._DeviceState()
    st.tensors, st.pslots, st.mslots = E._walk(m, names)
    assert E._cached_tensors(st) is st.tensors
    m.decoder.weight = nn.Parameter(m.decoder.weight.detach().clone())
    assert E._cached_tensors(st) is None
    st.tensors, st.pslots, st.mslots = E._walk(m, names)
    m.sm[0] = type(m.sm[0])(out_channels=16, in_channels=32, upsampling_depth=2)
    assert E._cached_tensors(st) is None


@pytest.mark.parametrize("wrap", [False, True])
def test_refresh_weights_forces_a_repack(wrap):
    m = P.SuDORMRF(**SMALL)
    cache = m.__dict__.setdefault("_b200_cache", {})
    for idx in (0, 1):
        cache[idx] = E._DeviceState()
        cache[idx].sig = (E._generation, ((1, 0),))
    P.refresh_weights(nn.DataParallel(m) if wrap else m)
    assert all(st.sig is None for st in cache.values())
    P.refresh_weights(P.SuDORMRF(**SMALL))          # a model that never ran: nothing to do


def test_captured_buffers_are_retired_not_freed():
    """A buffer a capture addressed goes to the retired list when replaced; one no capture saw is dropped."""
    st = E._DeviceState()
    a, b, c = torch.empty(8), torch.empty(8), torch.empty(16)
    E._replace(st, "packed", a)
    st.captured.add("packed")                   # what _hand_out records under stream capture
    E._replace(st, "packed", b)
    assert st.packed is b and len(st.retired) == 1 and st.retired[0] is a
    assert "packed" not in st.captured
    E._replace(st, "packed", c)                 # b was never captured: freed as before
    assert st.packed is c and len(st.retired) == 1
    E._replace(st, "workspace", a)
    st.captured.add("workspace")
    E._replace(st, "workspace", None)
    assert st.workspace is None and st.retired[-1] is a
    E.drop_cache(m := P.SuDORMRF(**SMALL))      # drop_cache on a model without a cache is a no-op
    assert "_b200_cache" not in m.__dict__
