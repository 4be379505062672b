"""Guard bands around the buffers a stage test hands to a kernel.

Every buffer sits between two bands of a fixed bit pattern: a write outside the tensor would land in the neighbouring
workspace segment of the model and show in no output, so the bands are checked after each call, and the inputs are
checked bitwise unchanged."""
import torch

GUARD = 1024                 # elements on either side: keeps the interior 16 B aligned (TMA) for every dtype used here
GUARD_BITS = 0x7FA5A5A5      # a NaN in fp32 and in the high word of an fp64


def guarded(src):
    """A contiguous copy of `src` (same device and dtype) inside a buffer with GUARD elements of GUARD_BITS on either
    side; the returned tensor is a view of that buffer."""
    n = src.numel()
    assert (n * src.element_size()) % 4 == 0
    buf = torch.empty(n + 2 * GUARD, dtype=src.dtype, device=src.device)
    buf.view(torch.int32).fill_(GUARD_BITS)
    t = buf[GUARD:GUARD + n].view(src.shape)
    t.copy_(src)
    return t


def assert_guards_intact(t, what):
    buf = t._base
    assert buf is not None and buf.numel() == t.numel() + 2 * GUARD, f"{what} was not made by guarded()"
    words = buf.view(torch.int32)
    es = buf.element_size()
    head = int((words[:GUARD * es // 4] != GUARD_BITS).sum())
    tail = int((words[(GUARD + t.numel()) * es // 4:] != GUARD_BITS).sum())
    assert head == 0 and tail == 0, f"{what}: {head} words written before and {tail} after the tensor"


class Guards:
    """Guarded device copies of one call's buffers.  check(): no guard was written, no input changed."""

    def __init__(self):
        self.outputs, self.inputs = {}, {}

    def output(self, name, src):
        self.outputs[name] = guarded(src)
        return self.outputs[name]

    def input(self, name, src):
        t = guarded(src)
        self.inputs[name] = (t, t.clone())
        return t

    def check(self):
        torch.cuda.synchronize()
        for name, t in self.outputs.items():
            assert_guards_intact(t, name)
        for name, (t, before) in self.inputs.items():
            assert_guards_intact(t, name)
            assert torch.equal(t.view(torch.uint8), before.view(torch.uint8)), f"input {name} was modified"
