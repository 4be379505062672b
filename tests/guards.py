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


# ---------------------------------------------------------------------------------------------------------------------
# scratch memory whose content on entry is chosen: exactly-sized byte buffers between guard bands
# ---------------------------------------------------------------------------------------------------------------------
POISON_NAN = 0x7FA5A5A5      # NaN in fp32, 7.6e306 when two words pair up as an fp64: propagates through arithmetic
POISON_HUGE = 0x7149F2CA     # 1e30 in fp32, 5.3e237 as an fp64: finite, so it survives what swallows a NaN
                             # (fmaxf-style ReLU, max, comparisons, the PReLU select)
BAND_BYTES = 4096            # guard band on either side of the interior


def _fill_words(t, pattern):
    """Fills a uint8 tensor whose base is 4 B aligned with a 32-bit pattern (little endian; a tail of 1-3 bytes gets
    the pattern's first bytes)."""
    n4 = t.numel() // 4 * 4
    word = pattern if pattern < 2 ** 31 else pattern - 2 ** 32
    if n4:
        t[:n4].view(torch.int32).fill_(word)
    for i in range(n4, t.numel()):
        t[i] = (pattern >> (8 * (i - n4))) & 0xFF


def poisoned(nbytes, pattern, align=256, device="cuda"):
    """A uint8 buffer of exactly `nbytes` whose base is `align`-aligned, every 32-bit word of it `pattern` (0: the clean
    run), between two BAND_BYTES bands of GUARD_BITS.  check_bands(t, what) verifies the bands afterwards."""
    assert nbytes > 0 and align % 4 == 0 and BAND_BYTES % 4 == 0
    buf = torch.empty(nbytes + 2 * BAND_BYTES + align + 3, dtype=torch.uint8, device=device)
    start = (-buf.data_ptr()) % 4                                    # CPU tensors may start anywhere
    off = start + BAND_BYTES + (-(buf.data_ptr() + start + BAND_BYTES)) % align
    _fill_words(buf[start:off], GUARD_BITS)
    tail = buf[off + nbytes:]
    tail_start = (-tail.data_ptr()) % 4
    tail[:tail_start].fill_(0xA5)
    _fill_words(tail[tail_start:], GUARD_BITS)
    t = buf[off:off + nbytes]
    _fill_words(t, pattern)
    assert t.data_ptr() % align == 0 and t.numel() == nbytes
    t._bands = (buf, off, nbytes, buf[:off].clone(), tail.clone())
    return t


def repoison(t, pattern):
    """Refills the interior of a poisoned() buffer (or any 4 B aligned uint8 tensor) in place."""
    _fill_words(t.view(-1), pattern)


def check_bands(t, what):
    """No byte of either band of a poisoned() buffer has changed."""
    buf, off, nbytes, head, tail = t._bands
    if buf.is_cuda:
        torch.cuda.synchronize()
    before = int((buf[:off] != head).sum())
    after = int((buf[off + nbytes:] != tail).sum())
    assert before == 0 and after == 0, f"{what}: {before} bytes written before and {after} after the buffer"


def poisoned_like(src, pattern):
    """A tensor of src's shape and dtype that fills a poisoned() buffer exactly (256 B aligned base)."""
    t = poisoned(src.numel() * src.element_size(), pattern, device=src.device)
    v = t.view(src.dtype).view(src.shape)
    v._bands = t._bands
    return v


def guarded_copy(src):
    """poisoned_like(src) holding src's values: an input whose neighbours are guard bands."""
    v = poisoned_like(src, 0)
    v.copy_(src)
    return v
