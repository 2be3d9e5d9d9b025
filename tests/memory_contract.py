"""Where the kernels write, and what they read: buffers for checking that an entry point writes exactly its outputs, leaves
its inputs alone and reads no workspace word it has not written.  Shared by tests/test_memory_contract_gpu.py,
tests/test_forced_plans_gpu.py and tests/forced_plans.py; tests/test_memory_contract_cpu.py shows on CPU tensors that
every check fires.

Sentinel.  Every buffer starts filled with the quiet NaN 0x7FC0A5A5.  GPU arithmetic only ever produces the canonical NaN
0x7FFFFFFF, so a word that still holds the sentinel after a call was never stored to.  A kernel that reads a workspace
word before writing it either copies the sentinel on (caught as unwritten) or computes with it; a second run on a zero
filled workspace then gives other bits.

Guards.  A checked buffer sits `offset_bytes` into a larger allocation with at least GUARD_BYTES of sentinel on both
sides: a store past either end of an output or a workspace changes a guard word.  Torch's allocator would otherwise put
a neighbouring tensor there, where an overrun goes unseen.
"""
import torch

SENTINEL = 0x7FC0A5A5
GUARD_BYTES = 4096


def _sentinel_bytes(nbytes, device):
    assert nbytes % 4 == 0
    return torch.full((nbytes // 4,), SENTINEL, dtype=torch.int32, device=device).view(torch.uint8)


class Guarded:
    """`nbytes` of memory `offset_bytes` (a multiple of 4) past an aligned start, inside sentinel guards.  `t` is the
    interior as a `dtype` tensor of `shape` (default: flat uint8); `fill` is 'sentinel' or 'zero' (the guards always hold
    the sentinel)."""

    def __init__(self, nbytes, offset_bytes=0, device='cuda', dtype=torch.uint8, shape=None, fill='sentinel'):
        assert offset_bytes % 4 == 0 and fill in ('sentinel', 'zero')
        self.nbytes = nbytes
        self.lo = GUARD_BYTES + offset_bytes
        self.hi = self.lo + nbytes
        total = (self.hi + GUARD_BYTES + 3) // 4 * 4
        self.buf = _sentinel_bytes(total, device)
        if fill == 'zero':
            self.buf[self.lo:self.hi].zero_()
        flat = self.buf[self.lo:self.hi].view(dtype)
        self.t = flat if shape is None else flat.view(shape)

    def ptr(self):
        return self.buf.data_ptr() + self.lo

    def guards_intact(self):
        ref = _sentinel_bytes(self.buf.numel(), self.buf.device)
        return torch.equal(self.buf[:self.lo], ref[:self.lo]) and torch.equal(self.buf[self.hi:], ref[self.hi:])

    def untouched(self):
        """The whole allocation, interior included, still holds the sentinel."""
        return torch.equal(self.buf, _sentinel_bytes(self.buf.numel(), self.buf.device))


def guarded(shape, offset_bytes=0, device='cuda'):
    """An fp32 output of `shape`, sentinel-filled, `offset_bytes` into its guarded allocation."""
    n = 1
    for s in shape:
        n *= s
    return Guarded(4 * n, offset_bytes, device, torch.float32, tuple(shape))


def workspace(nbytes, offset_bytes=0, fill='sentinel', device='cuda'):
    """A workspace of exactly `nbytes` (the queried size) at `offset_bytes` past a 16-byte boundary, guarded after and
    before.  nbytes is rounded up to whole words inside the guard, so a size that is not a multiple of 4 is not
    checked to the byte."""
    return Guarded((nbytes + 3) // 4 * 4, offset_bytes, device, torch.uint8, None, fill)


def words(t):
    """The 32-bit words of an fp32 / int32 tensor."""
    return t.contiguous().view(torch.int32)


def n_unwritten(t):
    """How many words of `t` still hold the sentinel."""
    return int((words(t) == SENTINEL).sum())


def same_bits(a, b):
    """Equal bit patterns at equal places, except that any NaN matches any NaN (0.0 and -0.0 differ)."""
    if a.shape != b.shape:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(words(a)[~na], words(b)[~nb])


def snapshot(tensors):
    """Copies of the inputs of a call, for unchanged()."""
    return [None if t is None else t.clone() for t in tensors]


def unchanged(before, after):
    """Every input still has exactly its bits (NaN payloads included)."""
    return all((a is None and b is None) or torch.equal(words(a), words(b)) for a, b in zip(before, after))


def assert_written(g, what):
    """An output after the call: nothing stored outside it, nothing in it left unwritten."""
    assert g.guards_intact(), f'{what}: a store landed outside the buffer'
    left = n_unwritten(g.t)
    assert left == 0, f'{what}: {left} of {g.t.numel()} elements never written'
