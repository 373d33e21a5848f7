"""Guard-band harness of the bounds tests (test_gpu_bounds.py, and test_bounds_harness_cpu.py on the CPU).

Every operand gets its own torch allocation laid out as [front guard | payload | back guard]. The guards are at least
64 KiB and at least one whole tile of the operand, so an over-read or over-write stays inside memory the test owns and
shows up without a fault:

* an input's guards (and the padding a kernel must not read) hold a poison that changes the answer if it is read: NaN
  for summed or multiplied operands, +Inf or 3e38 for maximised ones, a valid but wrong value for int32 operands;
* an output's or workspace's whole allocation is pre-filled with SENTINEL, a NaN payload no kernel produces. After the
  launch every guard byte must still hold what it held before (`check`), every byte the contract says is written must
  differ from the sentinel (`assert_written`) and every byte it says stays untouched must still hold it
  (`assert_untouched`).

The payload starts 256-byte aligned (TMA maps and the executor rely on it), plus `misalign` bytes for the scalar and
byte paths."""
from __future__ import annotations

import numpy as np

SENTINEL = 0x7FC0DEAD                       # a NaN payload: no kernel computes it, no copy of finite data produces it
NAN = 0x7FC00000
POS_INF = 0x7F800000
NEG_INF = 0xFF800000
BIG = int(np.array(3e38, np.float32).view(np.uint32))
FLOAT_POISONS = {"nan": np.float32(np.nan), "inf": np.float32(np.inf), "-inf": np.float32(-np.inf), "3e38": np.float32(3e38)}
GUARD_BYTES = 64 << 10
ALIGN = 256


def bits_of(value) -> int:
    """the 32-bit pattern of a float32 / int32 value or of an int already given as bits"""
    if isinstance(value, (float, np.floating)):
        return int(np.array(value, np.float32).view(np.uint32))
    return int(value) & 0xFFFFFFFF


class Guarded:
    """One allocation [front guard | payload of `nbytes` | back guard], every 32-bit word of it filled with `fill` (a float
    value or a bit pattern). `guard` is raised to GUARD_BYTES; pass the operand's tile size when that is larger."""

    def __init__(self, nbytes: int, fill=SENTINEL, guard: int = 0, misalign: int = 0, device: str = "cuda"):
        import torch
        self.nbytes = int(nbytes)
        self.guard = max(GUARD_BYTES, int(guard))
        self.guard += -self.guard % ALIGN
        total = self.guard + ALIGN + self.nbytes + misalign + self.guard
        total += -total % 4
        self.words = torch.empty(total // 4, dtype=torch.int32, device=device)
        self.fill_bits = bits_of(fill)
        self.words.fill_(np.array(self.fill_bits, np.uint32).view(np.int32).item())
        self.raw = self.words.view(torch.uint8)
        base = self.raw.data_ptr()
        self.start = self.guard + (-(base + self.guard) % ALIGN) + misalign
        self.end = self.start + self.nbytes
        self._snap = None

    @property
    def ptr(self) -> int:
        return self.raw.data_ptr() + self.start

    def view(self, dtype, shape=None):
        """the payload as a torch tensor of `dtype` (the payload offset must be a multiple of its size)"""
        import torch
        item = torch.empty((), dtype=dtype).element_size()
        assert self.start % item == 0 and self.nbytes % item == 0, "payload not aligned to the element size"
        v = self.raw[self.start:self.end].view(dtype)
        return v if shape is None else v.view(shape)

    def write(self, a: np.ndarray, at: int = 0):
        """copy the bytes of `a` into the payload from byte `at` on"""
        import torch
        b = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        assert at + b.size <= self.nbytes, "write past the payload"
        self.raw[self.start + at:self.start + at + b.size].copy_(torch.from_numpy(b.copy()))
        return self

    def fill_payload(self, value):
        """every 32-bit word of the payload set to `value` (float or bit pattern); the payload must be word aligned"""
        n = self.nbytes // 4
        return self.write(np.full(n, bits_of(value), np.uint32))

    def read(self, dtype=np.float32, shape=None) -> np.ndarray:
        a = self.raw[self.start:self.end].cpu().numpy().view(dtype)
        return a if shape is None else a.reshape(shape)

    def arm(self):
        """remember the guard bytes; `check` compares against this"""
        self._snap = (self.raw[:self.start].cpu().numpy().copy(), self.raw[self.end:].cpu().numpy().copy())
        return self

    def violations(self):
        """[(side, byte offset from the payload edge)] of every guard byte that changed since `arm` (the front side counts
        back from the payload start: offset 1 is the byte just before it)"""
        assert self._snap is not None, "arm() the buffer before the launch"
        front, back = self.raw[:self.start].cpu().numpy(), self.raw[self.end:].cpu().numpy()
        out = [("front", int(self.start - i)) for i in np.nonzero(front != self._snap[0])[0]]
        out += [("back", int(i)) for i in np.nonzero(back != self._snap[1])[0]]
        return out

    def check(self, name: str = "buffer"):
        v = self.violations()
        assert not v, f"{name}: {len(v)} guard bytes changed, first {v[:4]}"


def guarded_input(a: np.ndarray, fill, guard: int = 0, misalign: int = 0, device: str = "cuda") -> Guarded:
    """`a` between guards of `fill`, armed"""
    return Guarded(a.nbytes, fill=fill, guard=guard, misalign=misalign, device=device).write(a).arm()


def guarded_output(nbytes: int, guard: int = 0, misalign: int = 0, device: str = "cuda") -> Guarded:
    """`nbytes` of SENTINEL between guards of SENTINEL, armed"""
    return Guarded(nbytes, fill=SENTINEL, guard=guard, misalign=misalign, device=device).arm()


def sentinel_mask(a: np.ndarray) -> np.ndarray:
    """True for every 32-bit word of `a` that still holds SENTINEL"""
    return np.ascontiguousarray(a).view(np.uint32) == np.uint32(SENTINEL)


def assert_written(a: np.ndarray, what: str = "output"):
    m = sentinel_mask(a)
    assert not m.any(), f"{what}: {int(m.sum())} words the kernel must write still hold the sentinel, first at {np.argwhere(m)[:4].tolist()}"


def assert_untouched(a: np.ndarray, what: str = "output"):
    m = sentinel_mask(a)
    assert m.all(), f"{what}: {int((~m).sum())} words the kernel must not write were written, first at {np.argwhere(~m)[:4].tolist()}"


def assert_rows_bit_equal(clean: np.ndarray, other: np.ndarray, skip, what: str = "output"):
    """every row (axis 0) of `other` except those in `skip` carries the bits of `clean`"""
    c, o = np.ascontiguousarray(clean), np.ascontiguousarray(other)
    assert c.shape == o.shape
    keep = np.ones(c.shape[0], bool)
    keep[list(skip)] = False
    cb, ob = c.view(np.uint8).reshape(c.shape[0], -1), o.view(np.uint8).reshape(o.shape[0], -1)
    bad = [int(r) for r in np.nonzero(keep & (cb != ob).any(axis=1))[0]]
    assert not bad, f"{what}: rows {bad[:8]} changed when only rows {list(skip)} were poisoned"
