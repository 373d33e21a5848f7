"""The guard-band harness of test_gpu_bounds.py on CPU buffers: numpy stand-ins for kernels that write or read one element
out of bounds, and the check that reports each of them."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds_harness as bh  # noqa: E402


def _np(g):
    return g.raw.numpy()


def _copy(dst, src, n, lo=0):
    """the stand-in kernel: copies bytes [lo, n) of src's payload to dst's"""
    _np(dst)[dst.start + lo:dst.start + n] = _np(src)[src.start + lo:src.start + n]


def _pair(nbytes, misalign=0):
    src = bh.guarded_input(np.arange(nbytes, dtype=np.uint8), fill=bh.NAN, misalign=misalign, device="cpu")
    return src, bh.guarded_output(nbytes, misalign=misalign, device="cpu")


@pytest.mark.parametrize("misalign", [0, 1, 4])
def test_payload_is_aligned_and_guards_are_large(misalign):
    g = bh.Guarded(1000, misalign=misalign, guard=200_000, device="cpu")
    assert (g.ptr - misalign) % bh.ALIGN == 0
    assert g.start >= 200_000 and g.raw.numel() - g.end >= 200_000
    assert bh.Guarded(4, device="cpu").start >= bh.GUARD_BYTES


@pytest.mark.parametrize("misalign", [0, 1, 4])
def test_an_exact_copy_passes(misalign):
    src, dst = _pair(1003, misalign)
    _copy(dst, src, 1003)
    src.check("src")
    dst.check("dst")
    assert np.array_equal(dst.read(np.uint8), np.arange(1003, dtype=np.uint8))


@pytest.mark.parametrize("extra", [1, 4])
def test_a_write_past_the_end_is_reported(extra):
    src, dst = _pair(64)
    _np(dst)[dst.start:dst.end + extra] = 7                 # the kernel's length is `extra` bytes too long
    v = dst.violations()
    assert v and all(s == "back" for s, _ in v) and min(o for _, o in v) == 0
    with pytest.raises(AssertionError, match="guard bytes changed"):
        dst.check("dst")


def test_a_write_before_the_start_is_reported():
    src, dst = _pair(64)
    _np(dst)[dst.start - 4:dst.start] = 0                   # one float before the payload
    assert dst.violations() == [("front", 4), ("front", 3), ("front", 2), ("front", 1)]


def test_an_input_written_by_the_kernel_is_reported():
    src, dst = _pair(64)
    _np(src)[src.end] = 0xAB
    with pytest.raises(AssertionError):
        src.check("src")


def test_a_read_past_the_end_is_poisoned():
    """an over-read of one float picks up the guard's NaN and the sum shows it"""
    x = bh.guarded_input(np.ones(37, np.float32), fill=bh.NAN, device="cpu")
    whole = _np(x).view(np.float32)
    ok = whole[x.start // 4:x.end // 4].sum()
    over = whole[x.start // 4:x.end // 4 + 1].sum()
    under = whole[x.start // 4 - 1:x.end // 4].sum()
    assert ok == 37 and np.isnan(over) and np.isnan(under)


def test_a_maximum_over_a_read_past_the_end_is_poisoned():
    x = bh.guarded_input(np.zeros(5, np.float32), fill=bh.POS_INF, device="cpu")
    whole = _np(x).view(np.float32)
    assert whole[x.start // 4:x.end // 4].max() == 0 and whole[x.start // 4:x.end // 4 + 1].max() == np.inf


def test_a_missed_write_and_a_stray_write_are_reported():
    y = bh.guarded_output(4 * 12, device="cpu")
    out = _np(y)[y.start:y.end].view(np.float32).reshape(3, 4)
    out[:, :3] = 1.0                                        # columns [0, 3) are the contract, column 3 stays untouched
    bh.assert_written(y.read(shape=(3, 4))[:, :3])
    bh.assert_untouched(y.read(shape=(3, 4))[:, 3:])
    out[1, 3] = 0.0                                         # a stray write into the untouched column
    with pytest.raises(AssertionError, match="must not write"):
        bh.assert_untouched(y.read(shape=(3, 4))[:, 3:])
    out[2, 2] = np.array(bh.SENTINEL, np.uint32).view(np.float32)   # a missed write
    with pytest.raises(AssertionError, match="still hold the sentinel"):
        bh.assert_written(y.read(shape=(3, 4))[:, :3])


def test_row_isolation_check():
    clean = np.arange(12, dtype=np.float32).reshape(4, 3)
    other = clean.copy()
    other[2] = np.nan
    bh.assert_rows_bit_equal(clean, other, [2])
    other[0, 1] = np.float32(-0.0) if clean[0, 1] == 0 else np.nextafter(clean[0, 1], np.float32(9))
    with pytest.raises(AssertionError, match=r"rows \[0\]"):
        bh.assert_rows_bit_equal(clean, other, [2])


def test_poison_bit_patterns():
    assert np.isnan(np.array(bh.NAN, np.uint32).view(np.float32))
    assert np.isnan(np.array(bh.SENTINEL, np.uint32).view(np.float32))
    assert np.array(bh.POS_INF, np.uint32).view(np.float32) == np.inf
    assert np.array(bh.NEG_INF, np.uint32).view(np.float32) == -np.inf
    assert np.array(bh.BIG, np.uint32).view(np.float32) == np.float32(3e38)
    assert bh.bits_of(np.float32(np.nan)) == bh.NAN and bh.bits_of(-1) == 0xFFFFFFFF
