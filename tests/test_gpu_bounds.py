"""-m gpu: every raw kernel reads and writes only its own bytes, and one row's values never reach another row's bits.

Each operand sits in its own allocation between guard bands (bounds_harness.py): inputs between poison (NaN for summed
operands, +Inf for maximised ones, valid but wrong ids and mask values for int32 operands), outputs and workspaces between
and under the sentinel 0x7FC0DEAD. A case passes when the result matches fp64 / numpy, no guard byte changed, every
output word the contract writes was written and every word it leaves alone still holds the sentinel. Workspaces are
allocated at exactly the size the library reports, and their arrival counters must be zero after every launch.

Row isolation: a batched kernel is launched once clean and once with one row (sequence, image) poisoned with NaN, +Inf,
-Inf or 3e38; every other row must keep the clean launch's bits. The served path gets the same check for requests
coalesced into one batch and for tfsc_predict_device's rows past the batch."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds_harness as bh  # noqa: E402

pytestmark = pytest.mark.gpu
lib = t._lib.lib
TOL = 1e-4
POISONS = list(bh.FLOAT_POISONS)


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device; there is no CPU fallback"
    return torch


def _done(rc, what):
    t._lib.check(rc, what)
    _torch().cuda.synchronize()


def _err(got, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


def _inp(a, fill=bh.NAN, guard=0, misalign=0):
    return bh.guarded_input(np.ascontiguousarray(a), fill, guard=guard, misalign=misalign)


def _out(nbytes, guard=0, misalign=0):
    return bh.guarded_output(nbytes, guard=guard, misalign=misalign)


def _check(**bufs):
    for name, g in bufs.items():
        g.check(name)


def _poisoned(a, j, p):
    """a copy of `a` whose row j (axis 0) is all poison p"""
    b = np.array(a, copy=True)
    b[j] = bh.FLOAT_POISONS[p]
    return b


# ---------------------------------------------------------------------------------------------- X6 / X7 ----
def _segments(segs):
    arr = (t._lib.TfscCopySeg * max(1, len(segs)))()
    for i, (s, d, n) in enumerate(segs):
        arr[i].src, arr[i].dst, arr[i].bytes = s, d, n
    return arr


def test_copy_segments_guard_check_fires_on_a_long_segment():
    """a length 4 bytes past the payload writes into the destination's own back guard: the check must report it"""
    n = 4096
    src = bh.Guarded(n + 4, fill=0x01020304).write(np.arange(n, dtype=np.uint8)).arm()
    dst = _out(n)
    _done(lib.tfsc_k_copy_segments(_segments([(src.ptr, dst.ptr, n + 4)]), 1, None), "copy_segments")
    v = dst.violations()
    assert v and {s for s, _ in v} == {"back"} and max(o for _, o in v) < 4, v[:8]


def test_copy_segments_bit_exact_over_every_path():
    """more than 64 segments (two launches), zero-length ones, lengths = 0, 1, 2, 3 mod 4 and 0 mod 16, offsets 0, 4, 1
    (the 16-byte, 4-byte and byte paths), up to 1 MiB"""
    rng = np.random.default_rng(0)
    lengths = [0, 1, 2, 3, 4, 5, 6, 7, 15, 16, 17, 31, 32, 48, 63, 64, 65, 255, 256, 1000, 1001, 1002, 1003, 4096, 16383,
               16384, 16385, 65536 + 12, 1 << 20]
    cases = [(n, off) for off in (0, 4, 1) for n in lengths]
    rng.shuffle(cases)
    cases = cases[:40] + [(0, 0)] * 5 + cases[40:]
    assert len(cases) > 64
    bufs = []
    for n, off in cases:
        data = rng.integers(0, 256, n, dtype=np.uint8)
        src = bh.Guarded(n, fill=bh.NAN, misalign=off).write(data).arm()
        dst = _out(n, misalign=(off * 3) % 16)
        bufs.append((data, src, dst))
    segs = _segments([(s.ptr, d.ptr, len(data)) for data, s, d in bufs])
    _done(lib.tfsc_k_copy_segments(segs, len(bufs), None), "copy_segments")
    for i, (data, src, dst) in enumerate(bufs):
        _check(src=src, dst=dst)
        assert np.array_equal(dst.read(np.uint8), data), (i, len(data))


def test_copy_segments_all_zero_table():
    dst = _out(64)
    segs = _segments([(dst.ptr, dst.ptr, 0)] * 64 + [(dst.ptr, dst.ptr, 0)] * 3)
    _done(lib.tfsc_k_copy_segments(segs, 67, None), "copy_segments")
    dst.check("dst")
    bh.assert_untouched(dst.read(np.uint32))


# --------------------------------------------------------------------------------------------------- X1 ----
@pytest.mark.parametrize("n", [1, 3, 4, 5, (1 << 20) + 3])
@pytest.mark.parametrize("misalign", [0, 4])
def test_affine(n, misalign):
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
    xg, yg = _inp(x, misalign=misalign), _out(4 * n, misalign=misalign)
    ab = _inp(np.array([0.5, 2.0], np.float32))
    _done(lib.tfsc_k_affine(xg.ptr, yg.ptr, n, ab.ptr, ab.ptr + 4, None), "affine")
    _check(x=xg, y=yg, ab=ab)
    assert np.array_equal(yg.read(), np.float32(0.5) * x + np.float32(2.0))


# ----------------------------------------------------------------------------------------- X2 / X3 dense ----
def _counter_words(n):
    """the counter region both split-K layouts start their workspace with (the tensor-core plan has the more strips)"""
    return ((-(-n // 256)) * 4 + 255) // 256 * 64


def _dense(x, w, b, relu, variant, launches=2):
    """launches back to back on one workspace of exactly tfsc_k_dense_workspace bytes; returns y. variant None is
    tfsc_k_dense, "tc" tfsc_k_dense_tc, a number tfsc_k_dense_variant"""
    rows, k = x.shape
    n = w.shape[1]
    wsb = lib.tfsc_k_dense_workspace(rows, k, n)
    ws = bh.Guarded(wsb, fill=bh.SENTINEL).fill_payload(0).arm()
    xg = _inp(x, guard=64 * k * 4)
    wg, bg = _inp(w, guard=8 * n * 4), _inp(b)
    ys = []
    for _ in range(launches):
        yg = _out(4 * rows * n, guard=64 * n * 4)
        if variant is None:
            rc = lib.tfsc_k_dense(xg.ptr, wg.ptr, bg.ptr, yg.ptr, rows, k, n, int(relu), ws.ptr, wsb, None)
        elif variant == "tc":
            rc = lib.tfsc_k_dense_tc(xg.ptr, wg.ptr, bg.ptr, yg.ptr, rows, k, n, int(relu), ws.ptr, wsb, None)
        else:
            rc = lib.tfsc_k_dense_variant(variant, xg.ptr, wg.ptr, bg.ptr, yg.ptr, rows, k, n, int(relu), ws.ptr, wsb, None)
        _done(rc, f"dense {variant}")
        _check(x=xg, w=wg, b=bg, y=yg, workspace=ws)
        cw = min(_counter_words(n), wsb // 4)
        c = ws.read(np.uint32)[:cw]
        assert not c.any(), f"arrival counters not back at zero: {np.nonzero(c)[0][:8]}"
        y = yg.read(shape=(rows, n))
        bh.assert_written(y, "y")
        ys.append(y)
    for y in ys[1:]:
        assert np.array_equal(y.view(np.uint32), ys[0].view(np.uint32)), "a second launch on the same workspace changed y"
    return ys[0]


def _dense_case(rows, k, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    return x, w, b


def _dense_ref(x, w, b, relu):
    r = x.astype(np.float64) @ w.astype(np.float64) + b
    return np.maximum(r, 0) if relu else r


DENSE_ROWS = [1, 2, 3, 5, 8, 9, 16, 17, 48, 63, 64, 65, 128, 129]


@pytest.mark.parametrize("rows", DENSE_ROWS)
@pytest.mark.parametrize("k,n", [(128, 520), (129, 8), (132, 1032), (4097, 4104), (4099, 4100)])
def test_dense(rows, k, n):
    """tfsc_k_dense itself. k = 4097 is one past the SIMT kernel's 4096-row x stage (two or more K splits); n = 4100 is
    not a multiple of 8 and runs the generic kernel"""
    x, w, b = _dense_case(rows, k, n, rows * 31 + k + n)
    got = _dense(x, w, b, True, None)
    assert _err(got, _dense_ref(x, w, b, True)) <= TOL


@pytest.mark.parametrize("variant", [1, 2, 4, 5])
@pytest.mark.parametrize("rows", [1, 3, 8, 9, 65])
@pytest.mark.parametrize("k,n", [(128, 520), (4096, 1032)])
def test_dense_variants(variant, rows, k, n):
    x, w, b = _dense_case(rows, k, n, variant * 7 + rows * 31 + k + n)
    got = _dense(x, w, b, False, variant)
    assert _err(got, _dense_ref(x, w, b, False)) <= TOL


@pytest.mark.parametrize("variant", [0, 1, 2, 4])
@pytest.mark.parametrize("rows", [8, 65, 72])
def test_dense_mixed_passes_share_the_workspace_past_16384_columns(variant, rows):
    """past 16,384 columns the tensor-core plan has more than 64 strips, so its arrival counters spill past the first 256
    bytes of the workspace. A 64-row tensor-core pass and a <= 8-row split-K pass then share one workspace: each must
    find its counters at zero, launch after launch."""
    x, w, b = _dense_case(rows, 256, 16640, rows + variant)
    got = _dense(x, w, b, False, variant, launches=3)
    assert _err(got, _dense_ref(x, w, b, False)) <= TOL


@pytest.mark.parametrize("rows", [1, 9, 16, 17, 48, 63, 64])
@pytest.mark.parametrize("k,n", [(128, 256), (132, 1024), (4100, 4096)])
def test_dense_tc(rows, k, n):
    x, w, b = _dense_case(rows, k, n, rows * 13 + k + n)
    got = _dense(x, w, b, True, "tc")
    assert _err(got, _dense_ref(x, w, b, True)) <= TOL


@pytest.mark.parametrize("variant,rows,j", [(0, 8, 0), (0, 8, 7), (0, 8, 3), (0, 64, 0), (0, 64, 63), (0, 64, 31),
                                            (0, 129, 0), (0, 129, 128), (0, 129, 70), (1, 8, 4), (2, 8, 4), (4, 5, 4),
                                            ("tc", 48, 47), ("tc", 17, 16)])
@pytest.mark.parametrize("poison", POISONS)
def test_dense_row_isolation(variant, rows, j, poison):
    x, w, b = _dense_case(rows, 4096, 1024, rows + 5)
    clean = _dense(x, w, b, True, variant, launches=1)
    dirty = _dense(_poisoned(x, j, poison), w, b, True, variant, launches=1)
    bh.assert_rows_bit_equal(clean, dirty, [j], "y")


# -------------------------------------------------------------------------------------------------- gemm ----
def _gemm(fn, a_full, m, n, k, lda, bmat, bias, r, act):
    """A [m, lda] with columns [k, lda) and the rows past m poison, B [k, n] between NaN, C between sentinels"""
    ag = _inp(a_full, guard=128 * lda * 4)
    bg = _inp(bmat, guard=64 * n * 4)
    biasg = _inp(bias) if bias is not None else None
    rg = _inp(r, guard=128 * n * 4) if r is not None else None
    cg = _out(4 * m * n, guard=128 * n * 4)
    _done(getattr(lib, fn)(ag.ptr, bg.ptr, biasg.ptr if biasg else None, rg.ptr if rg else None, cg.ptr, m, n, k, lda, act, None), fn)
    _check(a=ag, b=bg, c=cg, **({"bias": biasg} if biasg else {}), **({"r": rg} if rg else {}))
    c = cg.read(shape=(m, n))
    bh.assert_written(c, "c")
    return c


def _gemm_case(m, n, k, lda, seed):
    rng = np.random.default_rng(seed)
    a = np.full((m, lda), np.nan, np.float32)
    a[:, :k] = rng.standard_normal((m, k))
    bmat = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float32)
    return a, bmat, bias, r


def _gemm_ref(a, k, bmat, bias, r, act):
    v = a[:, :k].astype(np.float64) @ bmat + bias + r
    return np.maximum(v, 0) if act == 1 else v


GEMM_TC = [(m, n, k, lda) for m, n in [(64, 64), (65, 96), (127, 160), (128, 224), (129, 64), (255, 96), (257, 224)]
           for k, lda in [(32, 32), (33, 36), (63, 124), (65, 68), (4099, 4100)]]


@pytest.mark.parametrize("m,n,k,lda", GEMM_TC)
def test_gemm_tc(m, n, k, lda):
    if lda % 4:
        pytest.skip("lda % 4 != 0 has no tensor-core map")
    a, bmat, bias, r = _gemm_case(m, n, k, lda, m + n + k)
    got = _gemm("tfsc_k_gemm_tc", a, m, n, k, lda, bmat, bias, r, 1)
    assert _err(got, _gemm_ref(a, k, bmat, bias, r, 1)) <= TOL


@pytest.mark.parametrize("m,n", [(64, 72), (65, 1000), (127, 72), (129, 1000), (257, 72)])
@pytest.mark.parametrize("k,lda", [(32, 32), (33, 37), (63, 123), (65, 65), (4099, 4103)])
def test_gemm(m, n, k, lda):
    a, bmat, bias, r = _gemm_case(m, n, k, lda, m + n + k + 1)
    got = _gemm("tfsc_k_gemm", a, m, n, k, lda, bmat, bias, r, 1)
    assert _err(got, _gemm_ref(a, k, bmat, bias, r, 1)) <= TOL


@pytest.mark.parametrize("fn,m,n,j", [("tfsc_k_gemm_tc", 257, 96, 0), ("tfsc_k_gemm_tc", 257, 96, 256), ("tfsc_k_gemm_tc", 257, 96, 127),
                                      ("tfsc_k_gemm_tc", 64, 64, 63), ("tfsc_k_gemm", 257, 1000, 128), ("tfsc_k_gemm", 129, 72, 0)])
@pytest.mark.parametrize("poison", POISONS)
def test_gemm_row_isolation(fn, m, n, j, poison):
    k = 4099 if fn == "tfsc_k_gemm" else 4100
    a, bmat, bias, r = _gemm_case(m, n, k, k, m + n)
    clean = _gemm(fn, a, m, n, k, k, bmat, bias, r, 0)
    dirty = _gemm(fn, _poisoned(a, j, poison), m, n, k, k, bmat, bias, r, 0)
    bh.assert_rows_bit_equal(clean, dirty, [j], "c")


@pytest.mark.parametrize("splits", ["2", "8"])
def test_gemm_tc_forced_split_k(splits):
    """the split-K and cluster-fold paths are picked for small tile grids only; force them (TFSC_GEMM_SPLITK is read once
    per process, hence the subprocess)"""
    if os.environ.get("TFSC_GEMM_SPLITK"):
        pytest.skip("already inside the forced-split run")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-k",
                          "test_gemm_tc or test_gemm_row_isolation"], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, TFSC_GEMM_SPLITK=splits), cwd=root)
    assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]


# ------------------------------------------------------------------------------------------ conv family ----
def _t64(a):
    import torch
    return torch.from_numpy(np.asarray(a, np.float64))


def _conv_ref(x, w, bias, stride, pad):
    import torch.nn.functional as F
    y = F.conv2d(_t64(x).permute(0, 3, 1, 2), _t64(w).permute(3, 2, 0, 1), _t64(bias), stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1).numpy()


@pytest.mark.parametrize("bsz,h,c,kh,stride,pad,cout", [(1, 15, 32, 3, 2, 1, 64), (3, 15, 32, 3, 2, 1, 96), (3, 9, 64, 1, 2, 0, 64)])
def test_conv_tc(bsz, h, c, kh, stride, pad, cout):
    rng = np.random.default_rng(h + c)
    x = rng.standard_normal((bsz, h, h, c)).astype(np.float32)
    w = (rng.standard_normal((kh, kh, c, cout)) / np.sqrt(kh * kh * c)).astype(np.float32)
    bias = rng.standard_normal(cout).astype(np.float32)
    oh = (h + 2 * pad - kh) // stride + 1
    xg, wg, bg = _inp(x, guard=h * h * c * 4), _inp(w), _inp(bias)
    yg = _out(4 * bsz * oh * oh * cout, guard=128 * cout * 4)
    _done(lib.tfsc_k_conv_tc(xg.ptr, wg.ptr, bg.ptr, None, yg.ptr, bsz, h, h, c, kh, kh, stride, pad, cout, 0, None), "conv_tc")
    _check(x=xg, w=wg, bias=bg, y=yg)
    y = yg.read(shape=(bsz, oh, oh, cout))
    bh.assert_written(y)
    assert _err(y, _conv_ref(x, w, bias, stride, pad)) <= TOL


@pytest.mark.parametrize("bsz,h,c,kh,stride,pad", [(1, 15, 3, 3, 2, 1), (3, 15, 5, 3, 2, 1), (3, 9, 4, 1, 2, 0), (3, 7, 8, 7, 2, 3)])
def test_im2col(bsz, h, c, kh, stride, pad):
    """the padding columns [KH*KW*C, ldc) are written as zeros and nothing past them"""
    rng = np.random.default_rng(h * c)
    x = rng.standard_normal((bsz, h, h, c)).astype(np.float32)
    oh = (h + 2 * pad - kh) // stride + 1
    kk = kh * kh * c
    ldc = kk + 5
    xg, cg = _inp(x), _out(4 * bsz * oh * oh * ldc)
    _done(lib.tfsc_k_im2col(xg.ptr, cg.ptr, bsz, h, h, c, kh, kh, stride, pad, ldc, None), "im2col")
    _check(x=xg, col=cg)
    col = cg.read(shape=(bsz * oh * oh, ldc))
    assert not col[:, kk:].any() and not np.signbit(col[:, kk:]).any()
    xp = np.pad(x, ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    ref = np.stack([xp[:, i:i + stride * oh:stride, j:j + stride * oh:stride, :] for i in range(kh) for j in range(kh)], axis=3)
    assert np.array_equal(col[:, :kk], ref.reshape(bsz * oh * oh, kk))


@pytest.mark.parametrize("bsz,h,c,kh,stride,pad", [(1, 15, 8, 3, 2, 1), (3, 15, 5, 3, 2, 1), (3, 9, 4, 1, 2, 0), (3, 112, 64, 3, 2, 1)])
def test_maxpool(bsz, h, c, kh, stride, pad):
    """+Inf guards: a window that reads past its image returns +Inf"""
    import torch.nn.functional as F
    x = np.random.default_rng(h).standard_normal((bsz, h, h, c)).astype(np.float32)
    oh = (h + 2 * pad - kh) // stride + 1
    xg, yg = _inp(x, fill=bh.POS_INF), _out(4 * bsz * oh * oh * c)
    _done(lib.tfsc_k_maxpool(xg.ptr, yg.ptr, bsz, h, h, c, kh, kh, stride, pad, None), "maxpool")
    _check(x=xg, y=yg)
    ref = F.max_pool2d(_t64(x).permute(0, 3, 1, 2), kh, stride, pad).permute(0, 2, 3, 1).numpy()
    assert np.array_equal(yg.read(shape=(bsz, oh, oh, c)), ref.astype(np.float32))


@pytest.mark.parametrize("bsz,hw,c", [(1, 49, 2048), (3, 49, 5), (3, 1, 7)])
def test_avgpool(bsz, hw, c):
    x = np.random.default_rng(c).standard_normal((bsz, hw, c)).astype(np.float32)
    xg, yg = _inp(x), _out(4 * bsz * c)
    _done(lib.tfsc_k_avgpool(xg.ptr, yg.ptr, bsz, hw, c, None), "avgpool")
    _check(x=xg, y=yg)
    assert _err(yg.read(shape=(bsz, c)), x.astype(np.float64).mean(axis=1)) <= 1e-5


def _depthwise(x, w, bias, k, s, p, misalign=0):
    bsz, h, _, c = x.shape
    oh = (h + 2 * p - k) // s + 1
    xg, wg, bg = _inp(x, misalign=misalign), _inp(w), _inp(bias)
    yg = _out(4 * bsz * oh * oh * c, misalign=misalign)
    _done(lib.tfsc_k_depthwise_conv(xg.ptr, wg.ptr, bg.ptr, yg.ptr, bsz, h, h, c, k, k, s, p, 0, None), "depthwise_conv")
    _check(x=xg, w=wg, bias=bg, y=yg)
    y = yg.read(shape=(bsz, oh, oh, c))
    bh.assert_written(y)
    return y


@pytest.mark.parametrize("bsz,h,c,k,s,p", [(1, 15, 32, 3, 2, 1), (3, 15, 5, 3, 2, 1), (3, 9, 8, 5, 2, 2), (3, 7, 3, 3, 1, 1)])
@pytest.mark.parametrize("misalign", [0, 4])
def test_depthwise_conv(bsz, h, c, k, s, p, misalign):
    import torch.nn.functional as F
    rng = np.random.default_rng(h + c + k)
    x = rng.standard_normal((bsz, h, h, c)).astype(np.float32)
    w = rng.standard_normal((k, k, c)).astype(np.float32)
    bias = rng.standard_normal(c).astype(np.float32)
    y = _depthwise(x, w, bias, k, s, p, misalign)
    ref = F.conv2d(_t64(x).permute(0, 3, 1, 2), _t64(w).permute(2, 0, 1).unsqueeze(1), _t64(bias), stride=s, padding=p, groups=c)
    assert _err(y, ref.permute(0, 2, 3, 1).numpy()) <= TOL
    for j in {0, bsz - 1}:
        for poison in POISONS:
            bh.assert_rows_bit_equal(y, _depthwise(_poisoned(x, j, poison), w, bias, k, s, p, misalign), [j])


@pytest.mark.parametrize("bsz,hw,c", [(1, 49, 32), (3, 49, 5), (3, 3, 7)])
def test_channel_scale(bsz, hw, c):
    rng = np.random.default_rng(hw + c)
    x = rng.standard_normal((bsz, hw, c)).astype(np.float32)
    gate = rng.random((bsz, c)).astype(np.float32)
    xg, gg, yg = _inp(x), _inp(gate), _out(4 * bsz * hw * c)
    _done(lib.tfsc_k_channel_scale(xg.ptr, gg.ptr, yg.ptr, bsz, hw, c, None), "channel_scale")
    _check(x=xg, gate=gg, y=yg)
    assert np.array_equal(yg.read(shape=(bsz, hw, c)), x * gate[:, None, :])


# ----------------------------------------------------------------------------------------------- Swin ----
def _window(qkv, bias, bsz, h, c, heads, ws, shift):
    qg, bg = _inp(qkv, guard=ws * h * 3 * c * 4), _inp(bias)
    yg = _out(4 * bsz * h * h * c)
    _done(lib.tfsc_k_window_attention(qg.ptr, bg.ptr, yg.ptr, bsz, h, h, c, heads, ws, shift, None), "window_attention")
    _check(qkv=qg, bias=bg, ctx=yg)
    y = yg.read(shape=(bsz, h, h, c))
    bh.assert_written(y)
    return y


def _window_ref(qkv, bias, heads, ws):
    """shift 0: plain attention inside each window, fp64"""
    bsz, h, _, c3 = qkv.shape
    c, d = c3 // 3, c3 // 3 // heads
    x = qkv.astype(np.float64).reshape(bsz, h // ws, ws, h // ws, ws, 3, heads, d).transpose(0, 1, 3, 5, 6, 2, 4, 7)
    x = x.reshape(bsz, h // ws, h // ws, 3, heads, ws * ws, d)
    q, k, v = x[:, :, :, 0], x[:, :, :, 1], x[:, :, :, 2]
    s = q @ np.swapaxes(k, -1, -2) / np.sqrt(d) + bias
    p = np.exp(s - s.max(-1, keepdims=True))
    o = (p / p.sum(-1, keepdims=True)) @ v                   # [b, wy, wx, heads, N, d]
    o = o.reshape(bsz, h // ws, h // ws, heads, ws, ws, d).transpose(0, 1, 4, 2, 5, 3, 6)
    return o.reshape(bsz, h, h, c)


@pytest.mark.parametrize("bsz,h,ws,shift", [(1, 14, 7, 0), (3, 14, 7, 0), (3, 14, 7, 3), (3, 8, 4, 2)])
def test_window_attention(bsz, h, ws, shift):
    heads, d = 2, 16
    c = heads * d
    rng = np.random.default_rng(h + ws + shift)
    qkv = rng.standard_normal((bsz, h, h, 3 * c)).astype(np.float32)
    bias = rng.standard_normal((heads, ws * ws, ws * ws)).astype(np.float32)
    y = _window(qkv, bias, bsz, h, c, heads, ws, shift)
    if shift == 0:
        assert _err(y, _window_ref(qkv, bias, heads, ws)) <= TOL
    for j in {0, bsz - 1}:
        for poison in POISONS:
            bh.assert_rows_bit_equal(y, _window(_poisoned(qkv, j, poison), bias, bsz, h, c, heads, ws, shift), [j])


@pytest.mark.parametrize("bsz,h,c", [(1, 14, 32), (3, 14, 5), (3, 2, 3)])
def test_patch_merge(bsz, h, c):
    x = np.random.default_rng(h * c).standard_normal((bsz, h, h, c)).astype(np.float32)
    xg, yg = _inp(x), _out(4 * x.size)
    _done(lib.tfsc_k_patch_merge(xg.ptr, yg.ptr, bsz, h, h, c, None), "patch_merge")
    _check(x=xg, y=yg)
    ref = np.concatenate([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], axis=-1)
    assert np.array_equal(yg.read(shape=ref.shape), ref)


# ------------------------------------------------------------------------------------------- attention ----
def _mask_rows(bsz, S, stride, seed):
    """one row fully masked (its padding 1s), one with its last keys masked (padding 1s), the rest random with
    padding 0s: a kernel that read [S, stride) would see a different mask"""
    rng = np.random.default_rng(seed)
    m = np.zeros((bsz, stride), np.int32)
    m[:, :S] = rng.random((bsz, S)) < 0.8
    m[:, 0] = 1
    if bsz > 1:
        m[1, :S] = 0
        m[1, S:] = 1
    if bsz > 2:
        m[2, S // 2:S] = 0
        m[2, S:] = 1
    return m


def _attn_ref(qkv, mask, heads, causal):
    bsz, S, H3 = qkv.shape
    H = H3 // 3
    d = H // heads
    q, k, v = (qkv[:, :, i * H:(i + 1) * H].astype(np.float64).reshape(bsz, S, heads, d).transpose(0, 2, 1, 3) for i in range(3))
    s = q @ np.swapaxes(k, -1, -2) / np.sqrt(d)
    if mask is not None:
        m = mask[:, :S]
        add = np.where(m == 0, -10000.0, 0.0)
        add[(m == 0).all(axis=1)] = 0.0
        s = s + add[:, None, None, :]
    if causal:
        s = np.where(np.tril(np.ones((S, S), bool)), s, -np.inf)
    p = np.exp(s - s.max(-1, keepdims=True))
    o = (p / p.sum(-1, keepdims=True)) @ v
    return o.transpose(0, 2, 1, 3).reshape(bsz, S, H)


def _attn(qkv, mask, heads, causal, stride):
    bsz, S, H3 = qkv.shape
    H = H3 // 3
    qg = _inp(qkv, guard=256 * H3 * 4)
    mg = _inp(mask, fill=1) if mask is not None else None
    cg = _out(4 * bsz * S * H, guard=256 * H * 4)
    fn = lib.tfsc_k_attention_causal if causal else lib.tfsc_k_attention_mask
    _done(fn(qg.ptr, mg.ptr if mg else None, stride, cg.ptr, bsz, S, H, heads, None), "attention")
    _check(qkv=qg, ctx=cg, **({"mask": mg} if mg else {}))
    ctx = cg.read(shape=(bsz, S, H))
    bh.assert_written(ctx, "ctx")
    return ctx


@pytest.mark.parametrize("S", [1, 31, 32, 33, 255, 256, 257, 512])
@pytest.mark.parametrize("causal", [False, True])
def test_attention(S, causal):
    bsz, heads, d = 3, 2, 64
    H = heads * d
    rng = np.random.default_rng(S + causal)
    qkv = rng.standard_normal((bsz, S, 3 * H)).astype(np.float32)
    stride = S + 7
    mask = _mask_rows(bsz, S, stride, S)
    got = _attn(qkv, mask, heads, causal, stride)
    assert _err(got, _attn_ref(qkv, mask, heads, causal)) <= TOL
    for j in (0, bsz - 1):
        for poison in POISONS:
            bh.assert_rows_bit_equal(got, _attn(_poisoned(qkv, j, poison), mask, heads, causal, stride), [j], "ctx")
        dead = mask.copy()
        dead[j] = 0
        bh.assert_rows_bit_equal(got, _attn(qkv, dead, heads, causal, stride), [j], "ctx")


@pytest.mark.parametrize("S", [31, 33, 257])
def test_attention_ids(S):
    """tfsc_k_attention: the ids are the mask (id 0 = [PAD]); the ids past the batch are a nonzero id"""
    bsz, heads, d = 3, 4, 16
    H = heads * d
    rng = np.random.default_rng(S)
    qkv = rng.standard_normal((bsz, S, 3 * H)).astype(np.float32)
    ids = rng.integers(1, 100, (bsz, S)).astype(np.int32)
    ids[1, S // 3:] = 0
    qg, ig = _inp(qkv, guard=256 * 3 * H * 4), _inp(ids, fill=5)
    cg = _out(4 * bsz * S * H)
    _done(lib.tfsc_k_attention(qg.ptr, ig.ptr, cg.ptr, bsz, S, H, heads, None), "attention")
    _check(qkv=qg, ids=ig, ctx=cg)
    assert _err(cg.read(shape=(bsz, S, H)), _attn_ref(qkv, (ids != 0).astype(np.int32), heads, False)) <= TOL


# ------------------------------------------------------------------------------------- LayerNorm / embed ----
def _ln_ref(x, gamma, beta, eps):
    x = x.astype(np.float64)
    mu = x.mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(((x - mu) ** 2).mean(-1, keepdims=True) + eps) * gamma + beta


def _ln(x, res, gamma, beta, misalign=0):
    tokens, H = x.shape
    xg, rg = _inp(x, misalign=misalign), (_inp(res, misalign=misalign) if res is not None else None)
    gg, bg = _inp(gamma), _inp(beta)
    yg = _out(4 * x.size, misalign=misalign)
    _done(lib.tfsc_k_layernorm(xg.ptr, rg.ptr if rg else None, gg.ptr, bg.ptr, yg.ptr, tokens, H, C.c_float(1e-12), None), "layernorm")
    _check(x=xg, gamma=gg, beta=bg, y=yg, **({"res": rg} if rg else {}))
    y = yg.read(shape=x.shape)
    bh.assert_written(y)
    return y


@pytest.mark.parametrize("H", [1, 63, 64, 768, 1023])
@pytest.mark.parametrize("misalign", [0, 4])
def test_layernorm(H, misalign):
    rng = np.random.default_rng(H)
    x, res = (rng.standard_normal((5, H)).astype(np.float32) for _ in range(2))
    gamma, beta = rng.standard_normal(H).astype(np.float32), rng.standard_normal(H).astype(np.float32)
    y = _ln(x, res, gamma, beta, misalign)
    assert _err(y, _ln_ref(x + res, gamma, beta, 1e-12)) <= TOL
    for j in (0, 2, 4):
        for poison in POISONS:
            bh.assert_rows_bit_equal(y, _ln(_poisoned(x, j, poison), res, gamma, beta, misalign), [j])


def _tables(vocab, S, H, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((vocab, H)).astype(np.float32), rng.standard_normal((S, H)).astype(np.float32),
            rng.standard_normal((2, H)).astype(np.float32))


@pytest.mark.parametrize("H", [63, 64])
@pytest.mark.parametrize("S", [1, 33])
def test_embed(H, S):
    """ids / types in [S, stride) and past the batch hold other valid ids; the tables sit between NaN guards"""
    bsz, vocab, stride = 3, 50, S + 3
    word, pos, typ = _tables(vocab, S, H, H + S)
    rng = np.random.default_rng(S)
    ids = np.full((bsz, stride), 7, np.int32)
    ids[:, :S] = rng.integers(0, vocab, (bsz, S))
    types = np.ones((bsz, stride), np.int32)
    types[:, :S] = rng.integers(0, 2, (bsz, S))
    types[:, S:] = 1 - types[:, :1]
    gamma, beta = np.ones(H, np.float32), np.zeros(H, np.float32)
    gs = [_inp(a) for a in (word, pos, typ, gamma, beta)]
    ig, tg = _inp(ids, fill=7), _inp(types, fill=1)
    yg = _out(4 * bsz * S * H)
    _done(lib.tfsc_k_embed(ig.ptr, tg.ptr, stride, *[g.ptr for g in gs], yg.ptr, bsz, S, H, vocab, C.c_float(1e-12), None), "embed")
    _check(ids=ig, types=tg, y=yg, **{f"t{i}": g for i, g in enumerate(gs)})
    e = word[ids[:, :S]].astype(np.float64) + pos[None] + typ[types[:, :S]]
    assert _err(yg.read(shape=(bsz, S, H)), _ln_ref(e, gamma, beta, 1e-12)) <= TOL

    yg2 = _out(4 * bsz * S * H)
    _done(lib.tfsc_k_embed_positions(ig.ptr, stride, gs[0].ptr, gs[1].ptr, yg2.ptr, bsz, S, H, vocab, None), "embed_positions")
    _check(ids=ig, y=yg2, word=gs[0], pos=gs[1])
    assert np.array_equal(yg2.read(shape=(bsz, S, H)), word[ids[:, :S]] + pos[None])


@pytest.mark.parametrize("S,H", [(1, 63), (33, 64), (65, 6)])
def test_last_token_and_mask_gather(S, H):
    """mask / ids columns [S, stride) would move the last token or add [MASK] candidates if they were read"""
    bsz, stride, tok, M = 3, S + 4, 7, min(S, 3)
    rng = np.random.default_rng(S * H)
    hidden = rng.standard_normal((bsz, S, H)).astype(np.float32)
    mask = _mask_rows(bsz, S, stride, S)
    hg, mg = _inp(hidden), _inp(mask, fill=1)
    pg, gg = _out(4 * bsz), _out(4 * bsz * H)
    _done(lib.tfsc_k_last_token(hg.ptr, mg.ptr, stride, bsz, S, H, pg.ptr, gg.ptr, None), "last_token")
    _check(hidden=hg, mask=mg, positions=pg, gathered=gg)
    want = np.array([int(np.nonzero(m[:S])[0].max()) if m[:S].any() else -1 for m in mask], np.int32)
    assert np.array_equal(pg.read(np.int32), want)
    g = gg.read(shape=(bsz, H))
    for r in range(bsz):
        assert np.array_equal(g[r], hidden[r, want[r]] if want[r] >= 0 else np.zeros(H, np.float32))

    ids = rng.integers(8, 100, (bsz, stride)).astype(np.int32)
    ids[:, S:] = tok
    ids[0, S - 1] = tok
    ids[2, 0] = tok
    ig = _inp(ids, fill=tok)
    pg2, gg2 = _out(4 * bsz * M), _out(4 * bsz * M * H)
    _done(lib.tfsc_k_mask_gather(hg.ptr, ig.ptr, mg.ptr, stride, bsz, S, H, M, tok, pg2.ptr, gg2.ptr, None), "mask_gather")
    _check(hidden=hg, ids=ig, mask=mg, positions=pg2, gathered=gg2)
    pos = pg2.read(np.int32, (bsz, M))
    gat = gg2.read(shape=(bsz, M, H))
    for r in range(bsz):
        cand = [p for p in range(S) if ids[r, p] == tok and mask[r, p] != 0][:M]
        assert pos[r].tolist() == cand + [-1] * (M - len(cand))
        for s in range(M):
            assert np.array_equal(gat[r, s], hidden[r, cand[s]] if s < len(cand) else np.zeros(H, np.float32))


# ---------------------------------------------------------------------------------------------- heads ----
def _topk64(x, k):
    return np.argsort(-x.astype(np.float64), kind="stable")[:k]


def _softmax64(x):
    x = x.astype(np.float64)
    e = np.exp(x - x.max())
    return e / e.sum()


@pytest.mark.parametrize("n", [1, 100, 32768])
@pytest.mark.parametrize("k", [1, 32])
@pytest.mark.parametrize("fill", [bh.NAN, bh.POS_INF])
def test_classify_head(n, k, fill):
    k = min(k, n)
    rows = 3
    logits = np.random.default_rng(n + k).standard_normal((rows, n)).astype(np.float32)
    lg = _inp(logits, fill=fill)
    pg, cg, ig, tg = _out(4 * rows * n), _out(8 * rows), _out(4 * rows * k), _out(4 * rows * k)
    _done(lib.tfsc_k_classify_head(lg.ptr, rows, n, k, pg.ptr, cg.ptr, ig.ptr, tg.ptr, None), "classify_head")
    _check(logits=lg, probs=pg, classes=cg, topk_idx=ig, topk_prob=tg)
    probs, idx = pg.read(shape=(rows, n)), ig.read(np.int32, (rows, k))
    for r in range(rows):
        assert _err(probs[r], _softmax64(logits[r])) <= 1e-5
        assert idx[r].tolist() == _topk64(logits[r], k).tolist()
    assert cg.read(np.int64).tolist() == [int(np.argmax(r)) for r in logits]
    assert np.array_equal(tg.read(shape=(rows, k)), np.take_along_axis(probs, idx, 1))


def _next(logits, ld, positions, vocab, k, slots=None):
    rows = positions.size // (slots or 1)
    lg = _inp(logits, fill=bh.NAN)
    pg = _inp(positions, fill=0)
    m = slots or 1
    ig, prg, tg = _out(4 * rows * m * k), _out(4 * rows * m * k), _out(4 * rows * m * k)
    if slots is None:
        rc = lib.tfsc_k_next_token_head(lg.ptr, ld, pg.ptr, rows, vocab, k, ig.ptr, prg.ptr, tg.ptr, None)
    else:
        rc = lib.tfsc_k_fill_mask_head(lg.ptr, ld, pg.ptr, rows, slots, vocab, k, ig.ptr, prg.ptr, tg.ptr, None)
    _done(rc, "head")
    _check(logits=lg, positions=pg, ids=ig, probs=prg, top_logits=tg)
    return ig.read(np.int32, (rows * m, k)), prg.read(shape=(rows * m, k)), tg.read(shape=(rows * m, k))


@pytest.mark.parametrize("vocab,ld", [(100, 104), (32768, 32800), (50257, 50272), (57344, 57344 + 33)])
@pytest.mark.parametrize("k", [1, 32])
@pytest.mark.parametrize("pad", ["nan", "inf"])
def test_next_token_and_fill_mask_heads(vocab, ld, k, pad):
    """logits columns [vocab, ld) hold NaN or +Inf: a head that read them would pick or weigh them"""
    rows = 3
    rng = np.random.default_rng(vocab + k)
    logits = np.full((rows, ld), bh.FLOAT_POISONS[pad], np.float32)
    logits[:, :vocab] = rng.standard_normal((rows, vocab))
    positions = np.array([5, -1, 0], np.int32)
    ids, probs, lgs = _next(logits, ld, positions, vocab, k)
    for r in range(rows):
        if positions[r] < 0:
            assert (ids[r] == -1).all() and (probs[r] == 0).all() and (lgs[r] == -np.finfo(np.float32).max).all()
            continue
        want = _topk64(logits[r, :vocab], k)
        assert ids[r].tolist() == want.tolist()
        assert np.array_equal(lgs[r], logits[r, want])
        assert _err(probs[r], _softmax64(logits[r, :vocab])[want]) <= 1e-5
    if vocab <= 32768:   # the fill-mask head (it takes vocabularies up to 32,768): 3 rows x 2 slots
        lg2 = np.concatenate([logits, logits[::-1]], axis=0)
        pos2 = np.stack([positions, positions[::-1]], axis=1).reshape(-1).astype(np.int32)
        ids, _, lgs = _next(lg2[[0, 3, 1, 4, 2, 5]], ld, pos2, vocab, k, slots=2)
        ids1, _, lgs1 = _next(logits, ld, positions, vocab, k)
        assert np.array_equal(ids[0::2], ids1) and np.array_equal(lgs[0::2], lgs1)


@pytest.mark.parametrize("poison", POISONS)
def test_head_row_isolation(poison):
    rows, vocab, k = 5, 1000, 8
    logits = np.random.default_rng(1).standard_normal((rows, vocab)).astype(np.float32)
    positions = np.arange(rows, dtype=np.int32)
    clean = _next(logits, vocab, positions, vocab, k)
    for j in (0, 2, 4):
        dirty = _next(_poisoned(logits, j, poison), vocab, positions, vocab, k)
        for a, b in zip(clean, dirty):
            bh.assert_rows_bit_equal(a, b, [j])


def test_span_head():
    """ids / types / mask in [S, stride) would add eligible tokens if read; spans against a brute-force reference"""
    rows, S, stride, k, maxlen, sep = 3, 40, 45, 32, 6, 3
    rng = np.random.default_rng(2)
    logits = rng.standard_normal((rows, S, 2)).astype(np.float32)
    ids = rng.integers(4, 100, (rows, stride)).astype(np.int32)
    ids[:, 10] = sep
    types = np.zeros((rows, stride), np.int32)
    types[:, 12:S] = 1
    types[:, S:] = 1
    mask = np.ones((rows, stride), np.int32)
    mask[:, S - 5:S] = 0
    mask[1] = 0
    mask[1, S:] = 1
    lg, ig, tg, mg = _inp(logits), _inp(ids, fill=9), _inp(types, fill=1), _inp(mask, fill=1)
    outs = [_out(4 * rows * S), _out(4 * rows * S), _out(4 * rows * k), _out(4 * rows * k), _out(4 * rows * k)]
    _done(lib.tfsc_k_span_head(lg.ptr, ig.ptr, mg.ptr, tg.ptr, stride, rows, S, maxlen, k, sep, *[o.ptr for o in outs], None), "span_head")
    _check(logits=lg, ids=ig, types=tg, mask=mg, **{f"out{i}": o for i, o in enumerate(outs)})
    st, en = outs[0].read(shape=(rows, S)), outs[1].read(shape=(rows, S))
    assert np.array_equal(st, logits[:, :, 0]) and np.array_equal(en, logits[:, :, 1])
    starts, ends, scores = outs[2].read(np.int32, (rows, k)), outs[3].read(np.int32, (rows, k)), outs[4].read(shape=(rows, k))
    for r in range(rows):
        ok = [p for p in range(S) if mask[r, p] != 0 and types[r, p] == 1 and ids[r, p] != sep]
        cand = sorted(((logits[r, i, 0] + logits[r, j, 1], i, j) for i in ok for j in ok if i <= j < i + maxlen),
                      key=lambda c: (-c[0], c[1], c[2]))[:k]
        cand += [(-np.finfo(np.float32).max, -1, -1)] * (k - len(cand))
        assert starts[r].tolist() == [c[1] for c in cand] and ends[r].tolist() == [c[2] for c in cand]
        assert np.array_equal(scores[r], np.array([c[0] for c in cand], np.float32))


@pytest.mark.parametrize("H", [63, 64])
def test_encoder_head(H):
    """mask columns [S, stride) are 1s and would enter the mean if read"""
    rows, S, stride = 3, 33, 37
    rng = np.random.default_rng(H)
    hidden = rng.standard_normal((rows, S, H)).astype(np.float32)
    pooled = rng.standard_normal((rows, H)).astype(np.float32)
    ids = rng.integers(1, 100, (rows, stride)).astype(np.int32)
    mask = _mask_rows(rows, S, stride, H)
    hg, pg, ig, mg = _inp(hidden), _inp(pooled), _inp(ids, fill=9), _inp(mask, fill=1)
    so, po, co, mo = _out(4 * hidden.size), _out(4 * rows * H), _out(4 * rows * H), _out(4 * rows * H)
    _done(lib.tfsc_k_encoder_head(hg.ptr, pg.ptr, ig.ptr, mg.ptr, stride, rows, S, H, 0, 0, so.ptr, po.ptr, co.ptr, mo.ptr, None),
          "encoder_head")
    _check(hidden=hg, pooled=pg, ids=ig, mask=mg, seq=so, pool=po, cls=co, mean=mo)
    assert np.array_equal(so.read(shape=hidden.shape), hidden) and np.array_equal(po.read(shape=pooled.shape), pooled)
    assert np.array_equal(co.read(shape=(rows, H)), hidden[:, 0])
    m = (mask[:, :S] != 0).astype(np.float64)
    ref = (m[:, :, None] * hidden).sum(1) / np.maximum(m.sum(1), 1e-9)[:, None]
    assert _err(mo.read(shape=(rows, H)), ref) <= 1e-5


# ------------------------------------------------------------------------------------------- generation ----
@pytest.mark.parametrize("S", [1, 63, 64, 65])
@pytest.mark.parametrize("extra", [0, 40])
@pytest.mark.parametrize("H,misalign", [(64, 0), (6, 0), (64, 4)])
def test_kv_cache_write(S, extra, H, misalign):
    """bit-exact copies into slots [0, S); slots [S, T) and everything past the batch keep the sentinel"""
    rows, T = 3, S + extra
    qkv = np.random.default_rng(S + H).standard_normal((rows, S, 3 * H)).astype(np.float32)
    qg = _inp(qkv, guard=64 * 3 * H * 4, misalign=misalign)
    kg, vg = (_out(4 * rows * T * H, guard=64 * H * 4, misalign=misalign) for _ in range(2))
    _done(lib.tfsc_k_kv_cache_write(qg.ptr, kg.ptr, vg.ptr, rows, S, T, H, None), "kv_cache_write")
    _check(qkv=qg, kc=kg, vc=vg)
    for g, part in ((kg, 1), (vg, 2)):
        c = g.read(shape=(rows, T, H))
        assert np.array_equal(c[:, :S].view(np.uint32), qkv[:, :, part * H:(part + 1) * H].view(np.uint32))
        bh.assert_untouched(c[:, S:], "cache slots past S")


def _decode_case(rows, S, t_, T, H, seed):
    rng = np.random.default_rng(seed)
    qkv = rng.standard_normal((rows, 3 * H)).astype(np.float32)
    pos = np.array([S - 1, S // 2, -1][:rows], np.int32)
    kc = np.full((rows, T, H), np.nan, np.float32)     # slots past each row's query: must not be read
    vc = kc.copy()
    for r in range(rows):
        q = pos[r] + 1 + t_
        kc[r, :q] = rng.standard_normal((q, H))
        vc[r, :q] = rng.standard_normal((q, H))
    mask = np.ones((rows, S + 3), np.int32)
    mask[:, S:] = 0
    mask[0, :S // 3] = 0
    return qkv, pos, kc, vc, mask


def _decode_ref(qkv, pos, kc, vc, mask, t_, heads):
    rows, H3 = qkv.shape
    H = H3 // 3
    d = H // heads
    out = np.zeros((rows, H))
    for r in range(rows):
        q = pos[r] + 1 + t_
        K = np.concatenate([kc[r, :q], qkv[None, r, H:2 * H]]).astype(np.float64)
        V = np.concatenate([vc[r, :q], qkv[None, r, 2 * H:]]).astype(np.float64)
        add = np.array([-10000.0 if j <= pos[r] and mask[r, j] == 0 else 0.0 for j in range(q + 1)])
        for h in range(heads):
            sl = slice(h * d, (h + 1) * d)
            s = K[:, sl] @ qkv[r, sl].astype(np.float64) / np.sqrt(d) + add
            p = np.exp(s - s.max())
            out[r, sl] = (p / p.sum()) @ V[:, sl]
    return out


@pytest.mark.parametrize("S,t_", [(60, 2), (60, 3), (60, 4), (120, 7), (120, 8), (1, 0)])
def test_decode_attention(S, t_):
    """an exact work buffer, launched twice; cache slots other than each row's query slot keep their bits"""
    rows, H, heads = 3, 128, 4
    L = S + t_ + 1
    T = L + 5
    qkv, pos, kc, vc, mask = _decode_case(rows, S, t_, T, H, S + t_)
    wb = lib.tfsc_k_decode_attention_work_bytes(rows, L, H, heads)
    assert wb > 0
    work = bh.Guarded(wb, fill=bh.SENTINEL).fill_payload(0).arm()
    qg, pg, mg = _inp(qkv, guard=64 * 3 * H * 4), _inp(pos, fill=0), _inp(mask, fill=0)
    kg, vg = _inp(kc, guard=64 * H * 4), _inp(vc, guard=64 * H * 4)
    ref = _decode_ref(qkv, pos, kc, vc, mask, t_, heads)
    ctxs = []
    for _ in range(2):
        cg = _out(4 * rows * H)
        _done(lib.tfsc_k_decode_attention(qg.ptr, kg.ptr, vg.ptr, pg.ptr, t_, mg.ptr, S + 3, S, T, cg.ptr, rows, H, heads,
                                          work.ptr, wb, None), "decode_attention")
        _check(qkv=qg, pos=pg, mask=mg, kc=kg, vc=vg, ctx=cg, work=work)
        assert not work.read(np.uint32)[:rows * heads].any(), "arrival counters not back at zero"
        ctxs.append(cg.read(shape=(rows, H)))
        assert _err(ctxs[-1], ref) <= TOL
    assert np.array_equal(ctxs[0].view(np.uint32), ctxs[1].view(np.uint32))
    for g, want, part in ((kg, kc, 1), (vg, vc, 2)):
        c = g.read(shape=(rows, T, H))
        for r in range(rows):
            q = pos[r] + 1 + t_
            assert np.array_equal(c[r, q].view(np.uint32), qkv[r, part * H:(part + 1) * H].view(np.uint32))
            other = np.delete(np.arange(T), q)
            assert np.array_equal(c[r, other].view(np.uint32), want[r, other].view(np.uint32))


@pytest.mark.parametrize("vocab,ld", [(100, 103), (50257, 50272)])
@pytest.mark.parametrize("pad", ["nan", "inf"])
@pytest.mark.parametrize("H", [64, 6])
def test_generate_select(vocab, ld, pad, H):
    """only column t of ids / log-probs and column 0 of length are written; logits [vocab, ld) are never read"""
    rows, t_, N, S = 3, 1, 4, 10
    rng = np.random.default_rng(vocab + H)
    logits = np.full((rows, ld), bh.FLOAT_POISONS[pad], np.float32)
    logits[:, :vocab] = rng.standard_normal((rows, vocab))
    pos = np.array([3, 0, 9], np.int32)
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((S + N, H)).astype(np.float32)
    lg, pg, wg, tg = _inp(logits), _inp(pos, fill=0), _inp(word), _inp(ptab)
    dg = bh.Guarded(4 * rows, fill=bh.SENTINEL).fill_payload(0).arm()
    ig, lpg, leng, yg = _out(4 * rows * N), _out(4 * rows * N), _out(4 * rows * 2), _out(4 * rows * H)
    _done(lib.tfsc_k_generate_select(lg.ptr, ld, vocab, pg.ptr, t_, 0, -1, dg.ptr, ig.ptr, N, lpg.ptr, N, leng.ptr, 2, wg.ptr, tg.ptr,
                                     yg.ptr, rows, H, None), "generate_select")
    _check(logits=lg, pos=pg, word=wg, pos_table=tg, done=dg, ids=ig, log_probs=lpg, length=leng, y=yg)
    ids, lp = ig.read(np.int32, (rows, N)), lpg.read(shape=(rows, N))
    length, y = leng.read(np.int32, (rows, 2)), yg.read(shape=(rows, H))
    g = np.argmax(logits[:, :vocab], axis=1)
    assert ids[:, t_].tolist() == g.tolist() and length[:, 0].tolist() == [t_ + 1] * rows
    x = logits[:, :vocab].astype(np.float64)
    ref_lp = x[np.arange(rows), g] - x.max(1) - np.log(np.exp(x - x.max(1, keepdims=True)).sum(1))
    assert np.max(np.abs(lp[:, t_] - ref_lp)) <= 1e-5
    assert np.array_equal(y, word[g] + ptab[pos + 1 + t_])
    other = [c for c in range(N) if c != t_]
    bh.assert_untouched(ids[:, other], "ids")
    bh.assert_untouched(lp[:, other], "log_probs")
    bh.assert_untouched(length[:, 1:], "length")


# ------------------------------------------------------------------------------ row isolation, the rest ----
def _assert_isolated(run, args, cases):
    """run(*args) returns outputs with the batch on axis 0. cases: [(j, dirty args)]; every row but j of every output
    keeps the clean launch's bits"""
    clean = run(*args)
    for j, dirty in cases:
        for i, (a, b) in enumerate(zip(clean, run(*dirty))):
            bh.assert_rows_bit_equal(a, b, [j], f"output {i}, row {j} poisoned")


def _float_cases(args, idx, js):
    """row j of the float inputs args[idx] set to each poison"""
    return [(j, [_poisoned(a, j, p) if i in idx else a for i, a in enumerate(args)]) for j in js for p in POISONS]


def _row_case(args, i, j, value):
    """row j of args[i] set to one value (an all-zero mask row, a row of one valid id)"""
    out = list(args)
    out[i] = np.array(out[i], copy=True)
    out[i][j] = value
    return j, out


def _conv_tc(x, w, bias, stride, pad):
    bsz, h, _, c = x.shape
    kh, cout = w.shape[0], w.shape[3]
    oh = (h + 2 * pad - kh) // stride + 1
    xg, wg, bg = _inp(x, guard=h * h * c * 4), _inp(w), _inp(bias)
    yg = _out(4 * bsz * oh * oh * cout, guard=128 * cout * 4)
    _done(lib.tfsc_k_conv_tc(xg.ptr, wg.ptr, bg.ptr, None, yg.ptr, bsz, h, h, c, kh, kh, stride, pad, cout, 0, None), "conv_tc")
    _check(x=xg, w=wg, bias=bg, y=yg)
    return (yg.read(shape=(bsz, oh, oh, cout)),)


def test_conv_tc_row_isolation():
    """8 x 8 outputs per image: images 0 and 1 share the first 128-row GEMM tile, image 2 has the second to itself"""
    rng = np.random.default_rng(4)
    x = rng.standard_normal((3, 15, 15, 32)).astype(np.float32)
    w = (rng.standard_normal((3, 3, 32, 64)) / 17).astype(np.float32)
    bias = rng.standard_normal(64).astype(np.float32)
    args = [x, w, bias, 2, 1]
    (y,) = _conv_tc(*args)
    assert _err(y, _conv_ref(x, w, bias, 2, 1)) <= TOL
    _assert_isolated(_conv_tc, args, _float_cases(args, [0], [0, 1, 2]))


def _pools(x, ldc_extra=5):
    """im2col (3 x 3, stride 2, pad 1), maxpool (same window), avgpool, channel_scale and patch_merge of x [b, h, h, c]"""
    bsz, h, _, c = x.shape
    oh = (h + 2 - 3) // 2 + 1
    ldc = 9 * c + ldc_extra
    gate = np.linspace(0.5, 1.5, bsz * c, dtype=np.float32).reshape(bsz, c)
    xg, xi, gg = _inp(x), _inp(x, fill=bh.POS_INF), _inp(gate)
    col, mp, ap = _out(4 * bsz * oh * oh * ldc), _out(4 * bsz * oh * oh * c), _out(4 * bsz * c)
    cs, pm = _out(4 * x.size), _out(4 * x.size)
    _done(lib.tfsc_k_im2col(xg.ptr, col.ptr, bsz, h, h, c, 3, 3, 2, 1, ldc, None), "im2col")
    _done(lib.tfsc_k_maxpool(xi.ptr, mp.ptr, bsz, h, h, c, 3, 3, 2, 1, None), "maxpool")
    _done(lib.tfsc_k_avgpool(xg.ptr, ap.ptr, bsz, h * h, c, None), "avgpool")
    _done(lib.tfsc_k_channel_scale(xg.ptr, gg.ptr, cs.ptr, bsz, h * h, c, None), "channel_scale")
    _done(lib.tfsc_k_patch_merge(xg.ptr, pm.ptr, bsz, h, h, c, None), "patch_merge")
    _check(x=xg, x_inf=xi, gate=gg, col=col, maxpool=mp, avgpool=ap, channel_scale=cs, patch_merge=pm)
    return (col.read(shape=(bsz, -1)), mp.read(shape=(bsz, -1)), ap.read(shape=(bsz, -1)), cs.read(shape=(bsz, -1)),
            pm.read(shape=(bsz, -1)))


@pytest.mark.parametrize("c", [4, 5])
def test_pool_family_row_isolation(c):
    x = np.random.default_rng(c).standard_normal((4, 14, 14, c)).astype(np.float32)
    _assert_isolated(_pools, [x], _float_cases([x], [0], [0, 2, 3]))


def _attn_ids(qkv, ids, heads):
    bsz, S, H3 = qkv.shape
    qg, ig, cg = _inp(qkv, guard=256 * H3 * 4), _inp(ids, fill=5), _out(4 * bsz * S * H3 // 3)
    _done(lib.tfsc_k_attention(qg.ptr, ig.ptr, cg.ptr, bsz, S, H3 // 3, heads, None), "attention")
    _check(qkv=qg, ids=ig, ctx=cg)
    return (cg.read(shape=(bsz, S, H3 // 3)),)


@pytest.mark.parametrize("S", [33, 257])
def test_attention_ids_row_isolation(S):
    rng = np.random.default_rng(S)
    qkv = rng.standard_normal((4, S, 3 * 64)).astype(np.float32)
    ids = rng.integers(1, 100, (4, S)).astype(np.int32)
    args = [qkv, ids, 4]
    _assert_isolated(_attn_ids, args, _float_cases(args, [0], [0, 1, 3]) + [_row_case(args, 1, j, 0) for j in (0, 1, 3)])


def _embeds(ids, types, tables, S):
    word, pos, typ, gamma, beta = tables
    bsz, stride = ids.shape
    H, vocab = word.shape[1], word.shape[0]
    gs = [_inp(a) for a in tables]
    ig, tg = _inp(ids, fill=7), _inp(types, fill=1)
    y1, y2 = _out(4 * bsz * S * H), _out(4 * bsz * S * H)
    _done(lib.tfsc_k_embed(ig.ptr, tg.ptr, stride, *[g.ptr for g in gs], y1.ptr, bsz, S, H, vocab, C.c_float(1e-12), None), "embed")
    _done(lib.tfsc_k_embed_positions(ig.ptr, stride, gs[0].ptr, gs[1].ptr, y2.ptr, bsz, S, H, vocab, None), "embed_positions")
    _check(ids=ig, types=tg, y1=y1, y2=y2, **{f"t{i}": g for i, g in enumerate(gs)})
    return y1.read(shape=(bsz, S * H)), y2.read(shape=(bsz, S * H))


@pytest.mark.parametrize("H", [63, 64])
def test_embed_row_isolation(H):
    """row j's ids all one valid id, its segment ids all 1"""
    S, vocab = 33, 50
    word, pos, typ = _tables(vocab, S, H, H)
    tables = (word, pos, typ, np.ones(H, np.float32), np.zeros(H, np.float32))
    rng = np.random.default_rng(H)
    ids = rng.integers(0, vocab, (4, S + 3)).astype(np.int32)
    types = rng.integers(0, 2, (4, S + 3)).astype(np.int32)
    args = [ids, types, tables, S]
    _assert_isolated(_embeds, args, [_row_case(args, 0, j, 3) for j in (0, 1, 3)] + [_row_case(args, 1, j, 1) for j in (0, 3)])


def _gathers(hidden, mask, ids, S, M, tok):
    bsz, _, H = hidden.shape
    stride = mask.shape[1]
    hg, mg, ig = _inp(hidden), _inp(mask, fill=1), _inp(ids, fill=tok)
    p1, g1, p2, g2 = _out(4 * bsz), _out(4 * bsz * H), _out(4 * bsz * M), _out(4 * bsz * M * H)
    _done(lib.tfsc_k_last_token(hg.ptr, mg.ptr, stride, bsz, S, H, p1.ptr, g1.ptr, None), "last_token")
    _done(lib.tfsc_k_mask_gather(hg.ptr, ig.ptr, mg.ptr, stride, bsz, S, H, M, tok, p2.ptr, g2.ptr, None), "mask_gather")
    _check(hidden=hg, mask=mg, ids=ig, p1=p1, g1=g1, p2=p2, g2=g2)
    return (p1.read(np.int32), g1.read(shape=(bsz, H)), p2.read(np.int32, (bsz, M)), g2.read(shape=(bsz, M * H)))


def test_last_token_and_mask_gather_row_isolation():
    S, H, M, tok = 33, 64, 3, 7
    rng = np.random.default_rng(5)
    hidden = rng.standard_normal((4, S, H)).astype(np.float32)
    mask = (rng.random((4, S + 4)) < 0.8).astype(np.int32)
    ids = rng.integers(8, 100, (4, S + 4)).astype(np.int32)
    ids[:, ::5] = tok
    args = [hidden, mask, ids, S, M, tok]
    _assert_isolated(_gathers, args, _float_cases(args, [0], [0, 2, 3]) + [_row_case(args, 1, j, 0) for j in (0, 3)] +
                     [_row_case(args, 2, j, tok) for j in (0, 3)])


def _classify(logits, k):
    rows, n = logits.shape
    lg = _inp(logits)
    pg, cg, ig, tg = _out(4 * rows * n), _out(8 * rows), _out(4 * rows * k), _out(4 * rows * k)
    _done(lib.tfsc_k_classify_head(lg.ptr, rows, n, k, pg.ptr, cg.ptr, ig.ptr, tg.ptr, None), "classify_head")
    _check(logits=lg, probs=pg, classes=cg, topk_idx=ig, topk_prob=tg)
    return pg.read(shape=(rows, n)), cg.read(np.int64), ig.read(np.int32, (rows, k)), tg.read(shape=(rows, k))


def _fill_mask(logits, positions, k):
    """logits [rows, M, vocab], positions [rows, M]"""
    rows, M, vocab = logits.shape
    ids, probs, lgs = _next(logits.reshape(rows * M, vocab), vocab, positions.reshape(-1), vocab, k, slots=M)
    return ids.reshape(rows, -1), probs.reshape(rows, -1), lgs.reshape(rows, -1)


def test_heads_row_isolation():
    """NaN rows leave the selection's sentinel index, which the heads clamp before reading the staged logits"""
    rng = np.random.default_rng(6)
    logits = rng.standard_normal((5, 1000)).astype(np.float32)
    _assert_isolated(_classify, [logits, 8], _float_cases([logits, 8], [0], [0, 2, 4]))
    slots = rng.standard_normal((5, 2, 1000)).astype(np.float32)
    positions = np.tile(np.array([[3, -1]], np.int32), (5, 1))
    positions[2] = [1, 4]
    args = [slots, positions, 8]
    _assert_isolated(_fill_mask, args, _float_cases(args, [0], [0, 2, 4]) + [_row_case(args, 1, 2, -1)])


def _span(logits, ids, types, mask, k, maxlen, sep):
    rows, S, _ = logits.shape
    stride = ids.shape[1]
    lg, ig, tg, mg = _inp(logits), _inp(ids, fill=9), _inp(types, fill=1), _inp(mask, fill=1)
    outs = [_out(4 * rows * S), _out(4 * rows * S), _out(4 * rows * k), _out(4 * rows * k), _out(4 * rows * k)]
    _done(lib.tfsc_k_span_head(lg.ptr, ig.ptr, mg.ptr, tg.ptr, stride, rows, S, maxlen, k, sep, *[o.ptr for o in outs], None), "span_head")
    _check(logits=lg, ids=ig, types=tg, mask=mg, **{f"out{i}": o for i, o in enumerate(outs)})
    return tuple(o.read(np.int32 if i in (2, 3) else np.float32, (rows, -1)) for i, o in enumerate(outs))


def _encoder(hidden, pooled, ids, mask):
    rows, S, H = hidden.shape
    stride = ids.shape[1]
    hg, pg, ig, mg = _inp(hidden), _inp(pooled), _inp(ids, fill=9), _inp(mask, fill=1)
    so, po, co, mo = _out(4 * hidden.size), _out(4 * rows * H), _out(4 * rows * H), _out(4 * rows * H)
    _done(lib.tfsc_k_encoder_head(hg.ptr, pg.ptr, ig.ptr, mg.ptr, stride, rows, S, H, 1, 1, so.ptr, po.ptr, co.ptr, mo.ptr, None),
          "encoder_head")
    _check(hidden=hg, pooled=pg, ids=ig, mask=mg, seq=so, pool=po, cls=co, mean=mo)
    return tuple(o.read(shape=(rows, -1)) for o in (so, po, co, mo))


def test_span_and_encoder_heads_row_isolation():
    rng = np.random.default_rng(7)
    rows, S, stride = 5, 40, 43
    logits = rng.standard_normal((rows, S, 2)).astype(np.float32)
    ids = rng.integers(4, 100, (rows, stride)).astype(np.int32)
    types = np.zeros((rows, stride), np.int32)
    types[:, 10:] = 1
    mask = np.ones((rows, stride), np.int32)
    args = [logits, ids, types, mask, 16, 6, 3]
    _assert_isolated(_span, args, _float_cases(args, [0], [0, 2, 4]) + [_row_case(args, 3, j, 0) for j in (0, 4)] +
                     [_row_case(args, 1, 2, 3)])
    hidden = rng.standard_normal((rows, S, 64)).astype(np.float32)
    pooled = rng.standard_normal((rows, 64)).astype(np.float32)
    args = [hidden, pooled, ids, mask]
    _assert_isolated(_encoder, args, _float_cases(args, [0, 1], [0, 2, 4]) + [_row_case(args, 3, j, 0) for j in (0, 4)])


def _kv(qkv, T):
    rows, S, H3 = qkv.shape
    H = H3 // 3
    qg = _inp(qkv, guard=64 * H3 * 4)
    kg, vg = _out(4 * rows * T * H, guard=64 * H * 4), _out(4 * rows * T * H, guard=64 * H * 4)
    _done(lib.tfsc_k_kv_cache_write(qg.ptr, kg.ptr, vg.ptr, rows, S, T, H, None), "kv_cache_write")
    _check(qkv=qg, kc=kg, vc=vg)
    return kg.read(shape=(rows, -1)), vg.read(shape=(rows, -1))


def _decode(qkv, kc, vc, pos, mask, t_, S, heads):
    rows, T, H = kc.shape
    L = S + t_ + 1
    wb = lib.tfsc_k_decode_attention_work_bytes(rows, L, H, heads)
    work = bh.Guarded(wb, fill=bh.SENTINEL).fill_payload(0).arm()
    qg, pg, mg = _inp(qkv, guard=64 * 3 * H * 4), _inp(pos, fill=0), _inp(mask, fill=0)
    kg, vg = _inp(kc, guard=64 * H * 4), _inp(vc, guard=64 * H * 4)
    cg = _out(4 * rows * H)
    _done(lib.tfsc_k_decode_attention(qg.ptr, kg.ptr, vg.ptr, pg.ptr, t_, mg.ptr, mask.shape[1], S, T, cg.ptr, rows, H, heads,
                                      work.ptr, wb, None), "decode_attention")
    _check(qkv=qg, pos=pg, mask=mg, kc=kg, vc=vg, ctx=cg, work=work)
    assert not work.read(np.uint32)[:rows * heads].any(), "arrival counters not back at zero"
    return cg.read(shape=(rows, H)), kg.read(shape=(rows, -1)), vg.read(shape=(rows, -1))


def _select(logits, pos, word, ptab, t_):
    rows, vocab = logits.shape
    H, N = word.shape[1], t_ + 2
    lg, pg, wg, tg = _inp(logits), _inp(pos, fill=0), _inp(word), _inp(ptab)
    dg = bh.Guarded(4 * rows, fill=bh.SENTINEL).fill_payload(0).arm()
    ig, lpg, leng, yg = _out(4 * rows * N), _out(4 * rows * N), _out(4 * rows), _out(4 * rows * H)
    _done(lib.tfsc_k_generate_select(lg.ptr, vocab, vocab, pg.ptr, t_, 0, -1, dg.ptr, ig.ptr, N, lpg.ptr, N, leng.ptr, 1, wg.ptr,
                                     tg.ptr, yg.ptr, rows, H, None), "generate_select")
    _check(logits=lg, pos=pg, word=wg, pos_table=tg, done=dg, ids=ig, log_probs=lpg, length=leng, y=yg)
    return (ig.read(np.int32, (rows, N)), lpg.read(shape=(rows, N)), leng.read(np.int32), yg.read(shape=(rows, H)),
            dg.read(np.int32))


@pytest.mark.parametrize("S,t_", [(60, 3), (120, 8)])
def test_generation_row_isolation(S, t_):
    """the KV cache write, decode attention over 64-key blocks (per-(row, head) counters and combine) and the select step,
    whose NaN rows leave an index the kernel clamps before it reads a table"""
    rows, H, heads = 5, 128, 4
    rng = np.random.default_rng(S)
    qkv = rng.standard_normal((rows, S, 3 * H)).astype(np.float32)
    _assert_isolated(_kv, [qkv, S + 9], _float_cases([qkv, S + 9], [0], [0, 2, 4]))
    L = S + t_ + 1
    T = L + 3
    pos = np.array([S - 1, S // 2, -1, 0, S - 2], np.int32)
    q1 = rng.standard_normal((rows, 3 * H)).astype(np.float32)
    kc = rng.standard_normal((rows, T, H)).astype(np.float32)
    vc = rng.standard_normal((rows, T, H)).astype(np.float32)
    mask = (rng.random((rows, S)) < 0.9).astype(np.int32)
    args = [q1, kc, vc, pos, mask, t_, S, heads]
    ctx = _decode(*args)[0]
    kc_ref = kc.copy()
    for r in range(rows):
        kc_ref[r, pos[r] + 1 + t_:] = np.nan
    assert _err(ctx, _decode_ref(q1, pos, kc_ref, vc, np.pad(mask, ((0, 0), (0, 3))), t_, heads)) <= TOL
    _assert_isolated(_decode, args, _float_cases(args, [0, 1, 2], [0, 2, 4]) + [_row_case(args, 4, j, 0) for j in (0, 4)])
    vocab = 1000
    logits = rng.standard_normal((rows, vocab)).astype(np.float32)
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((S + t_ + 2, H)).astype(np.float32)
    args = [logits, np.maximum(pos, 0), word, ptab, t_]
    _assert_isolated(_select, args, _float_cases(args, [0], [0, 2, 4]))


# ------------------------------------------------------------------------------------------ served path ----
DIMS = [64, 96, 48]


def _mlp_cfg(**kw):
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": DIMS, "modelProvider.synthetic.count": 2,
           "gpu.devices": [0], "gpu.arenaBytes": 64 << 20, "modelCache.size": 1 << 30, "serving.maxConcurrentModels": 2}
    cfg.update(kw)
    return cfg


@pytest.mark.parametrize("case", ["40+24", "1+62", "3+20+3"])
@pytest.mark.parametrize("poison", POISONS)
def test_coalesced_request_with_poison_leaves_the_others_bits(case, poison):
    """the requests coalesce into one batch, one of them poisoned; every other request gets the bits its rows get in the
    clean batch served as one request (the batch size picks the kernels, so that is the same launch sequence)"""
    sizes = [int(s) for s in case.split("+")]
    clean = np.random.default_rng(len(sizes)).standard_normal((sum(sizes), DIMS[0])).astype(np.float32)
    starts = np.cumsum([0] + sizes)
    bad = len(sizes) // 2
    x = clean.copy()
    x[starts[bad]:starts[bad + 1]] = bh.FLOAT_POISONS[poison]
    with t.Server(_mlp_cfg(**{"gpu.maxBatch": sum(sizes), "gpu.tickMicros": 3_000_000})) as srv, t.Server(_mlp_cfg()) as one:
        srv.predict("m1", "1", clean)            # resident; a full batch does not wait
        st0 = srv.stats()
        tickets = [srv.predict_submit("m1", "1", x[starts[i]:starts[i + 1]]) for i in range(len(sizes))]
        outs = [tk.wait(30.0) for tk in tickets]
        [tk.release() for tk in tickets]
        assert srv.stats()["batches"] - st0["batches"] == 1
        whole = one.predict("m1", "1", clean)
        man, blob = models.synth_mlp_blob(DIMS, seed=1001)
        assert _err(whole, models.forward(man, blob, clean, np.float64)) <= TOL
        for i in range(len(sizes)):
            if i == bad:
                assert outs[i].shape == (sizes[i], DIMS[-1])
                continue
            assert outs[i].tobytes() == whole[starts[i]:starts[i + 1]].tobytes(), (case, poison, i)


def test_predict_device_rows_past_the_batch():
    """x rows past B are NaN, y rows past B hold the sentinel: neither changes the rows below B, and rows past B stay"""
    B, extra = 5, 3
    x = np.random.default_rng(3).standard_normal((B, DIMS[0])).astype(np.float32)
    xfull = np.concatenate([x, np.full((extra, DIMS[0]), np.nan, np.float32)])
    with t.Server(_mlp_cfg()) as srv:
        want = srv.predict("m1", "1", x)
        srv.ensure(0, "m1", 1)
        xg = _inp(xfull)
        yg = _out(4 * (B + extra) * DIMS[-1])
        srv.predict_device(0, "m1", 1, xg.ptr, B, yg.ptr)
        srv.sync(0)
        _check(x=xg, y=yg)
        y = yg.read(shape=(B + extra, DIMS[-1]))
        man, blob = models.synth_mlp_blob(DIMS, seed=1001)
        assert _err(y[:B], models.forward(man, blob, x, np.float64)) <= TOL
        assert y[:B].tobytes() == want.tobytes()
        bh.assert_untouched(y[B:], "rows past the batch")


# ------------------------------------------------------------------------------------ served bundles ----
SERVED = ["resnet", "mobilenet_v2", "bert", "gpt2"]
GPT2_S = 32


@pytest.fixture(scope="module")
def served(tmp_path_factory):
    """small ResNet, MobileNetV2 and BERT bundles of test_gpu_batches.py and a small GPT-2 next-token bundle"""
    import gpt2_export as ge
    import test_gpu_batches as gb
    import test_gpu_gpt2 as gg
    tmp = tmp_path_factory.mktemp("served")
    fams = gb._write_families(tmp)
    gg._write_gpt2(tmp, GPT2_S, gg.SMALL, 44, name="gpt2")
    fams["gpt2"] = gb.Family("gpt2", gg.NAMES, lambda B, seed: ge.gpt2_inputs(B, GPT2_S, gg.SMALL["vocab"], seed=seed), None, None)
    return tmp, fams, gb


def _poisoned_requests(clean, lo, hi):
    """float inputs: rows [lo, hi) set to each poison; token inputs: their attention-mask rows all zero"""
    if isinstance(clean, dict):
        key = "input_mask" if "input_mask" in clean else "attention_mask"
        m = clean[key].copy()
        m[lo:hi] = 0
        return [("zero mask", dict(clean, **{key: m}))]
    out = []
    for p in POISONS:
        x = clean.copy()
        x[lo:hi] = bh.FLOAT_POISONS[p]
        out.append((p, x))
    return out


# The image nets pick their conv GEMMs' tile width and split-K from M = batch x OH x OW, so a request served alone runs
# other kernels than the batch it is coalesced into and its bits may differ in the last place even with no poison: there
# the request's values are compared with its served-alone values, and its bits with its rows of the clean batch. BERT's
# and GPT-2's routes give a row the same bits at these batch sizes, and there both comparisons are bit for bit.
ROUTED_BY_BATCH = {"resnet", "mobilenet_v2"}


@pytest.mark.parametrize("fam", SERVED)
def test_coalesced_bundle_requests_with_a_poisoned_one(served, fam):
    """three requests coalesce into one batch, the middle one poisoned (NaN, +-Inf, 3e38 images; an all-zero attention
    mask). It completes with a result or a clean error; each other request gets the bits of its rows in the clean batch
    served as one request, and the bits (values, for ROUTED_BY_BATCH) it gets served alone"""
    tmp, fams, gb = served
    f = fams[fam]
    sizes, bad = [2, 3, 2], 1
    starts = np.cumsum([0] + sizes)
    clean = f.inputs(sum(sizes), 31)
    with t.Server(gb._cfg(tmp, **{"gpu.maxBatch": sum(sizes), "gpu.tickMicros": 3_000_000})) as srv, t.Server(gb._cfg(tmp)) as one:
        whole = one.predict(f.name, "1", clean, outputs=f.outputs)
        alone = [one.predict(f.name, "1", gb._rows(clean, starts[i], starts[i + 1]), outputs=f.outputs) for i in range(len(sizes))]
        srv.predict(f.name, "1", clean, outputs=f.outputs)          # resident; a full batch does not wait
        for label, x in _poisoned_requests(clean, starts[bad], starts[bad + 1]):
            st0 = srv.stats()
            tickets = [srv.predict_submit(f.name, "1", gb._rows(x, starts[i], starts[i + 1]), outputs=f.outputs)
                       for i in range(len(sizes))]
            outs = []
            for tk in tickets:
                try:
                    outs.append(tk.wait(60.0))
                except t._lib.TfscError as e:
                    outs.append(e)
                finally:
                    tk.release()
            assert srv.stats()["batches"] - st0["batches"] == 1, (fam, label)
            r = outs[bad]
            if isinstance(r, Exception):
                assert r.code in (t._lib.E_INVALID, t._lib.E_INTERNAL), (fam, label, r)
            else:
                assert sorted(r) == sorted(f.outputs) and all(v.shape[0] == sizes[bad] for v in r.values()), (fam, label)
            for i in range(len(sizes)):
                if i == bad:
                    continue
                assert not isinstance(outs[i], Exception), (fam, label, i, outs[i])
                got = gb._bits(outs[i])
                assert got == gb._slice_bits(whole, starts[i], starts[i + 1]), (fam, label, i, "batch")
                if fam not in ROUTED_BY_BATCH:
                    assert got == gb._bits(alone[i]), (fam, label, i, "alone")
                    continue
                for name in ("logits", "probabilities"):
                    assert _err(outs[i][name], alone[i][name]) <= TOL, (fam, label, i, name)
