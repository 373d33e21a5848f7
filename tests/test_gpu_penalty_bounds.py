"""-m gpu: tfsc_k_generate_process reads and writes only its own bytes (the harness of test_gpu_bounds.py): guard bands on
every operand, logits padding past the vocabulary poisoned, the t = 0 step writing each row's prompt history and one token
and a later step only hist[hist_len0 + t], word / pos_table / y off 16-byte alignment, and rows whose logits, prompt or mask
change leaving every other row's bits alone."""
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds_harness as bh  # noqa: E402
import penalty_ref as pr  # noqa: E402
import test_gpu_bounds as tb  # noqa: E402

pytestmark = pytest.mark.gpu
lib = t._lib.lib
PROCS = [((1.3, 3, 2), None), ((0.8, 1, 0), (0.9, 40, 0.95))]
EOS = 2


def _process(logits, ld, vocab, pos, ids, mask, word, ptab, t_, proc, cfg, hist=None, hl0=None, misalign=0, seeds=None):
    """one guarded launch; logits [rows, ld] (columns from vocab on are the caller's poison), ids / mask [rows, S], hist
    [rows, S + 2] and hist_len0 [rows] from an earlier step (None: sentinel, for t = 0). Returns ids, log_probs [rows, t + 2],
    length, y, done, hist and hist_len0"""
    rows, S = ids.shape
    H, N, hld = word.shape[1], t_ + 2, S + 2
    lg, pg, ig_, mg = tb._inp(logits), tb._inp(pos, fill=0), tb._inp(ids, fill=0), tb._inp(mask, fill=1)
    sg = tb._inp(np.asarray(seeds, np.int32), fill=0) if cfg else None
    wg, tg = tb._inp(word, misalign=misalign), tb._inp(ptab, misalign=misalign)
    dg = bh.Guarded(4 * rows, fill=bh.SENTINEL).fill_payload(0).arm()
    hg = bh.Guarded(4 * rows * hld, fill=bh.SENTINEL)
    if hist is not None:
        hg.write(np.ascontiguousarray(hist, np.int32))
    hg.arm()
    h0 = bh.Guarded(4 * rows, fill=bh.SENTINEL)
    if hl0 is not None:
        h0.write(np.ascontiguousarray(hl0, np.int32))
    h0.arm()
    og, lpg, leng = tb._out(4 * rows * N), tb._out(4 * rows * N), tb._out(4 * rows)
    yg = tb._out(4 * rows * H, misalign=misalign)
    sampling = (sg.ptr, 1, *cfg) if cfg else (None, 0, 1.0, 0, 1.0)
    tb._done(lib.tfsc_k_generate_process(lg.ptr, ld, vocab, pg.ptr, t_, 0, EOS, dg.ptr, og.ptr, N, lpg.ptr, N, leng.ptr, 1, wg.ptr,
                                         tg.ptr, yg.ptr, rows, H, ig_.ptr, mg.ptr, S, hg.ptr, hld, h0.ptr, *proc, *sampling, None),
             "generate_process")
    bufs = dict(logits=lg, pos=pg, ids=ig_, mask=mg, word=wg, pos_table=tg, done=dg, hist=hg, hist_len0=h0, out_ids=og,
                log_probs=lpg, length=leng, y=yg)
    if sg is not None:
        bufs["seeds"] = sg
    tb._check(**bufs)
    return (og.read(np.int32, (rows, N)), lpg.read(shape=(rows, N)), leng.read(np.int32), yg.read(shape=(rows, H)),
            dg.read(np.int32), hg.read(np.int32, (rows, hld)), h0.read(np.int32))


def _case(vocab, ld, pad, H, seed):
    rows, S = 4, 12
    rng = np.random.default_rng(seed)
    logits = np.full((rows, ld), bh.FLOAT_POISONS[pad], np.float32)
    logits[:, :vocab] = rng.standard_normal((rows, vocab)) * 6
    ids = rng.integers(-3, vocab + 3, (rows, S)).astype(np.int32)
    ids[:, 6:] = ids[:, :6]                                                  # a repeated half: the n-gram ban has work
    mask = np.ones((rows, S), np.int32)
    mask[1, 8:] = 0                                                          # right-padded
    mask[2, :5] = 0                                                          # left-padded
    mask[3] = 0                                                              # fully padded
    pos = np.array([S - 1, 7, S - 1, -1], np.int32)
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((S + 4, H)).astype(np.float32)
    seeds = rng.integers(-2 ** 31, 2 ** 31, rows).astype(np.int32)
    return logits, ids, mask, pos, word, ptab, seeds


@pytest.mark.parametrize("vocab,ld", [(100, 103), (50257, 50272)])
@pytest.mark.parametrize("pad", ["nan", "inf"])
@pytest.mark.parametrize("H,misalign", [(64, 0), (64, 4), (6, 0)])
@pytest.mark.parametrize("proc,cfg", PROCS)
def test_generate_process(vocab, ld, pad, H, misalign, proc, cfg):
    """t = 0 writes each row's history and hist_len0 and one token after it, t = 1 only hist[hist_len0 + 1]; only column t
    of ids / log-probs is written; logits [vocab, ld) are never read: the tokens are the reference's"""
    logits, ids, mask, pos, word, ptab, seeds = _case(vocab, ld, pad, H, vocab + H + misalign)
    rows, S = ids.shape
    hld = S + 2
    out0 = _process(logits, ld, vocab, pos, ids, mask, word, ptab, 0, proc, cfg, misalign=misalign, seeds=seeds)
    hist0, hl0 = out0[5], out0[6]
    for r in range(rows):
        h = pr.history(ids[r], mask[r], int(pos[r]), vocab)
        assert hl0[r] == len(h), r
        assert hist0[r, :len(h)].tolist() == h, r
        bh.assert_untouched(hist0[r, len(h) + 1:], f"hist row {r}")
        want, amb = pr.pick(logits[r, :vocab], h, 0, *proc, EOS, seeds[r] if cfg else None, *(cfg or (1.0, 0, 1.0)))
        if pos[r] >= 0:
            assert amb or out0[0][r, 0] == want, (r, out0[0][r, 0], want)
            assert hist0[r, len(h)] == out0[0][r, 0], r
    t_ = 1
    out1 = _process(logits, ld, vocab, pos, ids, mask, word, ptab, t_, proc, cfg, hist=hist0, hl0=hl0, misalign=misalign, seeds=seeds)
    hist1 = out1[5]
    for r in range(rows):
        k = hl0[r] + t_
        others = [c for c in range(hld) if c != k]
        assert hist1[r, others].tobytes() == hist0[r, others].tobytes(), r
        assert hist1[r, k] != bh.SENTINEL and 0 <= hist1[r, k] < vocab, r
        if pos[r] >= 0:
            assert hist1[r, k] == out1[0][r, t_], r
    assert out1[6].tobytes() == hl0.tobytes()
    other = [c for c in range(t_ + 2) if c != t_]
    bh.assert_untouched(out1[0][:, other], "ids")
    bh.assert_untouched(out1[1][:, other], "log_probs")


@pytest.mark.parametrize("proc,cfg", PROCS + [((1.0, 0, 0), None)])
def test_process_row_isolation(proc, cfg):
    """a row of NaN, +-Inf or 3e38 logits, an all-zero mask or a prompt of one repeated id leaves every other row's bits"""
    vocab, ld, H = 1000, 1000, 128
    logits, ids, mask, pos, word, ptab, seeds = _case(vocab, ld, "nan", H, 7)
    pos = np.array([11, 7, 11, 5], np.int32)
    mask[3] = 1

    def run(logits, ids, mask):
        return _process(logits, ld, vocab, pos, ids, mask, word, ptab, 0, proc, cfg, seeds=seeds)
    args = [logits, ids, mask]
    cases = tb._float_cases(args, [0], [0, 2]) + [tb._row_case(args, 2, 1, 0), tb._row_case(args, 1, 3, 424)]
    tb._assert_isolated(run, args, cases)
