"""-m gpu: tfsc_k_generate_sample reads and writes only its own bytes (the harness of test_gpu_bounds.py): guard bands on
every operand, logits padding past the vocabulary and the gaps between strided seeds poisoned, word / pos_table / y off
16-byte alignment, and rows whose logits or seed change leaving every other row's bits alone."""
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds_harness as bh  # noqa: E402
import sampling_ref as sr  # noqa: E402
import test_gpu_bounds as tb  # noqa: E402

pytestmark = pytest.mark.gpu
lib = t._lib.lib
SEED_GAP = 0x5EED5EED                        # a valid seed, but not the row's: reading a gap changes the draw
CONFIGS = [(0.8, 40, 0.9), (1.3, 0, 0.95)]


def _sample(logits, ld, vocab, pos, word, ptab, seeds, t_, cfg, stride=1, misalign=0):
    """one guarded launch; logits [rows, ld] (columns from vocab on are the caller's poison), seeds at `stride` with the
    gaps poisoned. Returns ids, log_probs [rows, t + 2], length [rows], y [rows, H], done [rows]"""
    rows = len(pos)
    H, N = word.shape[1], t_ + 2
    sp = np.full((rows, stride), SEED_GAP, np.int32)
    sp[:, 0] = seeds
    lg, pg, sg = tb._inp(logits), tb._inp(pos, fill=0), tb._inp(sp, fill=SEED_GAP)
    wg, tg = tb._inp(word, misalign=misalign), tb._inp(ptab, misalign=misalign)
    dg = bh.Guarded(4 * rows, fill=bh.SENTINEL).fill_payload(0).arm()
    ig, lpg, leng = tb._out(4 * rows * N), tb._out(4 * rows * N), tb._out(4 * rows)
    yg = tb._out(4 * rows * H, misalign=misalign)
    tb._done(lib.tfsc_k_generate_sample(lg.ptr, ld, vocab, pg.ptr, t_, 0, -1, dg.ptr, ig.ptr, N, lpg.ptr, N, leng.ptr, 1, wg.ptr,
                                        tg.ptr, yg.ptr, rows, H, sg.ptr, stride, *cfg, None), "generate_sample")
    tb._check(logits=lg, pos=pg, seeds=sg, word=wg, pos_table=tg, done=dg, ids=ig, log_probs=lpg, length=leng, y=yg)
    return (ig.read(np.int32, (rows, N)), lpg.read(shape=(rows, N)), leng.read(np.int32), yg.read(shape=(rows, H)),
            dg.read(np.int32))


@pytest.mark.parametrize("vocab,ld", [(100, 103), (50257, 50272)])
@pytest.mark.parametrize("pad", ["nan", "inf"])
@pytest.mark.parametrize("H,misalign", [(64, 0), (64, 4), (6, 0)])
@pytest.mark.parametrize("cfg", CONFIGS)
def test_generate_sample(vocab, ld, pad, H, misalign, cfg):
    """only column t of ids / log-probs is written, every word of length and y is; logits [vocab, ld) and the seed gaps are
    never read: the draws are the reference's and those of a launch with packed seeds"""
    rows, t_, S = 4, 1, 10
    rng = np.random.default_rng(vocab + H + misalign)
    logits = np.full((rows, ld), bh.FLOAT_POISONS[pad], np.float32)
    logits[:, :vocab] = rng.standard_normal((rows, vocab)) * 6
    pos = np.array([3, 0, 9, 5], np.int32)
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((S + 4, H)).astype(np.float32)
    seeds = rng.integers(-2 ** 31, 2 ** 31, rows).astype(np.int32)
    ids, lp, length, y, done = _sample(logits, ld, vocab, pos, word, ptab, seeds, t_, cfg, stride=3, misalign=misalign)
    packed = _sample(logits, ld, vocab, pos, word, ptab, seeds, t_, cfg)
    for a, b in zip((ids, lp, length, y, done), packed):
        assert a.tobytes() == b.tobytes()
    g = ids[:, t_]
    for r in range(rows):
        want, amb = sr.draw(logits[r, :vocab], seeds[r], t_, *cfg)
        assert amb or g[r] == want, (r, g[r], want)
    x = logits[:, :vocab].astype(np.float64)
    ref_lp = x[np.arange(rows), g] - x.max(1) - np.log(np.exp(x - x.max(1, keepdims=True)).sum(1))
    assert np.max(np.abs(lp[:, t_] - ref_lp)) <= 1e-5
    assert length.tolist() == [t_ + 1] * rows and done.tolist() == [0] * rows
    assert np.array_equal(y, word[g] + ptab[pos + 1 + t_])
    other = [c for c in range(t_ + 2) if c != t_]
    bh.assert_untouched(ids[:, other], "ids")
    bh.assert_untouched(lp[:, other], "log_probs")


@pytest.mark.parametrize("cfg", CONFIGS + [(1.0, 0, 1.0)])
def test_sample_row_isolation(cfg):
    """a row of NaN, +-Inf or 3e38 logits (whose draw the kernel clamps before it reads a table), or another seed, leaves
    every other row's bits"""
    rows, t_, H, vocab = 5, 3, 128, 1000
    rng = np.random.default_rng(7)
    logits = rng.standard_normal((rows, vocab)).astype(np.float32) * 4
    pos = np.array([5, 0, 2, 7, 1], np.int32)
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((t_ + 10, H)).astype(np.float32)
    seeds = np.arange(rows, dtype=np.int32) * 101

    def run(logits, seeds):
        return _sample(logits, vocab, vocab, pos, word, ptab, seeds, t_, cfg, stride=2)
    args = [logits, seeds]
    cases = tb._float_cases(args, [0], [0, 2, 4]) + [tb._row_case(args, 1, j, 424242) for j in (0, 3)]
    tb._assert_isolated(run, args, cases)
