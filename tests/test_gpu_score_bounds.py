"""-m gpu: tfsc_k_token_score and tfsc_k_score_head read and write only their own bytes (the harness of test_gpu_bounds.py):
guard bands on every operand, logits padding past the vocabulary poisoned, the score kernel writing only the scored slots
of its chunk and the head only its outputs, and a row of NaN, +-Inf or 3e38 logits leaving every other row's bits alone."""
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds_harness as bh  # noqa: E402
import score_ref as sr  # noqa: E402
import test_gpu_bounds as tb  # noqa: E402

pytestmark = pytest.mark.gpu
lib = t._lib.lib


def _case(vocab, ld, pad, seed, S=10):
    rows = 4
    rng = np.random.default_rng(seed)
    logits = np.full((rows * S, ld), bh.FLOAT_POISONS[pad], np.float32)
    logits[:, :vocab] = rng.standard_normal((rows * S, vocab)) * 6
    ids = rng.integers(-3, vocab + 3, (rows, S)).astype(np.int32)
    mask = np.ones((rows, S), np.int32)
    mask[1, 7:] = 0                                                          # right-padded
    mask[2, :4] = 0                                                          # left-padded
    mask[2, 6] = 0                                                           # and holed
    mask[3] = 0                                                              # fully padded
    return logits, ids, mask


def _token_score(logits, ld, vocab, ids, mask, first, n, misalign=0):
    """one guarded launch over token rows [first, first + n); the log-probabilities and ranks [rows, S] start as sentinel"""
    rows, S = ids.shape
    lg = tb._inp(logits[first:first + n], misalign=misalign)
    ig, mg = tb._inp(ids, fill=0), tb._inp(mask, fill=1)
    lpg, rkg = tb._out(4 * rows * S), tb._out(4 * rows * S)
    tb._done(lib.tfsc_k_token_score(lg.ptr, ld, first, n, ig.ptr, mg.ptr, S, rows, S, vocab, lpg.ptr, rkg.ptr, None), "token_score")
    tb._check(logits=lg, ids=ig, mask=mg, log_probs=lpg, ranks=rkg)
    return lpg.read(shape=(rows, S)), rkg.read(np.int32, (rows, S))


@pytest.mark.parametrize("vocab,ld", [(100, 103), (50257, 50272)])
@pytest.mark.parametrize("pad", ["nan", "inf", "3e38"])
@pytest.mark.parametrize("first,n", [(0, 40), (3, 15), (17, 1), (25, 15)])
def test_token_score(vocab, ld, pad, first, n):
    """only slot next(p) of each attended p in the chunk is written, with the reference's rank; the padding columns are
    never read"""
    logits, ids, mask = _case(vocab, ld, pad, vocab + first)
    rows, S = ids.shape
    lp, rk = _token_score(logits, ld, vocab, ids, mask, first, n, misalign=4 * (first % 2))
    want_lp, want_rk, _s, _c = sr.score(logits.reshape(rows, S, ld), ids, mask, vocab)
    mine = np.zeros((rows, S), bool)
    for r in range(rows):
        for p, s in sr.scored_pairs(mask[r], S):
            mine[r, s] = first <= r * S + p < first + n
    bh.assert_untouched(lp[~mine], "log_probs outside the chunk's scored slots")
    bh.assert_untouched(rk[~mine], "ranks outside the chunk's scored slots")
    assert np.array_equal(rk[mine], want_rk[mine])
    assert np.all(np.abs(lp[mine] - want_lp[mine]) <= 2e-6 * np.maximum(1.0, np.abs(want_lp[mine])))


@pytest.mark.parametrize("misalign", [0, 4])
def test_score_head(misalign):
    """the head writes its outputs at their lds and nothing between them; it reads only the scored slots (the others hold
    NaN and a poison rank)"""
    rows, S, ld = 4, 10, 2 * 10 + 5
    _logits, _ids, mask = _case(100, 100, "nan", 3)
    scored = np.zeros((rows, S), bool)
    for r in range(rows):
        scored[r, [s for _p, s in sr.scored_pairs(mask[r], S)]] = True
    rng = np.random.default_rng(2)
    lp = np.where(scored, -rng.random((rows, S)) * 9, np.nan).astype(np.float32)
    rk = np.where(scored, rng.integers(0, 100, (rows, S)), 1 << 30).astype(np.int32)
    lpg, rkg, mg = tb._inp(lp), tb._inp(rk, fill=1 << 30), tb._inp(mask, fill=1)
    yg = tb._out(4 * rows * ld, misalign=misalign)
    y = yg.ptr
    tb._done(lib.tfsc_k_score_head(lpg.ptr, rkg.ptr, mg.ptr, S, rows, S, y, ld, y + 4 * S, ld, y + 8 * S, ld, y + 8 * S + 4, ld, None),
             "score_head")
    tb._check(log_probs=lpg, ranks=rkg, mask=mg, y=yg)
    out = yg.read(shape=(rows, ld))
    bh.assert_untouched(out[:, 2 * S + 2:], "the gap between rows")
    bh.assert_written(out[:, :2 * S + 2], "the outputs")
    assert np.array_equal(out[:, :S], np.where(scored, lp, 0).astype(np.float32))
    assert np.array_equal(out[:, S:2 * S].view(np.int32), np.where(scored, rk, -1))
    assert np.array_equal(out[:, 2 * S + 1].view(np.int32), scored.sum(axis=1))
    assert np.allclose(out[:, 2 * S], np.where(scored, lp, 0).astype(np.float64).sum(axis=1), rtol=1e-6)


def test_row_isolation():
    """a row of NaN, +-Inf or 3e38 logits, an all-zero mask row or out-of-range ids leave every other row's bits"""
    vocab, ld = 1000, 1000
    logits, ids, mask = _case(vocab, ld, "nan", 7)
    rows, S = ids.shape
    mask[3] = 1

    def run(logits, ids, mask):
        return _token_score(logits.reshape(rows * S, ld), ld, vocab, ids, mask, 0, rows * S)
    args = [logits.reshape(rows, S, ld), ids, mask]
    cases = tb._float_cases(args, [0], [0, 2]) + [tb._row_case(args, 2, 1, 0), tb._row_case(args, 1, 3, 10 ** 9)]
    tb._assert_isolated(run, args, cases)
