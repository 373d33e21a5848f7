"""Brute-force reference of the question-answering span head (test infrastructure): every candidate (i, j) of a row is
enumerated and sorted, nothing is shared with span.cu. A candidate is a pair of eligible tokens with i <= j < i + L, its
score the fp32 sum start[i] + end[j]; spans are ordered by score descending, then i, then j ascending, a NaN score is
never a candidate, and slots past the last candidate are (-1, -1, -FLT_MAX)."""
from __future__ import annotations

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def eligible(ids, mask, types, sep_id=None):
    """Token p is eligible when mask[p] != 0 (mask None: ids[p] != 0), types[p] == 1 and ids[p] != sep_id."""
    ids = np.asarray(ids)
    e = (np.asarray(mask) != 0) if mask is not None else (ids != 0)
    e = e & (np.asarray(types) == 1)
    if sep_id is not None:
        e = e & (ids != sep_id)
    return e


def _pairs(S, L):
    i, j = np.triu_indices(S)
    keep = j - i < L
    return i[keep], j[keep]


def span_ref(start, end, elig, L, k, dtype=np.float32):
    """(starts int32 [..., k], ends int32 [..., k], scores [..., k]) of rows start / end / elig [..., S]. The sums and
    scores are in `dtype`: float32 is the kernel's arithmetic, float64 ranks the exact logits of a reference model."""
    start = np.asarray(start, dtype)
    end = np.asarray(end, dtype)
    elig = np.asarray(elig, bool)
    lead, S = start.shape[:-1], start.shape[-1]
    s2, e2, g2 = start.reshape(-1, S), end.reshape(-1, S), elig.reshape(-1, S)
    i, j = _pairs(S, L)
    starts = np.full((len(s2), k), -1, np.int32)
    ends = np.full((len(s2), k), -1, np.int32)
    scores = np.full((len(s2), k), -FLT_MAX, dtype)
    for r in range(len(s2)):
        v = s2[r][i] + e2[r][j]                            # fp32 + fp32 -> fp32, as the kernel adds
        ok = g2[r][i] & g2[r][j] & ~np.isnan(v)
        vi, ii, jj = v[ok], i[ok], j[ok]
        order = np.lexsort((jj, ii, -vi))[:k]             # score descending, then i, then j ascending
        n = len(order)
        starts[r, :n], ends[r, :n], scores[r, :n] = ii[order], jj[order], vi[order]
    return starts.reshape(lead + (k,)), ends.reshape(lead + (k,)), scores.reshape(lead + (k,))


def qa_inputs(batch, seq, vocab, seed, sep_id):
    """SQuAD-shaped sentence pairs {input_ids, input_mask, segment_ids}, int32 [batch, seq]: a question in segment 0, a
    passage in segment 1 that ends in [SEP] = sep_id, then a [PAD] tail (rows padded from none up to half)."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(1, vocab, (batch, seq)).astype(np.int32)
    ids[ids == sep_id] = sep_id + 1 if sep_id + 1 < vocab else 1
    mask = np.ones((batch, seq), np.int32)
    seg = np.zeros((batch, seq), np.int32)
    for b in range(batch):
        end = seq - (b * seq) // (2 * batch)
        cut = max(1, min(end - 1, (end * (1 + b % 3)) // 6))
        ids[b, cut - 1] = sep_id                           # [SEP] after the question (segment 0)
        seg[b, cut:end] = 1
        ids[b, end - 1] = sep_id                           # the final [SEP] (segment 1)
        ids[b, end:], mask[b, end:] = 0, 0
    return {"input_ids": ids, "input_mask": mask, "segment_ids": seg}
