"""Reference of a processing generate bundle's step (DESIGN §3): the row's history, the repetition penalty, the no-repeat
n-gram bans and the minimum-length EOS ban on fp32 logits, then the greedy pick or the sampled one through sampling_ref, and
transformers' three processors on the same logits for comparison."""
import numpy as np

import sampling_ref as sr


def history(ids, mask, p, vocab):
    """the row's attended prompt ids in position order: positions j <= p whose mask is set (mask None: all), each clamped to
    [0, vocab)"""
    return [min(max(int(ids[j]), 0), vocab - 1) for j in range(p + 1) if mask is None or mask[j] != 0]


def banned_ngrams(h, n):
    """every h[i + n - 1] whose n - 1 tokens before it equal the history's last n - 1 tokens (n = 1: every id of h)"""
    L = len(h)
    if n < 1 or L < n - 1:
        return set()
    tail = list(h[L - n + 1:]) if n > 1 else []
    return {h[i + n - 1] for i in range(L - n + 1) if list(h[i:i + n - 1]) == tail}


def process(z, h, t, penalty=1.0, ngram=0, min_new=0, eos=-1, dtype=np.float32):
    """z' of the raw row z for history h at step t: z < 0 ? z * p : z / p once per id of h, then -inf at the banned n-gram
    ids, then -inf at eos while t < min_new; in fp32 (the kernel's bits) or, dtype float64, on fp64 reference logits"""
    z = np.asarray(z, dtype)
    out = z.copy()
    p = dtype(penalty)
    if h:
        u = np.unique(np.asarray(h, np.int64))
        with np.errstate(all="ignore"):
            out[u] = np.where(z[u] < 0, z[u] * p, z[u] / p).astype(dtype)
    for g in banned_ngrams(list(h), ngram):
        out[g] = -np.inf
    if t < min_new and eos >= 0:
        out[eos] = -np.inf
    return out


def argmax(z):
    """the next-token head's rank-order argmax: the largest value, ties to the lower id; all -inf: id 0"""
    return int(np.argmax(np.asarray(z, np.float32)))


def pick(z, h, t, penalty=1.0, ngram=0, min_new=0, eos=-1, seed=None, temperature=1.0, top_k=0, top_p=1.0):
    """(token, ambiguous) of the step: the argmax of z' (seed None or top_k = 1), or sampling_ref.draw on z' with the seed. All
    of z' -inf: id 0 and no draw."""
    zp = process(z, h, t, penalty, ngram, min_new, eos)
    if seed is None or top_k == 1 or np.all(zp == -np.inf):
        return argmax(zp), False
    # a top-k boundary past the finite logits keeps the same weights as one at their count: the -inf ids weigh 0
    finite = int(np.isfinite(zp).sum())
    k = min(top_k, finite) if top_k > 0 else 0
    return sr.draw(zp, seed, t, temperature, k, top_p)


def transformers_process(z, input_ids, prompt_len, penalty=None, ngram=None, min_new=None, eos=-1, dtype=np.float32):
    """transformers' RepetitionPenalty -> NoRepeatNGram -> MinNewTokensLength processors on the row z (fp32, or dtype
    float64) for input_ids (the prompt and the tokens so far); None leaves a processor out"""
    import torch
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor)
    ids = torch.tensor([list(input_ids)], dtype=torch.long)
    s = torch.from_numpy(np.asarray(z, dtype).copy())[None]
    if penalty is not None:
        s = RepetitionPenaltyLogitsProcessor(penalty)(ids, s)
    if ngram is not None:
        s = NoRepeatNGramLogitsProcessor(ngram)(ids, s)
    if min_new is not None:
        s = MinNewTokensLengthLogitsProcessor(prompt_len, min_new, eos)(ids, s)
    return s[0].numpy()
