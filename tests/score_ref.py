"""fp64 reference of score (GPT-2) bundles, test infrastructure: modelformat.gpt2_manifest's score graph interpreted with
gpt2_ref's helpers (the token_score op is the decoder's 1x1 conv over every token), and the scoring rule: every attended
position but a row's first is scored under the logits of the attended position before it. It shares no code with the
product beyond the manifest it reads."""
from __future__ import annotations

import numpy as np

import gpt2_ref as gr


def score_logits(man: dict, blob: np.ndarray, x, dtype=np.float64) -> np.ndarray:
    """logits [B, S, Vp] of a score bundle at every position in `dtype`; x as for gpt2_ref.gpt2_forward."""
    ops = [dict(o, op="conv", kh=1, kw=1) if o["op"] == "token_score" else o for o in man["ops"]]
    assert man["ops"][-1]["op"] == "token_score"
    _pos, y = gr.gpt2_forward(dict(man, ops=ops), blob, x, dtype)
    return y.reshape(y.shape[0], man["ops"][0]["h"], -1)


def scored_pairs(mask_row, S):
    """[(p, s)] of one row: s an attended position with an attended position below it, p = the largest such"""
    att = [j for j in range(S) if mask_row is None or mask_row[j] != 0]
    return list(zip(att[:-1], att[1:]))


def rank(z, t):
    """the number of ids that rank above t in the next-token head's order: z[j] > z[t], or equal with j < t"""
    z = np.asarray(z)
    return int(np.count_nonzero(z > z[t]) + np.count_nonzero(z[:t] == z[t]))


def score(logits, ids, mask, vocab):
    """(token_log_probs [B, S] fp64, token_ranks [B, S] int, token_log_prob_sum [B] fp64, token_count [B] int) from logits
    [B, S, >= vocab] (only the first vocab columns are read): the log-softmax at p of the clamped id at s, its rank in
    those logits, their sum and the count; 0 and -1 at unscored positions."""
    lg = np.asarray(logits)[..., :vocab]
    B, S = np.asarray(ids).reshape(len(lg), -1).shape
    ids = np.clip(np.asarray(ids).reshape(B, S), 0, vocab - 1)
    lp, rk = np.zeros((B, S)), np.full((B, S), -1, np.int64)
    for r in range(B):
        for p, s in scored_pairs(None if mask is None else np.asarray(mask).reshape(B, S)[r], S):
            z = lg[r, p].astype(np.float64)
            m = z.max()
            lp[r, s] = z[ids[r, s]] - m - np.log(np.exp(z - m).sum())
            rk[r, s] = rank(lg[r, p], ids[r, s])
    count = (rk >= 0).sum(axis=1)
    return lp, rk, lp.sum(axis=1), count


def score_forward(man: dict, blob: np.ndarray, x):
    """score() of a score bundle's fp64 forward on x"""
    roles = {i["role"]: i["name"] for i in man["signature"].get("inputs", [])}
    S = man["ops"][0]["h"]
    ids = np.asarray(x[roles["ids"]] if roles else x).reshape(-1, S)
    mask = np.asarray(x[roles["mask"]]).reshape(-1, S) if "mask" in roles else None
    return score(score_logits(man, blob, x), ids, mask, man["ops"][-1]["vocab"])
