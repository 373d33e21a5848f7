"""fp64 reference of greedy generation on GPT-2 generate bundles, test infrastructure: full recompute with gpt2_ref's
interpreter on each row's growing sequence, no KV cache. It shares no code with the product beyond the manifest it reads.

The rules: a row's prompt ends at p (its last attended position, S - 1 without a mask; -1: nothing to continue). Token g_t
sits at slot p + 1 + t with position embedding wpe[p + 1 + t], and it sees the prompt's attended keys and every generated
one. So step t runs the bundle's graph on prompt[:p + 1] + g[:t] with the prompt's mask and ones after it. g_t is the
argmax over the first vocab logits (ties to the lower id), its log-probability logit[g_t] - logsumexp(logits[:vocab]).
After eos_token_id (emitted and counted) a row's ids are -1 and its log-probabilities 0."""
from __future__ import annotations

import copy

import numpy as np

import gpt2_ref as gr


def _at_length(man: dict, L: int) -> dict:
    """the manifest on L tokens: the interpreter takes the sequence length from the embed op"""
    m = copy.deepcopy(man)
    m["ops"][0]["h"] = L
    return m


def generate_ref(man: dict, blob: np.ndarray, x, N: int, eos=None):
    """(ids [B, N] int32, log_probs [B, N] float64, length [B] int32) for x as gpt2_ref.gpt2_forward takes it."""
    roles = {i["role"]: i["name"] for i in man["signature"].get("inputs", [])}
    S = man["ops"][0]["h"]
    V = man["ops"][0]["vocab"]
    ids = np.asarray(x[roles["ids"]] if roles else x).reshape(-1, S)
    mask = np.asarray(x[roles["mask"]]).reshape(-1, S) if "mask" in roles else None
    B = ids.shape[0]
    out_ids = np.full((B, N), -1, np.int32)
    out_lp = np.zeros((B, N))
    length = np.zeros(B, np.int32)
    for b in range(B):
        p = S - 1 if mask is None else (int(np.nonzero(mask[b])[0].max()) if mask[b].any() else -1)
        if p < 0:
            continue
        seq = list(ids[b, :p + 1])
        msk = list(np.ones(p + 1, np.int32) if mask is None else mask[b, :p + 1])
        for t in range(N):
            L = len(seq)
            m = _at_length(man, L)
            feed = {roles["ids"]: np.array([seq], np.int32)} if roles else np.array([seq], np.int32)
            if "mask" in roles:
                feed[roles["mask"]] = np.array([msk], np.int32)
            pos, logits = gr.gpt2_forward(m, blob, feed)
            assert pos[0] == L - 1
            lg = logits[0, :V]
            g = int(np.argmax(lg))
            mx = lg.max()
            out_ids[b, t] = g
            out_lp[b, t] = lg[g] - (mx + np.log(np.exp(lg - mx).sum()))
            length[b] = t + 1
            if eos is not None and g == eos:
                break
            seq.append(g)
            msk.append(1)
    return out_ids, out_lp, length
