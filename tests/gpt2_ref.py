"""fp64 reference of next-token (GPT-2) bundles, test infrastructure: an interpreter of modelformat.gpt2_manifest's op list
(embedding without LayerNorm, LayerNorm, 1x1 convs with the tanh GELU, causal attention, last_token) and the next-token
head's top k (descending logit, ties to the lower id, as tf.math.top_k) with softmax probabilities over the first `vocab`
logits. It shares no code with the product beyond the manifest it reads."""
from __future__ import annotations

import math

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def gelu_tanh(x):
    return 0.5 * x * (1.0 + np.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def causal_attention_ref(qkv, heads, mask=None):
    """qkv [B, S, 3H] (q | k | v) -> ctx [B, S, H] in qkv's dtype: query i sees keys j <= i (exactly zero weight beyond),
    and a key whose mask is 0 gets -10000 unless every key of its sequence has mask 0 (BERT's additive mask)."""
    B, S, H3 = qkv.shape
    H = H3 // 3
    d = H // heads
    q, k, v = (qkv[..., i * H:(i + 1) * H].reshape(B, S, heads, d).transpose(0, 2, 1, 3) for i in range(3))
    sc = q @ k.transpose(0, 1, 3, 2) / math.sqrt(d)                      # [B, heads, S, S]
    if mask is not None:
        m = np.asarray(mask).reshape(B, S) == 0
        m &= ~m.all(axis=1, keepdims=True)
        sc = sc + np.where(m, -10000.0, 0.0)[:, None, None, :]
    hidden = np.triu(np.ones((S, S), bool), 1)
    sc = np.where(hidden, -np.inf, sc)
    p = np.exp(sc - sc.max(axis=-1, keepdims=True))
    p /= p.sum(axis=-1, keepdims=True)
    return (p @ v).transpose(0, 2, 1, 3).reshape(B, S, H)


def last_token_ref(hidden, mask):
    """positions [B] int32 (the highest position with mask != 0, S - 1 without a mask, -1 for none) and the gathered
    hidden states [B, H] (zeros for -1)."""
    B, S, H = hidden.shape
    if mask is None:
        pos = np.full(B, S - 1, np.int32)
    else:
        m = np.asarray(mask).reshape(B, S) != 0
        pos = np.where(m.any(axis=1), S - 1 - np.argmax(m[:, ::-1], axis=1), -1).astype(np.int32)
    gat = np.zeros((B, H), hidden.dtype)
    live = pos >= 0
    gat[live] = hidden[np.nonzero(live)[0], pos[live]]
    return pos, gat


def top_k_ref(logits, positions, vocab, k):
    """The next-token head on logits [B, Vp] (the first vocab columns count): ids [B, k] by a stable argsort of the negated
    fp32 logits, fp64 softmax probabilities over the vocab logits and the logits at those ids; a row with position -1 is
    (-1, 0, -FLT_MAX)."""
    lg = np.asarray(logits)[:, :vocab]
    B = lg.shape[0]
    ids = np.full((B, k), -1, np.int32)
    probs = np.zeros((B, k))
    vals = np.full((B, k), -FLT_MAX)
    for r in range(B):
        if positions[r] < 0:
            continue
        x = lg[r]
        order = np.argsort(-x, kind="stable")[:k]
        x64 = x.astype(np.float64)
        e = np.exp(x64 - x64.max())
        ids[r], probs[r], vals[r] = order, e[order] / e.sum(), x64[order]
    return ids, probs, vals


def gpt2_forward(man: dict, blob: np.ndarray, x, dtype=np.float64):
    """(positions [B] int32, logits [B, Vp]) of a next-token bundle in `dtype`. x: {name: int array [B, S]} for a bundle
    with signature.inputs, or the ids array of a single-input bundle."""
    roles = {i["role"]: i["name"] for i in man["signature"].get("inputs", [])}
    emb = man["ops"][0]
    S, H = emb["h"], emb["c"]
    ids = np.asarray(x[roles["ids"]] if roles else x).reshape(-1, S)
    mask = np.asarray(x[roles["mask"]]).reshape(-1, S) if "mask" in roles else None
    B = ids.shape[0]

    def t(off, *shape):
        return blob[off // 4: off // 4 + int(np.prod(shape))].astype(dtype).reshape(shape)

    bufs, pos = {}, None
    for o in man["ops"]:
        src = bufs.get(o["src"])
        if o["op"] == "embed":
            assert o.get("norm") is False
            y = t(o["word_offset"], o["vocab"], H)[np.clip(ids, 0, o["vocab"] - 1)] + t(o["pos_offset"], o["max_pos"], H)[:S]
        elif o["op"] == "layernorm":
            v = src + (bufs[o["res"]] if "res" in o else 0)
            mean = v.mean(axis=-1, keepdims=True)
            var = ((v - mean) ** 2).mean(axis=-1, keepdims=True)
            y = (v - mean) / np.sqrt(var + o["eps"]) * t(o["w_offset"], o["c"]) + t(o["b_offset"], o["c"])
        elif o["op"] == "conv":
            assert o["kh"] == o["kw"] == 1
            y = src @ t(o["w_offset"], o["c"], o["cout"]) + t(o["b_offset"], o["cout"])
            if "res" in o:
                y = y + bufs[o["res"]]
            act = o.get("act", "none")
            assert act in ("none", "gelu_tanh")
            y = gelu_tanh(y) if act == "gelu_tanh" else y
        elif o["op"] == "attention":
            assert o.get("causal") is True
            y = causal_attention_ref(src.reshape(B, S, -1), o["heads"], mask)
        elif o["op"] == "last_token":
            pos, y = last_token_ref(src.reshape(B, S, H), mask)
        else:
            raise ValueError(f"op {o['op']} is not part of a GPT-2 bundle")
        bufs[o["dst"]] = y
    return pos, bufs[-2].reshape(B, -1).astype(dtype)
