"""Reference forward of BERT graph bundles that declare several inputs (signature.inputs: input_ids / input_mask /
segment_ids), test infrastructure. It interprets the bundle's op list in fp64 (or fp32) with the attention and LayerNorm
arithmetic of oracle.models, reads the named inputs from a dict, adds the segment rows in the embedding and masks the keys
whose mask value is 0. It is independent of the product's packing code: nothing here concatenates a request row.

oracle.models.attention_ref masks every key whose value is 0 in the array it is given, so an explicit attention mask is
passed in place of the ids: a mask of all zeros adds the same constant to every score, i.e. the softmax of the raw scores,
which is the bundle's rule for a fully-masked sequence."""
from __future__ import annotations

import numpy as np

from oracle import models


def oracle_pair_manifest(seq, inputs, **arch):
    """The oracle's restatement of BERT (models.bert_ops / graph_manifest) with `inputs` declared as signature.inputs in
    place of signature.input (None: the single-input form)."""
    man = models.graph_manifest([seq], models.bert_ops(seq=seq, **arch), 4, ("input_ids", "logits"), "int32")
    if inputs is not None:
        man["signature"] = {"inputs": [{"name": i["name"], "role": i["role"]} for i in inputs], "output": "logits"}
    return man


def attention_mask_ref(qkv, mask, heads):
    """BERT attention on torch qkv[B, S, 3H] with an explicit mask[B, S]: key j of sequence b is masked iff mask[b, j] == 0."""
    return models.attention_ref(qkv, mask, heads)


def pair_forward(man: dict, blob: np.ndarray, x, dtype=np.float64) -> np.ndarray:
    """Logits [B, labels] of a BERT graph bundle. x: {name: int array [B, S]} for a bundle with signature.inputs (a missing
    mask role masks [PAD] = id 0, a missing type_ids role is segment 0), or the ids array of a single-input bundle."""
    import torch
    import torch.nn.functional as F
    td = torch.float64 if dtype == np.float64 else torch.float32
    S = man["input_shape"][0]
    roles = {i["role"]: i["name"] for i in man["signature"].get("inputs", [])}

    def named(role):
        if not roles:
            return torch.from_numpy(np.ascontiguousarray(x, np.int64)).reshape(-1, S) if role == "ids" else None
        return torch.from_numpy(np.ascontiguousarray(x[roles[role]], np.int64)).reshape(-1, S) if role in roles else None

    ids, types, mask = named("ids"), named("type_ids"), named("mask")
    if mask is None:
        mask = ids

    def vec(off, n):
        return torch.from_numpy(blob[off // 4: off // 4 + n]).to(td)

    bufs = {}
    for o in man["ops"]:
        src = bufs.get(o["src"])
        if o["op"] == "embed":
            Hd = o["c"]
            word = vec(o["word_offset"], o["vocab"] * Hd).view(o["vocab"], Hd)
            pos = vec(o["pos_offset"], o["max_pos"] * Hd).view(o["max_pos"], Hd)[:S]
            typ = vec(o["type_offset"], 2 * Hd).view(2, Hd)
            seg = typ[types.clamp(0, 1)] if types is not None else typ[0]
            e = word[ids.clamp(0, o["vocab"] - 1)] + pos.unsqueeze(0) + seg
            y = models.layer_norm_ref(e, vec(o["w_offset"], Hd), vec(o["b_offset"], Hd), o.get("eps", 1e-12))
        elif o["op"] == "layernorm":
            y = models.layer_norm_ref(src + bufs[o["res"]] if o.get("res", -100) != -100 else src, vec(o["w_offset"], o["c"]),
                                      vec(o["b_offset"], o["c"]), o.get("eps", 1e-12))
        elif o["op"] == "attention":
            y = attention_mask_ref(src, mask, o["heads"])
        elif o["op"] in ("conv", "dense"):
            c, cout = o["c"], o["cout"]
            w = vec(o["w_offset"], c * cout).view(c, cout)
            b = vec(o["b_offset"], cout)
            if o["op"] == "dense":   # the first c values of each example: the [CLS] token, or the whole vector
                y = (src.reshape(src.shape[0], -1)[:, :c] @ w + b).unsqueeze(1)
            else:                    # 1 x 1 conv over the tokens
                y = src @ w + b
            if o.get("res", -100) != -100:
                y = y + bufs[o["res"]]
            act = o.get("act", "none")
            y = torch.relu(y) if act == "relu" else F.gelu(y) if act == "gelu" else torch.tanh(y) if act == "tanh" else y
        else:
            raise ValueError(f"op {o['op']} is not part of a BERT bundle")
        bufs[o["dst"]] = y
    out = bufs[-2]
    return out.reshape(out.shape[0], -1).numpy().astype(dtype)
