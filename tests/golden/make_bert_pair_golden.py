"""Generates tests/golden/bert_pair_golden.json: fp64 logits of transformers' BertForSequenceClassification (seeded weights,
tests/torch_export.hf_bert) on sentence-pair inputs given as three tensors -- input_ids, input_mask (attention_mask) and
segment_ids (token_type_ids). The inputs hold segment ids 0 / 1, padded tails, real tokens masked out and id-0 tokens left
unmasked, so neither the mask nor the segments can be derived from the ids. Every sequence keeps at least one unmasked key
(transformers masks with finfo.min, the bundle with -10000: they agree only then). The tests rebuild the model live and
require these numbers when the library versions match.

    python tests/golden/make_bert_pair_golden.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import torch_export as te  # noqa: E402

CASES = {
    "bert_small_pair": dict(seed=4, input_seed=7, batch=8, seq=16, hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=32,
                            labels=3),
    "bert_base_pair": dict(seed=3, input_seed=8, batch=8),
}
ARCH = ("seq", "hidden", "layers", "heads", "inter", "vocab", "max_pos", "labels")


def pair_inputs(batch, seq, vocab, seed):
    """{input_ids, input_mask, segment_ids}, int32 [batch, seq]: row b is a sentence pair split at `cut`, padded after
    `end`; some rows mask real tokens out and keep id-0 tokens unmasked."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(1, vocab, (batch, seq)).astype(np.int32)
    mask = np.ones((batch, seq), np.int32)
    seg = np.zeros((batch, seq), np.int32)
    for b in range(batch):
        end = seq - (b * seq) // (2 * batch)              # row 0 unpadded, later rows up to half padding
        cut = max(1, (end * (2 + b % 3)) // 6)
        seg[b, cut:end] = 1
        ids[b, end:], mask[b, end:] = 0, 0                 # [PAD] tail
        if b % 2 == 1:
            mask[b, rng.integers(1, end, 2)] = 0           # real tokens masked out
        if b % 3 == 2:
            k = rng.integers(1, end, 2)
            ids[b, k], mask[b, k] = 0, 1                   # id 0 inside the sequence, still attended
    return {"input_ids": ids, "input_mask": mask, "segment_ids": seg}


def pair_reference(model, x):
    """transformers' own forward in fp64 with explicit attention_mask and token_type_ids."""
    import copy
    import torch
    m64 = copy.deepcopy(model).double()
    t = {k: torch.from_numpy(np.ascontiguousarray(v, np.int64)) for k, v in x.items()}
    with torch.no_grad():
        return m64(input_ids=t["input_ids"], attention_mask=t["input_mask"], token_type_ids=t["segment_ids"]).logits.numpy()


def pair_case(c):
    kw = {k: c[k] for k in ARCH if k in c}
    m = te.hf_bert(c["seed"], **kw)
    x = pair_inputs(c["batch"], kw.get("seq", 128), kw.get("vocab", 30522), c["input_seed"])
    return m, x, pair_reference(m, x)


if __name__ == "__main__":
    import torch
    import transformers
    out = {"versions": {"torch": torch.__version__, "transformers": transformers.__version__}, "cases": {}}
    for name, c in CASES.items():
        _m, _x, ref = pair_case(c)
        out["cases"][name] = {"config": c, "shape": list(ref.shape), "logits": [float(v) for v in ref.ravel()]}
        print(name, ref.shape, float(np.abs(ref).max()))
    with open(os.path.join(HERE, "bert_pair_golden.json"), "w") as f:
        json.dump(out, f)
