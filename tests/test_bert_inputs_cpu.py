"""BERT bundles with three inputs (input_ids, input_mask, segment_ids), CPU side: the fp64 reference on sentence-pair inputs
against transformers' BertForSequenceClassification, the committed fixture, and the two manifest writers."""
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_bert_pair_golden as pg  # noqa: E402
import torch_export as te  # noqa: E402

import bert_pair_ref as pr  # noqa: E402

INPUTS = t.modelformat.BERT_INPUTS


def _err(got, ref):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


def _arch(c):
    return {k: c[k] for k in pg.ARCH if k in c}


def _versions_match(g):
    import torch
    import transformers
    return {"torch": torch.__version__, "transformers": transformers.__version__} == g["versions"]


@pytest.mark.parametrize("name", ["bert_small_pair", "bert_base_pair"])
def test_oracle_pair_inputs_match_transformers(name, golden):
    c = pg.CASES[name]
    m, x, ref = pg.pair_case(c)
    g = golden("bert_pair_golden.json")
    if _versions_match(g):   # same seeds, same libraries -> the committed numbers
        assert np.max(np.abs(ref - np.array(g["cases"][name]["logits"]).reshape(g["cases"][name]["shape"]))) <= 1e-9
    # the inputs exercise what the ids alone cannot express
    assert (x["segment_ids"] == 1).any() and ((x["input_ids"] != 0) & (x["input_mask"] == 0)).any()
    assert ((x["input_ids"] == 0) & (x["input_mask"] == 1)).any() and (x["input_mask"].sum(1) > 0).all()
    arch = _arch(c)
    seq = arch.pop("seq", 128)
    oman = pr.oracle_pair_manifest(seq, INPUTS, **arch)
    blob = te.export_bert(m, oman)
    y = pr.pair_forward(oman, blob, x, np.float64)
    assert y.shape == ref.shape and _err(y, ref) <= 1e-6
    assert _err(pr.pair_forward(oman, blob, x, np.float32), ref) <= 1e-4
    # the same bundle with one input sees a different model input: mask from ids, segment 0
    man1 = pr.oracle_pair_manifest(seq, None, **arch)
    y1 = pr.pair_forward(man1, blob, x["input_ids"], np.float64)
    assert _err(y1, ref) > 1e-3
    # which the oracle's own interpreter of single-input bundles computes too
    assert _err(models.graph_forward(man1, blob, x["input_ids"], np.float64), y1) <= 1e-9


def test_fully_masked_sequence_is_softmax_of_raw_scores():
    """transformers adds finfo.min to masked keys; the bundle's rule for a sequence with every key masked is the softmax of
    its raw scores (no key masked), which the reference implements for an explicit mask as for ids."""
    import torch
    g = torch.Generator().manual_seed(3)
    qkv = torch.randn(2, 13, 3 * 32, generator=g, dtype=torch.float64)
    mask = torch.ones(2, 13, dtype=torch.int64)
    mask[1] = 0
    ctx = pr.attention_mask_ref(qkv, mask, 4)
    raw = models.attention_ref(qkv[1:], None, 4)
    assert torch.max(torch.abs(ctx[1:] - raw)) <= 1e-12
    # an all-ones mask masks nothing
    assert torch.max(torch.abs(pr.attention_mask_ref(qkv, torch.ones_like(mask), 4) - models.attention_ref(qkv, None, 4))) <= 1e-12


@pytest.mark.parametrize("inputs", [None, INPUTS, [{"name": "ids", "role": "ids"}, {"name": "am", "role": "mask"}]])
def test_manifest_writers_agree_on_inputs(inputs):
    arch = dict(seq=16, hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=32, labels=3)
    man = t.modelformat.bert_manifest(**arch, inputs=inputs)
    oman = pr.oracle_pair_manifest(arch.pop("seq"), inputs, **arch)
    assert man["signature"] == oman["signature"]
    assert man["weights_bytes"] == oman["weights_bytes"]
    assert [(o["op"], o.get("w_offset"), o.get("type_offset")) for o in man["ops"]] == \
           [(o["op"], o.get("w_offset"), o.get("type_offset")) for o in oman["ops"]]
    if inputs is None:
        assert man["signature"] == {"input": "input_ids", "output": "logits"}
    else:
        assert "input" not in man["signature"] and man["signature"]["inputs"] == inputs


def test_packed_order_is_byte_wise_sorted_names():
    assert t.modelformat.packed_input_order(INPUTS) == ["input_ids", "input_mask", "segment_ids"]
    # byte-wise, not locale or case-folded: upper case sorts before lower case, '_' (0x5f) before 'a'
    assert t.modelformat.packed_input_order([{"name": n} for n in ("b", "B", "a_", "a")]) == ["B", "a", "a_", "b"]
