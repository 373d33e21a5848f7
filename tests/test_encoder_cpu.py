"""Encoder (embedding) outputs -- sequence_output, pooled_output, cls_embedding, mean_embedding -- CPU side: every loader
rejection of an encoder bundle, packed_output_layout against the loader's layout (tfsc_manifest_check), the manifest
writer, the fp64 reference on hand cases, and encoder bundles exported from transformers' BertModel, with and without a
pooling layer, through the existing CPU interpreters."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bert_pair_ref as pr  # noqa: E402
import embed_export as ee  # noqa: E402
import embed_ref as er  # noqa: E402
import span_ref as sr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=1, heads=4, inter=128, vocab=100, max_pos=512)
ALL = [{"name": k, "kind": k} for k in mf.ENCODER_OUTPUT_KINDS]
NO_POOL = [o for o in ALL if o["kind"] != "pooled_output"]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _enc(seq=16, outputs=ALL, inputs=mf.BERT_INPUTS, pooler=True, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.bert_manifest(seq=seq, **arch, inputs=inputs, outputs=outputs, head="encoder", pooler=pooler)


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


# ------------------------------------------------------------------------------------------- layout ----
OUTPUT_SETS = [
    (ALL, True),
    (NO_POOL, False),
    ([{"name": "embedding", "kind": "mean_embedding", "normalize": True}], False),
    ([{"name": "z", "kind": "sequence_output"}, {"name": "a", "kind": "cls_embedding", "normalize": False},
      {"name": "pooled", "kind": "pooled_output"}], True),
    ([{"name": "Pooled", "kind": "pooled_output"}, {"name": "sentence", "kind": "mean_embedding"}], True),
    ([{"name": "last_hidden_state", "kind": "sequence_output"}], False),
]


@pytest.mark.parametrize("seq", [1, 16, 384])
@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(which, seq):
    outs, pooler = OUTPUT_SETS[which]
    man = _enc(seq=seq, outputs=outs, pooler=pooler)
    rc, got = _check(man)
    assert rc > 0, got
    H = SMALL["hidden"]
    layout = mf.packed_output_layout(outs, H, seq)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    assert [o["kind"] for o in got["outputs"]] == [next(x["kind"] for x in outs if x["name"] == n) for n, *_ in layout]
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == H and got["head_k"] == seq
    assert [x[0] for x in layout] == sorted((o["name"] for o in outs), key=lambda s: s.encode())


def test_encoder_manifest_writer():
    man = _enc(seq=16)
    last, prev = man["ops"][-1], man["ops"][-2]
    assert last["op"] == "dense" and last["act"] == "tanh" and last["src"] == 0 and last["dst"] == -2
    assert last["c"] == last["cout"] == 64 and prev["op"] == "layernorm" and prev["dst"] == 0
    rc, got = _check(man)
    assert rc > 0 and got["out_dim"] == 3 * 64 + 16 * 64 and got["in_dim"] == 3 * 16
    nop = _enc(seq=16, outputs=NO_POOL, pooler=False)
    assert nop["ops"][-1]["op"] == "layernorm" and nop["ops"][-1]["dst"] == -2 and not any(o["op"] == "dense" for o in nop["ops"])
    assert nop["weights_bytes"] < man["weights_bytes"]
    # the same bundles with one output answer the pooler [H] or the hidden states [S, 1, H], as any graph bundle
    rc, got = _check(_enc(seq=16, outputs=None))
    assert rc > 0 and got["out_dim"] == 64 and got["outputs"] == []
    rc, got = _check(_enc(seq=16, outputs=None, pooler=False))
    assert rc > 0 and got["out_dim"] == 16 * 64
    # the classifier and span variants are what they were
    assert mf.bert_manifest(seq=16, **SMALL) == mf.bert_manifest(seq=16, **SMALL, head="classify", pooler=False)
    # split_packed_rows gives sequence_output as [rows, S, H]
    S, H = 3, 4
    layout = mf.packed_output_layout(ALL, H, S)
    width = sum(w for _n, _o, w, _d in layout)
    words = np.arange(2 * width, dtype=np.float32).reshape(2, width)
    got = mf.split_packed_rows(words, ALL, H, S)
    off = dict((n, o) for n, o, _w, _d in layout)
    assert got["sequence_output"].shape == (2, S, H) and got["mean_embedding"].shape == (2, H)
    assert got["sequence_output"][1, 2, 3] == words[1, off["sequence_output"] + 2 * H + 3]
    assert got["cls_embedding"].tolist() == words[:, off["cls_embedding"]:off["cls_embedding"] + H].tolist()


def test_existing_layouts_are_unchanged():
    cls = [{"name": "classes", "kind": "classes"}, {"name": "logits", "kind": "logits"},
           {"name": "top", "kind": "top_k_classes", "k": 3}]
    assert mf.packed_output_layout(cls, 10) == [("classes", 0, 2, "int64"), ("logits", 2, 10, "float32"), ("top", 12, 3, "int32")]
    spans = [{"name": "start_logits", "kind": "start_logits"}, {"name": "span_scores", "kind": "span_scores", "k": 5}]
    assert mf.packed_output_layout(spans, 16) == [("span_scores", 0, 5, "float32"), ("start_logits", 5, 16, "float32")]


# ---------------------------------------------------------------------------------------- rejections ----
def test_encoder_kinds_need_a_graph_bundle(tmp_path):
    rng = np.random.default_rng(0)
    man = mf.write_mlp_bundle(str(tmp_path / "m" / "1"), [rng.standard_normal((8, 8)).astype(np.float32)],
                              [np.zeros(8, np.float32)], outputs=[{"name": "e", "kind": "cls_embedding"}])
    _refused(man, "encoder outputs need a graph bundle")
    aff = {"format": "tfsc-b200-v1", "template": "affine", "dtype": "float32", "weights_bytes": 512,
           "signature": {"input": "x", "outputs": NO_POOL}}
    _refused(aff, "encoder outputs need a graph bundle")


def test_encoder_kinds_need_embed_first():
    rn = mf.resnet50_manifest(image=32, classes=10, width=8, blocks=(1, 1, 1, 1), outputs=[{"name": "e", "kind": "mean_embedding"}])
    _refused(rn, "encoder outputs need a graph bundle whose first op is 'embed'")


def test_encoder_kinds_need_hidden_states_or_a_pooler():
    cls = mf.bert_manifest(seq=16, **SMALL, labels=2, inputs=mf.BERT_INPUTS, outputs=NO_POOL)       # pooler + classifier
    _refused(cls, "encoder outputs need a last op that writes the [16, 1, 64] hidden states, or a tanh pooler dense over "
                  "token 0 of the [16, 1, 64] hidden states the op before it writes (it writes [1, 1, 2])")
    qa = mf.bert_manifest(seq=16, **SMALL, inputs=mf.BERT_INPUTS, outputs=NO_POOL, head="span")
    _refused(qa, "(it writes [16, 1, 2])")
    man = _enc()
    man["ops"][-1]["act"] = "none"                                     # not a pooler
    _refused(man, "(it writes [1, 1, 64])")
    man = _enc()
    man["ops"][-1]["cout"] = 32                                        # a pooler of the wrong width
    man["weights_bytes"] += 1 << 20
    _refused(man, "(it writes [1, 1, 32])")
    man = _enc()
    extra = dict(man["ops"][-2], src=0, dst=2)                         # the op before the pooler does not write its source
    extra.pop("res")
    man["ops"].insert(-1, extra)
    _refused(man, "encoder outputs need a last op")


def test_pooled_output_needs_a_pooler():
    _refused(_enc(outputs=ALL, pooler=False), "pooled_output needs a bundle whose last op is the pooler")
    assert _check(_enc(outputs=NO_POOL, pooler=True))[0] > 0          # the other kinds are served with or without one


def test_encoder_kinds_do_not_mix():
    why = "encoder outputs (sequence_output, pooled_output, cls_embedding, mean_embedding) cannot be mixed with classification or span outputs"
    _refused(_enc(outputs=NO_POOL + [{"name": "logits", "kind": "logits"}]), why)
    _refused(_enc(outputs=[{"name": "start_logits", "kind": "start_logits"}] + NO_POOL), why)
    _refused(_enc(outputs=[{"name": "p", "kind": "probabilities"}, {"name": "c", "kind": "cls_embedding"}]), "('c' is cls_embedding)")


@pytest.mark.parametrize("case,why", [
    ("normalize_seq", "'normalize' belongs to cls_embedding and mean_embedding ('sequence_output' is sequence_output)"),
    ("normalize_pooled", "('pooled_output' is pooled_output)"),
    ("normalize_logits", "'normalize' belongs to cls_embedding and mean_embedding ('logits' is logits)"),
    ("normalize_int", "'mean_embedding' has a 'normalize' that is not true or false"),
    ("normalize_str", "'cls_embedding' has a 'normalize' that is not true or false"),
    ("k", "'k', 'max_answer_length' and 'sep_id' do not apply to encoder outputs ('mean_embedding' is mean_embedding)"),
    ("max_answer_length", "do not apply to encoder outputs ('sequence_output' is sequence_output)"),
    ("sep_id", "do not apply to encoder outputs ('cls_embedding' is cls_embedding)"),
    ("input_name", "'input_mask' is also an input name"),
])
def test_encoder_parameters(case, why):
    outs = {o["kind"]: dict(o) for o in ALL}
    if case == "normalize_seq":
        outs["sequence_output"]["normalize"] = True
    elif case == "normalize_pooled":
        outs["pooled_output"]["normalize"] = False
    elif case == "normalize_logits":
        man = mf.bert_manifest(seq=16, **SMALL, inputs=mf.BERT_INPUTS, outputs=[{"name": "logits", "kind": "logits", "normalize": True}])
        _refused(man, why)
        return
    elif case == "normalize_int":
        outs["mean_embedding"]["normalize"] = 1
    elif case == "normalize_str":
        outs["cls_embedding"]["normalize"] = "true"
    elif case == "k":
        outs["mean_embedding"]["k"] = 5
    elif case == "max_answer_length":
        outs["sequence_output"]["max_answer_length"] = 5
    elif case == "sep_id":
        outs["cls_embedding"]["sep_id"] = 102
    elif case == "input_name":
        outs["mean_embedding"]["name"] = "input_mask"
    _refused(_enc(outputs=list(outs.values())), why)


def _heads(hidden):  # a head width the attention kernels take at every S (d % 4 == 0, d <= 128)
    return next(h for h in range(1, hidden + 1) if hidden % h == 0 and (hidden // h) % 4 == 0 and hidden // h <= 128)


@pytest.mark.parametrize("seq,hidden", [(8193, 64), (16, 8200)])
def test_encoder_shape_limits(seq, hidden):
    man = _enc(seq=seq, hidden=hidden, heads=_heads(hidden), max_pos=max(512, seq), vocab=4, inter=8, outputs=NO_POOL, pooler=False)
    _refused(man, f"no encoder head kernel for S = {seq} and H = {hidden} (1 <= S <= 8192, 1 <= H <= 8192)")


def test_encoder_limits_accept_the_edges():
    for seq, hidden in ((1, 64), (512, 1024), (8192, 64), (16, 8192)):
        rc, got = _check(_enc(seq=seq, hidden=hidden, heads=_heads(hidden), max_pos=max(512, seq), vocab=4, inter=8, outputs=NO_POOL, pooler=False))
        assert rc > 0, got
    # S = 1: the pooler over the only token is still the pooler
    rc, got = _check(_enc(seq=1, outputs=ALL))
    assert rc > 0, got
    rc, got = _check(_enc(seq=8193, max_pos=8193, vocab=4, inter=8, outputs=None, pooler=False))  # no encoder outputs, no limit
    assert rc > 0, got


# ------------------------------------------------------------------------------------- fp64 reference ----
def test_embed_ref_hand_cases():
    h = np.array([[[1.0, 2.0], [3.0, 4.0], [100.0, -100.0]],
                  [[5.0, 6.0], [7.0, 8.0], [9.0, 10.0]]])
    mask = np.array([[1, 1, 0], [0, 0, 0]])
    ids = np.array([[101, 7, 0], [0, 0, 0]])
    m = er.mean_embedding(h, ids, mask)
    assert m[0].tolist() == [2.0, 3.0] and m[1].tolist() == [0.0, 0.0]        # a fully masked row is a zero vector
    assert er.normalize(m)[1].tolist() == [0.0, 0.0]                          # and normalising zero keeps it zero
    assert er.mean_embedding(h, ids)[0].tolist() == [2.0, 3.0]               # no mask: ids != 0
    # [PAD] at position 0 with a mask that keeps it: the mask decides
    assert er.mean_embedding(h, np.array([[0, 7, 8], [1, 1, 1]]), np.array([[1, 0, 0], [1, 1, 1]]))[0].tolist() == [1.0, 2.0]
    # a single token
    one = np.array([[[3.0, 4.0]]])
    assert er.mean_embedding(one, np.array([[5]]))[0].tolist() == [3.0, 4.0]
    assert er.mean_embedding(one, np.array([[5]]), norm=True)[0].tolist() == [0.6, 0.8]
    assert er.cls_embedding(one, norm=True)[0].tolist() == [0.6, 0.8] and er.cls_embedding(h)[1].tolist() == [5.0, 6.0]
    r = er.embed_ref(h, ids, mask, normalize_cls=True)
    assert np.allclose(np.linalg.norm(r["cls_embedding"], axis=1), 1.0) and np.array_equal(r["sequence_output"], h)


# ------------------------------------------------------------------------------------------ BertModel ----
@pytest.mark.parametrize("pooler", [True, False])
def test_encoder_bundles_match_transformers(pooler):
    S, B = 24, 4
    m = ee.hf_bert_model(61 + pooler, pooler=pooler, **SMALL)
    assert (m.pooler is not None) == pooler
    outs = ALL if pooler else NO_POOL
    # three inputs on sentence pairs: tests/bert_pair_ref.py
    man = _enc(seq=S, outputs=outs, pooler=pooler)
    blob = ee.export_bert_model(m, man)
    x = sr.qa_inputs(B, S, SMALL["vocab"], seed=8, sep_id=3)
    ref = ee.bert_model_reference(m, x["input_ids"], x["input_mask"], x["segment_ids"])
    y = pr.pair_forward(man, blob, x, np.float64)
    want = ref["pooler_output"] if pooler else ref["last_hidden_state"].reshape(B, -1)
    err = np.max(np.abs(y - want) / np.maximum(1.0, np.abs(want)))
    assert err <= 1e-6, err
    # one input (ids; the mask is ids != 0, segment 0): oracle.models.graph_forward
    man1 = _enc(seq=S, outputs=outs, pooler=pooler, inputs=None)
    blob1 = ee.export_bert_model(m, man1)
    ids = x["input_ids"] * x["input_mask"]
    ref1 = ee.bert_model_reference(m, ids)
    y1 = models.graph_forward(man1, blob1, ids, np.float64).reshape(B, -1)
    want1 = ref1["pooler_output"] if pooler else ref1["last_hidden_state"].reshape(B, -1)
    err = np.max(np.abs(y1 - want1) / np.maximum(1.0, np.abs(want1)))
    assert err <= 1e-6, err
    # the head's definitions, restated by embed_ref, are sentence-transformers' mean_pooling and F.normalize
    h = ref["last_hidden_state"]
    assert np.allclose(er.mean_embedding(h, x["input_ids"], x["input_mask"]), ref["mean"], rtol=1e-12, atol=1e-12)
    assert np.allclose(er.mean_embedding(h, x["input_ids"], x["input_mask"], norm=True), ref["mean_normalized"], rtol=1e-12, atol=1e-12)
    assert np.allclose(er.cls_embedding(h, norm=True), ref["cls_normalized"], rtol=1e-12, atol=1e-12)
