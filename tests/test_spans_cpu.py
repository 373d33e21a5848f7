"""Question-answering span outputs (start_logits, end_logits, span_starts, span_ends, span_scores), CPU side: the packed
layout of packed_output_layout against the loader's (tfsc_manifest_check), every loader rejection of a span bundle, the
brute-force span reference on hand-made rows, and a span bundle exported from transformers' BertForQuestionAnswering."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bert_pair_ref as pr  # noqa: E402
import span_ref as sr  # noqa: E402
import qa_export as qe  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=1, heads=4, inter=128, vocab=100, max_pos=512)


def spans(k=5, L=10, sep=None, names=("span_starts", "span_ends", "span_scores")):
    out = []
    for n, kind in zip(names, ("span_starts", "span_ends", "span_scores")):
        o = {"name": n, "kind": kind, "k": k, "max_answer_length": L}
        if sep is not None:
            o["sep_id"] = sep
        out.append(o)
    return out


LOGITS = [{"name": "start_logits", "kind": "start_logits"}, {"name": "end_logits", "kind": "end_logits"}]
FULL = LOGITS + spans()


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _qa(seq=16, outputs=FULL, inputs=mf.BERT_INPUTS, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.bert_manifest(seq=seq, **arch, inputs=inputs, outputs=outputs, head="span")


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


# ------------------------------------------------------------------------------------------- layout ----
OUTPUT_SETS = [
    FULL,
    LOGITS,
    spans(k=32, L=1),
    [{"name": "end_logits", "kind": "end_logits"}] + spans(k=1, L=384, sep=102, names=("b", "a", "c")),
    [{"name": "Start", "kind": "start_logits"}, {"name": "zé", "kind": "span_scores", "k": 20, "max_answer_length": 30}],
]


@pytest.mark.parametrize("seq", [1, 16, 384])
@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(which, seq):
    # max_answer_length <= S
    outs = [dict(o, max_answer_length=min(o["max_answer_length"], seq)) if "max_answer_length" in o else o
            for o in OUTPUT_SETS[which]]
    man = _qa(seq=seq, outputs=outs)
    rc, got = _check(man)
    assert rc > 0, got
    layout = mf.packed_output_layout(outs, seq)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    assert [o["kind"] for o in got["outputs"]] == [next(x["kind"] for x in outs if x["name"] == n) for n, *_ in layout]
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == seq
    assert got["head_k"] == next((o["k"] for o in outs if "k" in o), 0)
    assert [x[0] for x in layout] == sorted((o["name"] for o in outs), key=lambda s: s.encode())


def test_span_manifest_writer():
    man = _qa(seq=16)
    last = man["ops"][-1]
    assert last["op"] == "conv" and last["src"] == 0 and last["dst"] == -2 and last["cout"] == 2 and last["kh"] == 1
    assert not any(o["op"] == "dense" for o in man["ops"])            # no pooler, no classifier
    rc, got = _check(man)
    assert rc > 0 and got["out_dim"] == 16 + 16 + 5 + 5 + 5 and got["in_dim"] == 3 * 16
    # the same bundle with one output is served as [S, 1, 2] interleaved logits, as before
    rc, got = _check(_qa(seq=16, outputs=None))
    assert rc > 0 and got["out_dim"] == 32 and got["outputs"] == []
    # split_packed_rows cuts the span kinds with their dtypes
    layout = mf.packed_output_layout(FULL, 4)
    width = sum(w for _n, _o, w, _d in layout)
    words = np.zeros((2, width), np.uint32)
    for name, off, w, _dt in layout:
        if name == "span_starts":
            words[:, off:off + w] = np.uint32(0xFFFFFFFF)           # -1
        elif name == "start_logits":
            words[:, off:off + w] = np.float32([1.5, 2, 3, 4]).view(np.uint32)
    got = mf.split_packed_rows(words, FULL, 4)
    assert got["span_starts"].dtype == np.int32 and (got["span_starts"] == -1).all() and got["span_starts"].shape == (2, 5)
    assert got["span_ends"].dtype == np.int32 and got["span_scores"].dtype == np.float32
    assert got["start_logits"].tolist() == [[1.5, 2, 3, 4]] * 2


# ---------------------------------------------------------------------------------------- rejections ----
def test_span_kinds_need_a_graph_bundle(tmp_path):
    rng = np.random.default_rng(0)
    man = mf.write_mlp_bundle(str(tmp_path / "m" / "1"), [rng.standard_normal((8, 2)).astype(np.float32)],
                              [np.zeros(2, np.float32)], outputs=LOGITS)
    _refused(man, "span outputs need a graph bundle")
    aff = {"format": "tfsc-b200-v1", "template": "affine", "dtype": "float32", "weights_bytes": 512,
           "signature": {"input": "x", "outputs": spans()}}
    _refused(aff, "span outputs need a graph bundle")


def test_span_kinds_need_embed_and_type_ids():
    rn = mf.resnet50_manifest(image=32, classes=10, width=8, blocks=(1, 1, 1, 1), outputs=FULL)
    _refused(rn, "span outputs need a graph bundle whose first op is 'embed'")
    _refused(_qa(inputs=None), "span outputs need a 'type_ids' input")
    _refused(_qa(inputs=mf.BERT_INPUTS[:2]), "span outputs need a 'type_ids' input")


def test_span_kinds_need_per_token_start_end_logits():
    cls = mf.bert_manifest(seq=16, **SMALL, labels=2, inputs=mf.BERT_INPUTS, outputs=FULL)    # pooler + classifier: [2]
    _refused(cls, "span outputs need a last op that writes [16, 1, 2] start / end logits per token (it writes [1, 1, 2])")
    man = _qa()
    man["ops"][-1]["cout"] = 3
    _refused(man, "(it writes [16, 1, 3])")


def test_span_and_classification_kinds_do_not_mix():
    _refused(_qa(outputs=LOGITS + [{"name": "classes", "kind": "classes"}]), "cannot be mixed with classification outputs")
    _refused(_qa(outputs=[{"name": "logits", "kind": "logits"}] + LOGITS), "cannot be mixed with classification outputs")


@pytest.mark.parametrize("case,why", [
    ("no_k", "'span_starts' needs an integer 'k', the same for every span output"),
    ("k_float", "needs an integer 'k'"),
    ("k_mismatch", "'span_scores' needs an integer 'k', the same for every span output"),
    ("no_len", "'span_starts' needs an integer 'max_answer_length', the same for every span output"),
    ("len_mismatch", "'span_ends' needs an integer 'max_answer_length'"),
    ("sep_mismatch", "'span_ends' has a 'sep_id' that is not a token id >= 0 or differs"),
    ("sep_partial", "'span_ends' has a 'sep_id'"),
    ("sep_negative", "'span_starts' has a 'sep_id' that is not a token id >= 0"),
    ("k_on_logits", "'k', 'max_answer_length' and 'sep_id' belong to span_starts, span_ends and span_scores ('start_logits' is start_logits)"),
    ("sep_on_logits", "('end_logits' is end_logits)"),
])
def test_span_parameters(case, why):
    outs = [dict(o) for o in FULL]
    starts, ends, scores = outs[2], outs[3], outs[4]
    if case == "no_k":
        del starts["k"]
    elif case == "k_float":
        starts["k"] = 2.5
    elif case == "k_mismatch":
        scores["k"] = 6
    elif case == "no_len":
        del starts["max_answer_length"]
    elif case == "len_mismatch":
        ends["max_answer_length"] = 29
    elif case == "sep_mismatch":
        starts["sep_id"], ends["sep_id"], scores["sep_id"] = 102, 103, 102
    elif case == "sep_partial":
        starts["sep_id"] = 102
    elif case == "sep_negative":
        starts["sep_id"] = -1
    elif case == "k_on_logits":
        outs[0]["k"] = 5
    elif case == "sep_on_logits":
        outs[1]["sep_id"] = 102
    _refused(_qa(outputs=outs), why)


@pytest.mark.parametrize("seq,k,L", [(16, 0, 5), (16, 33, 5), (16, -1, 5), (16, 5, 0), (16, 5, 17), (4097, 5, 30)])
def test_span_shape_limits(seq, k, L):
    man = _qa(seq=seq, outputs=LOGITS + spans(k=k, L=L), max_pos=max(512, seq))
    _refused(man, f"no span kernel for S = {seq}, max_answer_length = {L} and k = {k} (1 <= S <= 4096, "
                  "1 <= max_answer_length <= S, 1 <= k <= 32)")


def test_span_limits_accept_the_edges():
    for seq, k, L in ((1, 1, 1), (4096, 32, 4096), (384, 20, 30)):
        rc, got = _check(_qa(seq=seq, outputs=spans(k=k, L=L), max_pos=max(512, seq)))
        assert rc > 0, got
    rc, got = _check(_qa(seq=4097, outputs=None, max_pos=4097))    # no span outputs: no span limit
    assert rc > 0, got
    _refused(_qa(seq=4097, outputs=LOGITS, max_pos=4097), "no span kernel for S = 4097")


def test_existing_wording_is_kept():
    cls = [{"name": "logits", "kind": "logits", "k": 3}]
    _refused(mf.bert_manifest(seq=16, **SMALL, inputs=mf.BERT_INPUTS, outputs=cls), "'k' belongs to the top-k outputs only")
    _refused(_qa(outputs=[{"name": "x", "kind": "softmax"}]), "unknown kind 'softmax'")
    _refused(_qa(outputs=FULL + [{"name": "e2", "kind": "end_logits"}]), "1 to 5 outputs")


# ------------------------------------------------------------------------------------- span reference ----
def test_span_ref_hand_cases():
    f32 = np.float32
    start = f32([0, 5, 1, 2])
    end = f32([0, 1, 4, 2])
    el = np.array([0, 1, 1, 1], bool)
    s, e, v = sr.span_ref(start, end, el, L=4, k=7)
    # candidates: (1,1)=6 (1,2)=9 (1,3)=7 (2,2)=5 (2,3)=3 (3,3)=4
    assert s.tolist() == [1, 1, 1, 2, 3, 2, -1] and e.tolist() == [2, 3, 1, 2, 3, 3, -1]
    assert v.tolist()[:6] == [9, 7, 6, 5, 4, 3] and v[6] == -sr.FLT_MAX and v.dtype == np.float32
    # L = 1: single tokens only
    s, e, v = sr.span_ref(start, end, el, L=1, k=3)
    assert s.tolist() == [1, 2, 3] and e.tolist() == [1, 2, 3] and v.tolist() == [6, 5, 4]
    # ties: equal scores go to the lower start, then the lower end
    s, e, v = sr.span_ref(f32([1, 1, 1]), f32([1, 1, 1]), np.ones(3, bool), L=3, k=6)
    assert list(zip(s.tolist(), e.tolist())) == [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)] and (v == 2).all()
    # no eligible token
    s, e, v = sr.span_ref(start, end, np.zeros(4, bool), L=4, k=2)
    assert s.tolist() == [-1, -1] and e.tolist() == [-1, -1] and (v == -sr.FLT_MAX).all()
    # NaN scores are not candidates
    s, e, v = sr.span_ref(f32([np.nan, 1]), f32([1, 1]), np.ones(2, bool), L=2, k=3)
    assert s.tolist() == [1, -1, -1] and e.tolist() == [1, -1, -1]
    # the sum is fp32: 1 + 2^-24 rounds to 1, so both spans tie and order by index
    s, e, v = sr.span_ref(f32([1, 1]), f32([2 ** -24, 0]), np.ones(2, bool), L=1, k=2)
    assert s.tolist() == [0, 1] and (v == 1).all()


def test_eligibility_and_sep_id():
    ids = np.array([101, 7, 102, 8, 9, 102, 0, 0])
    mask = np.array([1, 1, 1, 1, 0, 1, 0, 1])
    types = np.array([0, 0, 0, 1, 1, 1, 1, 1])
    assert sr.eligible(ids, mask, types).tolist() == [0, 0, 0, 1, 0, 1, 0, 1]
    assert sr.eligible(ids, mask, types, sep_id=102).tolist() == [0, 0, 0, 1, 0, 0, 0, 1]
    assert sr.eligible(ids, None, types, sep_id=102).tolist() == [0, 0, 0, 1, 1, 0, 0, 0]
    start = np.arange(8, dtype=np.float32)
    s, e, _v = sr.span_ref(start, start, sr.eligible(ids, mask, types, sep_id=102), L=8, k=4)
    assert list(zip(s.tolist(), e.tolist())) == [(7, 7), (3, 7), (3, 3), (-1, -1)]
    # row-batched form
    s2, e2, v2 = sr.span_ref(np.stack([start, start]), np.stack([start, start]),
                             np.stack([sr.eligible(ids, mask, types, 102)] * 2), L=8, k=4)
    assert s2.shape == (2, 4) and s2[1].tolist() == s.tolist()


def test_span_ref_matches_an_exhaustive_loop():
    rng = np.random.default_rng(3)
    for S, L, k in ((7, 3, 5), (13, 13, 32), (9, 1, 2)):
        st = np.round(rng.uniform(-2, 2, S)).astype(np.float32)       # ties
        en = np.round(rng.uniform(-2, 2, S)).astype(np.float32)
        el = rng.uniform(size=S) < 0.7
        cands = sorted(((-(float(np.float32(st[i] + en[j]))), i, j) for i in range(S) for j in range(i, min(S, i + L))
                        if el[i] and el[j]))[:k]
        s, e, v = sr.span_ref(st, en, el, L, k)
        assert [(i, j) for _v, i, j in cands] == [(a, b) for a, b in zip(s.tolist(), e.tolist()) if a >= 0]
        assert [-x for x, _i, _j in cands] == v[:len(cands)].tolist()


# ----------------------------------------------------------------------------- BertForQuestionAnswering ----
def test_qa_bundle_matches_transformers():
    S, B, sep = 48, 4, 3
    m = qe.hf_bert_qa(21, **SMALL)
    assert getattr(m, "qa_outputs", None) is not None and m.bert.pooler is None
    man = _qa(seq=S, outputs=FULL)
    blob = qe.export_bert_qa(m, man)
    x = sr.qa_inputs(B, S, SMALL["vocab"], seed=5, sep_id=sep)
    st64, en64 = qe.bert_qa_reference(m, x["input_ids"], x["input_mask"], x["segment_ids"])
    y = pr.pair_forward(man, blob, x, np.float64).reshape(B, S, 2)
    err = np.max(np.abs(y - np.stack([st64, en64], -1)) / np.maximum(1.0, np.abs(np.stack([st64, en64], -1))))
    assert err <= 1e-6, err
    # spans of the fp64 logits keep their order once rounded to fp32 where the score gaps are wide
    el = sr.eligible(x["input_ids"], x["input_mask"], x["segment_ids"], sep)
    assert el.any(axis=1).all() and not el[np.arange(B), (x["input_mask"].sum(1) - 1)].any()   # the final [SEP] is out
    s, e, v = sr.span_ref(st64.astype(np.float32), en64.astype(np.float32), el, L=30, k=5)
    assert (s >= 0).all() and (e >= s).all() and (e - s < 30).all() and (np.diff(v, axis=1) <= 0).all()
