"""Fill-mask (masked-language-model) outputs -- masked_positions, masked_top_k_ids, masked_top_k_probabilities,
masked_top_k_logits -- CPU side: every loader rejection of a fill-mask bundle (tfsc_manifest_check), packed_output_layout
against the loader's layout, the manifest writer, the fp64 reference on hand cases, and a BertForMaskedLM export through
the CPU reference within 1e-6 of transformers fp64."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mlm_export as me  # noqa: E402
import mlm_ref as mr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=1, heads=4, inter=128, vocab=100, max_pos=512)
MASK_ID = 4
K = 5
ALL = [{"name": "masked_positions", "kind": "masked_positions"}] + \
      [{"name": k, "kind": k, "k": K} for k in mf.MLM_OUTPUT_KINDS[1:]]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _mlm(seq=16, slots=3, outputs=ALL, inputs=mf.BERT_INPUTS, mask_token_id=MASK_ID, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.bert_manifest(seq=seq, **arch, inputs=inputs, outputs=outputs, head="mlm", slots=slots, mask_token_id=mask_token_id)


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


# ------------------------------------------------------------------------------------------- layout ----
OUTPUT_SETS = [
    ALL,
    [{"name": "masked_positions", "kind": "masked_positions"}],
    [{"name": "ids", "kind": "masked_top_k_ids", "k": 1}],
    [{"name": "z", "kind": "masked_top_k_logits", "k": 32}, {"name": "a", "kind": "masked_top_k_probabilities", "k": 32}],
    [{"name": "Pos", "kind": "masked_positions"}, {"name": "top", "kind": "masked_top_k_ids", "k": 3}],
]


@pytest.mark.parametrize("slots", [1, 3, 16])
@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(which, slots):
    outs = OUTPUT_SETS[which]
    rc, got = _check(_mlm(seq=16, slots=slots, outputs=outs))
    assert rc > 0, got
    layout = mf.packed_output_layout(outs, slots)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    assert [o["kind"] for o in got["outputs"]] == [next(x["kind"] for x in outs if x["name"] == n) for n, *_ in layout]
    k = next((o["k"] for o in outs if "k" in o), 0)
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == slots and got["head_k"] == k
    assert got["in_dim"] == 3 * 16


def test_mlm_manifest_writer():
    man = _mlm(seq=16, slots=3, vocab=100)
    g, dense, ln, dec = man["ops"][-4:]
    assert g == dict(g, op="mask_gather", src=0, dst=1, h=16, w=1, c=64, slots=3, mask_token_id=MASK_ID)
    assert man["ops"][-5]["op"] == "layernorm" and man["ops"][-5]["dst"] == 0
    assert dense["h"] == 3 and dense["act"] == "gelu" and dense["cout"] == 64 and ln["h"] == 3
    assert dec["h"] == 3 and dec["cout"] == 128 and dec["dst"] == -2              # Vp: 100 rounded up to a multiple of 32
    assert _mlm(vocab=30522)["ops"][-1]["cout"] == 30528
    # split_packed_rows gives the top-k kinds as [rows, M, k]
    M = 3
    layout = mf.packed_output_layout(ALL, M)
    width = sum(w for _n, _o, w, _d in layout)
    words = np.arange(2 * width, dtype=np.float32).reshape(2, width)
    got = mf.split_packed_rows(words, ALL, M)
    off = dict((n, o) for n, o, _w, _d in layout)
    assert got["masked_top_k_ids"].shape == (2, M, K) and got["masked_top_k_ids"].dtype == np.int32
    assert got["masked_positions"].shape == (2, M) and got["masked_positions"].dtype == np.int32
    assert got["masked_top_k_logits"][1, 2, 4] == words[1, off["masked_top_k_logits"] + 2 * K + 4]


def test_existing_layouts_are_unchanged():
    enc = [{"name": "sequence_output", "kind": "sequence_output"}, {"name": "cls", "kind": "cls_embedding"}]
    assert mf.packed_output_layout(enc, 4, 3) == [("cls", 0, 4, "float32"), ("sequence_output", 4, 12, "float32")]
    cls = [{"name": "classes", "kind": "classes"}, {"name": "top", "kind": "top_k_classes", "k": 3}]
    assert mf.packed_output_layout(cls, 10) == [("classes", 0, 2, "int64"), ("top", 2, 3, "int32")]


# ---------------------------------------------------------------------------------------- rejections ----
def test_mlm_kinds_need_a_graph_bundle(tmp_path):
    rng = np.random.default_rng(0)
    man = mf.write_mlp_bundle(str(tmp_path / "m" / "1"), [rng.standard_normal((8, 8)).astype(np.float32)],
                              [np.zeros(8, np.float32)], outputs=[{"name": "p", "kind": "masked_positions"}])
    _refused(man, "fill-mask outputs need a graph bundle")
    aff = {"format": "tfsc-b200-v1", "template": "affine", "dtype": "float32", "weights_bytes": 512,
           "signature": {"input": "x", "outputs": ALL}}
    _refused(aff, "fill-mask outputs need a graph bundle")


def test_mlm_kinds_need_embed_first():
    rn = mf.resnet50_manifest(image=32, classes=10, width=8, blocks=(1, 1, 1, 1), outputs=[{"name": "p", "kind": "masked_positions"}])
    _refused(rn, "fill-mask outputs need a graph bundle whose first op is 'embed'")


def test_mlm_kinds_need_one_mask_gather():
    man = mf.bert_manifest(seq=16, **SMALL, inputs=mf.BERT_INPUTS, outputs=ALL, head="encoder", pooler=False)
    _refused(man, "fill-mask outputs need exactly one mask_gather op (the bundle has 0)")
    man = _mlm()
    man["ops"].insert(-3, dict(man["ops"][-4], src=0, dst=3))         # a second gather
    _refused(man, "fill-mask outputs need exactly one mask_gather op (the bundle has 2)")


def test_mask_gather_needs_fill_mask_outputs():
    why = "a mask_gather op needs fill-mask outputs"
    _refused(_mlm(outputs=None), why)
    _refused(_mlm(outputs=[{"name": "logits", "kind": "logits"}]), why)
    _refused(_mlm(outputs=[{"name": "s", "kind": "sequence_output"}]), why)


def test_gather_source_and_slots():
    man = _mlm()
    man["ops"][-4]["h"], man["ops"][-4]["c"] = 32, 32                   # [32, 1, 32]: the element count, not the shape
    man["ops"][-3]["c"] = 32
    _refused(man, "the mask_gather op needs the [16, 1, 64] hidden states of a scratch buffer (it reads [32, 1, 32] of buffer 0)")
    for slots in (0, 17):
        man = _mlm()
        man["ops"][-4]["slots"] = slots
        _refused(man, f"mask_gather needs 1 <= slots <= h (slots = {slots}, h = 16)")
    assert _check(_mlm(slots=16))[0] > 0 and _check(_mlm(slots=1))[0] > 0


@pytest.mark.parametrize("tok", [0, -1, 100, 1000])
def test_mask_token_id_range(tok):
    _refused(_mlm(mask_token_id=tok), f"mask_token_id {tok} is not a token id in [1, 100)")


def test_last_op_writes_the_slot_logits():
    man = _mlm()
    man["ops"][-1]["cout"] = 96                                          # Vp < vocab
    _refused(man, "fill-mask outputs need a last op that writes [3, 1, Vp] logits, Vp >= 100 (it writes [3, 1, 96])")
    man = _mlm()
    man["ops"] = man["ops"][:-1]
    man["ops"][-1]["dst"] = -2                                           # ends in the transform's LayerNorm: [3, 1, 64]
    _refused(man, "(it writes [3, 1, 64])")
    assert _check(_mlm(vocab=96))[0] > 0                                 # Vp = vocab is fine


def test_mlm_kinds_do_not_mix():
    why = ("fill-mask outputs (masked_positions, masked_top_k_ids, masked_top_k_probabilities, masked_top_k_logits) cannot be"
           " mixed with classification, span or encoder outputs")
    for other in ({"name": "logits", "kind": "logits"}, {"name": "start_logits", "kind": "start_logits"},
                  {"name": "cls", "kind": "cls_embedding"}, {"name": "top", "kind": "top_k_classes", "k": 5}):
        _refused(_mlm(outputs=ALL + [other]), why)
        _refused(_mlm(outputs=[other] + ALL), why)


@pytest.mark.parametrize("case,why", [
    ("k_missing", "'masked_top_k_ids' needs an integer 'k' >= 1, the same for every fill-mask top-k output"),
    ("k_mismatch", "'masked_top_k_logits' needs an integer 'k' >= 1, the same for every fill-mask top-k output"),
    ("k_float", "'masked_top_k_probabilities' needs an integer 'k'"),
    ("k_negative_first", "'masked_top_k_ids' needs an integer 'k' >= 1"),
    ("k_zero", "'masked_top_k_ids' needs an integer 'k' >= 1"),
    ("k_on_positions", "'k' belongs to masked_top_k_ids, masked_top_k_probabilities and masked_top_k_logits ('masked_positions' is"
                       " masked_positions)"),
    ("normalize", "'normalize', 'max_answer_length' and 'sep_id' do not apply to fill-mask outputs ('masked_top_k_ids' is"
                  " masked_top_k_ids)"),
    ("max_answer_length", "do not apply to fill-mask outputs ('masked_positions' is masked_positions)"),
    ("sep_id", "do not apply to fill-mask outputs ('masked_top_k_logits' is masked_top_k_logits)"),
    ("input_name", "'input_mask' is also an input name"),
])
def test_mlm_parameters(case, why):
    outs = {o["kind"]: dict(o) for o in ALL}
    if case == "k_missing":
        del outs["masked_top_k_ids"]["k"]
    elif case == "k_mismatch":
        outs["masked_top_k_logits"]["k"] = K + 1
    elif case == "k_float":
        outs["masked_top_k_probabilities"]["k"] = 2.5
    elif case == "k_negative_first":                                  # a negative k first, then a valid one: still refused
        outs["masked_top_k_ids"]["k"] = -3
    elif case == "k_zero":
        outs = {k_: dict(o, k=0) if "k" in o else o for k_, o in outs.items()}
    elif case == "k_on_positions":
        outs["masked_positions"]["k"] = K
    elif case == "normalize":
        outs["masked_top_k_ids"]["normalize"] = True
    elif case == "max_answer_length":
        outs["masked_positions"]["max_answer_length"] = 5
    elif case == "sep_id":
        outs["masked_top_k_logits"]["sep_id"] = 102
    elif case == "input_name":
        outs["masked_positions"]["name"] = "input_mask"
    _refused(_mlm(outputs=list(outs.values())), why)


@pytest.mark.parametrize("vocab,k,ok", [(1, 1, True), (32768, 32, True), (32769, 5, False), (100, 33, False),
                                        (4, 5, False), (5, 5, True)])
def test_fill_mask_limits(vocab, k, ok):
    outs = [{"name": "ids", "kind": "masked_top_k_ids", "k": k}]
    man = _mlm(vocab=vocab, hidden=32, inter=8, outputs=outs, mask_token_id=min(MASK_ID, vocab - 1) if vocab > 1 else 1)
    rc, got = _check(man)
    if ok and vocab > 1:
        assert rc > 0, got
    elif vocab == 1:                                                   # no token id is in [1, 1)
        assert rc == t._lib.E_INVALID and "is not a token id in [1, 1)" in got
    else:
        assert rc == t._lib.E_INVALID and "no fill-mask kernels for S = 16, H = 32, M = 3" in got, got


def test_positions_alone_need_no_k():
    rc, got = _check(_mlm(outputs=[{"name": "p", "kind": "masked_positions"}], vocab=40000 // 2))
    assert rc > 0 and got["head_k"] == 0 and got["out_dim"] == 3


# ------------------------------------------------------------------------------------- fp64 reference ----
def test_reference_hand_cases():
    h = np.arange(2 * 5 * 2, dtype=np.float64).reshape(2, 5, 2)
    ids = np.array([[7, 9, 7, 7, 1], [1, 2, 3, 4, 5]])
    mask = np.array([[1, 1, 0, 1, 1], [1, 1, 1, 1, 1]])
    pos, gat = mr.mask_gather_ref(h, ids, mask, 7, 2)
    assert pos.tolist() == [[0, 3], [-1, -1]]                          # position 2 is masked out; row 1 has no [MASK]
    assert gat[0].tolist() == [h[0, 0].tolist(), h[0, 3].tolist()] and (gat[1] == 0).all()
    pos, _ = mr.mask_gather_ref(h, ids, None, 7, 2)
    assert pos.tolist() == [[0, 2], [-1, -1]]                          # no mask input: first M in ascending p
    logits = np.array([[[1.0, 3.0, 3.0, -1.0, 50.0], [0.0, 0.0, 0.0, 0.0, 0.0]]], np.float32)
    ids_, probs, vals = mr.top_k_ref(logits, np.array([[4, -1]]), 4, 3)
    assert ids_.tolist() == [[[1, 2, 0], [-1, -1, -1]]]               # ties to the lower id; the padding column 4 is ignored
    e = np.exp(np.array([1.0, 3.0, 3.0, -1.0]) - 3.0)
    assert np.allclose(probs[0, 0], e[[1, 2, 0]] / e.sum(), rtol=1e-15) and probs[0, 1].tolist() == [0, 0, 0]
    assert vals[0, 0].tolist() == [3.0, 3.0, 1.0] and (vals[0, 1] == -mr.FLT_MAX).all()


# -------------------------------------------------------------------------------------- BertForMaskedLM ----
@pytest.mark.parametrize("inputs", [mf.BERT_INPUTS, None])
def test_mlm_bundle_matches_transformers(inputs):
    S, B, M = 24, 4, 3
    m = me.hf_mlm_model(91, **SMALL)
    man = _mlm(seq=S, slots=M, inputs=inputs)
    blob = me.export_mlm_model(m, man)
    x = mr.mlm_inputs(B, S, SMALL["vocab"], 2, seed=5, mask_token_id=MASK_ID)
    if inputs is None:                                                 # one input: the mask is ids != 0, segment 0
        xin = x["input_ids"]
        ref = me.mlm_reference(m, xin)
        mask = None
    else:
        xin = x
        ref = me.mlm_reference(m, x["input_ids"], x["input_mask"], x["segment_ids"])
        mask = x["input_mask"]
    pos, logits = mr.mlm_forward(man, blob, xin, np.float64)
    want_pos, _ = mr.mask_gather_ref(np.zeros((B, S, 1)), x["input_ids"], mask, MASK_ID, M)
    assert pos.tolist() == want_pos.tolist() and (pos >= 0).any() and (pos < 0).any()
    V = SMALL["vocab"]
    assert logits.shape == (B, M, 128) and not logits[:, :, V:][pos >= 0].any()     # zero padding columns, zero bias
    for r in range(B):
        for s in range(M):
            if pos[r, s] < 0:
                continue
            want = ref[r, pos[r, s]]
            err = np.max(np.abs(logits[r, s, :V] - want) / np.maximum(1.0, np.abs(want)))
            assert err <= 1e-6, (r, s, err)
    ids, _p, _v = mr.top_k_ref(logits, pos, V, K)
    ids_hf, _p, _v = mr.top_k_ref(np.stack([ref[r, np.maximum(pos[r], 0)] for r in range(B)]), pos, V, K)
    assert ids.tolist() == ids_hf.tolist()
