"""Multi-output signatures (signature.outputs), CPU side: the Python writers and packed_output_layout against the loader's
own layout rule (tfsc_manifest_check), the loader's rejections, the writers' round trip, and oracle/wire.py on
PredictResponses that carry int64_val / int_val."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import wire

mf = t.modelformat
lib = t._lib.lib
FULL = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"},
        {"name": "classes", "kind": "classes"}, {"name": "top_k_classes", "kind": "top_k_classes", "k": 5},
        {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": 5}]
SMALL_BERT = dict(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, max_pos=64, labels=7)


def _check(man: dict):
    """(rc, parsed layout or the loader's message)"""
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _mlp_man(tmp_path, n_out, outputs, **kw):
    rng = np.random.default_rng(0)
    w = [rng.standard_normal((8, 16)).astype(np.float32), rng.standard_normal((16, n_out)).astype(np.float32)]
    b = [np.zeros(16, np.float32), np.zeros(n_out, np.float32)]
    return mf.write_mlp_bundle(str(tmp_path / "m" / "1"), w, b, outputs=outputs, **kw)


OUTPUT_SETS = [
    FULL,
    [{"name": "scores", "kind": "probabilities"}, {"name": "Label", "kind": "classes"}],     # "L" < "s": uppercase first
    [{"name": "b_top", "kind": "top_k_classes", "k": 3}, {"name": "a_p", "kind": "top_k_probabilities", "k": 3},
     {"name": "a", "kind": "logits"}],                                                       # "a" < "a_p" < "b_top"
    [{"name": "cls", "kind": "classes"}],
    [{"name": "zé", "kind": "logits"}, {"name": "zz", "kind": "classes"}],              # UTF-8 0xC3 sorts after "z"
]


@pytest.mark.parametrize("n", [5, 13, 1001])
@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(tmp_path, which, n):
    outs = OUTPUT_SETS[which]
    man = _mlp_man(tmp_path, n, outs)
    rc, got = _check(man)
    assert rc > 0, got
    layout = mf.packed_output_layout(outs, n)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == n
    # the packed order is byte-wise sorted UTF-8, not code-point or locale order
    assert [x[0] for x in layout] == sorted((o["name"] for o in outs), key=lambda s: s.encode())


def test_graph_writers_match_loader():
    man = mf.bert_manifest(**SMALL_BERT, inputs=mf.BERT_INPUTS, outputs=FULL)
    rc, got = _check(man)
    assert rc > 0, got
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == mf.packed_output_layout(FULL, 7)
    assert got["out_dim"] == 7 + 7 + 2 + 5 + 5 and got["in_dim"] == 3 * 16
    assert "output" not in man["signature"] and man["signature"]["outputs"] == FULL
    rn = mf.resnet50_manifest(image=32, classes=10, width=8, blocks=(1, 1, 1, 1), outputs=FULL[:3])
    rc, got = _check(rn)
    assert rc > 0, got
    assert [(o["name"], o["offset"], o["width"]) for o in got["outputs"]] == [("classes", 0, 2), ("logits", 2, 10), ("probabilities", 12, 10)]
    # without outputs the manifests are what they were: one output, out_dim = the logits width
    assert mf.resnet50_manifest(image=32, classes=10, width=8, blocks=(1, 1, 1, 1))["signature"] == {"input": "x", "output": "y"}
    rc, got = _check(mf.bert_manifest(**SMALL_BERT))
    assert rc > 0 and got["out_dim"] == 7 and got["outputs"] == []


def test_manifest_round_trips_through_writer(tmp_path):
    man = _mlp_man(tmp_path, 40, FULL, input_name="features")
    with open(tmp_path / "m" / "1" / "tfsc_model.json") as f:
        on_disk = json.load(f)
    assert on_disk == man and on_disk["signature"] == {"input": "features", "outputs": FULL}
    assert os.path.getsize(tmp_path / "m" / "1" / "weights.bin") == man["weights_bytes"]
    rc, got = _check(on_disk)
    assert rc > 0 and got["head_n"] == 40 and got["head_k"] == 5


def test_split_packed_rows():
    outs, n, rows = FULL, 4, 3
    layout = mf.packed_output_layout(outs, n)
    width = sum(w for _n, _o, w, _d in layout)
    words = np.zeros((rows, width), np.uint32)
    logits = np.arange(rows * n, dtype=np.float32).reshape(rows, n)
    for name, off, w, _dt in layout:
        if name == "classes":
            words[:, off] = [7, 8, 9]                      # low word; the high word stays 0
        elif name == "logits":
            words[:, off:off + w] = logits.view(np.uint32)
        elif name == "top_k_classes":
            words[:, off:off + w] = np.arange(w, dtype=np.uint32)
    got = mf.split_packed_rows(words.view(np.float32), outs, n)
    assert got["classes"].dtype == np.int64 and got["classes"].tolist() == [7, 8, 9]
    assert np.array_equal(got["logits"], logits) and got["top_k_classes"].dtype == np.int32
    assert got["top_k_classes"].tolist() == [list(range(5))] * rows


def _bad(tmp_path, outs, n=10, **kw):
    rc, msg = _check(_mlp_man(tmp_path, n, outs, **kw))
    assert rc == t._lib.E_INVALID, msg
    return msg


def test_loader_rejections(tmp_path):
    P = {"name": "p", "kind": "probabilities"}
    assert "unknown kind 'softmax'" in _bad(tmp_path, [{"name": "p", "kind": "softmax"}])
    assert "duplicate name 'p'" in _bad(tmp_path, [P, {"name": "p", "kind": "classes"}])
    assert "duplicate kind 'probabilities'" in _bad(tmp_path, [P, {"name": "q", "kind": "probabilities"}])
    assert "needs an integer 'k'" in _bad(tmp_path, [{"name": "t", "kind": "top_k_classes"}])
    assert "needs an integer 'k'" in _bad(tmp_path, [{"name": "t", "kind": "top_k_classes", "k": 3},
                                                     {"name": "u", "kind": "top_k_probabilities", "k": 4}])
    assert "'k' belongs to the top-k outputs" in _bad(tmp_path, [{"name": "p", "kind": "probabilities", "k": 3}])
    for n, k in ((10, 0), (10, 11), (64, 33), (32769, 1)):
        assert "no head kernel" in _bad(tmp_path, [{"name": "t", "kind": "top_k_classes", "k": k}], n=n)
    assert "1 to 5 outputs" in _bad(tmp_path, [])
    assert "1 to 5 outputs" in _bad(tmp_path, FULL + [{"name": "x2", "kind": "logits"}])
    assert "also an input name" in _bad(tmp_path, [{"name": "x", "kind": "logits"}])
    # 'outputs' together with 'output'
    man = _mlp_man(tmp_path, 10, [P])
    man["signature"]["output"] = "y"
    rc, msg = _check(man)
    assert rc == t._lib.E_INVALID and "mutually exclusive" in msg
    # an affine bundle has no logits row
    aff = mf.write_affine_bundle(str(tmp_path / "a" / "1"), 0.5, 2.0)
    aff["signature"] = {"input": "x", "outputs": [P]}
    rc, msg = _check(aff)
    assert rc == t._lib.E_INVALID and "mlp or graph" in msg
    # a graph whose response is not one vector per row (a conv feature map)
    g = mf._graph_manifest([4, 4, 3], [{"op": "conv", "src": -1, "dst": -2, "h": 4, "w": 4, "c": 3, "kh": 1, "kw": 1,
                                        "stride": 1, "pad": 0, "cout": 8, "act": "none"}], 1, outputs=[P])
    rc, msg = _check(g)
    assert rc == t._lib.E_INVALID and "rank 3" in msg
    # the multi-input BERT bundle: an output named like one of its inputs
    rc, msg = _check(mf.bert_manifest(**SMALL_BERT, inputs=mf.BERT_INPUTS, outputs=[{"name": "input_mask", "kind": "classes"}]))
    assert rc == t._lib.E_INVALID and "also an input name" in msg


def _varints(vals):
    out = b""
    for v in vals:
        v &= (1 << 64) - 1
        while v >= 0x80:
            out += bytes([(v & 0x7F) | 0x80])
            v >>= 7
        out += bytes([v])
    return out


def _ld(field, payload):
    return _varints([(field << 3) | 2, len(payload)]) + payload


def test_oracle_decodes_int64_and_int_val():
    """The bytes the server writes for a multi-output response: float_val packed (5), int64_val packed (10), int_val packed
    (7), the map in sorted name order."""
    def tensor(dtype, shape, field, payload):
        sh = b"".join(_ld(2, _varints([(1 << 3) | 0, d])) for d in shape)
        return _varints([(1 << 3) | 0, dtype]) + _ld(2, sh) + _ld(field, payload)

    probs = np.array([[0.25, 0.75], [0.5, 0.5]], np.float32)
    body = b""
    for name, tb in (("classes", tensor(9, [2], 10, _varints([1, 0]))),
                     ("probabilities", tensor(1, [2, 2], 5, probs.astype("<f4").tobytes())),
                     ("top_k_classes", tensor(3, [2, 2], 7, _varints([1, 0, 0, 1])))):
        body += _ld(1, _ld(1, name.encode()) + _ld(2, tb))
    body += _ld(2, wire.encode_model_spec("m", 3, "serving_default"))
    spec, outs = wire.decode_predict_response(body)
    assert spec[0] == "m" and list(outs) == ["classes", "probabilities", "top_k_classes"]
    assert outs["classes"].dtype == np.int64 and outs["classes"].tolist() == [1, 0]
    assert outs["top_k_classes"].dtype == np.int32 and outs["top_k_classes"].tolist() == [[1, 0], [0, 1]]
    assert np.array_equal(outs["probabilities"], probs)
    assert struct.unpack("<f", outs["probabilities"][0, 0].tobytes())[0] == 0.25
