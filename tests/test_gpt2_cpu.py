"""GPT-2 next-token bundles, CPU side: every loader refusal of the new fields, op and output kinds (tfsc_manifest_check),
the writer at GPT-2 small / medium / large shapes, packed_output_layout against the loader's layout, and a seeded
GPT2LMHeadModel export through the fp64 reference within 1e-6 of transformers fp64."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpt2_export as ge  # noqa: E402
import gpt2_ref as gr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=64)
K = 5
ALL = [{"name": "next_token_position", "kind": "next_token_position"}] + \
      [{"name": k, "kind": k, "k": K} for k in mf.NEXT_TOKEN_OUTPUT_KINDS[1:]]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _gpt2(seq=16, outputs=ALL, inputs=mf.GPT2_INPUTS, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=outputs)


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


def _op(man, kind, i=0):
    return [o for o in man["ops"] if o["op"] == kind][i]


# ------------------------------------------------------------------------------------------- writer / layout ----
@pytest.mark.parametrize("arch", [(768, 12, 12), (1024, 24, 16), (1280, 36, 20)], ids=["small", "medium", "large"])
def test_writer_at_gpt2_shapes(arch):
    hidden, layers, heads = arch
    man = mf.gpt2_manifest(seq=1024, hidden=hidden, layers=layers, heads=heads, outputs=ALL)
    rc, got = _check(man)
    assert rc > 0, got
    assert got["head_n"] == 50257 and got["head_k"] == K and got["in_dim"] == 1024
    assert man["ops"][-1]["cout"] == 50272 and len(man["ops"]) == 1 + 7 * layers + 3
    assert sum(o.get("causal", False) for o in man["ops"]) == layers
    assert sum(o.get("act") == "gelu_tanh" for o in man["ops"]) == layers
    rc, got = _check(mf.gpt2_manifest(seq=1024, hidden=hidden, layers=1, heads=heads, inputs=mf.GPT2_INPUTS, outputs=ALL))
    assert rc > 0 and got["in_dim"] == 2 * 1024, got


OUTPUT_SETS = [
    ALL,
    [{"name": "next_token_position", "kind": "next_token_position"}],
    [{"name": "ids", "kind": "next_token_top_k_ids", "k": 1}],
    [{"name": "z", "kind": "next_token_top_k_logits", "k": 32}, {"name": "a", "kind": "next_token_top_k_probabilities", "k": 32}],
    [{"name": "Pos", "kind": "next_token_position"}, {"name": "top", "kind": "next_token_top_k_ids", "k": 3}],
]


@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(which):
    outs = OUTPUT_SETS[which]
    rc, got = _check(_gpt2(outputs=outs))
    assert rc > 0, got
    layout = mf.packed_output_layout(outs, 1000)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    k = next((o["k"] for o in outs if "k" in o), 0)
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == 1000 and got["head_k"] == k
    words = np.arange(3 * got["out_dim"], dtype=np.int32).reshape(3, -1)
    split = mf.split_packed_rows(words, outs, 1000)
    kinds = {o["name"]: o["kind"] for o in outs}
    for name, off, width, _dt in layout:
        assert split[name].shape == ((3,) if kinds[name] == "next_token_position" else (3, width))
        assert np.array_equal(split[name].reshape(3, -1).view(np.int32), words[:, off:off + width])


def test_existing_bundles_are_unchanged():
    """a BERT bundle says nothing of causal / norm, so it keeps attending to every key and its LayerNorm embedding"""
    man = mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100)
    assert not any("causal" in o or "norm" in o for o in man["ops"])
    assert _check(man)[0] > 0


# ---------------------------------------------------------------------------------------------- refusals ----
def test_causal_must_be_a_bool_on_attention():
    man = _gpt2()
    _op(man, "attention")["causal"] = 1
    _refused(man, "attention has a 'causal' that is not true or false")
    man = _gpt2()
    _op(man, "conv")["causal"] = True
    _refused(man, "conv takes no 'causal' (attention only)")


def test_causal_needs_the_tiled_kernels():
    man = _gpt2(hidden=72, heads=12)                                   # d = 6
    _refused(man, "no causal attention kernel for S = 16, hidden 72, 12 heads")
    man = _gpt2(hidden=72, heads=12)
    _op(man, "attention")["causal"] = False                            # the row kernel serves the non-causal op
    for o in man["ops"]:
        o.pop("causal", None)
    assert _check(man)[0] > 0


def test_norm_must_be_a_bool_on_embed():
    man = _gpt2()
    man["ops"][0]["norm"] = "no"
    _refused(man, "embed has a 'norm' that is not true or false")
    man = _gpt2()
    _op(man, "layernorm")["norm"] = False
    _refused(man, "layernorm takes no 'norm' (embed only)")


def test_norm_false_reads_no_type_ids():
    man = _gpt2(inputs=mf.GPT2_INPUTS + [{"name": "segment_ids", "role": "type_ids"}])
    _refused(man, "signature.inputs: an embed op with norm false reads no type_ids input")


def test_norm_false_reads_only_word_and_position_tables():
    man = _gpt2()
    man["ops"][0]["pos_offset"] = man["weights_bytes"]
    _refused(man, "bad embed op")


def test_gelu_tanh_is_a_gemm_activation():
    man = _gpt2()
    assert _check(man)[0] > 0
    dw = {"format": "tfsc-b200-v1", "template": "graph", "dtype": "float32", "input_shape": [8, 8, 16], "n_buffers": 1,
          "weights_bytes": 4096, "ops": [{"op": "depthwise_conv", "src": -1, "dst": -2, "h": 8, "w": 8, "c": 16, "kh": 3,
                                          "kw": 3, "pad": 1, "act": "gelu_tanh"}]}
    _refused(dw, "depthwise_conv act 'gelu_tanh' is not none, relu, relu6, silu or sigmoid")


def test_last_token_needs_next_token_outputs():
    man = _gpt2(outputs=None)
    _refused(man, "graph manifest: a last_token op needs next-token outputs")


def test_one_last_token():
    man = _gpt2()
    lt = _op(man, "last_token")
    man["ops"].insert(man["ops"].index(lt), dict(lt, dst=2))
    _refused(man, "next-token outputs need exactly one last_token op (the bundle has 2)")


def test_last_token_source():
    man = _gpt2()
    lt = _op(man, "last_token")
    lt["h"], lt["w"] = 8, 2                                            # the same element count, not [S, 1, H]
    _refused(man, "the last_token op needs the [16, 1, 64] hidden states of a scratch buffer (it reads [8, 2, 64] of buffer 0)")


def test_last_op_writes_the_vocabulary_row():
    man = _gpt2()
    man["ops"][-1]["cout"] = 992
    _refused(man, "next-token outputs need a last op that writes [1, 1, Vp] logits, Vp >= 1000")


@pytest.mark.parametrize("vocab,k,ok", [(57344, 32, True), (57345, 1, False), (50257, 32, True), (50257, 33, False),
                                        (4, 4, True), (4, 5, False)])
def test_next_token_limits(vocab, k, ok):
    outs = [{"name": "ids", "kind": "next_token_top_k_ids", "k": k}]
    man = _gpt2(seq=4, layers=1, vocab=vocab, outputs=outs)
    if ok:
        assert _check(man)[0] > 0
    else:
        _refused(man, f"no next-token head for vocab = {vocab} and k = {k} (1 <= vocab <= 57344, 1 <= k <= min(vocab, 32))")


def test_next_token_kinds_do_not_mix():
    for other in ({"name": "l", "kind": "logits"}, {"name": "m", "kind": "masked_positions"}):
        _refused(_gpt2(outputs=ALL[:1] + [other]), "next-token outputs (next_token_position, next_token_top_k_ids,")
        _refused(_gpt2(outputs=[other] + ALL[:1]), "cannot be mixed with classification, span, encoder or fill-mask outputs")


def test_next_token_needs_a_graph_bundle(tmp_path):
    man = mf.write_mlp_bundle(str(tmp_path / "m" / "1"), [np.zeros((4, 4), np.float32)], [np.zeros(4, np.float32)], outputs=ALL[:1])
    _refused(man, "signature.outputs: next-token outputs need a graph bundle")


@pytest.mark.parametrize("entry,why", [
    ({"name": "a", "kind": "next_token_top_k_ids"}, "'a' needs an integer 'k' >= 1, the same for every next-token top-k output"),
    ({"name": "a", "kind": "next_token_top_k_ids", "k": 0}, "needs an integer 'k' >= 1"),
    ({"name": "a", "kind": "next_token_top_k_ids", "k": 4}, "needs an integer 'k' >= 1"),             # K elsewhere
    ({"name": "a", "kind": "next_token_position", "k": K}, "'k' belongs to next_token_top_k_ids"),
    ({"name": "a", "kind": "next_token_top_k_ids", "k": K, "normalize": True}, "do not apply to next-token outputs"),
    ({"name": "a", "kind": "next_token_top_k_ids", "k": K, "max_answer_length": 3}, "do not apply to next-token outputs"),
    ({"name": "a", "kind": "next_token_top_k_ids", "k": K, "sep_id": 3}, "do not apply to next-token outputs"),
    ({"name": "a", "kind": "next_token_top_k"}, "unknown next-token kind 'next_token_top_k' (next_token_position,"),
])
def test_next_token_fields(entry, why):
    outs = [{"name": "z", "kind": "next_token_top_k_logits", "k": K}, entry]
    _refused(_gpt2(outputs=outs), why)


def test_unknown_kind_message_is_unchanged():
    got = _refused(_gpt2(outputs=[{"name": "a", "kind": "nope"}]), "unknown kind 'nope' (logits,")
    assert got.endswith("masked_top_k_logits)")


# ----------------------------------------------------------------------------------------- fp64 reference ----
def test_reference_hand_cases():
    rng = np.random.default_rng(0)
    qkv = rng.standard_normal((2, 5, 3 * 8))
    ctx = gr.causal_attention_ref(qkv, 2)
    assert np.allclose(ctx[:, 0], qkv[:, 0, 16:])                       # query 0 sees key 0 alone
    qkv2 = qkv.copy()
    qkv2[:, 3:] += 1.0
    assert np.array_equal(gr.causal_attention_ref(qkv2, 2)[:, :3], ctx[:, :3])
    h = rng.standard_normal((3, 4, 2))
    pos, gat = gr.last_token_ref(h, np.array([[1, 1, 0, 0], [0, 0, 1, 1], [0, 0, 0, 0]]))
    assert pos.tolist() == [1, 3, -1] and np.array_equal(gat[0], h[0, 1]) and not gat[2].any()
    ids, probs, vals = gr.top_k_ref(np.array([[1.0, 3.0, 3.0, 2.0, 9.0], [0, 0, 0, 0, 0]], np.float32), [0, -1], 4, 3)
    assert ids.tolist() == [[1, 2, 3], [-1, -1, -1]] and probs[1].sum() == 0 and vals[1, 0] == -gr.FLT_MAX


@pytest.mark.parametrize("inputs", [mf.GPT2_INPUTS, None], ids=["mask", "ids_only"])
def test_gpt2_bundle_matches_transformers(inputs):
    pytest.importorskip("transformers")
    S, B = 12, 6
    model = ge.hf_gpt2_model(3, **SMALL)
    man = _gpt2(seq=S, inputs=inputs)
    blob = ge.export_gpt2_model(model, man)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], 5)
    mask = x["attention_mask"] if inputs else None
    if inputs is None:
        x = x["input_ids"]
        ids = x
    else:
        ids = x["input_ids"]
        assert (mask[1] == 0).any() and (mask[2, 0] == 0)               # right- and left-padded rows
    pos, logits = gr.gpt2_forward(man, blob, x)
    ref = ge.gpt2_reference(model, ids, mask)
    want_pos = np.full(B, S - 1) if mask is None else [max(np.nonzero(m)[0]) for m in mask]
    assert pos.tolist() == list(want_pos)
    V = SMALL["vocab"]
    at = ref[np.arange(B), pos]
    err = np.abs(logits[:, :V] - at).max()
    assert err <= 1e-6, err
    assert not logits[:, V:].any()
    ids_ref = np.argsort(-at, axis=1, kind="stable")[:, :K]
    ids_got, _p, _v = gr.top_k_ref(logits, pos, V, K)
    assert np.array_equal(ids_got, ids_ref)


def test_left_padding_keeps_positions():
    """transformers counts positions 0..S-1 whatever the padding, so a left-padded row is not the unpadded one shifted"""
    pytest.importorskip("transformers")
    S = 8
    model = ge.hf_gpt2_model(4, **SMALL)
    man = _gpt2(seq=S)
    blob = ge.export_gpt2_model(model, man)
    ids = np.array([[0, 0, 0, 7, 8, 9, 10, 11], [7, 8, 9, 10, 11, 0, 0, 0]], np.int32)
    mask = np.array([[0, 0, 0, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 0, 0, 0]], np.int32)
    pos, logits = gr.gpt2_forward(man, blob, {"input_ids": ids, "attention_mask": mask})
    ref = ge.gpt2_reference(model, ids, mask)
    assert pos.tolist() == [7, 4]
    assert np.abs(logits[:, :SMALL["vocab"]] - ref[[0, 1], [7, 4]]).max() <= 1e-6
    assert np.abs(logits[0] - logits[1]).max() > 1e-3
