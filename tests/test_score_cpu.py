"""GPT-2 score bundles, CPU side: the fp64 reference (score_ref) against transformers' GPT2LMHeadModel log-softmax and its
shifted-label loss, every loader refusal of the token_score op and the score kinds with its message, the writer at GPT-2
small / medium / large shapes, the packed layout against the loader's, and the forward hop's signature of a score bundle."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpt2_export as ge  # noqa: E402
import score_ref as sr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=64)
ALL = [{"name": k, "kind": k} for k in mf.SCORE_OUTPUT_KINDS]


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


# ----------------------------------------------------------------------------------------- fp64 reference ----
def _rows(S):
    """ids and mask [6, S]: unpadded, right-padded, left-padded, holed, one attended token, and holes at both ends"""
    rng = np.random.default_rng(S)
    ids = rng.integers(0, SMALL["vocab"], (6, S)).astype(np.int32)
    mask = np.ones((6, S), np.int32)
    mask[1, S - 4:] = 0
    mask[2, :5] = 0
    mask[3, [2, 3, 7, S - 2]] = 0
    mask[4, :] = 0
    mask[4, 6] = 1
    mask[5, [0, 1, 5, S - 1]] = 0
    return ids, mask


def test_reference_hand_cases():
    assert sr.scored_pairs([0, 1, 1, 0, 1, 0], 6) == [(1, 2), (2, 4)]
    assert sr.scored_pairs(None, 3) == [(0, 1), (1, 2)]
    assert sr.scored_pairs([0, 0, 1], 3) == [] and sr.scored_pairs([0, 0, 0], 3) == []
    z = np.array([1.0, 3.0, 3.0, -2.0, 3.0], np.float32)
    assert [sr.rank(z, i) for i in range(5)] == [3, 0, 1, 4, 2]
    logits = np.log(np.array([[[0.5, 0.25, 0.25, 9], [0.1, 0.2, 0.7, 9], [1, 1, 1, 9]]]))
    lp, rk, total, count = sr.score(logits, np.array([[2, 0, 7]]), None, 3)   # the padding column is never read
    assert np.allclose(lp, [[0, np.log(0.5), np.log(0.7)]]) and rk.tolist() == [[-1, 0, 0]]
    assert np.isclose(total[0], np.log(0.35)) and count.tolist() == [2]


@pytest.mark.parametrize("inputs", [mf.GPT2_INPUTS, None], ids=["mask", "ids_only"])
def test_reference_matches_transformers_log_softmax(inputs):
    pytest.importorskip("transformers")
    import torch
    S = 12
    model = ge.hf_gpt2_model(7, **SMALL)
    man = _gpt2(seq=S, inputs=inputs)
    blob = ge.export_gpt2_model(model, man)
    ids, mask = _rows(S)
    x = {"input_ids": ids, "attention_mask": mask} if inputs else ids
    lp, rk, total, count = sr.score_forward(man, blob, x)
    ref = ge.gpt2_reference(model, ids, mask if inputs else None)
    ls = torch.log_softmax(torch.from_numpy(ref), -1).numpy()
    m = mask if inputs else np.ones_like(mask)
    n = 0
    for r in range(len(ids)):
        for p, s in sr.scored_pairs(m[r], S):
            assert abs(lp[r, s] - ls[r, p, ids[r, s]]) <= 1e-6, (r, s)
            assert rk[r, s] == int((ref[r, p] > ref[r, p, ids[r, s]]).sum() + (ref[r, p, :ids[r, s]] == ref[r, p, ids[r, s]]).sum())
            n += 1
    assert n == count.sum() and n > 30
    assert np.allclose(total, lp.sum(axis=1)) and (rk[lp == 0] == -1).all()
    assert count.tolist() == ([S - 1] * 6 if inputs is None else [S - 1, S - 5, S - 6, S - 5, 0, S - 5])


def test_mean_log_prob_is_transformers_loss():
    """an independent pin: on unpadded and right-padded rows, -sum / count is transformers' shifted-label loss with
    labels -100 where the mask is 0 (its causal-LM loss: the labels shifted left by one, cross entropy with ignore_index
    -100, taken here on the fp64 logits, since the model's own loss upcasts them to fp32 only)"""
    pytest.importorskip("transformers")
    import torch
    S = 12
    model = ge.hf_gpt2_model(8, **SMALL)
    man = _gpt2(seq=S)
    blob = ge.export_gpt2_model(model, man)
    ids, mask = _rows(S)
    ids, mask = ids[:2], mask[:2]
    _lp, _rk, total, count = sr.score_forward(man, blob, {"input_ids": ids, "attention_mask": mask})
    logits = torch.from_numpy(ge.gpt2_reference(model, ids, mask))
    labels = torch.where(torch.from_numpy(mask) == 0, -100, torch.from_numpy(ids.astype(np.int64)))
    for r in range(2):
        loss = torch.nn.functional.cross_entropy(logits[r, :-1], labels[r, 1:], ignore_index=-100).item()
        assert abs(-total[r] / count[r] - loss) <= 1e-9, (r, -total[r] / count[r], loss)


# ------------------------------------------------------------------------------------------- writer / layout ----
@pytest.mark.parametrize("arch", [(768, 12, 12), (1024, 24, 16), (1280, 36, 20)], ids=["small", "medium", "large"])
def test_writer_at_gpt2_shapes(arch):
    hidden, layers, heads = arch
    man = mf.gpt2_manifest(seq=1024, hidden=hidden, layers=layers, heads=heads, inputs=mf.GPT2_INPUTS, outputs=ALL)
    rc, got = _check(man)
    assert rc > 0, got
    assert got["head_n"] == 1024 and got["head_k"] == 0 and got["in_dim"] == 2048 and got["out_dim"] == 2 * 1024 + 2
    assert len(man["ops"]) == 1 + 7 * layers + 2 and not any(o["op"] == "last_token" for o in man["ops"])
    lnf, ts = man["ops"][-2:]
    assert lnf["op"] == "layernorm" and lnf["h"] == 1024 and ts["src"] == lnf["dst"]
    assert ts == dict(ts, op="token_score", dst=-2, h=1024, w=1, c=hidden, cout=50272, vocab=50257)


def test_export_fills_the_score_bundle():
    """export_gpt2_model reads ops[-3:] as (ignored, ln_f, decoder): the score bundle's blob is the next-token bundle's"""
    pytest.importorskip("transformers")
    model = ge.hf_gpt2_model(2, **SMALL)
    a, b = _gpt2(), _gpt2(outputs=[{"name": "n", "kind": "next_token_position"}])
    ba, bb = ge.export_gpt2_model(model, a), ge.export_gpt2_model(model, b)
    for oa, ob in zip(a["ops"][:-2], b["ops"][:-3]):
        for key in ("w_offset", "b_offset", "word_offset", "pos_offset"):
            if key in oa:
                n = oa["c"] * oa.get("cout", 1) if key == "w_offset" and "cout" in oa else oa.get("c", 1)
                assert np.array_equal(ba[oa[key] // 4:][:n], bb[ob[key] // 4:][:n])
    for key, n in (("w_offset", 64 * 1024), ("b_offset", 1024)):
        assert np.array_equal(ba[a["ops"][-1][key] // 4:][:n], bb[b["ops"][-1][key] // 4:][:n])


OUTPUT_SETS = [ALL, [{"name": "lp", "kind": "token_log_probs"}], [{"name": "n", "kind": "token_count"}],
               [{"name": "Sum", "kind": "token_log_prob_sum"}, {"name": "ranks", "kind": "token_ranks"}]]


@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(which):
    outs = OUTPUT_SETS[which]
    rc, got = _check(_gpt2(outputs=outs))
    assert rc > 0, got
    layout = mf.packed_output_layout(outs, 16)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == 16 and got["head_k"] == 0
    words = np.arange(3 * got["out_dim"], dtype=np.int32).reshape(3, -1)
    split = mf.split_packed_rows(words, outs, 16)
    kinds = {o["name"]: o["kind"] for o in outs}
    for name, off, width, _dt in layout:
        assert split[name].shape == ((3, 16) if kinds[name] in ("token_log_probs", "token_ranks") else (3,))
        assert np.array_equal(split[name].reshape(3, -1).view(np.int32), words[:, off:off + width])


def _roundtrip(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_signature_roundtrip(json.dumps(man).encode(), buf, len(buf))
    assert rc > 0, lib.tfsc_last_error().decode()
    return json.loads(buf.value)


@pytest.mark.parametrize("seq,inputs", [(16, mf.GPT2_INPUTS), (1024, None), (7, mf.GPT2_INPUTS)])
def test_signature_roundtrip(seq, inputs):
    """the ingress rank lays the score outputs out from the signature alone (an unusable layout would leave out_dim 0)"""
    got = _roundtrip(_gpt2(seq=seq, inputs=inputs, max_pos=max(64, seq)))
    assert got["owner"] == got["ingress"]
    assert got["owner"]["out_dim"] == 2 * seq + 2 and got["owner"]["in_dim"] == seq * (2 if inputs else 1)


# ---------------------------------------------------------------------------------------------- refusals ----
def test_score_kinds_do_not_mix():
    for other in ({"name": "l", "kind": "logits"}, {"name": "n", "kind": "next_token_position"},
                  {"name": "g", "kind": "generated_ids", "max_new_tokens": 2}):
        for outs in (ALL[:1] + [other], [other] + ALL[:1]):
            _refused(_gpt2(outputs=outs), "signature.outputs: score outputs (token_log_probs, token_ranks, token_log_prob_sum,"
                                          " token_count) cannot be mixed with classification, span, encoder, fill-mask,"
                                          " next-token or generate outputs")


@pytest.mark.parametrize("field", ["k", "max_new_tokens", "eos_token_id", "temperature", "top_k", "top_p", "repetition_penalty",
                                   "no_repeat_ngram_size", "min_new_tokens", "normalize", "max_answer_length", "sep_id"])
def test_score_entries_take_no_fields(field):
    outs = [dict(ALL[0]), dict(ALL[1], **{field: 1})]
    _refused(_gpt2(outputs=outs), f"signature.outputs: '{field}' does not apply to score outputs ('token_ranks' is token_ranks)")


def test_unknown_token_kind_is_told_the_score_kinds():
    got = _refused(_gpt2(outputs=[{"name": "a", "kind": "token_probs"}]), "signature.outputs: unknown score kind 'token_probs' (")
    assert got.endswith("(token_log_probs, token_ranks, token_log_prob_sum, token_count)")


def test_unknown_kind_message_is_unchanged():
    got = _refused(_gpt2(outputs=[{"name": "a", "kind": "nope"}]), "unknown kind 'nope' (logits,")
    assert got.endswith("masked_top_k_logits)") and "token_" not in got


def test_token_score_needs_score_outputs():
    man = _gpt2()
    del man["signature"]["outputs"]
    man["signature"]["output"] = "logits"
    _refused(man, "graph manifest: a token_score op needs score outputs (token_log_probs, token_ranks, token_log_prob_sum,"
                  " token_count)")


def test_token_score_with_other_outputs():
    man = _gpt2()
    man["signature"]["outputs"] = [{"name": "n", "kind": "next_token_position"}]
    _refused(man, "graph manifest: a token_score op needs score outputs")


def test_score_outputs_need_one_token_score_op():
    man = _gpt2(outputs=[{"name": "n", "kind": "next_token_position"}])
    man["signature"]["outputs"] = ALL
    _refused(man, "graph manifest: a score bundle scores every token: it has no last_token or mask_gather op")
    man = _gpt2()
    man["ops"][-1] = dict(man["ops"][-1], op="conv", kh=1, kw=1, stride=1, pad=0)
    del man["ops"][-1]["vocab"]
    _refused(man, "signature.outputs: score outputs need exactly one token_score op (the bundle has 0)")
    man = _gpt2()
    man["ops"].insert(len(man["ops"]) - 1, dict(man["ops"][-1], dst=2))
    _refused(man, "signature.outputs: score outputs need exactly one token_score op (the bundle has 2)")


def test_token_score_is_the_last_op():
    man = _gpt2()
    ts = man["ops"].pop()
    man["ops"].insert(len(man["ops"]) - 1, ts)              # token_score, then ln_f writing the response
    man["ops"][-1]["dst"] = -2
    _refused(man, "signature.outputs: score outputs need the token_score op to be the last op")


def test_token_score_source():
    man = _gpt2(inputs=None)
    man["ops"][-1]["src"] = -1
    man["ops"][-1]["c"] = 1                                   # the request itself: [16] ids
    _refused(man, "the token_score op needs the [16, 1, 64] hidden states of a scratch buffer (it reads [16, 1, 1] of buffer -1)")
    man = _gpt2()
    ts = man["ops"][-1]
    ts["h"], ts["c"] = 8, 128
    ts["cout"] = 512                                           # [8, 1, 128]: the same element count, not [S, 1, H]
    _refused(man, "the token_score op needs the [16, 1, 64] hidden states of a scratch buffer (it reads [8, 1, 128] of buffer 1)")


def test_token_score_geometry():
    for field, v in (("kh", 3), ("w", 2), ("stride", 2), ("pad", 1)):
        man = _gpt2()
        man["ops"][-1][field] = v
        _refused(man, "graph manifest: token_score projects each of its h tokens: w = 1, kh = kw = stride = 1, pad = 0")
    man = _gpt2()
    man["ops"][-1]["act"] = "relu"
    _refused(man, "graph manifest: token_score takes no activation (act 'relu')")
    man = _gpt2()
    man["ops"][-1]["res"] = 0
    _refused(man, "graph manifest: token_score takes no residual input")


def test_token_score_vocab_and_width():
    man = _gpt2()
    man["ops"][-1]["vocab"] = 999
    _refused(man, "signature.outputs: the token_score op's vocab = 999 differs from the embed op's vocab = 1000")
    man = _gpt2()
    man["ops"][-1]["cout"] = 992
    _refused(man, "signature.outputs: the token_score op writes cout = 992 logits per token, below vocab = 1000")
    man = _gpt2()
    man["ops"][-1]["cout"] = 1000                             # unpadded: accepted (the GEMM route)
    assert _check(man)[0] > 0


def test_token_score_weights_in_range():
    man = _gpt2()
    man["ops"][-1]["b_offset"] = man["weights_bytes"]
    _refused(man, "graph manifest: weights out of range or misaligned")


def test_score_needs_causal_attention():
    man = _gpt2()
    _op(man, "attention", 1)["causal"] = False
    _refused(man, "signature.outputs: score outputs need causal attention (op 10 is not causal)")


@pytest.mark.parametrize("vocab,ok", [(57344, True), (57345, False), (1, True)])
def test_score_vocab_limit(vocab, ok):
    man = _gpt2(seq=4, layers=1, vocab=vocab)
    if ok:
        assert _check(man)[0] > 0
    else:
        _refused(man, f"signature.outputs: no score kernels for S = 4 and vocab = {vocab} (1 <= S <= 16384, 1 <= vocab <= 57344)")


def test_score_needs_a_graph_bundle(tmp_path):
    man = mf.write_mlp_bundle(str(tmp_path / "m" / "1"), [np.zeros((4, 4), np.float32)], [np.zeros(4, np.float32)], outputs=ALL[:1])
    _refused(man, "signature.outputs: score outputs need a graph bundle")


def test_score_bundle_takes_no_seed():
    _refused(_gpt2(inputs=mf.GPT2_SAMPLING_INPUTS), "signature.inputs: a 'seed' input belongs to sampling generate bundles")


def test_single_input_score_bundle():
    rc, got = _check(_gpt2(inputs=None))
    assert rc > 0 and got["in_dim"] == 16, got
