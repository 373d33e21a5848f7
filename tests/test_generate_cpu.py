"""GPT-2 generate bundles, CPU side: every loader refusal of the generate outputs (tfsc_manifest_check), the messages that
were there before them, the writer at GPT-2 small / medium / large shapes, packed_output_layout against the loader's layout,
and the fp64 greedy reference (generate_ref) against transformers' GPT2LMHeadModel.generate in fp64."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import generate_ref as gen  # noqa: E402
import gpt2_export as ge  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=64)
N = 6


def _outs(n=N, eos=None, kinds=mf.GENERATE_OUTPUT_KINDS):
    return [dict({"name": k, "kind": k, "max_new_tokens": n}, **({} if eos is None else {"eos_token_id": eos})) for k in kinds]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _gpt2(seq=16, outputs=None, inputs=mf.GPT2_INPUTS, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=_outs() if outputs is None else outputs)


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


# ------------------------------------------------------------------------------------------- writer / layout ----
@pytest.mark.parametrize("arch", [(768, 12, 12), (1024, 24, 16), (1280, 36, 20)], ids=["small", "medium", "large"])
def test_writer_at_gpt2_shapes(arch):
    hidden, layers, heads = arch
    for seq, n in ((128, 32), (993, 32), (1, 1024)):
        man = mf.gpt2_manifest(seq=seq, hidden=hidden, layers=layers, heads=heads, inputs=mf.GPT2_INPUTS, outputs=_outs(n, eos=50256))
        rc, got = _check(man)
        assert rc > 0, got
        assert got["head_n"] == 50257 and got["head_k"] == n and got["in_dim"] == 2 * seq
        assert got["out_dim"] == 2 * n + 1


OUTPUT_SETS = [
    _outs(),
    _outs(kinds=["generated_length"]),
    _outs(1, kinds=["generated_ids"]),
    [{"name": "z", "kind": "generated_log_probs", "max_new_tokens": 9}, {"name": "a", "kind": "generated_ids", "max_new_tokens": 9,
                                                                          "eos_token_id": 3}],
]


@pytest.mark.parametrize("which", range(len(OUTPUT_SETS)))
def test_layout_matches_loader(which):
    outs = OUTPUT_SETS[which]
    rc, got = _check(_gpt2(outputs=outs))
    assert rc > 0, got
    layout = mf.packed_output_layout(outs, 1000)
    assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout
    n = outs[0]["max_new_tokens"]
    assert got["out_dim"] == sum(w for _n, _o, w, _d in layout) and got["head_n"] == 1000 and got["head_k"] == n
    words = np.arange(3 * got["out_dim"], dtype=np.int32).reshape(3, -1)
    split = mf.split_packed_rows(words, outs, 1000)
    kinds = {o["name"]: o["kind"] for o in outs}
    for name, off, width, _dt in layout:
        assert split[name].shape == ((3,) if kinds[name] == "generated_length" else (3, n))
        assert np.array_equal(split[name].reshape(3, -1).view(np.int32), words[:, off:off + width])


def test_next_token_bundle_of_the_same_graph_is_unchanged():
    nt = [{"name": "next_token_top_k_ids", "kind": "next_token_top_k_ids", "k": 5}]
    rc, got = _check(_gpt2(outputs=nt))
    assert rc > 0 and got["head_k"] == 5 and got["out_dim"] == 5


# ---------------------------------------------------------------------------------------------- refusals ----
@pytest.mark.parametrize("entry,why", [
    ({"name": "a", "kind": "generated_ids"}, "'a' needs an integer 'max_new_tokens' >= 1, the same for every generate output"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": 0}, "needs an integer 'max_new_tokens' >= 1"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": 2.5}, "needs an integer 'max_new_tokens' >= 1"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": N + 1}, "the same for every generate output"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": N, "eos_token_id": -1}, "has an 'eos_token_id' that is not a token id"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": N, "eos_token_id": "x"}, "has an 'eos_token_id' that is not a token id"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": N, "k": 3}, "do not apply to generate outputs"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": N, "normalize": True}, "do not apply to generate outputs"),
    ({"name": "a", "kind": "generated_ids", "max_new_tokens": N, "sep_id": 2}, "do not apply to generate outputs"),
    ({"name": "a", "kind": "generated_idz"}, "unknown generate kind 'generated_idz' (generated_ids, generated_log_probs, "
                                             "generated_length)"),
])
def test_generate_fields(entry, why):
    outs = [{"name": "z", "kind": "generated_log_probs", "max_new_tokens": N}, entry]
    _refused(_gpt2(outputs=outs), why)


def test_eos_must_agree_and_fit_the_vocabulary():
    outs = _outs(eos=7)
    outs[1]["eos_token_id"] = 8
    _refused(_gpt2(outputs=outs), "differs from the other generate outputs'")
    outs = _outs(eos=7)
    del outs[1]["eos_token_id"]                                         # only the owner needs it: giving it once is enough
    assert _check(_gpt2(outputs=outs))[0] > 0
    _refused(_gpt2(outputs=_outs(eos=1000)), "signature.outputs: eos_token_id = 1000 is not below vocab = 1000")
    assert _check(_gpt2(outputs=_outs(eos=999)))[0] > 0


def test_generate_kinds_do_not_mix():
    for other in ({"name": "l", "kind": "logits"}, {"name": "m", "kind": "masked_positions"},
                  {"name": "n", "kind": "next_token_position"}, {"name": "s", "kind": "sequence_output"}):
        why = ("signature.outputs: generate outputs (generated_ids, generated_log_probs, generated_length) cannot be mixed with"
               " classification, span, encoder, fill-mask or next-token outputs")
        _refused(_gpt2(outputs=_outs()[:1] + [other]), why)
        _refused(_gpt2(outputs=[other] + _outs()[:1]), why)


def test_earlier_messages_are_unchanged():
    got = _refused(_gpt2(outputs=[{"name": "a", "kind": "nope"}]), "signature.outputs: unknown kind 'nope' (logits,")
    assert got.endswith("masked_top_k_logits)") and "generated" not in got and "next_token" not in got
    got = _refused(_gpt2(outputs=[{"name": "a", "kind": "next_token_nope"}]), "unknown next-token kind 'next_token_nope'")
    assert got.endswith("(next_token_position, next_token_top_k_ids, next_token_top_k_probabilities, next_token_top_k_logits)")
    nt = [{"name": "p", "kind": "next_token_position"}]
    _refused(_gpt2(outputs=nt + [{"name": "l", "kind": "logits"}]),
             "signature.outputs: next-token outputs (next_token_position, next_token_top_k_ids, next_token_top_k_probabilities,"
             " next_token_top_k_logits) cannot be mixed with classification, span, encoder or fill-mask outputs ('l' is logits)")
    for outs, head in ((nt, "next-token"), (None, "generate")):
        man = _gpt2(outputs=outs)
        man["ops"][-1]["cout"] = 992
        _refused(man, f"signature.outputs: {head} outputs need a last op that writes [1, 1, Vp] logits, Vp >= 1000 (it writes"
                      " [1, 1, 992])")


def test_last_token_and_embed():
    man = _gpt2(outputs=None)
    lt = [o for o in man["ops"] if o["op"] == "last_token"][0]
    man["ops"].insert(man["ops"].index(lt), dict(lt, dst=2))
    _refused(man, "signature.outputs: generate outputs need exactly one last_token op (the bundle has 2)")
    man = mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100)
    man["signature"] = {k: v for k, v in man["signature"].items() if k != "output"} | {"outputs": _outs()}
    _refused(man, "generate outputs need exactly one last_token op")


def test_decoder_ops():
    man = _gpt2()
    man["ops"][3]["causal"] = False                                    # attention to every key: a decoder it is not
    _refused(man, "generate outputs need a decoder of layernorm, 1x1 conv and causal attention ops on the [16, 1, c] tokens"
                  " between the embed and the last_token op (op 3 is not)")
    assert _check(dict(man, signature=_gpt2(outputs=[{"name": "p", "kind": "next_token_position"}])["signature"]))[0] > 0


def test_embed_without_layernorm():
    man = _gpt2()
    emb = man["ops"][0]
    emb["norm"] = True
    emb["w_offset"] = emb["b_offset"] = emb["type_offset"] = 0
    _refused(man, "signature.outputs: generate outputs need an embed op with norm false (word + position embeddings)")


@pytest.mark.parametrize("seq,n,ok", [(16, 49, True), (16, 50, False), (64, 1, True), (1, 64, True), (1, 65, False)])
def test_positions_fit(seq, n, ok):
    man = _gpt2(seq=seq, outputs=_outs(n))
    if ok:
        assert _check(man)[0] > 0
    else:
        _refused(man, f"signature.outputs: S + max_new_tokens - 1 = {seq + n - 1} positions exceed the embed op's max_pos = 64")


@pytest.mark.parametrize("vocab,n,ok", [(57344, 1, True), (57345, 1, False), (50257, 16384, True), (50257, 16385, False)])
def test_generate_limits(vocab, n, ok):
    man = _gpt2(seq=1, layers=1, vocab=vocab, max_pos=16400, outputs=_outs(n))
    if ok:
        assert _check(man)[0] > 0
    else:
        _refused(man, f"no generate head for vocab = {vocab} and max_new_tokens = {n} (1 <= vocab <= 57344, 1 <= max_new_tokens <= 16384)")


def test_decode_attention_keys():
    _refused(_gpt2(seq=16000, layers=1, max_pos=17000, outputs=_outs(1000)),
             "signature.outputs: no decode attention kernel for 16999 keys, hidden 64, 4 heads")


# ----------------------------------------------------------------------------------------- fp64 reference ----
def _hf_greedy(model, ids, n, eos):
    import torch
    m64 = model.double()
    x = torch.from_numpy(np.asarray(ids, np.int64))[None]
    with torch.no_grad():
        out = m64.generate(x, attention_mask=torch.ones_like(x), do_sample=False, num_beams=1, max_new_tokens=n,
                           eos_token_id=eos, pad_token_id=0 if eos is None else eos)
    return out[0, x.shape[1]:].numpy()


@pytest.mark.parametrize("eos_pick", [None, 2])
def test_reference_matches_transformers_generate(eos_pick):
    """unpadded rows, and right-padded rows run alone with their attended prompt, give transformers' greedy ids"""
    pytest.importorskip("transformers")
    import copy
    S, B, n = 10, 6, 8
    model = ge.hf_gpt2_model(5, **SMALL)
    man = _gpt2(seq=S, outputs=_outs(n))
    blob = ge.export_gpt2_model(model, man)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], 9)
    rows = [r for r in range(B) if x["attention_mask"][r, 0] == 1]          # unpadded and right-padded
    ids0, _lp, _ln = gen.generate_ref(man, blob, {k: v[rows] for k, v in x.items()}, n)
    eos = None if eos_pick is None else int(ids0[0, eos_pick])              # a token the reference emits mid-sequence
    ids, lp, length = gen.generate_ref(man, blob, {k: v[rows] for k, v in x.items()}, n, eos=eos)
    for i, r in enumerate(rows):
        p = int(np.nonzero(x["attention_mask"][r])[0].max())
        want = _hf_greedy(copy.deepcopy(model), x["input_ids"][r, :p + 1], n, eos)
        got = ids[i, :length[i]]
        assert np.array_equal(got, want[:length[i]]), (r, got, want)
        assert (ids[i, length[i]:] == -1).all() and (lp[i, length[i]:] == 0).all() and (lp[i, :length[i]] <= 0).all()
        if eos is not None and eos in got:
            assert got[-1] == eos and length[i] == list(got).index(eos) + 1
    if eos is not None:
        assert length[0] == eos_pick + 1 or eos in ids0[0, :eos_pick]


def test_reference_fully_padded_row():
    model = ge.hf_gpt2_model(6, **SMALL)
    man = _gpt2(seq=8, outputs=_outs(3))
    blob = ge.export_gpt2_model(model, man)
    x = ge.gpt2_inputs(2, 8, SMALL["vocab"], 1)
    x["attention_mask"][1] = 0
    ids, lp, length = gen.generate_ref(man, blob, x, 3)
    assert length.tolist() == [3, 0] and (ids[1] == -1).all() and (lp[1] == 0).all()
