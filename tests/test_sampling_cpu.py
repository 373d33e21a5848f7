"""GPT-2 sampling generate bundles, CPU side: the Philox4x32-10 reference against Random123's known answers, the reference
sampler's kept set against transformers' warpers, every loader refusal of the sampling fields and the seed input, the
messages and layouts of bundles without a seed, and the packed layout with one."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sampling_ref as sr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=64)
N = 6
IDS_SEED = [{"name": "input_ids", "role": "ids"}, {"name": "seed", "role": "seed"}]


def _outs(n=N, **fields):
    return [dict({"name": k, "kind": k, "max_new_tokens": n}, **fields) for k in mf.GENERATE_OUTPUT_KINDS]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _gpt2(seq=16, outputs=None, inputs=mf.GPT2_SAMPLING_INPUTS, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=_outs(top_k=40) if outputs is None else outputs)


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


# ------------------------------------------------------------------------------------------------- Philox ----
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert sr.philox4x32_10(ctr, key) == want


def test_uniform_is_53_bits_of_the_first_two_words():
    x = sr.philox4x32_10((3, 0, 0, 0), (7, 0))
    assert sr.uniform53(7, 3) == (x[0] >> 5) * 2 ** 26 + (x[1] >> 6) and 0 <= sr.uniform53(7, 3) < 2 ** 53
    assert sr.uniform53(-1, 0) == sr.uniform53(0xFFFFFFFF, 0)              # the seed is its int32 bits


# --------------------------------------------------------------------------------------- reference sampler ----
@pytest.mark.parametrize("temperature,top_k,top_p", [(1.0, 0, 1.0), (0.7, 40, 1.0), (1.0, 0, 0.9), (1.3, 200, 0.95),
                                                     (0.5, 5, 0.5), (1.7, 1000, 0.9)])
def test_kept_set_matches_transformers_warpers(temperature, top_k, top_p):
    pytest.importorskip("transformers")
    rng = np.random.default_rng(int(temperature * 10) + top_k)
    checked = 0
    for r in range(40):
        z = (rng.standard_normal(1000) * (1 + r % 4)).astype(np.float32)
        kept, w, amb = sr.kept_set(z, temperature, top_k, top_p)
        assert np.all(np.diff(z[kept].astype(np.float64)) <= 0) and np.all(w > 0)
        if amb:
            continue
        assert sorted(kept.tolist()) == sorted(sr.warpers_kept(z, temperature, top_k, top_p).tolist()), r
        checked += 1
    assert checked >= 36


def test_kept_set_rank_order_and_ties():
    z = np.array([1.0, 3.0, 3.0, 2.0, 3.0], np.float32)
    assert sr.rank_order(z).tolist() == [1, 2, 4, 3, 0]
    assert sr.kept_set(z, 1.0, 2)[0].tolist() == [1, 2]                 # ties at the boundary: the lower ids
    kept, w, _a = sr.kept_set(z, 1.0, 0, 0.5)                           # three weights of 1: half needs two
    assert kept.tolist() == [1, 2] and w.tolist() == [1.0, 1.0]
    assert sr.kept_set(z, 1.0, 0, 1e-9)[0].tolist() == [1]              # at least one token


def test_draw_top_k_one_is_the_argmax_and_the_distribution_holds():
    rng = np.random.default_rng(0)
    z = rng.standard_normal(50).astype(np.float32)
    assert all(sr.draw(z, s, 0, 1.3, 1, 0.5) == (int(np.argmax(z)), False) for s in range(20))
    probs = sr.kept_probabilities(z, 0.8, 10, 0.9)
    counts = {}
    for s in range(4000):
        g, _a = sr.draw(z, s, 2, 0.8, 10, 0.9)
        counts[g] = counts.get(g, 0) + 1
    assert set(counts) <= set(probs)
    for g, p in probs.items():
        assert abs(counts.get(g, 0) / 4000 - p) <= 5 * (p * (1 - p) / 4000) ** 0.5 + 1e-3, g


# ------------------------------------------------------------------------------------------------ loader ----
def test_sampling_bundle_layout():
    rc, got = _check(_gpt2())
    assert rc > 0, got
    assert got["in_dim"] == 2 * 16 + 1 and got["head_k"] == N and got["out_dim"] == 2 * N + 1
    rc, got = _check(_gpt2(inputs=IDS_SEED, outputs=_outs(temperature=0.8)))
    assert rc > 0 and got["in_dim"] == 16 + 1, got


@pytest.mark.parametrize("fields", [dict(temperature=1), dict(top_k=0), dict(top_p=1), dict(temperature=0.01, top_k=1000, top_p=1e-3),
                                    dict(temperature=1e30, top_k=1), dict(temperature=1e-37)])
def test_sampling_fields_accepted(fields):
    rc, got = _check(_gpt2(outputs=_outs(**fields)))
    assert rc > 0, got


@pytest.mark.parametrize("field,value,why", [
    ("temperature", 0, "'generated_ids' has a 'temperature' that is not a finite number > 0"),
    ("temperature", -1.5, "has a 'temperature' that is not a finite number > 0"),
    ("temperature", 1e300, "has a 'temperature' that is not a finite number > 0"),
    ("temperature", "hot", "has a 'temperature' that is not a finite number > 0"),
    ("temperature", 1e-39, "has a 'temperature' that is not a finite number > 0 with a finite fp32 reciprocal"),  # subnormal
    ("top_k", 2.5, "'generated_ids' has a 'top_k' that is not an integer >= 0 (0: off)"),
    ("top_k", -1, "has a 'top_k' that is not an integer >= 0"),
    ("top_k", 1001, "signature.outputs: top_k = 1001 exceeds vocab = 1000"),
    ("top_p", 0, "'generated_ids' has a 'top_p' outside (0, 1] (1: off)"),
    ("top_p", 1.01, "has a 'top_p' outside (0, 1]"),
    ("top_p", True, "has a 'top_p' outside (0, 1]"),
])
def test_sampling_field_refusals(field, value, why):
    _refused(_gpt2(outputs=_outs(**{field: value})), why)


@pytest.mark.parametrize("field,a,b", [("temperature", 0.7, 0.8), ("top_k", 4, 5), ("top_p", 0.9, 0.95)])
def test_sampling_fields_must_agree(field, a, b):
    outs = _outs(**{field: a})
    outs[2][field] = b
    _refused(_gpt2(outputs=outs), f"has a '{field}' that differs from the other generate outputs'")
    outs = _outs(**{field: a})
    del outs[0][field]                                                  # one entry giving it is enough
    assert _check(_gpt2(outputs=outs))[0] > 0


def test_seed_input_refusals():
    _refused(_gpt2(inputs=mf.GPT2_INPUTS), "signature.outputs: a sampling generate bundle (temperature, top_k or top_p) needs an"
                                           " input with the role 'seed' (int32 [batch, 1])")
    _refused(_gpt2(inputs=None), "needs an input with the role 'seed'")
    why = "signature.inputs: a 'seed' input belongs to sampling generate bundles (generate outputs with temperature, top_k or top_p)"
    _refused(_gpt2(outputs=_outs()), why)                               # greedy generate
    _refused(_gpt2(outputs=[{"name": "ids", "kind": "next_token_top_k_ids", "k": 3}]), why)
    bert_in = [{"name": "input_ids", "role": "ids"}, {"name": "input_mask", "role": "mask"}, {"name": "seed", "role": "seed"}]
    _refused(mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, inputs=bert_in), why)
    _refused(mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, inputs=bert_in,
                              outputs=[{"name": "probabilities", "kind": "probabilities"}]), why)


def test_earlier_generate_checks_come_first():
    man = _gpt2(inputs=mf.GPT2_INPUTS, outputs=_outs(top_k=5, eos_token_id=1000))
    _refused(man, "signature.outputs: eos_token_id = 1000 is not below vocab = 1000")
    _refused(_gpt2(seq=16, outputs=_outs(50, top_k=5)), "S + max_new_tokens - 1 = 65 positions exceed the embed op's max_pos = 64")


def test_bundles_without_a_seed_are_unchanged():
    rc, got = _check(mf.gpt2_manifest(seq=16, **SMALL, inputs=mf.GPT2_INPUTS, outputs=_outs()))
    assert rc > 0 and got["in_dim"] == 32 and got["out_dim"] == 2 * N + 1
    rc, got = _check(mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, inputs=mf.BERT_INPUTS))
    assert rc > 0 and got["in_dim"] == 48
    man = _gpt2(inputs=[{"name": "input_ids", "role": "ids"}, {"name": "x", "role": "dice"}])
    _refused(man, "signature.inputs: unknown role 'dice' (ids, mask, type_ids)")
    _refused(_gpt2(inputs=mf.BERT_INPUTS + [{"name": "seed", "role": "seed"}]), "signature.inputs must list 1 to 3 inputs")
    # the fields belong to generate entries: a next-token entry ignores them, as it ignores any other unknown field
    rc, got = _check(_gpt2(inputs=mf.GPT2_INPUTS, outputs=[{"name": "ids", "kind": "next_token_top_k_ids", "k": 3, "top_k": 9}]))
    assert rc > 0, got


# ---------------------------------------------------------------------------------------- forward hop signature ----
def _roundtrip(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_signature_roundtrip(json.dumps(man).encode(), buf, len(buf))
    assert rc > 0, lib.tfsc_last_error().decode()
    return json.loads(buf.value)


@pytest.mark.parametrize("inputs,widths", [
    (mf.GPT2_SAMPLING_INPUTS, {"attention_mask": (0, 16), "input_ids": (16, 16), "seed": (32, 1)}),
    (IDS_SEED, {"input_ids": (0, 16), "seed": (16, 1)}),
    ([{"name": "a_seed", "role": "seed"}, {"name": "ids", "role": "ids"}], {"a_seed": (0, 1), "ids": (1, 16)}),
])
def test_signature_roundtrip_of_a_sampling_bundle(inputs, widths):
    """the ingress rank rebuilds the owner's offsets and widths from the roles in the signature the owner sends"""
    got = _roundtrip(_gpt2(inputs=inputs, outputs=_outs(temperature=0.8)))
    assert got["owner"] == got["ingress"], got
    assert got["owner"]["in_dim"] == 2 * 16 + 1 - 16 * (len(inputs) == 2) and got["owner"]["out_dim"] == 2 * N + 1
    assert {i["name"]: (i["offset"], i["width"]) for i in got["owner"]["inputs"]} == widths
    assert [i["role"] for i in got["owner"]["inputs"] if i["name"].endswith("seed")] == [3]


def test_signature_roundtrip_without_a_seed():
    got = _roundtrip(mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, inputs=mf.BERT_INPUTS))
    assert got["owner"] == got["ingress"] and got["owner"]["in_dim"] == 48
    assert [(i["offset"], i["width"]) for i in got["owner"]["inputs"]] == [(0, 16), (16, 16), (32, 16)]
    got = _roundtrip(mf.gpt2_manifest(seq=16, **SMALL, inputs=mf.GPT2_INPUTS, outputs=_outs()))
    assert got["owner"] == got["ingress"] and [(i["offset"], i["width"]) for i in got["owner"]["inputs"]] == [(0, 16), (16, 16)]
