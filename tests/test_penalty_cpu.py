"""GPT-2 processing generate bundles (repetition_penalty, no_repeat_ngram_size, min_new_tokens), CPU side: the reference
(penalty_ref) against transformers' three processors bit for bit on fp32 logits, its history and picks, every loader refusal
of the fields with its message, the field-agreement rule, bundles without the fields answered as before, and the forward
hop's signature of a processing bundle."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import penalty_ref as pr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=64)
N = 6
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "manifest_check_golden.json")


def _outs(n=N, **fields):
    return [dict({"name": k, "kind": k, "max_new_tokens": n}, **fields) for k in mf.GENERATE_OUTPUT_KINDS]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, buf.value.decode()) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _gpt2(seq=16, outputs=None, inputs=mf.GPT2_INPUTS, **kw):
    arch = dict(SMALL)
    arch.update(kw)
    return mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=_outs(repetition_penalty=1.3) if outputs is None else outputs)


def _refused(man, why):
    rc, got = _check(man)
    assert rc == t._lib.E_INVALID, got
    assert why in got, got
    return got


# --------------------------------------------------------------------------------- reference vs transformers ----
def _row(rng, vocab):
    """fp32 logits with negative, zero, -0 and tied values"""
    z = (rng.standard_normal(vocab) * 4).astype(np.float32)
    z[rng.integers(0, vocab, vocab // 10)] = 0.0
    z[rng.integers(0, vocab, vocab // 20)] = -0.0
    z[rng.integers(0, vocab, vocab // 10)] = np.float32(1.5)
    z[rng.integers(0, vocab, vocab // 10)] = np.float32(-2.25)
    return z


@pytest.mark.parametrize("vocab", [50, 50257])
@pytest.mark.parametrize("penalty", [0.7, 1.0, 1.17, 1.3, 2.9])
def test_penalty_matches_transformers(vocab, penalty):
    pytest.importorskip("transformers")
    rng = np.random.default_rng(int(penalty * 100) + vocab)
    for r in range(6):
        z = _row(rng, vocab)
        L = int(rng.integers(1, 300))
        h = rng.integers(0, min(vocab, 40 + 400 * r), L).tolist()          # duplicates
        want = pr.transformers_process(z, h, L, penalty=penalty)
        got = pr.process(z, h, 0, penalty=penalty)
        assert got.tobytes() == want.tobytes(), (penalty, r)


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_no_repeat_ngram_matches_transformers(n):
    pytest.importorskip("transformers")
    rng = np.random.default_rng(n)
    for r in range(30):
        vocab = 30
        z = _row(rng, vocab)
        L = int(rng.integers(0, 60))
        h = rng.integers(0, 3 + r % 5, L).tolist()                          # small alphabets: many repeated n-grams
        want = pr.transformers_process(z, h, L, ngram=n)
        got = pr.process(z, h, 0, ngram=n)
        assert got.tobytes() == want.tobytes(), (n, r, h)
    assert pr.banned_ngrams([1, 2, 3, 1, 2], 3) == {3}
    assert pr.banned_ngrams([4, 4, 4], 2) == {4} and pr.banned_ngrams([5, 6, 5], 1) == {5, 6}
    assert pr.banned_ngrams([1, 2], 4) == set()


@pytest.mark.parametrize("m", [1, 3, 5])
def test_min_new_tokens_matches_transformers(m):
    pytest.importorskip("transformers")
    rng = np.random.default_rng(m)
    prompt = rng.integers(0, 100, 9).tolist()
    for t_ in range(7):                                                   # t on both sides of m
        z = _row(rng, 100)
        ids = prompt + rng.integers(0, 100, t_).tolist()
        want = pr.transformers_process(z, ids, len(prompt), min_new=m, eos=17)
        got = pr.process(z, ids, t_, min_new=m, eos=17)
        assert got.tobytes() == want.tobytes(), (m, t_)
        assert (got[17] == -np.inf) == (t_ < m)


def test_all_three_in_transformers_order():
    pytest.importorskip("transformers")
    rng = np.random.default_rng(5)
    prompt = rng.integers(0, 40, 20).tolist()
    for t_ in range(8):
        z = _row(rng, 40)
        ids = prompt + rng.integers(0, 40, t_).tolist()
        for n in (1, 2, 3):
            want = pr.transformers_process(z, ids, len(prompt), penalty=1.3, ngram=n, min_new=4, eos=3)
            got = pr.process(z, ids, t_, penalty=1.3, ngram=n, min_new=4, eos=3)
            assert got.tobytes() == want.tobytes(), (t_, n)


def test_history_and_picks():
    ids = np.array([5, -3, 70000, 9, 9, 1], np.int32)
    assert pr.history(ids, None, 3, 100) == [5, 0, 99, 9]                 # clamped as the embedding clamps
    assert pr.history(ids, [1, 0, 1, 0, 1, 1], 5, 100) == [5, 99, 9, 1]
    assert pr.history(ids, [1] * 6, -1, 100) == []                        # no attended token
    z = np.array([1.0, 3.0, 3.0, -2.0], np.float32)
    assert pr.pick(z, [], 0) == (1, False)                                # ties to the lower id
    assert pr.pick(z, [1], 0, penalty=2.0) == (2, False)
    assert pr.pick(z, [0, 1, 2, 3], 0, ngram=1) == (0, False)             # everything banned: id 0
    assert pr.pick(z, [0, 1, 2, 3], 0, ngram=1, seed=3, temperature=0.7, top_k=2) == (0, False)
    assert pr.pick(z, [], 0, seed=3, top_k=1) == (1, False)
    assert pr.process(z, [0, 3], 0, penalty=1.0).tobytes() == z.tobytes()  # p = 1 is the identity


# ------------------------------------------------------------------------------------------------ loader ----
def test_processing_bundle_layout_is_the_plain_bundles():
    for fields, inputs in ((dict(repetition_penalty=1.3), mf.GPT2_INPUTS), (dict(no_repeat_ngram_size=3), None),
                           (dict(min_new_tokens=2, eos_token_id=7), mf.GPT2_INPUTS),
                           (dict(repetition_penalty=1.2, no_repeat_ngram_size=2, min_new_tokens=6, eos_token_id=7, top_k=5),
                            mf.GPT2_SAMPLING_INPUTS)):
        plain = {k: v for k, v in fields.items() if k not in ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens")}
        rc, got = _check(_gpt2(inputs=inputs, outputs=_outs(**fields)))
        assert rc > 0, got
        assert (rc, got) == _check(_gpt2(inputs=inputs, outputs=_outs(**plain))), fields


@pytest.mark.parametrize("fields", [dict(repetition_penalty=1), dict(repetition_penalty=0.01), dict(repetition_penalty=1e30),
                                    dict(repetition_penalty=1.2e-38), dict(no_repeat_ngram_size=1),
                                    dict(no_repeat_ngram_size=21), dict(min_new_tokens=1, eos_token_id=0),
                                    dict(min_new_tokens=6, eos_token_id=999)])
def test_processing_fields_accepted(fields):
    rc, got = _check(_gpt2(outputs=_outs(**fields)))
    assert rc > 0, got


@pytest.mark.parametrize("fields,why", [
    (dict(repetition_penalty=0), "signature.outputs: 'generated_ids' has a 'repetition_penalty' that is not a finite number > 0"
                                 " with a finite, normal fp32 value (1: off)"),
    (dict(repetition_penalty=-1.3), "has a 'repetition_penalty' that is not a finite number > 0"),
    (dict(repetition_penalty=1e300), "has a 'repetition_penalty' that is not a finite number > 0"),
    (dict(repetition_penalty=1e39), "has a 'repetition_penalty' that is not a finite number > 0"),  # fp32 inf
    (dict(repetition_penalty=1e-39), "has a 'repetition_penalty' that is not a finite number > 0"),  # fp32 subnormal
    (dict(repetition_penalty=1e-50), "has a 'repetition_penalty' that is not a finite number > 0"),  # fp32 zero
    (dict(repetition_penalty="1.3"), "has a 'repetition_penalty' that is not a finite number > 0"),
    (dict(repetition_penalty=True), "has a 'repetition_penalty' that is not a finite number > 0"),
    (dict(no_repeat_ngram_size=0), "signature.outputs: 'generated_ids' has a 'no_repeat_ngram_size' that is not an integer >= 1"),
    (dict(no_repeat_ngram_size=2.5), "has a 'no_repeat_ngram_size' that is not an integer >= 1"),
    (dict(no_repeat_ngram_size=-3), "has a 'no_repeat_ngram_size' that is not an integer >= 1"),
    (dict(no_repeat_ngram_size=22), "signature.outputs: no_repeat_ngram_size = 22 exceeds S + max_new_tokens - 1 = 21"),
    (dict(min_new_tokens=0, eos_token_id=1), "signature.outputs: 'generated_ids' has a 'min_new_tokens' that is not an integer >= 1"),
    (dict(min_new_tokens="2", eos_token_id=1), "has a 'min_new_tokens' that is not an integer >= 1"),
    (dict(min_new_tokens=7, eos_token_id=1), "signature.outputs: min_new_tokens = 7 exceeds max_new_tokens = 6"),
    (dict(min_new_tokens=2), "signature.outputs: min_new_tokens needs an eos_token_id: it bans the EOS token until that many"
                             " tokens are generated"),
])
def test_processing_field_refusals(fields, why):
    _refused(_gpt2(outputs=_outs(**fields)), why)


@pytest.mark.parametrize("field,a,b", [("repetition_penalty", 1.3, 1.2), ("no_repeat_ngram_size", 3, 2), ("min_new_tokens", 2, 3)])
def test_processing_fields_must_agree(field, a, b):
    outs = _outs(eos_token_id=5, **{field: a})
    outs[2][field] = b
    _refused(_gpt2(outputs=outs), f"signature.outputs: '{outs[2]['name']}' has a '{field}' that differs from the other generate"
                                  " outputs'")
    outs = _outs(eos_token_id=5, **{field: a})
    del outs[0][field]                                                  # one entry giving it is enough
    assert _check(_gpt2(outputs=outs))[0] > 0


def test_earlier_generate_and_sampling_checks_come_first():
    _refused(_gpt2(outputs=_outs(eos_token_id=1000, min_new_tokens=9)), "eos_token_id = 1000 is not below vocab = 1000")
    _refused(_gpt2(outputs=_outs(50, no_repeat_ngram_size=99)), "S + max_new_tokens - 1 = 65 positions exceed the embed op's max_pos")
    _refused(_gpt2(outputs=_outs(top_k=1001, no_repeat_ngram_size=99)), "top_k = 1001 exceeds vocab = 1000")
    _refused(_gpt2(outputs=_outs(top_p=0.5, min_new_tokens=9)), "needs an input with the role 'seed'")
    _refused(_gpt2(outputs=_outs(temperature=0, repetition_penalty=0)), "has a 'temperature' that is not a finite number > 0")
    # a seed belongs to sampling bundles whatever the repetition fields
    _refused(_gpt2(inputs=mf.GPT2_SAMPLING_INPUTS, outputs=_outs(repetition_penalty=1.3)),
             "signature.inputs: a 'seed' input belongs to sampling generate bundles")


def test_other_heads_ignore_the_fields():
    man = _gpt2(outputs=[{"name": "ids", "kind": "next_token_top_k_ids", "k": 3, "repetition_penalty": 0, "min_new_tokens": -1}])
    assert _check(man)[0] > 0


def test_bundles_without_the_fields_answer_as_before():
    """tfsc_manifest_check's code and output, layout or message, as the library answered before processing bundles
    existed (tests/golden/make_manifest_check_golden.py)"""
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert len(golden) >= 10
    for name, g in golden.items():
        assert _check(g["manifest"]) == (g["rc"], g["output"]), name


# ---------------------------------------------------------------------------------------- forward hop signature ----
def _roundtrip(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_signature_roundtrip(json.dumps(man).encode(), buf, len(buf))
    assert rc > 0, lib.tfsc_last_error().decode()
    return json.loads(buf.value)


@pytest.mark.parametrize("inputs,fields", [
    (mf.GPT2_INPUTS, dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=2, eos_token_id=4)),
    (None, dict(no_repeat_ngram_size=2)),
    (mf.GPT2_SAMPLING_INPUTS, dict(repetition_penalty=1.1, temperature=0.8, top_p=0.9)),
])
def test_signature_roundtrip_of_a_processing_bundle(inputs, fields):
    plain = {k: v for k, v in fields.items() if k not in ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens")}
    got = _roundtrip(_gpt2(inputs=inputs, outputs=_outs(**fields)))
    assert got == _roundtrip(_gpt2(inputs=inputs, outputs=_outs(**plain)))
    assert got["owner"] == got["ingress"]
