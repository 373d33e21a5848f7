"""The loader's verdict on signature.outputs, pinned: every case of make_manifest_verdicts.cases() (a base bundle, its
outputs and edits) gets exactly the verdict tests/golden/manifest_verdicts.json stores for it from tfsc_manifest_check --
the return code and the packed layout or the error text, so which of several faults is reported cannot move either. For
every accepted case, modelformat.packed_output_layout gives the loader's layout."""
import json
import os
import sys

import tfservingcache_b200 as t

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_manifest_verdicts as mv  # noqa: E402

mf = t.modelformat


def _golden():
    with open(os.path.join(os.path.dirname(mv.__file__), "manifest_verdicts.json")) as f:
        g = json.load(f)
    cases = mv.cases()
    assert g["recipes_sha256"] == mv.recipes_digest(cases), "the cases changed: regenerate the golden (make_manifest_verdicts.py)"
    assert len(g["verdicts"]) == len(cases)
    return [(c, tuple(g["results"][i])) for c, i in zip(cases, g["verdicts"])]


CASES = _golden()


def test_the_golden_covers_every_kind_and_both_verdicts():
    assert len(CASES) > 2500
    assert {o["kind"] for c, _v in CASES if c.get("outputs") for o in c["outputs"] if isinstance(o, dict) and "kind" in o} >= \
        set(mv.KINDS)
    assert sum(rc >= 0 for _c, (rc, _s) in CASES) > 300 and sum(rc == t._lib.E_INVALID for _c, (rc, _s) in CASES) > 2000


def test_loader_verdicts_are_unchanged():
    wrong = []
    for c, want in CASES:
        got = mv.verdict(t._lib.lib, mv.manifest(c))
        if got != want:
            wrong.append((c, want, got))
    assert not wrong, f"{len(wrong)} of {len(CASES)} verdicts changed, first: {wrong[0]}"


def test_packed_output_layout_matches_the_loader():
    accepted = [(c, s) for c, (rc, s) in CASES if rc >= 0 and c.get("outputs")]
    assert accepted
    for c, s in accepted:
        if len({o["k"] for o in c["outputs"] if "k" in o}) > 1:
            continue  # a negative top-k k followed by a valid one: the loader keeps the valid one, the writer never emits this
        got = json.loads(s)
        layout = mf.packed_output_layout(c["outputs"], got["head_n"], got["head_k"])
        assert [(o["name"], o["offset"], o["width"], o["dtype"]) for o in got["outputs"]] == layout, c
        assert got["out_dim"] == sum(w for _n, _o, w, _d in layout), c
