"""Generates tests/golden/manifest_verdicts.json: the loader's verdict on manifests that declare signature.outputs, as
tfsc_manifest_check returns it -- the return code and either the packed layout JSON or the error text. Each case is a
recipe, not a manifest: a base bundle written by modelformat (BASES), the outputs to declare, and edits to its ops or
top-level fields (apply_edits). The recipes are cases() below; the golden holds each distinct verdict once, the verdict of
every case in case order, and a digest of the case list. tests/test_manifest_verdicts.py rebuilds every manifest from
its recipe and requires the same return code and the same string, so a change to the loader cannot move a message or
change which of several faults is reported without changing the golden. A change to cases() needs a golden regenerated
from a build of the loader the cases were pinned against.

The cases cover every kind alone, every ordered pair of kinds, every kind with each of the entry fields k,
max_answer_length, sep_id and normalize set to a spread of values, pairs whose second entry carries a faulty field, two
entries of one family that disagree, and the bundle-shape edits of the test_*_cpu.py suites.

    python tests/golden/make_manifest_verdicts.py [path/to/libtfsc_b200.so]

The library defaults to the package's build, tfservingcache_b200/libtfsc_b200.so.
"""
import copy
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tfservingcache_b200 import modelformat as mf  # noqa: E402

SMALL = dict(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, max_pos=512, labels=3)
INPUTS = {"none": None, "bert": mf.BERT_INPUTS, "bert2": mf.BERT_INPUTS[:2]}


def _bert(head, **kw):
    arch = dict(SMALL, inputs="bert")
    arch.update(kw)
    arch["inputs"] = INPUTS[arch["inputs"]]
    return mf.bert_manifest(**arch, head=head)


def _mlp(labels=10):
    with tempfile.TemporaryDirectory() as d:
        import numpy as np
        return mf.write_mlp_bundle(d, [np.zeros((8, 16), np.float32), np.zeros((16, labels), np.float32)],
                                   [np.zeros(16, np.float32), np.zeros(labels, np.float32)])


def _affine():
    with tempfile.TemporaryDirectory() as d:
        return mf.write_affine_bundle(d, 2.0, 3.0)


BASES = {
    "mlp": _mlp,                                                        # 10 logits
    "affine": _affine,
    "resnet": lambda **kw: mf.resnet50_manifest(**dict(dict(image=32, classes=10, width=8, blocks=(1, 1, 1, 1)), **kw)),
    "bert": lambda **kw: _bert("classify", **dict(dict(inputs="none"), **kw)),
    "bert_in": lambda **kw: _bert("classify", **kw),
    "qa": lambda **kw: _bert("span", **kw),
    "enc": lambda **kw: _bert("encoder", **kw),
    "enc_nopool": lambda **kw: _bert("encoder", pooler=False, **kw),
    "mlm": lambda **kw: _bert("mlm", **dict(dict(slots=3, mask_token_id=4), **kw)),
}

CLASSIFY = ["logits", "probabilities", "classes", "top_k_classes", "top_k_probabilities"]
SPAN = ["start_logits", "end_logits", "span_starts", "span_ends", "span_scores"]
ENCODER = ["sequence_output", "pooled_output", "cls_embedding", "mean_embedding"]
MLM = ["masked_positions", "masked_top_k_ids", "masked_top_k_probabilities", "masked_top_k_logits"]
FAMILIES = {"mlp": CLASSIFY, "qa": SPAN, "enc": ENCODER, "mlm": MLM}
KINDS = CLASSIFY + SPAN + ENCODER + MLM
HOME = {k: base for base, kinds in FAMILIES.items() for k in kinds}      # the base a kind is served by
TOPK = {"top_k_classes", "top_k_probabilities", "masked_top_k_ids", "masked_top_k_probabilities", "masked_top_k_logits"}
SPAN_RESULT = ("span_starts", "span_ends", "span_scores")
FIELDS = ("k", "max_answer_length", "sep_id", "normalize")
ABSENT = "<absent>"
VALUES = (ABSENT, 0, 1, 5, -1, 2.5, True, "x")
FAULTY = {"k": 2.5, "max_answer_length": -1, "sep_id": -1, "normalize": "x"}


def entry(kind, name=None, **fields):
    """A well-formed signature.outputs entry of `kind` (k = 3, max_answer_length = 5 where the kind takes them), with
    `fields` set on top (ABSENT deletes one)."""
    e = {"name": name or kind, "kind": kind}
    if kind in TOPK or kind in SPAN_RESULT:
        e["k"] = 3
    if kind in SPAN_RESULT:
        e["max_answer_length"] = 5
    for f, v in fields.items():
        if v == ABSENT:
            e.pop(f, None)
        else:
            e[f] = v
    return e


def apply_edits(man, edits):
    """Edits, in order: ["op", i, key, value] sets ops[i][key] (value None deletes it); ["cut", i] keeps ops[:i];
    ["insert", i, j, {overrides}] inserts a copy of ops[j] with overrides (None deletes a key) before ops[i]; ["top", key,
    value] sets a top-level field (None deletes it); ["add", key, delta] adds to one; ["sig", key, value] sets a signature
    field (None deletes it)."""
    for e in edits:
        if e[0] == "op":
            _set(man["ops"][e[1]], e[2], e[3])
        elif e[0] == "cut":
            man["ops"] = man["ops"][:e[1]]
        elif e[0] == "insert":
            op = dict(man["ops"][e[2]])
            for k, v in e[3].items():
                _set(op, k, v)
            man["ops"].insert(e[1], op)
        elif e[0] == "top":
            _set(man, e[1], e[2])
        elif e[0] == "add":
            man[e[1]] += e[2]
        elif e[0] == "sig":
            _set(man["signature"], e[1], e[2])
        else:
            raise ValueError(f"unknown edit {e!r}")
    return man


def _set(d, k, v):
    if v is None:
        d.pop(k, None)
    else:
        d[k] = v


_base_cache = {}


def manifest(case):
    """The manifest a case's recipe describes: {"base": name or [name, {kwargs}], "outputs": list or None, "edits": [...]}."""
    base = case["base"]
    name, kw = (base, {}) if isinstance(base, str) else base
    key = json.dumps([name, kw], sort_keys=True)
    if key not in _base_cache:
        _base_cache[key] = BASES[name](**kw)
    man = copy.deepcopy(_base_cache[key])
    if case.get("outputs") is not None:
        sig = {k: v for k, v in man["signature"].items() if k != "output"}
        sig["outputs"] = case["outputs"]
        man["signature"] = sig
    return apply_edits(man, case.get("edits", []))


def cases():
    out = []

    def add(base, outputs, edits=()):
        out.append({"base": base, "outputs": outputs, "edits": list(edits)})

    # every kind alone, on every base
    for base in BASES:
        for k in KINDS:
            add(base, [entry(k)])
    # every ordered pair, on the first kind's base
    for a in KINDS:
        for b in KINDS:
            if a != b:
                add(HOME[a], [entry(a), entry(b)])
    # each family whole, in both orders, on every base
    for base in BASES:
        for kinds in FAMILIES.values():
            add(base, [entry(k) for k in kinds])
            add(base, [entry(k) for k in reversed(kinds)])
    # every kind with each entry field set to each value, on its base
    seen = set()
    for k in KINDS:
        for f in FIELDS:
            for v in VALUES:
                c = {"base": HOME[k], "outputs": [entry(k, **{f: v})], "edits": []}
                if json.dumps(c) not in seen:                          # json: 1 and True are different values
                    seen.add(json.dumps(c))
                    out.append(c)
    # a pair whose second entry carries one faulty field: which message wins
    for a in KINDS:
        for b in KINDS:
            if a != b:
                for f in FIELDS:
                    add(HOME[a], [entry(a), entry(b, **{f: FAULTY[f]})])
    # a stray normalize: true after each kind
    for a in KINDS:
        for b in KINDS:
            if a != b:
                add(HOME[a], [entry(a), entry(b, normalize=True)])
    # two entries of one family that disagree (or agree in another spelling)
    for a, b in (("top_k_classes", "top_k_probabilities"), ("top_k_probabilities", "top_k_classes")):
        for va, vb in ((3, 4), (3, 3.0), (-1, 3), (3, -1), (0, 0), (-2, -2), (3, ABSENT)):
            add("mlp", [entry(a, k=va), entry(b, k=vb)])
    for a in SPAN_RESULT:
        for b in SPAN_RESULT:
            if a != b:
                for f, va, vb in (("k", 3, 4), ("k", -1, -1), ("k", 0, 0), ("max_answer_length", 5, 6),
                                  ("max_answer_length", 0, 0), ("sep_id", 102, ABSENT), ("sep_id", ABSENT, 102),
                                  ("sep_id", 102, 103), ("sep_id", 102, 102), ("sep_id", 0, 0)):
                    add("qa", [entry(a, **{f: va}), entry(b, **{f: vb})])
    for a in ("masked_top_k_ids", "masked_top_k_probabilities", "masked_top_k_logits"):
        for b in ("masked_top_k_ids", "masked_top_k_probabilities", "masked_top_k_logits"):
            if a != b:
                for va, vb in ((3, 4), (-3, 3), (3, 3.0), (100, 100), (32, 32), (33, 33)):
                    add("mlm", [entry(a, k=va), entry(b, k=vb)])
    for va, vb in ((True, False), (False, True), (True, True), (1, True), (True, "true")):
        add("enc", [entry("cls_embedding", normalize=va), entry("mean_embedding", normalize=vb)])
        add("enc", [entry("mean_embedding", normalize=va), entry("cls_embedding", normalize=vb)])
    # malformed lists and entries
    for outs in ([], [entry(k) for k in CLASSIFY] + [entry("logits", name="l2")], ["logits"], [{"kind": "logits"}],
                 [{"name": "", "kind": "logits"}], [{"name": "a", "kind": "softmax"}], [{"name": "a"}],
                 [entry("logits"), entry("logits", name="other")], [entry("logits"), entry("probabilities", name="logits")],
                 [entry("logits", name="x")], [entry("start_logits", name="input_ids")], [entry("logits", name="input_ids")]):
        for base in ("mlp", "qa", "bert", "bert_in"):
            add(base, outs)
    add("mlp", [entry("logits")], [["sig", "output", "y"]])
    add("mlp", None, [["sig", "outputs", {"name": "a", "kind": "logits"}]])
    # limits: N, k, S, max_answer_length, H, M, vocab
    for labels in (1, 2, 3, 32768, 32769):
        for k in (1, 2, 3, 32, 33):
            add(["mlp", {"labels": labels}], [entry("top_k_classes", k=k)])
            add(["bert", {"labels": labels}], [entry("logits"), entry("top_k_probabilities", k=k)])
        add(["mlp", {"labels": labels}], [entry("logits")])
    for seq, k, L in ((1, 1, 1), (16, 0, 5), (16, 33, 5), (16, -1, 5), (16, 5, 0), (16, 5, 17), (16, 32, 16),
                      (4096, 32, 4096), (4097, 5, 30)):
        add(["qa", {"seq": seq, "max_pos": max(512, seq)}], [entry("start_logits"), entry("span_ends", k=k, max_answer_length=L)])
    add(["qa", {"seq": 4097, "max_pos": 4097}], [entry("start_logits"), entry("end_logits")])
    add(["qa", {"seq": 4097, "max_pos": 4097}], None)
    for seq, hidden, heads in ((1, 64, 4), (8192, 64, 4), (8193, 64, 4), (16, 8192, 64), (16, 8200, 82)):
        kw = {"seq": seq, "hidden": hidden, "heads": heads, "max_pos": max(512, seq), "vocab": 4, "inter": 8}
        add(["enc_nopool", kw], [entry("sequence_output"), entry("mean_embedding")])
    add(["enc", {"seq": 1}], [entry(k) for k in ENCODER])
    for vocab, k in ((1, 1), (32768, 32), (32769, 5), (100, 33), (4, 5), (5, 5)):
        kw = {"vocab": vocab, "hidden": 32, "inter": 8, "mask_token_id": min(4, vocab - 1) if vocab > 1 else 1}
        add(["mlm", kw], [entry("masked_top_k_ids", k=k)])
    for seq, slots in ((16, 1), (16, 16), (1, 1), (16, 17), (16, 0)):
        add(["mlm", {"seq": seq, "slots": slots}], [entry(k) for k in MLM])
        add(["mlm", {"seq": seq, "slots": slots}], [entry("masked_positions")])
    for tok in (0, -1, 1, 99, 100, 1000):
        add(["mlm", {"mask_token_id": tok}], [entry("masked_positions")])
    # bundle shapes: the base bundles' structural checks
    for base in ("qa", "enc", "enc_nopool", "mlm"):
        for inputs in ("none", "bert2"):
            for kinds in FAMILIES.values():
                add([base, {"inputs": inputs}], [entry(k) for k in kinds])
    add("qa", [entry(k) for k in SPAN], [["op", -1, "cout", 3]])
    add("qa", [entry(k) for k in SPAN], [["op", -1, "h", 8]])
    add("enc", [entry(k) for k in ENCODER], [["op", -1, "act", "none"]])
    add("enc", [entry(k) for k in ENCODER], [["op", -1, "cout", 32], ["add", "weights_bytes", 1 << 20]])
    add("enc", [entry(k) for k in ENCODER], [["insert", -1, -2, {"src": 0, "dst": 2, "res": None}]])
    add("enc", [entry("cls_embedding")], [["insert", -1, -2, {"src": 0, "dst": 2, "res": None}]])
    add("enc", [entry("pooled_output")], [["op", -1, "src", 2], ["op", -2, "dst", 2]])
    add("enc_nopool", [entry("cls_embedding")], [["op", -1, "c", 32]])
    for outs in (None, [entry("logits")], [entry("sequence_output")], [entry("start_logits")], [entry("masked_positions")]):
        add("mlm", outs)
    add("mlm", [entry(k) for k in MLM], [["op", -4, "h", 32], ["op", -4, "c", 32], ["op", -3, "c", 32]])
    add("mlm", [entry(k) for k in MLM], [["op", -4, "src", 3], ["op", -5, "dst", 3]])
    add("mlm", [entry(k) for k in MLM], [["op", -4, "slots", 0]])
    add("mlm", [entry(k) for k in MLM], [["op", -4, "slots", 17]])
    add("mlm", [entry(k) for k in MLM], [["op", -1, "cout", 96]])
    add("mlm", [entry(k) for k in MLM], [["cut", -1], ["op", -1, "dst", -2]])
    add("mlm", [entry(k) for k in MLM], [["insert", -3, -4, {"src": 0, "dst": 3}]])
    add(["mlm", {"vocab": 96}], [entry(k) for k in MLM])
    for base in ("bert", "bert_in", "resnet"):
        add(base, [entry("masked_positions")], [["insert", 1, 0, {"op": "mask_gather", "src": 0, "dst": 1, "slots": 1}]])
    add("qa", [entry("logits")])
    add("qa", [entry("top_k_classes", k=2)])
    return out


def verdict(lib, man):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return rc, (buf.value if rc >= 0 else lib.tfsc_last_error()).decode()


def load(path):
    lib = C.CDLL(path)
    lib.tfsc_manifest_check.restype = C.c_int
    lib.tfsc_manifest_check.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    lib.tfsc_last_error.restype = C.c_char_p
    return lib


def recipes_digest(cs):
    """sha256 of the case list: the golden's verdicts are stored in this order"""
    return hashlib.sha256(json.dumps(cs, sort_keys=True).encode()).hexdigest()


if __name__ == "__main__":
    lib = load(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tfservingcache_b200", "libtfsc_b200.so"))
    cs = cases()
    results, index, verdicts = [], {}, []
    for c in cs:
        v = verdict(lib, manifest(c))
        if v not in index:                                             # many cases share a verdict: store each once
            index[v] = len(results)
            results.append(v)
        verdicts.append(index[v])
    rows = [", ".join(map(str, verdicts[i:i + 40])) for i in range(0, len(verdicts), 40)]
    with open(os.path.join(HERE, "manifest_verdicts.json"), "w") as f:
        f.write('{"recipes_sha256": "%s",\n"results": [\n' % recipes_digest(cs) +
                ",\n".join(json.dumps(list(v)) for v in results) + '\n],\n"verdicts": [\n' + ",\n".join(rows) + "\n]}\n")
    print(len(cs), "cases,", sum(results[i][0] >= 0 for i in verdicts), "accepted,", len(results), "distinct verdicts")
