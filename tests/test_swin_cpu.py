"""Swin Transformer bundles, CPU side: every loader refusal of the window_attention and patch_merge ops
(tfsc_manifest_check), the writer for swin_t / swin_s / swin_b, its topology, and the numpy fp64 whole-bundle forward on
exported torchvision weights within 1e-6 of torchvision's fp64 forward."""
import copy
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import swin_export as se  # noqa: E402
import swin_ref as sr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
CLASSIFY = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"},
            {"name": "classes", "kind": "classes"}, {"name": "top_k_classes", "kind": "top_k_classes", "k": 5},
            {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": 5}]
VARIANTS = {"swin_t": {}, "swin_s": dict(depths=(2, 2, 18, 2)), "swin_b": dict(embed_dim=128, heads=(4, 8, 16, 32))}


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _block(wa=None, pm=None, h=14, c=8, heads=2, window=7, shift=3):
    """[h, h, 3c] -> window_attention -> patch_merge -> avgpool -> dense 3"""
    a = {"op": "window_attention", "src": -1, "dst": 0, "h": h, "w": h, "c": 3 * c, "heads": heads, "window": window, "shift": shift}
    a.update(wa or {})
    m = {"op": "patch_merge", "src": 0, "dst": 1, "h": a["h"], "w": a["w"], "c": c}
    m.update(pm or {})
    ops = [a, m, {"op": "avgpool", "src": 1, "dst": 2, "h": m["h"] // 2, "w": m["w"] // 2, "c": 4 * c},
           {"op": "dense", "src": 2, "dst": -2, "h": 1, "w": 1, "c": 4 * c, "cout": 3, "act": "none"}]
    return mf._graph_manifest([a["h"], a["w"], a["c"]], ops, 3)


def _refused(man, why):
    rc, err = _check(man)
    assert rc == t._lib.E_INVALID and why in err, err


def test_the_block_loads():
    rc, res = _check(_block())
    assert rc >= 0 and res["out_dim"] == 3 and res["in_dim"] == 14 * 14 * 24, res


@pytest.mark.parametrize("h,w,c,heads,window,shift", [(56, 56, 96, 3, 7, 0), (56, 56, 96, 3, 7, 3), (7, 7, 768, 24, 7, 0),
                                                      (24, 24, 1024, 32, 12, 6), (12, 36, 384, 12, 12, 11), (14, 28, 64, 2, 7, 1),
                                                      (16, 16, 16, 1, 16, 15), (3, 3, 4, 4, 1, 0), (7, 7, 448, 7, 7, 6),
                                                      (12, 12, 78, 2, 12, 5)])
def test_window_attention_limits_accept(h, w, c, heads, window, shift):
    op = {"op": "window_attention", "src": -1, "dst": -2, "h": h, "w": w, "c": 3 * c, "heads": heads, "window": window, "shift": shift}
    rc, res = _check(mf._graph_manifest([h, w, 3 * c], [op], 1))
    assert rc >= 0 and res["out_dim"] == h * w * c, res


@pytest.mark.parametrize("h,c,heads,window", [(17, 16, 1, 17), (7, 520, 8, 7), (12, 80, 2, 12), (14, 64, 1, 14)])
def test_window_attention_limits_refuse(h, c, heads, window):
    """a window over 16, a head over 64 columns, or K and V of a window beyond 48 KB of shared memory"""
    _refused(_block(wa={"h": h, "w": h, "c": 3 * c, "heads": heads, "window": window, "shift": 0}), "no window_attention kernel for")


def test_window_attention_refusals():
    _refused(_block(wa={"c": 25}), "window_attention expects a packed [h, w, 3C] qkv source (c = 25)")
    _refused(_block(wa={"heads": 3}), "window_attention needs heads that divide C = 8 (heads 3)")
    _refused(_block(wa={"heads": 0}), "window_attention needs heads that divide C = 8 (heads 0)")
    for h, w in ((15, 14), (14, 15), (10, 10)):
        _refused(_block(wa={"h": h, "w": w}, pm={"h": 14, "w": 14}),
                 f"window_attention needs a feature map that is a multiple of the window (h x w = {h} x {w}, window 7)")
    for s in (-1, 7, 8):
        _refused(_block(shift=s), f"window_attention shift {s} is outside [0, window) (h x w = 14 x 14, window 7)")
    for ws in (0, -7):
        _refused(_block(window=ws, shift=0), "no window_attention kernel for")
    _refused(_block(wa={"res": -1}), "window_attention takes no residual input")
    _refused(_block(wa={"act": "gelu"}), "window_attention takes no activation (act 'gelu')")
    man = _block()
    man["ops"][0]["bias_offset"] += 4
    _refused(man, "window_attention bias table out of range or not 256-byte aligned")
    man = _block()
    man["ops"][0]["bias_offset"] = man["weights_bytes"]
    _refused(man, "window_attention bias table out of range or not 256-byte aligned")
    man = _block()
    man["weights_bytes"] = man["ops"][0]["bias_offset"] + 2 * 49 * 49 * 4 - 4
    _refused(man, "window_attention bias table out of range or not 256-byte aligned")
    man = _block()                                                                     # the source holds [14, 14, 24] per image
    man["ops"][0].update(h=7, w=28)
    assert _check(man)[0] >= 0
    man["ops"][0].update(h=7, w=7)
    _refused(man, "op input size does not match its producer")


def test_patch_merge_refusals():
    _refused(_block(pm={"h": 7, "w": 28}), "patch_merge needs an even h and w (h x w = 7 x 28)")
    _refused(_block(pm={"h": 28, "w": 7}), "patch_merge needs an even h and w (h x w = 28 x 7)")
    _refused(_block(pm={"cout": 16}), "patch_merge writes 4c = 32 channels (cout 16)")
    assert _check(_block(pm={"cout": 32}))[0] >= 0
    _refused(_block(pm={"res": -1}), "patch_merge takes no residual input")
    _refused(_block(pm={"act": "relu"}), "patch_merge takes no activation (act 'relu')")
    _refused(_block(pm={"h": 14, "w": 14, "c": 16}), "op input size does not match its producer")
    big = {"op": "patch_merge", "src": -1, "dst": -2, "h": 65536, "w": 65536, "c": 1}
    _refused(mf._graph_manifest([65536, 65536, 1], [big], 1), "no patch_merge kernel for 65536 x 65536 x 1 (h * w * c < 2^31)")


# ------------------------------------------------------------------------------------------------ writer ----
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_writer_is_accepted(variant):
    rc, res = _check(mf.swin_manifest(**VARIANTS[variant]))
    assert rc >= 0 and res["out_dim"] == 1000 and res["in_dim"] == 224 * 224 * 3, res
    rc, res = _check(mf.swin_manifest(classes=21, outputs=CLASSIFY, **VARIANTS[variant]))
    assert rc >= 0 and res["head_n"] == 21 and res["head_k"] == 5, res


def test_swin_b_at_384_with_window_12_is_accepted():
    man = mf.swin_manifest(image=384, embed_dim=128, heads=(4, 8, 16, 32), window=12)
    assert _check(man)[0] >= 0
    assert [(o["h"], o["shift"]) for o in man["ops"] if o["op"] == "window_attention"][-2:] == [(12, 0), (12, 0)]


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_topology(variant):
    kw = VARIANTS[variant]
    depths, heads, dim = kw.get("depths", (2, 2, 6, 2)), kw.get("heads", (3, 6, 12, 24)), kw.get("embed_dim", 96)
    ops = mf.swin_manifest(**kw)["ops"]
    count = {k: sum(o["op"] == k for o in ops) for k in ("conv", "layernorm", "window_attention", "patch_merge", "avgpool", "dense")}
    blocks = sum(depths)
    assert count == {"conv": 1 + 4 * blocks + 3, "layernorm": 1 + 2 * blocks + 3 + 1, "window_attention": blocks, "patch_merge": 3,
                     "avgpool": 1, "dense": 1}
    assert len(ops) == sum(count.values())
    wa = [o for o in ops if o["op"] == "window_attention"]
    stages = [(56 >> s, dim << s, heads[s]) for s, n in enumerate(depths) for _ in range(n)]
    assert [(o["h"], o["w"], o["c"] // 3, o["heads"]) for o in wa] == [(h, h, c, nh) for h, c, nh in stages]
    assert all(o["c"] // 3 // o["heads"] == 32 and o["window"] == 7 for o in wa)
    # odd blocks shift by 3, except at 7 x 7 where the window covers the map (torchvision turns the shift off there)
    assert [o["shift"] for o in wa] == [3 if j % 2 and h > 7 else 0 for (h, _c, _n), j in zip(stages, [j for n in depths for j in range(n)])]
    assert [(o["h"], o["c"]) for o in ops if o["op"] == "patch_merge"] == [(56, dim), (28, 2 * dim), (14, 4 * dim)]
    # each patch merge: LayerNorm(4C), then the reduction 4C -> 2C
    for i, o in enumerate(ops):
        if o["op"] == "patch_merge":
            assert ops[i + 1]["op"] == "layernorm" and ops[i + 1]["c"] == 4 * o["c"]
            assert ops[i + 2]["op"] == "conv" and (ops[i + 2]["c"], ops[i + 2]["cout"]) == (4 * o["c"], 2 * o["c"])
    assert ops[0]["kh"] == ops[0]["stride"] == 4 and ops[0]["pad"] == 0 and ops[0]["cout"] == dim
    assert all(o["eps"] == 1e-5 for o in ops if o["op"] == "layernorm")
    assert max(max(o.get("src", -1), o["dst"]) for o in ops) == 3


# ----------------------------------------------------------------------------------- fp64 restatement ----
def test_ref_ops_on_hand_cases():
    x = np.arange(2 * 4 * 4 * 3, dtype=np.float64).reshape(2, 4, 4, 3)
    y = sr.patch_merge(x)
    assert y.shape == (2, 2, 2, 12)
    assert np.array_equal(y[1, 1, 0], np.concatenate([x[1, 2, 0], x[1, 3, 0], x[1, 2, 1], x[1, 3, 1]]))
    ids = sr.shift_regions(14, 14, 7, 3)
    assert ids[0, 0] == 0 and ids[7, 7] == 4 and ids[11, 11] == 8 and ids[6, 13] == 2 and ids[13, 0] == 6
    # one token per window: the output is v of the same pixel, whatever the shift
    qkv = np.random.default_rng(0).standard_normal((1, 3, 3, 6))
    assert np.allclose(sr.window_attention(qkv, np.zeros((1, 1, 1)), 1, 1, 0), qkv[..., 4:])


@pytest.mark.parametrize("kw,image", [(dict(embed_dim=32, depths=(2, 2), heads=(1, 2)), 56),
                                      (dict(embed_dim=32, depths=(1, 2, 2), heads=(2, 2, 4), window=4), 64),
                                      ({}, 224)])
def test_reference_forward_matches_torchvision(kw, image):
    m = se.torchvision_swin(11, classes=10, **kw)
    man = mf.swin_manifest(image=image, classes=10, **kw)
    assert sum(o["shift"] > 0 for o in man["ops"] if o["op"] == "window_attention") >= 1
    # torchvision's parameters are the bundle's minus the expanded bias tables, plus their compact tables, minus the
    # reductions' zero biases
    bundle = sum(o.get("kh", 1) * o.get("kw", 1) * o["c"] * o["cout"] + o["cout"] for o in man["ops"] if o["op"] in ("conv", "dense"))
    bundle += sum(2 * o["c"] for o in man["ops"] if o["op"] == "layernorm")
    reductions = sum(o["cout"] for i, o in enumerate(man["ops"]) if i >= 2 and man["ops"][i - 2]["op"] == "patch_merge")
    tables = sum(p.numel() for n, p in m.named_parameters() if n.endswith("relative_position_bias_table"))
    assert sum(p.numel() for p in m.parameters()) == bundle - reductions + tables
    blob = se.export_swin(m, copy.deepcopy(man))
    x = se.images(3, image, 13)
    ref = se.reference(m, x)
    got = sr.forward(man, blob, x)
    assert ref.shape == got.shape == (3, 10)
    assert float(np.max(np.abs(got - ref) / np.maximum(1.0, np.abs(ref)))) <= 1e-6
    assert ref.std() > 0.02                                              # not a constant net
