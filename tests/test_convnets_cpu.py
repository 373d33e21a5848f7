"""MobileNetV2 / EfficientNet bundles, CPU side: every loader refusal of the depthwise_conv and channel_scale ops
(tfsc_manifest_check), the limits of depthwise_supported, both manifest writers across image sizes and multipliers, and the
numpy fp64 whole-bundle forward on exported torchvision weights within 1e-6 of torchvision's fp64 forward."""
import copy
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import convnet_export as ce  # noqa: E402
import convnet_ref as cr  # noqa: E402

mf = t.modelformat
lib = t._lib.lib
CLASSIFY = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"},
            {"name": "classes", "kind": "classes"}, {"name": "top_k_classes", "kind": "top_k_classes", "k": 5},
            {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": 5}]


def _check(man: dict):
    buf = C.create_string_buffer(1 << 16)
    rc = lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return (rc, json.loads(buf.value)) if rc >= 0 else (rc, lib.tfsc_last_error().decode())


def _se_block(dw=None, scale=None):
    """[8, 8, 4] -> depthwise 3x3 relu6 -> SE (avgpool, 1x1 4 -> 2 silu, 1x1 2 -> 4 sigmoid, channel_scale) -> pool -> dense 3"""
    d = {"op": "depthwise_conv", "src": -1, "dst": 0, "h": 8, "w": 8, "c": 4, "kh": 3, "kw": 3, "stride": 1, "pad": 1, "act": "relu6"}
    d.update(dw or {})
    oh = (d["h"] + 2 * d["pad"] - d["kh"]) // d["stride"] + 1
    s = {"op": "channel_scale", "src": 0, "gate": 1, "dst": 2, "h": oh, "w": oh, "c": 4}
    s.update(scale or {})
    ops = [d, {"op": "avgpool", "src": 0, "dst": 1, "h": oh, "w": oh, "c": 4},
           {"op": "conv", "src": 1, "dst": 3, "h": 1, "w": 1, "c": 4, "cout": 2, "act": "silu"},
           {"op": "conv", "src": 3, "dst": 1, "h": 1, "w": 1, "c": 2, "cout": 4, "act": "sigmoid"}, s,
           {"op": "avgpool", "src": 2, "dst": 3, "h": s["h"], "w": s["w"], "c": 4},
           {"op": "dense", "src": 3, "dst": -2, "h": 1, "w": 1, "c": 4, "cout": 3, "act": "none"}]
    return mf._graph_manifest([d["h"], d["w"], 4], ops, 4)


def _refused(man, why):
    rc, err = _check(man)
    assert rc == t._lib.E_INVALID and why in err, err


def test_the_se_block_loads():
    rc, res = _check(_se_block())
    assert rc >= 0 and res["out_dim"] == 3


@pytest.mark.parametrize("k,stride,pad,h", [(1, 1, 0, 1), (3, 2, 1, 7), (5, 2, 2, 113), (7, 1, 3, 7), (7, 2, 3, 1), (7, 2, 0, 7),
                                            (2, 1, 1, 8), (4, 2, 2, 9)])
def test_depthwise_limits_accept(k, stride, pad, h):
    assert _check(_se_block(dw={"kh": k, "kw": k, "stride": stride, "pad": pad, "h": h, "w": h}))[0] >= 0


@pytest.mark.parametrize("k,stride,pad,h", [(8, 1, 0, 8), (3, 3, 1, 8), (3, 1, 2, 8), (7, 1, 4, 8), (1, 1, 1, 8), (5, 1, 0, 4)])
def test_depthwise_limits_refuse(k, stride, pad, h):
    _refused(_se_block(dw={"kh": k, "kw": k, "stride": stride, "pad": pad, "h": h, "w": h}), "no depthwise_conv kernel for")


def test_depthwise_refusals():
    _refused(_se_block(dw={"cout": 8}), "depthwise_conv writes its c = 4 channels (cout 8)")
    _refused(_se_block(dw={"res": -1}), "depthwise_conv takes no residual input")
    for act in ("gelu", "tanh", "swish", "hard_swish", ""):
        _refused(_se_block(dw={"act": act}), f"depthwise_conv act '{act}' is not none, relu, relu6, silu or sigmoid")
    for act in ("none", "relu", "relu6", "silu", "sigmoid"):
        assert _check(_se_block(dw={"act": act}))[0] >= 0
    man = _se_block()
    man["ops"][0]["w_offset"] += 4
    _refused(man, "weights out of range or misaligned")
    man = _se_block()
    man["ops"][0]["b_offset"] = man["weights_bytes"]
    _refused(man, "weights out of range or misaligned")
    man = _se_block()
    man["weights_bytes"] = man["ops"][0]["w_offset"] + 3 * 3 * 4 * 4 - 4
    _refused(man, "weights out of range or misaligned")


def test_channel_scale_refusals():
    why = "channel_scale needs a gate that an earlier op wrote to a scratch buffer with c = 4 values per image"
    _refused(_se_block(scale={"gate": -1}), why + " (gate -1)")                     # the request tensor
    _refused(_se_block(scale={"gate": 0}), why + " (gate 0)")                       # [8, 8, 4] per image, not [4]
    _refused(_se_block(scale={"gate": 7}), why + " (gate 7)")                       # no such buffer
    man = _se_block(scale={"gate": 3})                                                  # written with 2 values
    _refused(man, why + " (gate 3)")
    man = _se_block()
    del man["ops"][4]["gate"]
    _refused(man, why + " (gate -100)")
    _refused(_se_block(scale={"dst": 1}), "channel_scale cannot write its gate buffer (gate == dst == 1)")
    _refused(_se_block(scale={"h": 4, "w": 4}), "channel_scale reads 256 values per image, not h * w * c = 64")
    _refused(_se_block(scale={"act": "sigmoid"}), "channel_scale takes no activation (act 'sigmoid')")
    _refused(_se_block(scale={"act": "bogus"}), "channel_scale takes no activation (act 'bogus')")
    _refused(_se_block(scale={"res": 0}), "channel_scale takes no residual input")


def test_existing_ops_keep_reading_unknown_acts_as_none():
    man = _se_block()
    man["ops"][2]["act"] = "swish"
    assert _check(man)[0] >= 0


def _depthwise_shapes(man):
    return sorted({(o["c"], o["h"], o["kh"], o["stride"], o["pad"]) for o in man["ops"] if o["op"] == "depthwise_conv"},
                  key=lambda s: (s[1] * -1, s[0], s[2], s[3]))


def test_mobilenet_v2_topology():
    man = mf.mobilenet_v2_manifest()
    ops = man["ops"]
    assert sum(o["op"] in ("conv", "depthwise_conv") for o in ops) == 52 and sum(o["op"] == "depthwise_conv" for o in ops) == 17
    assert set(_depthwise_shapes(man)) == {(32, 112, 3, 1, 1), (96, 112, 3, 2, 1), (144, 56, 3, 1, 1), (144, 56, 3, 2, 1),
                                           (192, 28, 3, 1, 1), (192, 28, 3, 2, 1), (384, 14, 3, 1, 1), (576, 14, 3, 1, 1),
                                           (576, 14, 3, 2, 1), (960, 7, 3, 1, 1)}
    assert {o.get("act") for o in ops if o["op"] != "avgpool"} == {"relu6", "none"}
    assert sum("res" in o for o in ops) == 10


def test_efficientnet_b0_topology():
    man = mf.efficientnet_manifest()
    ops = man["ops"]
    assert sum(o["op"] in ("conv", "depthwise_conv") for o in ops) == 81 and sum(o["op"] == "depthwise_conv" for o in ops) == 16
    assert sum(o["op"] == "channel_scale" for o in ops) == 16
    assert set(_depthwise_shapes(man)) == {(32, 112, 3, 1, 1), (96, 112, 3, 2, 1), (144, 56, 3, 1, 1), (144, 56, 5, 2, 2),
                                           (240, 28, 3, 2, 1), (240, 28, 5, 1, 2), (480, 14, 3, 1, 1), (480, 14, 5, 1, 2),
                                           (672, 14, 5, 1, 2), (672, 14, 5, 2, 2), (1152, 7, 3, 1, 1), (1152, 7, 5, 1, 2)}
    assert {o.get("act") for o in ops if o["op"] not in ("avgpool", "channel_scale")} == {"silu", "sigmoid", "none"}


@pytest.mark.parametrize("image", [32, 64, 97, 224, 260])
@pytest.mark.parametrize("width", [0.35, 0.5, 1.0, 1.4])
def test_mobilenet_v2_writer_is_accepted(image, width):
    rc, res = _check(mf.mobilenet_v2_manifest(image=image, classes=17, width_mult=width))
    assert rc >= 0 and res["out_dim"] == 17 and res["in_dim"] == image * image * 3, res
    rc, res = _check(mf.mobilenet_v2_manifest(image=image, classes=1000, width_mult=width, outputs=CLASSIFY))
    assert rc >= 0 and res["head_n"] == 1000 and res["head_k"] == 5, res


# torchvision's (width_mult, depth_mult) of B0-B7, and reduced variants
@pytest.mark.parametrize("width,depth", [(1.0, 1.0), (1.0, 1.1), (1.1, 1.2), (1.2, 1.4), (1.4, 1.8), (1.6, 2.2), (1.8, 2.6),
                                         (2.0, 3.1), (0.5, 0.5), (0.25, 0.34)])
@pytest.mark.parametrize("image", [64, 224, 300])
def test_efficientnet_writer_is_accepted(width, depth, image):
    rc, res = _check(mf.efficientnet_manifest(image=image, classes=1000, width_mult=width, depth_mult=depth, outputs=CLASSIFY))
    assert rc >= 0 and res["head_n"] == 1000 and res["in_dim"] == image * image * 3, res


def test_efficientnet_b7_depths():
    man = mf.efficientnet_manifest(image=600, width_mult=2.0, depth_mult=3.1)
    assert sum(o["op"] == "depthwise_conv" for o in man["ops"]) == sum(int(np.ceil(n * 3.1)) for n in (1, 2, 2, 3, 3, 4, 1))


# ----------------------------------------------------------------------------------- fp64 restatement ----
def test_depthwise_ref_on_a_hand_case():
    x = np.arange(2 * 3 * 3 * 2, dtype=np.float64).reshape(2, 3, 3, 2)
    w = np.zeros((3, 3, 2))
    w[1, 1, 0], w[0, 0, 1] = 2.0, 1.0                                   # channel 0: 2 * centre; channel 1: the top-left tap
    y = cr.depthwise_conv(x, w, np.array([0.5, -1.0]), 1, 1)
    assert np.array_equal(y[..., 0], 2 * x[..., 0] + 0.5)
    assert y[0, 0, 0, 1] == -1.0 and y[0, 1, 1, 1] == x[0, 0, 0, 1] - 1.0
    assert np.array_equal(cr.depthwise_conv(x, w, np.zeros(2), 2, 1).shape, (2, 2, 2, 2))
    assert np.allclose(cr.act(np.array([-1.0, 3.0, 7.0]), "relu6"), [0, 3, 6])
    assert np.allclose(cr.act(np.array([0.0]), "silu"), [0]) and np.allclose(cr.act(np.array([0.0]), "sigmoid"), [0.5])
    g = np.array([[2.0, 0.5], [1.0, -1.0]])
    assert np.array_equal(cr.channel_scale(x, g), x * g[:, None, None, :])


@pytest.mark.parametrize("net,image,classes,width,depth", [("mobilenet_v2", 224, 1000, 1.0, 1.0), ("efficientnet", 224, 1000, 1.0, 1.0),
                                                           ("mobilenet_v2", 64, 10, 0.35, 1.0), ("efficientnet", 64, 10, 0.5, 0.5)])
def test_reference_forward_matches_torchvision(net, image, classes, width, depth):
    if net == "mobilenet_v2":
        m = ce.torchvision_mobilenet_v2(11, width, classes)
        man = mf.mobilenet_v2_manifest(image, classes, width)
    else:
        m = ce.torchvision_efficientnet(12, width, depth, classes)
        man = mf.efficientnet_manifest(image, classes, width, depth)
    # torchvision's parameters are the bundle's (BatchNorm folded: one bias per channel) plus one more per BatchNorm channel
    bundle = sum(o["kh"] * o["kw"] * o["c"] * (o["cout"] if o["op"] == "conv" else 1) + o.get("cout", o["c"])
                 for o in man["ops"] if o["op"] in ("conv", "depthwise_conv")) + sum(o["c"] * o["cout"] + o["cout"] for o in man["ops"] if o["op"] == "dense")
    bn = sum(b.num_features for b in m.modules() if type(b).__name__ == "BatchNorm2d")
    assert sum(p.numel() for p in m.parameters()) == bundle + bn
    blob = ce.export_convnet(m, copy.deepcopy(man))
    x = ce.images(3, image, 13)
    ref = ce.reference(m, x)
    got = cr.forward(man, blob, x)
    assert ref.shape == got.shape == (3, classes)
    assert float(np.max(np.abs(got - ref) / np.maximum(1.0, np.abs(ref)))) <= 1e-6
    assert ref.std() > 0.02                                              # not a constant net
