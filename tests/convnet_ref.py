"""numpy fp64 restatement of the image-net graph ops (test infrastructure): depthwise_conv, channel_scale, the relu6 / silu /
sigmoid activations, and a whole-bundle forward over a manifest and its blob (conv, depthwise_conv, channel_scale,
avgpool, dense), so that a served MobileNetV2 / EfficientNet bundle can be pinned to fp64 without the executor's code."""
from __future__ import annotations

import numpy as np

ACTS = {0: "none", 1: "relu", 4: "relu6", 5: "silu", 6: "sigmoid"}


def act(x: np.ndarray, name: str) -> np.ndarray:
    if name == "relu":
        return np.maximum(x, 0.0)
    if name == "relu6":
        return np.minimum(np.maximum(x, 0.0), 6.0)
    if name == "silu":
        return x / (1.0 + np.exp(-x))
    if name == "sigmoid":
        return 1.0 / (1.0 + np.exp(-x))
    if name == "tanh":
        return np.tanh(x)
    assert name == "none", name
    return x


def _taps(x, kh, kw, stride, pad):
    """(i, j, x[:, i::stride, j::stride, :] of the zero-padded input, OH x OW) for every tap of a kh x kw window"""
    b, h, w, c = x.shape
    oh, ow = (h + 2 * pad - kh) // stride + 1, (w + 2 * pad - kw) // stride + 1
    xp = np.zeros((b, h + 2 * pad, w + 2 * pad, c), np.float64)
    xp[:, pad:pad + h, pad:pad + w] = x
    for i in range(kh):
        for j in range(kw):
            yield i, j, xp[:, i:i + stride * (oh - 1) + 1:stride, j:j + stride * (ow - 1) + 1:stride]


def depthwise_conv(x, w, bias, stride, pad, act_name="none"):
    """x [B, H, W, C], w [kh, kw, C], bias [C] -> act(y) [B, OH, OW, C] in fp64"""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    y = sum(xs * w[i, j] for i, j, xs in _taps(x, w.shape[0], w.shape[1], stride, pad))
    return act(y + np.asarray(bias, np.float64), act_name)


def conv(x, w, bias, stride, pad, act_name="none", res=None):
    """x [B, H, W, C], w [kh, kw, C, cout] (HWIO) -> act(conv + bias (+ res)) [B, OH, OW, cout] in fp64"""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    y = sum(xs @ w[i, j] for i, j, xs in _taps(x, w.shape[0], w.shape[1], stride, pad)) + np.asarray(bias, np.float64)
    return act(y if res is None else y + res, act_name)


def channel_scale(x, gate):
    """x [B, H, W, C] * gate [B, C] per channel"""
    return np.asarray(x, np.float64) * np.asarray(gate, np.float64).reshape(len(x), 1, 1, -1)


def forward(man: dict, blob: np.ndarray, x: np.ndarray) -> np.ndarray:
    """fp64 forward of a float-input graph bundle built from conv, depthwise_conv, channel_scale, avgpool and dense ops:
    the logits [B, N] of the op that writes the response"""
    blob = np.asarray(blob, np.float32)
    bufs = {-1: np.asarray(x, np.float64).reshape(len(x), *man["input_shape"])}
    B = len(x)

    def tensor(off, n):
        return blob[off // 4: off // 4 + n].astype(np.float64)

    for o in man["ops"]:
        src = bufs[o.get("src", -1)]
        h, w, c = o.get("h", 1), o.get("w", 1), o["c"]
        kind, a = o["op"], o.get("act", "none")
        res = bufs[o["res"]] if "res" in o else None
        if kind == "conv":
            kh, kw, cout, s, p = o.get("kh", 1), o.get("kw", 1), o["cout"], o.get("stride", 1), o.get("pad", 0)
            wt = tensor(o["w_offset"], kh * kw * c * cout).reshape(kh, kw, c, cout)
            oh, ow = (h + 2 * p - kh) // s + 1, (w + 2 * p - kw) // s + 1
            y = conv(src.reshape(B, h, w, c), wt, tensor(o["b_offset"], cout), s, p, a,
                     None if res is None else res.reshape(B, oh, ow, cout))
        elif kind == "depthwise_conv":
            kh, kw = o["kh"], o["kw"]
            y = depthwise_conv(src.reshape(B, h, w, c), tensor(o["w_offset"], kh * kw * c).reshape(kh, kw, c), tensor(o["b_offset"], c),
                               o.get("stride", 1), o.get("pad", 0), a)
        elif kind == "channel_scale":
            y = channel_scale(src.reshape(B, h, w, c), bufs[o["gate"]].reshape(B, c))
        elif kind == "avgpool":
            y = src.reshape(B, h * w, c).mean(axis=1).reshape(B, 1, 1, c)
        elif kind == "dense":
            cout = o["cout"]
            y = src.reshape(B, -1)[:, :c] @ tensor(o["w_offset"], c * cout).reshape(c, cout) + tensor(o["b_offset"], cout)
            y = act(y if res is None else y + res.reshape(B, cout), a).reshape(B, 1, 1, cout)
        else:
            raise ValueError(f"convnet_ref has no op '{kind}'")
        bufs[o["dst"]] = y
    return bufs[-2].reshape(B, -1)
