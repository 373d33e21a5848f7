"""numpy fp64 restatement of the Swin graph ops (test infrastructure): window_attention, patch_merge and LayerNorm, and a
whole-bundle forward over a manifest and its blob that takes conv, avgpool and dense from convnet_ref. The attention
follows torchvision's steps (roll, window partition, attention, reverse partition, roll back) rather than the kernel's
addressing, so that a served Swin bundle and the raw kernels can be pinned to fp64 without the executor's code."""
from __future__ import annotations

import numpy as np
from scipy.special import erf

import convnet_ref as cr


def gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def layernorm(x, gamma, beta, eps):
    """over the last axis, biased variance"""
    x = np.asarray(x, np.float64)
    mu = x.mean(axis=-1, keepdims=True)
    return (x - mu) / np.sqrt(((x - mu) ** 2).mean(axis=-1, keepdims=True) + eps) * gamma + beta


def shift_regions(H, W, ws, s):
    """torchvision's shift-mask region id of every position of the rolled map [H, W]"""
    ids = np.zeros((H, W), np.int64)
    for i, (h0, h1) in enumerate(((0, H - ws), (H - ws, H - s), (H - s, H))):
        for j, (w0, w1) in enumerate(((0, W - ws), (W - ws, W - s), (W - s, W))):
            ids[h0:h1, w0:w1] = 3 * i + j
    return ids


def _partition(x, ws):
    """[B, H, W, ...] -> [B, nW, ws * ws, ...] (windows row-major, tokens row-major within a window)"""
    B, H, W = x.shape[:3]
    rest = x.shape[3:]
    x = x.reshape(B, H // ws, ws, W // ws, ws, *rest)
    return np.moveaxis(x, 3, 2).reshape(B, (H // ws) * (W // ws), ws * ws, *rest)


def window_attention(qkv, bias, heads, ws, shift):
    """qkv [B, H, W, 3C] (q | k | v), bias [heads, N, N] -> ctx [B, H, W, C] in fp64"""
    qkv, bias = np.asarray(qkv, np.float64), np.asarray(bias, np.float64)
    B, H, W, C3 = qkv.shape
    C = C3 // 3
    d, N = C // heads, ws * ws
    x = _partition(np.roll(qkv, (-shift, -shift), axis=(1, 2)), ws)              # [B, nW, N, 3C]
    x = x.reshape(B, -1, N, 3, heads, d).transpose(3, 0, 1, 4, 2, 5)              # [3, B, nW, heads, N, d]
    q, k, v = x
    s = q @ np.swapaxes(k, -1, -2) / np.sqrt(d) + bias
    if shift:
        ids = _partition(shift_regions(H, W, ws, shift)[None], ws)[0]             # [nW, N]
        s = s + np.where(ids[:, :, None] != ids[:, None, :], -100.0, 0.0)[None, :, None]
    p = np.exp(s - s.max(axis=-1, keepdims=True))
    o = (p / p.sum(axis=-1, keepdims=True)) @ v                                   # [B, nW, heads, N, d]
    o = o.transpose(0, 1, 3, 2, 4).reshape(B, H // ws, W // ws, ws, ws, C)
    o = o.transpose(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)
    return np.roll(o, (shift, shift), axis=(1, 2))


def patch_merge(x):
    """[B, H, W, C] -> [B, H/2, W/2, 4C]: x0 | x1 | x2 | x3 as torchvision's PatchMerging"""
    return np.concatenate([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], axis=-1)


def forward(man: dict, blob: np.ndarray, x: np.ndarray) -> np.ndarray:
    """fp64 forward of a float-input graph bundle built from conv, layernorm, window_attention, patch_merge, avgpool and
    dense ops: the logits [B, N] of the op that writes the response"""
    blob = np.asarray(blob, np.float32)
    B = len(x)
    bufs = {-1: np.asarray(x, np.float64).reshape(B, *man["input_shape"])}

    def tensor(off, n):
        return blob[off // 4: off // 4 + n].astype(np.float64)

    for o in man["ops"]:
        src = bufs[o.get("src", -1)]
        h, w, c = o.get("h", 1), o.get("w", 1), o["c"]
        kind, a = o["op"], o.get("act", "none")
        if kind == "layernorm":
            res = 0.0 if "res" not in o else bufs[o["res"]].reshape(B, h, w, c)
            y = layernorm(src.reshape(B, h, w, c) + res, tensor(o["w_offset"], c), tensor(o["b_offset"], c), o["eps"])
        elif kind == "window_attention":
            n = o["window"] ** 2
            y = window_attention(src.reshape(B, h, w, c), tensor(o["bias_offset"], o["heads"] * n * n).reshape(o["heads"], n, n),
                                 o["heads"], o["window"], o["shift"])
        elif kind == "patch_merge":
            y = patch_merge(src.reshape(B, h, w, c))
        elif kind == "conv":
            kh, kw, cout, s, p = o.get("kh", 1), o.get("kw", 1), o["cout"], o.get("stride", 1), o.get("pad", 0)
            oh, ow = (h + 2 * p - kh) // s + 1, (w + 2 * p - kw) // s + 1
            res = None if "res" not in o else bufs[o["res"]].reshape(B, oh, ow, cout)
            y = cr.conv(src.reshape(B, h, w, c), tensor(o["w_offset"], kh * kw * c * cout).reshape(kh, kw, c, cout),
                        tensor(o["b_offset"], cout), s, p, "none", res)
            y = gelu(y) if a == "gelu" else cr.act(y, a)
        else:                                                                      # avgpool, dense
            y = cr.forward({"input_shape": [h, w, c], "ops": [dict(o, src=-1, dst=-2)]}, blob, src).reshape(B, 1, 1, -1)
        bufs[o["dst"]] = y
    return bufs[-2].reshape(B, -1)

