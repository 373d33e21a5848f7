"""Numeric oracle for the executor the reference delegates to (TF-Serving, external and
unpinned: deploy/docker-compose/docker-compose.yaml:22-37).  TEST INFRASTRUCTURE ONLY: nothing under
tfservingcache_b200/ imports it.  numpy / torch-CPU restatement of the forward pass of each model
template the GPU build executes, reading the same ``weights.bin`` blob + ``tfsc_model.json`` manifest
the product pages into HBM (independent parse).

Pin status: TF-Serving itself cannot run here or on the GPU box, so the only number that comes from it is
the half_plus_two known answer [1,2,5] -> [2.5,3,4.5] (deploy/docker-compose/readme.md:40-42).  Since
round 2 the graph templates are pinned on the libraries that DEFINE the two model families instead:
torchvision's ResNet and transformers' BertForSequenceClassification (seeded, every parameter randomised,
fp64 forward) are reproduced to 1e-7 / 1e-15 from bundles exported by tests/torch_export.py
(tests/test_model_pins.py, committed numbers tests/golden/model_torch_golden.json).  The dense-MLP and
affine templates are plain ``x @ W + b`` / ``a*x + b`` in fp64.

Also holds the seeded synthetic weight generator (integer hash -> uniform fp32), restated
bit-exactly by the product's synthetic provider (csrc/provider.cc) so that 1 GB models never
have to be stored: value(seed, tensor, i) = (u24(mix32(i + k)) * 2^-24 * 2 - 1) * scale.
"""
from __future__ import annotations

import json
import math
import os

import numpy as np

M32 = 0xFFFFFFFF


def mix32(x):
    """lowbias32 integer hash on uint32 (numpy array or int)."""
    if isinstance(x, (int, np.integer)):
        x = int(x) & M32
        x ^= x >> 16
        x = (x * 0x7FEB352D) & M32
        x ^= x >> 15
        x = (x * 0x846CA68B) & M32
        x ^= x >> 16
        return x
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    return x


def tensor_key(seed: int, tensor_id: int) -> int:
    return mix32((seed * 0x9E3779B9 + tensor_id * 0x85EBCA6B + 0x165667B1) & M32)


def synth_tensor(seed: int, tensor_id: int, n: int, scale: float, start: int = 0) -> np.ndarray:
    k = tensor_key(seed, tensor_id)
    i = (np.arange(start, start + n, dtype=np.uint64) + np.uint64(k)) & np.uint64(M32)
    h = mix32(i)
    u = (h >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return (u * np.float32(2.0) - np.float32(1.0)) * np.float32(scale)


def weight_scale(fan_in: int) -> float:
    return float(np.float32(math.sqrt(3.0 / float(fan_in))))


BIAS_SCALE = float(np.float32(0.1))


def align256(x: int) -> int:
    return (x + 255) & ~255


def mlp_manifest(dims, activations=None) -> dict:
    """Layout restated from the product format (DESIGN.md 'model bundle'): per layer W[in,out]
    row-major fp32 then b[out], every tensor 256-byte aligned."""
    n_layers = len(dims) - 1
    if activations is None:
        activations = ["relu"] * (n_layers - 1) + ["linear"]
    off, layers = 0, []
    for l in range(n_layers):
        fi, fo = dims[l], dims[l + 1]
        w_off = off
        off = align256(off + fi * fo * 4)
        b_off = off
        off = align256(off + fo * 4)
        layers.append({"in": fi, "out": fo, "activation": activations[l],
                       "w_offset": w_off, "b_offset": b_off})
    return {"format": "tfsc-b200-v1", "template": "mlp", "dtype": "float32",
            "signature": {"input": "x", "output": "y"}, "layers": layers, "weights_bytes": off}


def synth_mlp_blob(dims, seed: int, activations=None):
    man = mlp_manifest(dims, activations)
    blob = np.zeros(man["weights_bytes"] // 4, dtype=np.float32)
    for l, L in enumerate(man["layers"]):
        w = synth_tensor(seed, 2 * l, L["in"] * L["out"], weight_scale(L["in"]))
        b = synth_tensor(seed, 2 * l + 1, L["out"], BIAS_SCALE)
        blob[L["w_offset"] // 4: L["w_offset"] // 4 + w.size] = w
        blob[L["b_offset"] // 4: L["b_offset"] // 4 + b.size] = b
    return man, blob


def affine_manifest() -> dict:
    return {"format": "tfsc-b200-v1", "template": "affine", "dtype": "float32",
            "signature": {"input": "x", "output": "y"}, "a_offset": 0, "b_offset": 256,
            "weights_bytes": 512}


def affine_blob(a: float, b: float):
    man = affine_manifest()
    blob = np.zeros(man["weights_bytes"] // 4, dtype=np.float32)
    blob[0] = a
    blob[64] = b
    return man, blob


def load_bundle(version_dir: str):
    with open(os.path.join(version_dir, "tfsc_model.json")) as f:
        man = json.load(f)
    blob = np.fromfile(os.path.join(version_dir, "weights.bin"), dtype=np.float32)
    return man, blob


def forward(man: dict, blob: np.ndarray, x: np.ndarray, dtype=np.float32) -> np.ndarray:
    """Forward pass in ``dtype`` (float32 = the reference executor's arithmetic type; float64 is
    the arbiter for tolerance questions)."""
    t = man["template"]
    if t == "affine":
        a = dtype(blob[man["a_offset"] // 4])
        b = dtype(blob[man["b_offset"] // 4])
        return (x.astype(dtype) * a + b).astype(dtype)
    if t == "mlp":
        h = x.astype(dtype)
        for L in man["layers"]:
            w = blob[L["w_offset"] // 4: L["w_offset"] // 4 + L["in"] * L["out"]].reshape(L["in"], L["out"])
            b = blob[L["b_offset"] // 4: L["b_offset"] // 4 + L["out"]]
            h = h @ w.astype(dtype) + b.astype(dtype)
            if L["activation"] == "relu":
                h = np.maximum(h, dtype(0))
        return h
    if t == "graph":
        return graph_forward(man, blob, x, dtype)
    raise ValueError(f"unknown template {t}")


def resnet50_ops(image=224, classes=1000):
    """Independent restatement of the ResNet-50 v1.5 topology (He et al. 2015; stride on the 3x3 conv as in
    torchvision / the TF official model), expressed in the bundle's op list."""
    ops = []
    cfg = [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)]
    size = image
    ops.append(dict(op="conv", src=-1, dst=0, h=size, w=size, c=3, kh=7, kw=7, stride=2, pad=3, cout=64, act="relu"))
    size = (size + 2 * 3 - 7) // 2 + 1
    ops.append(dict(op="maxpool", src=0, dst=1, h=size, w=size, c=64, kh=3, kw=3, stride=2, pad=1))
    size = (size + 2 - 3) // 2 + 1
    cur, cin = 1, 64
    for planes, n_blocks, first_stride in cfg:
        for blk in range(n_blocks):
            stride = first_stride if blk == 0 else 1
            others = [i for i in range(5) if i != cur]
            t1, t2, t3, t4 = others[0], others[1], others[2], others[3]
            out_size = (size + 2 - 3) // stride + 1
            ops.append(dict(op="conv", src=cur, dst=t1, h=size, w=size, c=cin, kh=1, kw=1, stride=1, pad=0, cout=planes, act="relu"))
            ops.append(dict(op="conv", src=t1, dst=t2, h=size, w=size, c=planes, kh=3, kw=3, stride=stride, pad=1, cout=planes, act="relu"))
            shortcut = cur
            if blk == 0:
                ops.append(dict(op="conv", src=cur, dst=t3, h=size, w=size, c=cin, kh=1, kw=1, stride=stride, pad=0, cout=4 * planes, act="none"))
                shortcut = t3
            ops.append(dict(op="conv", src=t2, dst=t4, res=shortcut, h=out_size, w=out_size, c=planes, kh=1, kw=1, stride=1, pad=0,
                            cout=4 * planes, act="relu"))
            cur, cin, size = t4, 4 * planes, out_size
    t1 = [i for i in range(5) if i != cur][0]
    ops.append(dict(op="avgpool", src=cur, dst=t1, h=size, w=size, c=cin))
    ops.append(dict(op="dense", src=t1, dst=-2, h=1, w=1, c=cin, cout=classes, act="none"))
    return ops


def graph_manifest(input_shape, ops, n_buffers=5, signature=("x", "y"), input_dtype="float32"):
    off = 0
    for o in ops:
        if o["op"] in ("conv", "dense"):
            k = o.get("kh", 1) * o.get("kw", 1) * o["c"]
            o["w_offset"] = off
            off = align256(off + k * o["cout"] * 4)
            o["b_offset"] = off
            off = align256(off + o["cout"] * 4)
        elif o["op"] in ("layernorm", "embed"):
            o["w_offset"] = off
            off = align256(off + o["c"] * 4)
            o["b_offset"] = off
            off = align256(off + o["c"] * 4)
            if o["op"] == "embed":
                o["word_offset"] = off
                off = align256(off + o["vocab"] * o["c"] * 4)
                o["pos_offset"] = off
                off = align256(off + o["max_pos"] * o["c"] * 4)
                o["type_offset"] = off
                off = align256(off + 2 * o["c"] * 4)
    return {"format": "tfsc-b200-v1", "template": "graph", "dtype": "float32", "input_dtype": input_dtype,
            "signature": {"input": signature[0], "output": signature[1]},
            "input_shape": list(input_shape), "n_buffers": n_buffers, "ops": ops, "weights_bytes": off}


EMBED_SCALE = float(np.float32(0.05))


def synth_graph_blob(man: dict, seed: int) -> np.ndarray:
    """Tensor ids of op i: 8*i + {0 kernel / gamma, 1 bias / beta, 2 word, 3 pos, 4 type}."""
    blob = np.zeros(man["weights_bytes"] // 4, dtype=np.float32)

    def put(off, arr):
        blob[off // 4: off // 4 + arr.size] = arr

    for i, o in enumerate(man["ops"]):
        if o["op"] in ("conv", "dense"):
            fan_in = o.get("kh", 1) * o.get("kw", 1) * o["c"]
            put(o["w_offset"], synth_tensor(seed, 8 * i, fan_in * o["cout"], weight_scale(fan_in)))
            put(o["b_offset"], synth_tensor(seed, 8 * i + 1, o["cout"], BIAS_SCALE))
        elif o["op"] in ("layernorm", "embed"):
            put(o["w_offset"], synth_tensor(seed, 8 * i, o["c"], BIAS_SCALE) + np.float32(1.0))
            put(o["b_offset"], synth_tensor(seed, 8 * i + 1, o["c"], BIAS_SCALE))
            if o["op"] == "embed":
                put(o["word_offset"], synth_tensor(seed, 8 * i + 2, o["vocab"] * o["c"], EMBED_SCALE))
                put(o["pos_offset"], synth_tensor(seed, 8 * i + 3, o["max_pos"] * o["c"], EMBED_SCALE))
                put(o["type_offset"], synth_tensor(seed, 8 * i + 4, 2 * o["c"], EMBED_SCALE))
    return blob


def bert_ops(seq=128, hidden=768, layers=12, heads=12, inter=3072, vocab=30522, max_pos=512, labels=2):
    """Independent restatement of BERT-base (Devlin et al. 2018; google-research/bert modeling.py structure:
    embeddings + LayerNorm, L x [self-attention, add & norm, GELU feed-forward, add & norm], tanh pooler on the
    first token, linear classifier) in the bundle's op list."""
    def lin(src, dst, cin, cout, act="none"):
        return dict(op="conv", src=src, dst=dst, h=seq, w=1, c=cin, kh=1, kw=1, stride=1, pad=0, cout=cout, act=act)
    ops = [dict(op="embed", src=-1, dst=0, h=seq, w=1, c=hidden, vocab=vocab, max_pos=max_pos, eps=1e-12)]
    for _layer in range(layers):
        ops.append(lin(0, 1, hidden, 3 * hidden))
        ops.append(dict(op="attention", src=1, dst=2, h=seq, w=1, c=3 * hidden, heads=heads))
        ops.append(lin(2, 3, hidden, hidden))
        ops.append(dict(op="layernorm", src=3, res=0, dst=2, h=seq, w=1, c=hidden, eps=1e-12))
        ops.append(lin(2, 1, hidden, inter, "gelu"))
        ops.append(lin(1, 3, inter, hidden))
        ops.append(dict(op="layernorm", src=3, res=2, dst=0, h=seq, w=1, c=hidden, eps=1e-12))
    ops.append(dict(op="dense", src=0, dst=1, h=1, w=1, c=hidden, cout=hidden, act="tanh"))
    ops.append(dict(op="dense", src=1, dst=-2, h=1, w=1, c=hidden, cout=labels, act="none"))
    return ops


def layer_norm_ref(v, gamma, beta, eps):
    """LayerNorm over the last axis of the torch tensor v, in v's dtype: two-pass mean and (biased) variance,
    (v - mean) / sqrt(var + eps) * gamma + beta."""
    import torch
    mean = v.mean(dim=-1, keepdim=True)
    var = ((v - mean) ** 2).mean(dim=-1, keepdim=True)
    return (v - mean) / torch.sqrt(var + eps) * gamma + beta


def attention_ref(qkv, ids, heads: int):
    """BERT multi-head self-attention (google-research/bert modeling.py attention_layer) on a torch tensor
    qkv[B, S, 3H] = q | k | v, in qkv's dtype: per head softmax(q k^T / sqrt(d) + mask) v with d = H / heads, where the
    additive mask is -10000 on every key whose token id is 0 ([PAD]); ids[B, S] or None (no mask). Returns ctx[B, S, H]."""
    import torch
    Bn, S, C3 = qkv.shape
    Hd = C3 // 3
    dh = Hd // heads
    q, k, v = (qkv[..., i * Hd:(i + 1) * Hd].reshape(Bn, S, heads, dh).permute(0, 2, 1, 3) for i in range(3))
    sc = q @ k.transpose(-1, -2) / math.sqrt(dh)
    if ids is not None:
        sc = sc + ((torch.as_tensor(ids) == 0).to(qkv.dtype) * -10000.0)[:, None, None, :]
    p = torch.softmax(sc, dim=-1)
    return (p @ v).permute(0, 2, 1, 3).reshape(Bn, S, Hd)


def graph_forward(man: dict, blob: np.ndarray, x: np.ndarray, dtype=np.float64) -> np.ndarray:
    """Interpreter of a graph bundle with torch-CPU functional ops (conv2d / max_pool2d) in `dtype`; NHWC in and
    out, NCHW inside."""
    import torch
    import torch.nn.functional as F
    td = torch.float64 if dtype == np.float64 else torch.float32
    ish = man["input_shape"]
    is_ids = man.get("input_dtype", "float32") == "int32"
    if is_ids:
        ids = torch.from_numpy(np.ascontiguousarray(x, dtype=np.int64)).reshape(-1, *ish)
        bufs = {-1: ids}
    else:
        xb = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).reshape(-1, *ish).to(td)
        bufs = {-1: xb.permute(0, 3, 1, 2).contiguous()}

    def vec(off, n):
        return torch.from_numpy(blob[off // 4: off // 4 + n]).to(td)

    def layer_norm(v, o):  # v: [B, C, S, 1]
        g, bta = vec(o["w_offset"], o["c"]), vec(o["b_offset"], o["c"])
        return layer_norm_ref(v.permute(0, 2, 3, 1), g, bta, o.get("eps", 1e-12)).permute(0, 3, 1, 2)

    for o in man["ops"]:
        src = bufs[o["src"]]
        if o["op"] == "embed":
            S, Hd = o["h"], o["c"]
            word = vec(o["word_offset"], o["vocab"] * Hd).view(o["vocab"], Hd)
            pos = vec(o["pos_offset"], o["max_pos"] * Hd).view(o["max_pos"], Hd)[:S]
            typ = vec(o["type_offset"], 2 * Hd).view(2, Hd)[0]
            e = word[src.clamp(0, o["vocab"] - 1)] + pos.unsqueeze(0) + typ          # [B, S, H]
            y = layer_norm(e.permute(0, 2, 1).unsqueeze(-1), o)
        elif o["op"] == "layernorm":
            v = src + (bufs[o["res"]] if o.get("res", -100) != -100 else 0)
            y = layer_norm(v, o)
        elif o["op"] == "attention":
            qkv = src.squeeze(-1).permute(0, 2, 1)                                    # [B, S, 3H]
            ctx = attention_ref(qkv, bufs[-1] if is_ids else None, o["heads"])         # the mask comes from the request's ids
            y = ctx.permute(0, 2, 1).unsqueeze(-1)
        elif o["op"] in ("conv", "dense"):
            kh, kw, c, cout = o.get("kh", 1), o.get("kw", 1), o["c"], o["cout"]
            w = torch.from_numpy(blob[o["w_offset"] // 4: o["w_offset"] // 4 + kh * kw * c * cout].reshape(kh, kw, c, cout)).to(td)
            b = torch.from_numpy(blob[o["b_offset"] // 4: o["b_offset"] // 4 + cout]).to(td)
            if o["op"] == "dense":
                flat = src.permute(0, 2, 3, 1).reshape(src.shape[0], -1)[:, :c]      # first token / the whole vector
                y = flat @ w.reshape(c, cout) + b
                y = y.reshape(src.shape[0], cout, 1, 1)
            else:
                y = F.conv2d(src, w.permute(3, 2, 0, 1).contiguous(), b, stride=o["stride"], padding=o["pad"])
            if o.get("res", -100) != -100:
                y = y + bufs[o["res"]]
            if o.get("act", "none") == "relu":
                y = torch.relu(y)
            elif o.get("act") == "gelu":
                y = F.gelu(y)
            elif o.get("act") == "tanh":
                y = torch.tanh(y)
        elif o["op"] == "maxpool":
            y = F.max_pool2d(src, (o["kh"], o["kw"]), stride=o["stride"], padding=o["pad"])
        elif o["op"] == "avgpool":
            y = src.mean(dim=(2, 3), keepdim=True)
        else:
            raise ValueError(o["op"])
        bufs[o["dst"]] = y
    out = bufs[-2]
    out = out.permute(0, 2, 3, 1).reshape(out.shape[0], -1) if out.shape[2] * out.shape[3] == 1 else out.permute(0, 2, 3, 1)
    return out.numpy().astype(dtype)
