"""Writer for the native model bundle ("tfsc-b200-v1"): <baseDir>/<name>/<version>/
{tfsc_model.json, weights.bin}.  weights.bin is what gets paged verbatim into the HBM arena: per
dense layer W[in,out] row-major fp32 (the TF dense-kernel layout) then b[out], every tensor
256-byte aligned."""
from __future__ import annotations

import json
import math
import os

import numpy as np


def _align256(x: int) -> int:
    return (x + 255) & ~255


# signature.outputs kinds as the loader's kind table (csrc/model.cc) has them: kind -> (head, dtype, per-row dims in n and
# k). n is the last op's per-row width (classify), S (span), H (encoder), the mask_gather op's slots M (fill-mask) or the
# vocabulary (next-token); k is the entries' "k" (the same on every top-k or span result entry), or S for an encoder. The span result kinds also carry
# "max_answer_length" and optionally "sep_id" (a graph bundle with a type_ids input, ending in [S, 1, 2] start / end
# logits); cls_embedding and mean_embedding may carry "normalize": true; classes is one int64 (2 words) and
# next_token_position one int32. The generate kinds (greedy generation on a GPT-2 bundle, n = the vocabulary) carry
# "max_new_tokens" = N as their k, the same on every entry, and optionally "eos_token_id"; generated_length is one int32.
# The score kinds (scoring the input of a GPT-2 bundle, n = S) take a name and a kind only: token_log_probs and token_ranks
# hold one value per position, token_log_prob_sum and token_count one per row.
OUTPUT_KIND_TABLE = {
    "logits": ("classify", "float32", "n"), "probabilities": ("classify", "float32", "n"), "classes": ("classify", "int64", ""),
    "top_k_classes": ("classify", "int32", "k"), "top_k_probabilities": ("classify", "float32", "k"),
    "start_logits": ("span", "float32", "n"), "end_logits": ("span", "float32", "n"), "span_starts": ("span", "int32", "k"),
    "span_ends": ("span", "int32", "k"), "span_scores": ("span", "float32", "k"),
    "sequence_output": ("encoder", "float32", "kn"), "pooled_output": ("encoder", "float32", "n"),
    "cls_embedding": ("encoder", "float32", "n"), "mean_embedding": ("encoder", "float32", "n"),
    "masked_positions": ("fill_mask", "int32", "n"), "masked_top_k_ids": ("fill_mask", "int32", "nk"),
    "masked_top_k_probabilities": ("fill_mask", "float32", "nk"), "masked_top_k_logits": ("fill_mask", "float32", "nk"),
    "next_token_position": ("next_token", "int32", ""), "next_token_top_k_ids": ("next_token", "int32", "k"),
    "next_token_top_k_probabilities": ("next_token", "float32", "k"), "next_token_top_k_logits": ("next_token", "float32", "k"),
    "generated_ids": ("generate", "int32", "k"), "generated_log_probs": ("generate", "float32", "k"),
    "generated_length": ("generate", "int32", ""),
    "token_log_probs": ("score", "float32", "n"), "token_ranks": ("score", "int32", "n"),
    "token_log_prob_sum": ("score", "float32", ""), "token_count": ("score", "int32", ""),
}
(OUTPUT_KINDS, SPAN_OUTPUT_KINDS, ENCODER_OUTPUT_KINDS, MLM_OUTPUT_KINDS, NEXT_TOKEN_OUTPUT_KINDS, GENERATE_OUTPUT_KINDS,
 SCORE_OUTPUT_KINDS) = (tuple(k for k, v in OUTPUT_KIND_TABLE.items() if v[0] == head)
                        for head in ("classify", "span", "encoder", "fill_mask", "next_token", "generate", "score"))


def _signature(sig: dict, outputs):
    """signature.outputs replaces signature.output: a list of {"name", "kind"} (+ "k" for the top-k kinds, + "k",
    "max_answer_length" [, "sep_id"] for the span kinds)."""
    if outputs is None:
        return sig
    sig = {k: v for k, v in sig.items() if k != "output"}
    sig["outputs"] = [dict(o) for o in outputs]
    return sig


def _dims(o, n, seq):
    head, _dtype, dims = OUTPUT_KIND_TABLE[o["kind"]]
    k = o.get("max_new_tokens") if head == "generate" else o.get("k")
    return [int(n if d == "n" else seq if head == "encoder" else k) for d in dims]


def packed_output_layout(outputs, n, seq=None):
    """(name, element offset, width, dtype) of every output in a packed response row, in packed order (byte-wise sorted
    names). Offsets and widths count 32-bit words: a kind's per-row dims (OUTPUT_KIND_TABLE) in n, the entry's "k" (or
    "max_new_tokens") and,
    for the encoder kinds, seq = S; classes is one little-endian int64 in 2 words."""
    out, off = [], 0
    for o in sorted(outputs, key=lambda o: o["name"].encode()):
        dtype = OUTPUT_KIND_TABLE[o["kind"]][1]
        width = math.prod(_dims(o, n, seq)) * (2 if dtype == "int64" else 1)
        out.append((o["name"], off, width, dtype))
        off += width
    return out


def split_packed_rows(rows_words: np.ndarray, outputs, n, seq=None) -> dict:
    """{name: array} from packed rows ([rows, out_dim] of any 4-byte dtype, e.g. the float32 view of tfsc_predict_device's y).
    n and seq as for packed_output_layout; the rank-2 kinds come out as [rows, *dims]: sequence_output [rows, seq, n], the
    fill-mask top-k kinds [rows, n, k]."""
    w = np.ascontiguousarray(rows_words).view(np.uint32).reshape(len(rows_words), -1)
    dims = {o["name"]: _dims(o, n, seq) for o in outputs}
    res = {}
    for name, off, width, dtype in packed_output_layout(outputs, n, seq):
        part = np.ascontiguousarray(w[:, off:off + width])
        if dtype == "int64" or not dims[name]:       # the scalar kinds: one value per row
            res[name] = part.view("<i8" if dtype == "int64" else "<i4").reshape(-1)
        else:
            res[name] = part.view("<i4" if dtype == "int32" else "<f4")
        if len(dims[name]) == 2:
            res[name] = res[name].reshape(len(w), *dims[name])
    return res


def write_mlp_bundle(version_dir: str, weights, biases, activations=None, input_name="x", output_name="y", extra_signatures=None,
                     outputs=None):
    n = len(weights)
    if activations is None:
        activations = ["relu"] * (n - 1) + ["linear"]
    off, layers = 0, []
    for w, b, act in zip(weights, biases, activations):
        fi, fo = w.shape
        w_off = off
        off = _align256(off + fi * fo * 4)
        b_off = off
        off = _align256(off + fo * 4)
        layers.append({"in": int(fi), "out": int(fo), "activation": act, "w_offset": w_off, "b_offset": b_off})
    blob = np.zeros(off // 4, dtype=np.float32)
    for L, w, b in zip(layers, weights, biases):
        blob[L["w_offset"] // 4: L["w_offset"] // 4 + w.size] = np.asarray(w, np.float32).ravel()
        blob[L["b_offset"] // 4: L["b_offset"] // 4 + b.size] = np.asarray(b, np.float32).ravel()
    man = {"format": "tfsc-b200-v1", "template": "mlp", "dtype": "float32",
           "signature": _signature({"input": input_name, "output": output_name}, outputs), "layers": layers, "weights_bytes": off}
    if extra_signatures:   # classify / regress signatures: [{"name", "method": "classify"|"regress", "feature"}]
        man["extra_signatures"] = list(extra_signatures)
    _write(version_dir, man, blob)
    return man


def write_affine_bundle(version_dir: str, a: float, b: float, input_name="x", output_name="y", extra_signatures=None):
    blob = np.zeros(128, dtype=np.float32)
    blob[0], blob[64] = a, b
    man = {"format": "tfsc-b200-v1", "template": "affine", "dtype": "float32",
           "signature": {"input": input_name, "output": output_name}, "a_offset": 0, "b_offset": 256,
           "weights_bytes": 512}
    if extra_signatures:
        man["extra_signatures"] = list(extra_signatures)
    _write(version_dir, man, blob)
    return man


def _write(version_dir: str, man: dict, blob: np.ndarray):
    os.makedirs(version_dir, exist_ok=True)
    with open(os.path.join(version_dir, "tfsc_model.json"), "w") as f:
        json.dump(man, f)
    blob.astype("<f4").tofile(os.path.join(version_dir, "weights.bin"))


def _graph_manifest(input_shape, ops, n_buffers, input_name="x", output_name="y", input_dtype="float32", inputs=None, outputs=None):
    off = 0

    def take(nbytes):
        nonlocal off
        o = off
        off = _align256(off + nbytes)
        return o

    for op in ops:
        if op["op"] in ("conv", "dense", "token_score"):
            k = op.get("kh", 1) * op.get("kw", 1) * op["c"]
            op["w_offset"] = take(k * op["cout"] * 4)
            op["b_offset"] = take(op["cout"] * 4)
        elif op["op"] == "depthwise_conv":                  # kernel [kh, kw, c], bias [c]
            op["w_offset"] = take(op["kh"] * op["kw"] * op["c"] * 4)
            op["b_offset"] = take(op["c"] * 4)
        elif op["op"] == "window_attention":                # relative-position bias expanded to [heads, N, N]
            op["bias_offset"] = take(op["heads"] * op["window"] ** 4 * 4)
        elif op["op"] == "embed" and op.get("norm", True) is False:   # word and position tables only
            op["word_offset"] = take(op["vocab"] * op["c"] * 4)
            op["pos_offset"] = take(op["max_pos"] * op["c"] * 4)
        elif op["op"] in ("layernorm", "embed"):
            op["w_offset"] = take(op["c"] * 4)      # gamma
            op["b_offset"] = take(op["c"] * 4)      # beta
            if op["op"] == "embed":
                op["word_offset"] = take(op["vocab"] * op["c"] * 4)
                op["pos_offset"] = take(op["max_pos"] * op["c"] * 4)
                op["type_offset"] = take(2 * op["c"] * 4)
    sig = {"input": input_name, "output": output_name}
    if inputs is not None:   # several named inputs with roles: "inputs" replaces "input"
        sig = {"inputs": [{"name": i["name"], "role": i["role"]} for i in inputs], "output": output_name}
    return {"format": "tfsc-b200-v1", "template": "graph", "dtype": "float32", "input_dtype": input_dtype,
            "signature": _signature(sig, outputs), "input_shape": list(input_shape),
            "n_buffers": n_buffers, "ops": ops, "weights_bytes": off}


def resnet50_manifest(image=224, classes=1000, width=64, blocks=(3, 4, 6, 3), outputs=None):
    """ResNet-50 v1.5 (torchvision topology: stride on the 3x3 conv) as a graph bundle, NHWC, BatchNorm folded into
    kernel + bias. Buffers: 0 = block input / identity, 1 = 1x1 out, 2 = 3x3 out, 3 = block out, 4 = downsample.
    outputs: signature.outputs (a list of {"name", "kind"[, "k"]}) in place of the single logits output."""
    ops, h = [], image
    ops.append({"op": "conv", "src": -1, "dst": 0, "h": h, "w": h, "c": 3, "kh": 7, "kw": 7, "stride": 2, "pad": 3,
                "cout": width, "act": "relu"})
    h = (h + 6 - 7) // 2 + 1
    ops.append({"op": "maxpool", "src": 0, "dst": 1, "h": h, "w": h, "c": width, "kh": 3, "kw": 3, "stride": 2, "pad": 1})
    h = (h + 2 - 3) // 2 + 1
    cur, cin = 1, width          # `cur` = buffer holding the block input
    free = [0, 2, 3, 4]
    for li, nb in enumerate(blocks):
        planes = width * (2 ** li)
        for bi in range(nb):
            stride = 2 if (bi == 0 and li > 0) else 1
            a, b, c_, d = [x for x in range(5) if x != cur][:4]
            ho = (h + 2 - 3) // stride + 1
            ops.append({"op": "conv", "src": cur, "dst": a, "h": h, "w": h, "c": cin, "kh": 1, "kw": 1, "stride": 1, "pad": 0,
                        "cout": planes, "act": "relu"})
            ops.append({"op": "conv", "src": a, "dst": b, "h": h, "w": h, "c": planes, "kh": 3, "kw": 3, "stride": stride,
                        "pad": 1, "cout": planes, "act": "relu"})
            ident = cur
            if bi == 0:  # projection shortcut
                ops.append({"op": "conv", "src": cur, "dst": c_, "h": h, "w": h, "c": cin, "kh": 1, "kw": 1, "stride": stride,
                            "pad": 0, "cout": planes * 4, "act": "none"})
                ident = c_
            ops.append({"op": "conv", "src": b, "dst": d, "res": ident, "h": ho, "w": ho, "c": planes, "kh": 1, "kw": 1,
                        "stride": 1, "pad": 0, "cout": planes * 4, "act": "relu"})
            cur, cin, h = d, planes * 4, ho
    a = [x for x in range(5) if x != cur][0]
    ops.append({"op": "avgpool", "src": cur, "dst": a, "h": h, "w": h, "c": cin})
    ops.append({"op": "dense", "src": a, "dst": -2, "h": 1, "w": 1, "c": cin, "cout": classes, "act": "none"})
    return _graph_manifest([image, image, 3], ops, 5, outputs=outputs)


def _make_divisible(v: float, divisor: int = 8) -> int:
    """torchvision's channel rounding: the nearest multiple of `divisor`, at least `divisor`, never 10 % below v."""
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


def _conv(src, dst, h, c, cout, k=1, stride=1, act="none", res=None):
    o = {"op": "conv", "src": src, "dst": dst, "h": h, "w": h, "c": c, "kh": k, "kw": k, "stride": stride, "pad": (k - 1) // 2,
         "cout": cout, "act": act}
    if res is not None:
        o["res"] = res
    return o


def _depthwise(src, dst, h, c, k, stride, act):
    return {"op": "depthwise_conv", "src": src, "dst": dst, "h": h, "w": h, "c": c, "kh": k, "kw": k, "stride": stride,
            "pad": (k - 1) // 2, "act": act}


def _classifier(ops, cur, h, cin, last, classes, act, n_buffers, image, outputs):
    """the 1x1 conv to `last` channels, global average pool and the dense classifier that end both image nets"""
    a, b = [x for x in range(n_buffers) if x != cur][:2]
    ops.append(_conv(cur, a, h, cin, last, act=act))
    ops.append({"op": "avgpool", "src": a, "dst": b, "h": h, "w": h, "c": last})
    ops.append({"op": "dense", "src": b, "dst": -2, "h": 1, "w": 1, "c": last, "cout": classes, "act": "none"})
    return _graph_manifest([image, image, 3], ops, n_buffers, outputs=outputs)


def mobilenet_v2_manifest(image=224, classes=1000, width_mult=1.0, outputs=None):
    """MobileNetV2 (Sandler et al. 2018; torchvision topology, symmetric padding) as a graph bundle, NHWC, BatchNorm folded
    into kernel + bias, ReLU6 after every conv but the projections. An inverted-residual block is a 1x1 expansion (absent at
    expansion 1), a 3x3 depthwise conv and a 1x1 projection with the block input as residual when the shape allows.
    Dropout is identity at inference. Buffers: the block input and three others. outputs as for resnet50_manifest."""
    setting = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]
    cin = _make_divisible(32 * width_mult)
    ops, h, cur = [_conv(-1, 0, image, 3, cin, k=3, stride=2, act="relu6")], (image - 1) // 2 + 1, 0
    for t, c, n, s in setting:
        cout = _make_divisible(c * width_mult)
        for i in range(n):
            stride, hidden = (s if i == 0 else 1), int(round(cin * t))
            a, b, d = [x for x in range(4) if x != cur]
            src = cur
            if t != 1:
                ops.append(_conv(cur, a, h, cin, hidden, act="relu6"))
                src = a
            ho = (h - 1) // stride + 1
            ops.append(_depthwise(src, b, h, hidden, 3, stride, "relu6"))
            ops.append(_conv(b, d, ho, hidden, cout, res=cur if stride == 1 and cin == cout else None))
            cur, cin, h = d, cout, ho
    return _classifier(ops, cur, h, cin, _make_divisible(1280 * max(1.0, width_mult)), classes, "relu6", 4, image, outputs)


def efficientnet_manifest(image=224, classes=1000, width_mult=1.0, depth_mult=1.0, outputs=None):
    """EfficientNet (Tan & Le 2019; torchvision topology, symmetric padding) as a graph bundle, NHWC, BatchNorm folded into
    kernel + bias, SiLU activations. The default multipliers give B0; torchvision's (width_mult, depth_mult) of B1-B7 give
    those topologies (image size is the caller's). An MBConv block is a 1x1 expansion (absent at expansion 1), a k x k
    depthwise conv, squeeze-and-excitation (global average pool, a 1x1 conv to max(1, block input / 4) channels with SiLU, a
    1x1 conv back with sigmoid, channel_scale by that gate) and a 1x1 projection with the block input as residual when the
    shape allows. Stochastic depth and dropout are identity at inference. Buffers: the block input and three others, the SE
    pool / gate in the one the projection writes. outputs as for resnet50_manifest."""
    setting = [(1, 3, 1, 32, 16, 1), (6, 3, 2, 16, 24, 2), (6, 5, 2, 24, 40, 2), (6, 3, 2, 40, 80, 3), (6, 5, 1, 80, 112, 3),
               (6, 5, 2, 112, 192, 4), (6, 3, 1, 192, 320, 1)]
    cin = _make_divisible(32 * width_mult)
    ops, h, cur = [_conv(-1, 0, image, 3, cin, k=3, stride=2, act="silu")], (image - 1) // 2 + 1, 0
    for e, k, s, _ci, co, n in setting:
        cout = _make_divisible(co * width_mult)
        for i in range(int(math.ceil(n * depth_mult))):
            stride, exp, sq = (s if i == 0 else 1), _make_divisible(cin * e), max(1, cin // 4)
            a, b, d = [x for x in range(4) if x != cur]
            src = cur
            if exp != cin:
                ops.append(_conv(cur, a, h, cin, exp, act="silu"))
                src = a
            ho = (h - 1) // stride + 1
            ops.append(_depthwise(src, b, h, exp, k, stride, "silu"))
            ops.append({"op": "avgpool", "src": b, "dst": d, "h": ho, "w": ho, "c": exp})
            ops.append(_conv(d, a, 1, exp, sq, act="silu"))
            ops.append(_conv(a, d, 1, sq, exp, act="sigmoid"))
            ops.append({"op": "channel_scale", "src": b, "gate": d, "dst": a, "h": ho, "w": ho, "c": exp})
            ops.append(_conv(a, d, ho, exp, cout, res=cur if stride == 1 and cin == cout else None))
            cur, cin, h = d, cout, ho
    return _classifier(ops, cur, h, cin, 4 * cin, classes, "silu", 4, image, outputs)


def swin_manifest(image=224, classes=1000, embed_dim=96, depths=(2, 2, 6, 2), heads=(3, 6, 12, 24), window=7, outputs=None):
    """Swin Transformer V1 (Liu et al. 2021; torchvision's SwinTransformer topology) as a graph bundle, NHWC. The defaults
    give swin_t; depths (2, 2, 18, 2) give swin_s, embed_dim 128 with heads (4, 8, 16, 32) swin_b. The stem is a 4x4 /
    stride-4 conv and a LayerNorm. A block is LayerNorm, the qkv projection, window_attention (shifted by window // 2 in
    every second block, unshifted where the window covers the whole map, as torchvision does), the output projection with
    the block input as residual, LayerNorm, the MLP (4x, GELU) with the attention output as residual. Between stages,
    patch_merge, LayerNorm(4C) and the bias-free reduction 4C -> 2C (a zero bias). The end is LayerNorm, the global average
    pool and the dense classifier. Every Linear is a 1x1 conv over the h * w tokens ([h * w, 1, c]). Token maps must be
    multiples of the window at every stage (no padding). Buffers: the block input and three others. outputs as for
    resnet50_manifest."""
    def ln(src, dst, n, c):
        return {"op": "layernorm", "src": src, "dst": dst, "h": n, "w": 1, "c": c, "eps": 1e-5}

    def linear(src, dst, n, c, cout, act="none", res=None):
        o = {"op": "conv", "src": src, "dst": dst, "h": n, "w": 1, "c": c, "kh": 1, "kw": 1, "stride": 1, "pad": 0, "cout": cout,
             "act": act}
        if res is not None:
            o["res"] = res
        return o

    h, c = image // 4, embed_dim
    ops = [{"op": "conv", "src": -1, "dst": 0, "h": image, "w": image, "c": 3, "kh": 4, "kw": 4, "stride": 4, "pad": 0,
            "cout": c, "act": "none"}, ln(0, 1, h * h, c)]
    cur = 1
    for stage, (depth, nh) in enumerate(zip(depths, heads)):
        n = h * h
        a, b, d = [x for x in range(4) if x != cur]
        for i in range(depth):
            shift = window // 2 if i % 2 == 1 and window < h else 0
            ops += [ln(cur, a, n, c), linear(a, b, n, c, 3 * c),
                    {"op": "window_attention", "src": b, "dst": a, "h": h, "w": h, "c": 3 * c, "heads": nh, "window": window,
                     "shift": shift},
                    linear(a, d, n, c, c, res=cur), ln(d, a, n, c), linear(a, b, n, c, 4 * c, act="gelu"),
                    linear(b, cur, n, 4 * c, c, res=d)]
        if stage + 1 < len(depths):
            ops += [{"op": "patch_merge", "src": cur, "dst": a, "h": h, "w": h, "c": c}, ln(a, b, n // 4, 4 * c),
                    linear(b, cur, n // 4, 4 * c, 2 * c)]
            h, c = h // 2, 2 * c
    a, b = [x for x in range(4) if x != cur][:2]
    ops += [ln(cur, a, h * h, c), {"op": "avgpool", "src": a, "dst": b, "h": h, "w": h, "c": c},
            {"op": "dense", "src": b, "dst": -2, "h": 1, "w": 1, "c": c, "cout": classes, "act": "none"}]
    return _graph_manifest([image, image, 3], ops, 4, outputs=outputs)


def write_graph_bundle(version_dir: str, manifest: dict, blob: np.ndarray):
    _write(version_dir, manifest, np.asarray(blob, np.float32))


BERT_INPUTS = [{"name": "input_ids", "role": "ids"}, {"name": "input_mask", "role": "mask"},
               {"name": "segment_ids", "role": "type_ids"}]


def packed_input_order(inputs):
    """Names of `inputs` in the order their rows are concatenated in a request row: byte-wise sorted."""
    return sorted((i["name"] for i in inputs), key=lambda n: n.encode())


def bert_manifest(seq=128, hidden=768, layers=12, heads=12, inter=3072, vocab=30522, max_pos=512, labels=2, inputs=None,
                  outputs=None, head="classify", pooler=True, slots=1, mask_token_id=103):
    """BERT-base fine-tune variant (Devlin et al. 2018) as a graph bundle: token ids int32 [B, seq] -> logits
    [B, labels]. A sequence is an "image" with h = seq tokens, w = 1, c = width; dense layers are 1x1 convs.
    With inputs=None the bundle takes the ids only: the attention mask is derived from them ([PAD] = 0), token_type is 0.
    With inputs = a list of {"name", "role"} (roles "ids", "mask", "type_ids"; e.g. BERT_INPUTS) it declares those int32
    [B, seq] inputs, and the kernels read the attention mask and the segment ids from the request.
    With outputs = a list of {"name", "kind"[, "k"]} (kinds in OUTPUT_KINDS) the bundle answers those outputs, computed
    from the logits on the GPU, in place of the single "logits" output.
    head="span" makes the question-answering variant (BertForQuestionAnswering): no pooler and no classifier, the last op
    is the per-token qa_outputs Linear(hidden, 2), a 1x1 conv from buffer 0 writing [B, seq, 1, 2] start / end logits.
    Its span outputs (SPAN_OUTPUT_KINDS) need inputs with a "type_ids" role.
    head="encoder" makes the encoder without a classifier (BertModel), answering ENCODER_OUTPUT_KINDS: with pooler=True
    the last op is the pooler (a tanh dense over token 0 of buffer 0, writing [B, hidden]) and the hidden states are
    buffer 0; with pooler=False (BertModel(add_pooling_layer=False)) the last LayerNorm writes the [B, seq, 1, hidden]
    hidden states as the response.
    head="mlm" makes the masked-language-model variant (BertForMaskedLM), answering MLM_OUTPUT_KINDS: after the encoder a
    mask_gather op copies the hidden states of the first `slots` = M tokens whose id is mask_token_id to buffer 1
    ([B, M, 1, hidden]), then the prediction head runs on those M slots: the transform (a 1x1 conv hidden -> hidden with
    GELU), its LayerNorm, and the decoder (a 1x1 conv hidden -> Vp writing [B, M, 1, Vp] logits), Vp = vocab rounded up
    to a multiple of 32 so that the projection runs on the tensor-core GEMM; its columns from vocab on are zero padding.
    Buffers: 0 hidden, 1 qkv / ffn-intermediate, 2 context / post-attention, 3 dense output."""
    ops = [{"op": "embed", "src": -1, "dst": 0, "h": seq, "w": 1, "c": hidden, "vocab": vocab, "max_pos": max_pos, "eps": 1e-12}]

    def dense(src, dst, cin, cout, act="none", res=None):
        o = {"op": "conv", "src": src, "dst": dst, "h": seq, "w": 1, "c": cin, "kh": 1, "kw": 1, "stride": 1, "pad": 0,
             "cout": cout, "act": act}
        if res is not None:
            o["res"] = res
        return o

    for _ in range(layers):
        ops.append(dense(0, 1, hidden, 3 * hidden))                                     # fused Q|K|V projection
        ops.append({"op": "attention", "src": 1, "dst": 2, "h": seq, "w": 1, "c": 3 * hidden, "heads": heads})
        ops.append(dense(2, 3, hidden, hidden))                                         # attention output projection
        ops.append({"op": "layernorm", "src": 3, "res": 0, "dst": 2, "h": seq, "w": 1, "c": hidden, "eps": 1e-12})
        ops.append(dense(2, 1, hidden, inter, act="gelu"))
        ops.append(dense(1, 3, inter, hidden))
        ops.append({"op": "layernorm", "src": 3, "res": 2, "dst": 0, "h": seq, "w": 1, "c": hidden, "eps": 1e-12})
    if head == "encoder":
        if pooler:
            ops.append({"op": "dense", "src": 0, "dst": -2, "h": 1, "w": 1, "c": hidden, "cout": hidden, "act": "tanh"})
        else:
            ops[-1]["dst"] = -2                                                          # the last LayerNorm answers
    elif head == "mlm":
        M, vp = slots, (vocab + 31) // 32 * 32
        ops.append({"op": "mask_gather", "src": 0, "dst": 1, "h": seq, "w": 1, "c": hidden, "slots": M,
                    "mask_token_id": mask_token_id})

        def slot_dense(src, dst, cout, act="none"):
            return {"op": "conv", "src": src, "dst": dst, "h": M, "w": 1, "c": hidden, "kh": 1, "kw": 1, "stride": 1, "pad": 0,
                    "cout": cout, "act": act}
        ops.append(slot_dense(1, 2, hidden, act="gelu"))                                # cls.predictions.transform.dense
        ops.append({"op": "layernorm", "src": 2, "dst": 3, "h": M, "w": 1, "c": hidden, "eps": 1e-12})
        ops.append(slot_dense(3, -2, vp))                                                # decoder (tied to word_embeddings)
    elif head == "span":
        ops.append(dense(0, -2, hidden, 2))                                              # qa_outputs: start | end per token
    else:
        ops.append({"op": "dense", "src": 0, "dst": 1, "h": 1, "w": 1, "c": hidden, "cout": hidden, "act": "tanh"})  # pooler on [CLS]
        ops.append({"op": "dense", "src": 1, "dst": -2, "h": 1, "w": 1, "c": hidden, "cout": labels, "act": "none"})
    return _graph_manifest([seq], ops, 4, input_name="input_ids", output_name="logits", input_dtype="int32", inputs=inputs,
                           outputs=outputs)


GPT2_INPUTS = [{"name": "input_ids", "role": "ids"}, {"name": "attention_mask", "role": "mask"}]
# a sampling generate bundle's inputs: GPT2_INPUTS and the per-request seed, int32 [B, 1] (one value per row)
GPT2_SAMPLING_INPUTS = GPT2_INPUTS + [{"name": "seed", "role": "seed"}]


def gpt2_manifest(seq=1024, hidden=768, layers=12, heads=12, vocab=50257, max_pos=1024, inputs=None, outputs=None):
    """GPT-2 (Radford et al. 2019; transformers' GPT2LMHeadModel topology) as a next-token graph bundle: token ids int32
    [B, seq] -> the vocabulary logits of each row's last attended token, answered through NEXT_TOKEN_OUTPUT_KINDS. The
    defaults give GPT-2 small; (1024, 24, 16), (1280, 36, 20) and (1600, 48, 25) as (hidden, layers, heads) give medium,
    large and XL. The embedding is wte[id] + wpe[s] without LayerNorm ("norm": false). A block is ln_1, c_attn (a 1x1 conv
    H -> 3H, packed q | k | v), causal attention, c_proj with the block input as residual, ln_2, c_fc (H -> 4H, tanh GELU)
    and c_proj with the residual. Then a last_token op copies each row's last attended token (the highest position whose
    mask is set, else seq - 1), ln_f runs on that one token, and the decoder, wte transposed and zero-padded to Vp = vocab
    rounded up to a multiple of 32 with a zero bias, writes [B, 1, 1, Vp] logits (columns from vocab on are padding).
    With inputs=None the bundle takes the ids only and attends to every position; inputs=GPT2_INPUTS adds an
    "attention_mask" that hides keys whose mask is 0 and picks the last attended token. Positions are 0..seq-1 whatever
    the padding, as transformers' default position ids. Every LayerNorm has eps 1e-5. With GENERATE_OUTPUT_KINDS outputs
    (each entry with "max_new_tokens": N and optionally "eos_token_id") the same graph is a greedy generation bundle:
    seq + N - 1 <= max_pos. Entries that also give "temperature" (a finite number > 0, default 1), "top_k" (an integer
    0 <= top_k <= vocab, 0 = off) or "top_p" (0 < top_p <= 1, 1 = off), the same on every entry that gives one, make it a
    sampling bundle: each token is drawn from the temperature / top-k / top-p distribution with the row's seed, so its
    inputs need a "seed" role (GPT2_SAMPLING_INPUTS: an int32 [B, 1] "seed" beside the ids and mask, or
    [{"name": "input_ids", "role": "ids"}, {"name": "seed", "role": "seed"}] without a mask). Entries that give
    "repetition_penalty" (a finite number > 0 whose fp32 value is normal; 1 = off), "no_repeat_ngram_size" (an integer
    1 <= n <= seq + N - 1) or "min_new_tokens" (an integer 1 <= m <= N; needs "eos_token_id"), the same on every entry that
    gives one, make it a processing bundle, greedy or sampling: each step penalises the ids of the row's history (its
    attended prompt ids and the tokens so far), bans every token that would repeat an n-gram of it and bans EOS before
    step m, as transformers' processors of the same names, and picks the token from the processed logits;
    generated_log_probs stay the model's raw log-probabilities.
    With SCORE_OUTPUT_KINDS outputs the bundle scores its input instead: after the same blocks ln_f runs on all seq tokens
    and a token_score op (the decoder's weights, [seq, 1, hidden] -> Vp logits per token, projected in chunks) gives each
    attended token but a row's first its log-probability and rank under the logits of the attended position before it
    (token_log_probs and token_ranks [seq], 0 and -1 at the other positions), and their sum and count per row.
    Buffers: 0 residual stream, 1 normed / attention context, 2 qkv / MLP hidden, 3 post-attention residual."""
    ops = [{"op": "embed", "src": -1, "dst": 0, "h": seq, "w": 1, "c": hidden, "vocab": vocab, "max_pos": max_pos, "norm": False}]

    def ln(src, dst, n):
        return {"op": "layernorm", "src": src, "dst": dst, "h": n, "w": 1, "c": hidden, "eps": 1e-5}

    def conv(src, dst, n, cin, cout, act="none", res=None):
        o = {"op": "conv", "src": src, "dst": dst, "h": n, "w": 1, "c": cin, "kh": 1, "kw": 1, "stride": 1, "pad": 0,
             "cout": cout, "act": act}
        if res is not None:
            o["res"] = res
        return o

    for _ in range(layers):
        ops += [ln(0, 1, seq), conv(1, 2, seq, hidden, 3 * hidden),
                {"op": "attention", "src": 2, "dst": 1, "h": seq, "w": 1, "c": 3 * hidden, "heads": heads, "causal": True},
                conv(1, 3, seq, hidden, hidden, res=0), ln(3, 1, seq), conv(1, 2, seq, hidden, 4 * hidden, act="gelu_tanh"),
                conv(2, 0, seq, 4 * hidden, hidden, res=3)]
    vp = (vocab + 31) // 32 * 32
    if outputs is not None and any(o.get("kind") in SCORE_OUTPUT_KINDS for o in outputs):
        ops += [ln(0, 1, seq), {"op": "token_score", "src": 1, "dst": -2, "h": seq, "w": 1, "c": hidden, "cout": vp, "vocab": vocab}]
    else:
        ops += [{"op": "last_token", "src": 0, "dst": 1, "h": seq, "w": 1, "c": hidden}, ln(1, 2, 1), conv(2, -2, 1, hidden, vp)]
    return _graph_manifest([seq], ops, 4, input_name="input_ids", output_name="logits", input_dtype="int32", inputs=inputs,
                           outputs=outputs)
