"""Independent numeric pins for Swin Transformer (test infrastructure): a seeded torchvision SwinTransformer (V1) with every
parameter randomised, exported into the bundle of modelformat.swin_manifest, and torchvision's own forward in fp64 as
the reference. Nothing here shares code with the product beyond the manifest it fills."""
from __future__ import annotations

import numpy as np


def torchvision_swin(seed: int, embed_dim=96, depths=(2, 2, 6, 2), heads=(3, 6, 12, 24), window=7, classes=1000):
    """Linear / conv weights N(0, 1 / fan_in), biases N(0, 0.1), LayerNorm gamma 1 + N(0, 0.1) and beta N(0, 0.1), the
    relative-position bias tables N(0, 1); stochastic depth and dropout are identity in eval mode"""
    import torch
    from torchvision.models.swin_transformer import SwinTransformer
    torch.manual_seed(seed)
    m = SwinTransformer(patch_size=[4, 4], embed_dim=embed_dim, depths=list(depths), num_heads=list(heads), window_size=[window, window],
                        stochastic_depth_prob=0.0, num_classes=classes)
    gen = torch.Generator().manual_seed(seed + 7)

    def rnd(p, scale, shift=0.0):
        return torch.randn(p.shape, generator=gen, dtype=torch.float32) * scale + shift

    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (torch.nn.Conv2d, torch.nn.Linear)):
                mod.weight.copy_(rnd(mod.weight, (1.0 / mod.weight[0].numel()) ** 0.5))
                if mod.bias is not None:
                    mod.bias.copy_(rnd(mod.bias, 0.1))
            elif isinstance(mod, torch.nn.LayerNorm):
                mod.weight.copy_(rnd(mod.weight, 0.1, 1.0))
                mod.bias.copy_(rnd(mod.bias, 0.1))
            elif hasattr(mod, "relative_position_bias_table"):
                mod.relative_position_bias_table.copy_(rnd(mod.relative_position_bias_table, 1.0))
    return m.eval()


def _tensors(model):
    """what the bundle's weight-carrying ops hold, in op order: ("conv", kernel [kh, kw, cin, cout], bias),
    ("layernorm", gamma, beta), ("window_attention", bias [heads, N, N])"""
    import torch
    from torchvision.models.swin_transformer import PatchMerging

    def lin(mod):
        w = mod.weight.detach().double()
        b = mod.bias.detach().double() if mod.bias is not None else torch.zeros(w.shape[0], dtype=torch.float64)
        return ("conv", w.T[None, None], b)                                      # Linear [out, in] -> [1, 1, in, out]

    def ln(mod):
        return ("layernorm", mod.weight.detach().double(), mod.bias.detach().double())

    stem = model.features[0]
    out = [("conv", stem[0].weight.detach().double().permute(2, 3, 1, 0), stem[0].bias.detach().double()), ln(stem[2])]
    for layer in list(model.features)[1:]:
        if isinstance(layer, PatchMerging):
            out += [ln(layer.norm), lin(layer.reduction)]
            continue
        for blk in layer:
            out += [ln(blk.norm1), lin(blk.attn.qkv), ("window_attention", blk.attn.get_relative_position_bias()[0].detach().double()),
                    lin(blk.attn.proj), ln(blk.norm2), lin(blk.mlp[0]), lin(blk.mlp[3])]
    return out + [ln(model.norm), ("dense", model.head.weight.detach().double().T, model.head.bias.detach().double())]


def export_swin(model, manifest: dict) -> np.ndarray:
    """Fill the blob of a swin_manifest bundle from the torchvision model of the same configuration"""
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)
    ops = [o for o in manifest["ops"] if o["op"] in ("conv", "dense", "layernorm", "window_attention")]
    tensors = _tensors(model)
    assert len(ops) == len(tensors), (len(ops), len(tensors))

    def put(off, v):
        v = v.contiguous().float().numpy().ravel()
        blob[off // 4: off // 4 + v.size] = v

    for o, (kind, *vals) in zip(ops, tensors):
        assert kind == o["op"], (kind, o["op"])
        if kind == "window_attention":
            assert tuple(vals[0].shape) == (o["heads"], o["window"] ** 2, o["window"] ** 2)
            put(o["bias_offset"], vals[0])
            continue
        if kind == "conv":
            assert tuple(vals[0].shape) == (o["kh"], o["kw"], o["c"], o["cout"]), (tuple(vals[0].shape), o)
        put(o["w_offset"], vals[0])
        put(o["b_offset"], vals[1])
    return blob


def reference(model, x_nhwc: np.ndarray) -> np.ndarray:
    """torchvision's own forward in fp64 on NHWC fp32 input"""
    import copy
    import torch
    m64 = copy.deepcopy(model).double()
    with torch.no_grad():
        return m64(torch.from_numpy(np.ascontiguousarray(x_nhwc)).double().permute(0, 3, 1, 2)).numpy()


def images(batch: int, size: int, seed: int) -> np.ndarray:
    """seeded NHWC fp32 images, roughly normalised pixels"""
    return np.random.default_rng(seed).standard_normal((batch, size, size, 3)).astype(np.float32)
