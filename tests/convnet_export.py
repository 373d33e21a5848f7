"""Independent numeric pins for the image nets (test infrastructure): seeded torchvision MobileNetV2 and EfficientNet with
every parameter and BatchNorm statistic randomised, exported into the bundles of modelformat.mobilenet_v2_manifest /
efficientnet_manifest (BatchNorm folded into kernel + bias), and torchvision's own forward in fp64 as the reference.
Nothing here shares code with the product beyond the manifest it fills."""
from __future__ import annotations

import numpy as np


def _randomise(m, seed: int):
    """conv / linear weights N(0, 1 / fan_in) (the default init of a depthwise conv is k*k-fold too small to keep
    activations O(1)), biases N(0, 0.1), BatchNorm gamma 1 + N(0, 0.1), beta and mean N(0, 0.1), var |1 + N(0, 0.1)| + 0.5"""
    import torch
    gen = torch.Generator().manual_seed(seed + 7)

    def rnd(p, scale, shift=0.0):
        return torch.randn(p.shape, generator=gen, dtype=torch.float32) * scale + shift

    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (torch.nn.Conv2d, torch.nn.Linear)):
                fan_in = mod.weight[0].numel()
                mod.weight.copy_(rnd(mod.weight, (1.0 / fan_in) ** 0.5))
                if mod.bias is not None:
                    mod.bias.copy_(rnd(mod.bias, 0.1))
            elif isinstance(mod, torch.nn.BatchNorm2d):
                mod.weight.copy_(rnd(mod.weight, 0.1, 1.0))
                mod.bias.copy_(rnd(mod.bias, 0.1))
                mod.running_mean.copy_(rnd(mod.running_mean, 0.1))
                mod.running_var.copy_(rnd(mod.running_var, 0.1, 1.0).abs() + 0.5)
    return m.eval()


def torchvision_mobilenet_v2(seed: int, width_mult=1.0, classes=1000):
    import torch
    from torchvision.models import mobilenet_v2
    torch.manual_seed(seed)
    return _randomise(mobilenet_v2(weights=None, width_mult=width_mult, num_classes=classes), seed)


def torchvision_efficientnet(seed: int, width_mult=1.0, depth_mult=1.0, classes=1000):
    """efficientnet_b0 at the default multipliers; other multipliers build the same family with torchvision's configuration"""
    import torch
    from torchvision.models import efficientnet_b0
    from torchvision.models.efficientnet import EfficientNet, _efficientnet_conf
    torch.manual_seed(seed)
    if (width_mult, depth_mult) == (1.0, 1.0):
        m = efficientnet_b0(weights=None, num_classes=classes)
    else:
        setting, last = _efficientnet_conf("efficientnet_b0", width_mult=width_mult, depth_mult=depth_mult)
        m = EfficientNet(setting, 0.2, num_classes=classes, last_channel=last)
    return _randomise(m, seed)


def _conv_pairs(model):
    """(conv, bn or None) in execution order: every bias-free conv is followed by its BatchNorm; the SE convs carry a bias"""
    import torch
    mods = [m for m in model.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.BatchNorm2d))]
    pairs, i = [], 0
    while i < len(mods):
        conv = mods[i]
        assert isinstance(conv, torch.nn.Conv2d)
        if conv.bias is not None:
            pairs.append((conv, None))
            i += 1
        else:
            assert isinstance(mods[i + 1], torch.nn.BatchNorm2d)
            pairs.append((conv, mods[i + 1]))
            i += 2
    return pairs


def export_convnet(model, manifest: dict) -> np.ndarray:
    """Fill the blob of a mobilenet_v2_manifest / efficientnet_manifest bundle from the torchvision model of the same
    configuration: conv kernels [kh, kw, cin, cout], depthwise kernels [kh, kw, c], BatchNorm folded in fp64, then fp32."""
    import torch
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)
    convs = [o for o in manifest["ops"] if o["op"] in ("conv", "depthwise_conv")]
    pairs = _conv_pairs(model)
    assert len(convs) == len(pairs), (len(convs), len(pairs))
    for o, (conv, bn) in zip(convs, pairs):
        w = conv.weight.detach().double()                          # [cout, cin / groups, kh, kw]
        if bn is None:
            scale, b = torch.ones(w.shape[0], dtype=torch.float64), conv.bias.detach().double()
        else:
            scale = bn.weight.detach().double() / (bn.running_var.detach().double() + bn.eps).sqrt()
            b = bn.bias.detach().double() - bn.running_mean.detach().double() * scale
        w = w * scale[:, None, None, None]
        assert conv.stride[0] == o["stride"] and conv.padding[0] == o["pad"] and conv.kernel_size == (o["kh"], o["kw"])
        if o["op"] == "depthwise_conv":
            assert conv.groups == o["c"] == w.shape[0] and w.shape[1] == 1
            w = w[:, 0].permute(1, 2, 0)                           # [kh, kw, c]
        else:
            assert conv.groups == 1 and tuple(w.shape[:2]) == (o["cout"], o["c"])
            w = w.permute(2, 3, 1, 0)                              # [kh, kw, cin, cout]
        w = w.contiguous().float().numpy().ravel()
        blob[o["w_offset"] // 4: o["w_offset"] // 4 + w.size] = w
        blob[o["b_offset"] // 4: o["b_offset"] // 4 + b.numel()] = b.float().numpy()
    fc = [o for o in manifest["ops"] if o["op"] == "dense"]
    lin = [m for m in model.classifier.modules() if isinstance(m, torch.nn.Linear)]
    assert len(fc) == len(lin) == 1
    w = lin[0].weight.detach().float().numpy().T.copy()              # Linear stores [out, in]; the bundle wants [in, out]
    blob[fc[0]["w_offset"] // 4: fc[0]["w_offset"] // 4 + w.size] = w.ravel()
    blob[fc[0]["b_offset"] // 4: fc[0]["b_offset"] // 4 + fc[0]["cout"]] = lin[0].bias.detach().float().numpy()
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
