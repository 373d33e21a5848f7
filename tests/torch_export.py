"""Independent numeric pins (test infrastructure): build the BASELINE configs[1] / configs[3] models with the
libraries that DEFINE them -- torchvision.models.resnet50 and transformers.BertForSequenceClassification -- export
their parameters into the product's bundle format, and let those libraries' own forward pass (fp64) be the reference.
The oracle (oracle/models.py) and the GPU executor must both reproduce it within 1e-4, so a topology mistake shared by
the oracle and the product manifests (same author) can no longer hide.

TF-Serving itself (the reference's executor, deploy/docker-compose/docker-compose.yaml:22-37) is absent from this image and
from the GPU box; torchvision / transformers are present on both, so these checks run live in `-m "not gpu"` and `-m gpu`.
Nothing here imports oracle/ or shares code with tfservingcache_b200/modelformat.py beyond the manifest it fills.
"""
from __future__ import annotations

import numpy as np


def _rand_like(p, gen, scale, shift=0.0):
    import torch
    return torch.randn(p.shape, generator=gen, dtype=torch.float32) * scale + shift


# ------------------------------------------------------------------------------ ResNet-50 (torchvision) ----
def torchvision_resnet(seed: int, blocks=(3, 4, 6, 3), classes=1000):
    """torchvision ResNet (Bottleneck, v1.5: stride on the 3x3 conv) with seeded weights and NON-trivial BatchNorm
    statistics / affine parameters, so that folding BN into conv kernel + bias is exercised. eval() mode."""
    import torch
    from torchvision.models.resnet import Bottleneck, ResNet
    torch.manual_seed(seed)
    m = ResNet(Bottleneck, list(blocks), num_classes=classes)
    gen = torch.Generator().manual_seed(seed + 7)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.weight.copy_(_rand_like(mod.weight, gen, 0.1, 1.0))
                mod.bias.copy_(_rand_like(mod.bias, gen, 0.1))
                mod.running_mean.copy_(_rand_like(mod.running_mean, gen, 0.1))
                mod.running_var.copy_(_rand_like(mod.running_var, gen, 0.1, 1.0).abs() + 0.5)
        m.fc.bias.copy_(_rand_like(m.fc.bias, gen, 0.1))
    return m.eval()


def _fold(conv, bn):
    """conv + eval-mode BatchNorm -> (kernel [kh,kw,cin,cout], bias [cout]) in fp64 then fp32."""
    w = conv.weight.detach().double()                      # [cout, cin, kh, kw]
    scale = bn.weight.detach().double() / (bn.running_var.detach().double() + bn.eps).sqrt()
    wf = (w * scale[:, None, None, None]).permute(2, 3, 1, 0).contiguous()
    bf = bn.bias.detach().double() - bn.running_mean.detach().double() * scale
    return wf.float().numpy(), bf.float().numpy()


def export_resnet(model, manifest: dict) -> np.ndarray:
    """Fill the bundle blob of `manifest` (modelformat.resnet50_manifest with the same blocks / classes) from a
    torchvision ResNet, in execution order: stem, then per block conv1, conv2, [downsample], conv3, then fc."""
    pairs = [(model.conv1, model.bn1)]
    for layer in (model.layer1, model.layer2, model.layer3, model.layer4):
        for blk in layer:
            pairs += [(blk.conv1, blk.bn1), (blk.conv2, blk.bn2)]
            if blk.downsample is not None:
                pairs.append((blk.downsample[0], blk.downsample[1]))
            pairs.append((blk.conv3, blk.bn3))
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)
    convs = [o for o in manifest["ops"] if o["op"] == "conv"]
    assert len(convs) == len(pairs), (len(convs), len(pairs))
    for o, (conv, bn) in zip(convs, pairs):
        w, b = _fold(conv, bn)
        assert w.shape == (o["kh"], o["kw"], o["c"], o["cout"]) and conv.stride[0] == o["stride"] and conv.padding[0] == o["pad"]
        blob[o["w_offset"] // 4: o["w_offset"] // 4 + w.size] = w.ravel()
        blob[o["b_offset"] // 4: o["b_offset"] // 4 + b.size] = b
    fc = [o for o in manifest["ops"] if o["op"] == "dense"]
    assert len(fc) == 1
    w = model.fc.weight.detach().float().numpy().T.copy()   # Linear stores [out, in]; the bundle wants [in, out]
    blob[fc[0]["w_offset"] // 4: fc[0]["w_offset"] // 4 + w.size] = w.ravel()
    blob[fc[0]["b_offset"] // 4: fc[0]["b_offset"] // 4 + fc[0]["cout"]] = model.fc.bias.detach().float().numpy()
    return blob


def resnet_reference(model, x_nhwc: np.ndarray) -> np.ndarray:
    """torchvision's own forward in fp64 on NHWC fp32 input."""
    import copy
    import torch
    m64 = copy.deepcopy(model).double()
    with torch.no_grad():
        return m64(torch.from_numpy(np.ascontiguousarray(x_nhwc)).double().permute(0, 3, 1, 2)).numpy()


# ------------------------------------------------------------------------- BERT (transformers) ----
def hf_bert(seed: int, seq=128, hidden=768, layers=12, heads=12, inter=3072, vocab=30522, max_pos=512, labels=2):
    """transformers.BertForSequenceClassification with every parameter randomised (the default init zeroes all biases
    and sets LayerNorm to identity, which would leave those code paths unpinned). eval() mode, erf GELU."""
    import torch
    from transformers import BertConfig, BertForSequenceClassification
    cfg = BertConfig(vocab_size=vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                     intermediate_size=inter, max_position_embeddings=max_pos, type_vocab_size=2, num_labels=labels,
                     hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                     pad_token_id=0)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m = BertForSequenceClassification(cfg)
    gen = torch.Generator().manual_seed(seed + 11)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "LayerNorm.weight" in name:
                p.copy_(_rand_like(p, gen, 0.1, 1.0))
            elif name.endswith("bias"):
                p.copy_(_rand_like(p, gen, 0.1))
            elif "embeddings" in name:
                p.copy_(_rand_like(p, gen, 0.05))
            else:
                p.copy_(_rand_like(p, gen, (1.0 / p.shape[1]) ** 0.5))
    return m.eval()


def export_bert(model, manifest: dict) -> np.ndarray:
    """Fill the bundle blob of modelformat.bert_manifest(...) from a HF BERT: fused Q|K|V projection, Linear weights
    transposed to [in, out]."""
    bert = model.bert
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)

    def put(off, arr):
        a = np.ascontiguousarray(arr.detach().float().numpy() if hasattr(arr, "detach") else arr, np.float32).ravel()
        blob[off // 4: off // 4 + a.size] = a

    def lin(o, weights, biases):
        import torch
        w = torch.cat([w_.detach().t() for w_ in weights], dim=1)          # [in, sum(out)]
        b = torch.cat([b_.detach() for b_ in biases])
        assert tuple(w.shape) == (o["c"], o["cout"])
        put(o["w_offset"], w.contiguous())
        put(o["b_offset"], b)

    ops = iter(manifest["ops"])
    o = next(ops)
    assert o["op"] == "embed"
    emb = bert.embeddings
    put(o["w_offset"], emb.LayerNorm.weight)
    put(o["b_offset"], emb.LayerNorm.bias)
    put(o["word_offset"], emb.word_embeddings.weight)
    put(o["pos_offset"], emb.position_embeddings.weight)
    put(o["type_offset"], emb.token_type_embeddings.weight)
    for layer in bert.encoder.layer:
        att, so = layer.attention.self, layer.attention.output
        lin(next(ops), [att.query.weight, att.key.weight, att.value.weight], [att.query.bias, att.key.bias, att.value.bias])
        assert next(ops)["op"] == "attention"
        lin(next(ops), [so.dense.weight], [so.dense.bias])
        o = next(ops)
        assert o["op"] == "layernorm"
        put(o["w_offset"], so.LayerNorm.weight)
        put(o["b_offset"], so.LayerNorm.bias)
        lin(next(ops), [layer.intermediate.dense.weight], [layer.intermediate.dense.bias])
        lin(next(ops), [layer.output.dense.weight], [layer.output.dense.bias])
        o = next(ops)
        assert o["op"] == "layernorm"
        put(o["w_offset"], layer.output.LayerNorm.weight)
        put(o["b_offset"], layer.output.LayerNorm.bias)
    lin(next(ops), [bert.pooler.dense.weight], [bert.pooler.dense.bias])
    lin(next(ops), [model.classifier.weight], [model.classifier.bias])
    assert next(ops, None) is None
    return blob


def bert_reference(model, ids: np.ndarray) -> np.ndarray:
    """transformers' own forward in fp64: attention mask = (id != [PAD]=0), token types 0."""
    import copy
    import torch
    m64 = copy.deepcopy(model).double()
    t = torch.from_numpy(np.ascontiguousarray(ids, np.int64))
    with torch.no_grad():
        return m64(input_ids=t, attention_mask=(t != 0).long(), token_type_ids=torch.zeros_like(t)).logits.numpy()
