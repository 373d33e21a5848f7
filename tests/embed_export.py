"""transformers.BertModel as an independent numeric pin for encoder bundles (test infrastructure): a seeded model with every
parameter randomised, with or without its pooling layer, exported into a modelformat.bert_manifest(..., head="encoder")
blob, and its own fp64 forward as the reference. Sentence embeddings follow sentence-transformers' mean_pooling and
torch.nn.functional.normalize."""
from __future__ import annotations

import numpy as np

from torch_export import _rand_like


def hf_bert_model(seed: int, pooler=True, hidden=768, layers=12, heads=12, inter=3072, vocab=30522, max_pos=512):
    """BertModel(add_pooling_layer=pooler) with every parameter randomised (the default init zeroes all biases and sets
    LayerNorm to identity, which would leave those code paths unpinned). eval() mode, erf GELU."""
    import torch
    from transformers import BertConfig, BertModel
    cfg = BertConfig(vocab_size=vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                     intermediate_size=inter, max_position_embeddings=max_pos, type_vocab_size=2, hidden_act="gelu",
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12, pad_token_id=0)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m = BertModel(cfg, add_pooling_layer=pooler)
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


def export_bert_model(model, manifest: dict) -> np.ndarray:
    """Fill the blob of modelformat.bert_manifest(..., head="encoder") from a BertModel: embeddings, fused Q|K|V
    projection, Linear weights transposed to [in, out], and the pooler as the last dense op when the bundle has one."""
    import torch
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)

    def put(off, arr):
        a = np.ascontiguousarray(arr.detach().float().numpy(), np.float32).ravel()
        blob[off // 4: off // 4 + a.size] = a

    def lin(o, weights, biases):
        w = torch.cat([w_.detach().t() for w_ in weights], dim=1)          # [in, sum(out)]
        assert tuple(w.shape) == (o["c"], o["cout"])
        put(o["w_offset"], w.contiguous())
        put(o["b_offset"], torch.cat([b_.detach() for b_ in biases]))

    def norm(o, ln):
        assert o["op"] in ("layernorm", "embed")
        put(o["w_offset"], ln.weight)
        put(o["b_offset"], ln.bias)

    ops = iter(manifest["ops"])
    o = next(ops)
    emb = model.embeddings
    norm(o, emb.LayerNorm)
    put(o["word_offset"], emb.word_embeddings.weight)
    put(o["pos_offset"], emb.position_embeddings.weight)
    put(o["type_offset"], emb.token_type_embeddings.weight)
    for layer in model.encoder.layer:
        att, so = layer.attention.self, layer.attention.output
        lin(next(ops), [att.query.weight, att.key.weight, att.value.weight], [att.query.bias, att.key.bias, att.value.bias])
        assert next(ops)["op"] == "attention"
        lin(next(ops), [so.dense.weight], [so.dense.bias])
        norm(next(ops), so.LayerNorm)
        lin(next(ops), [layer.intermediate.dense.weight], [layer.intermediate.dense.bias])
        lin(next(ops), [layer.output.dense.weight], [layer.output.dense.bias])
        norm(next(ops), layer.output.LayerNorm)
    if model.pooler is not None:
        o = next(ops)
        assert o["op"] == "dense" and o["act"] == "tanh" and o["dst"] == -2
        lin(o, [model.pooler.dense.weight], [model.pooler.dense.bias])
    assert next(ops, None) is None
    return blob


def bert_model_reference(model, ids: np.ndarray, mask=None, types=None) -> dict:
    """transformers' own BertModel forward in fp64: last_hidden_state [B, S, H], pooler_output [B, H] (with a pooler), and
    sentence-transformers' mean_pooling of the hidden states with its attention mask (the ids != 0 without one) and the
    L2-normalised mean and [CLS] vectors."""
    import copy
    import torch
    import torch.nn.functional as F
    m64 = copy.deepcopy(model).double()

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.int64))
    am = t(mask) if mask is not None else (t(ids) != 0).long()
    with torch.no_grad():
        out = m64(input_ids=t(ids), attention_mask=am, token_type_ids=None if types is None else t(types))
        h = out.last_hidden_state
        m = am.unsqueeze(-1).expand(h.size()).double()
        mean = torch.sum(h * m, 1) / torch.clamp(m.sum(1), min=1e-9)
        res = {"last_hidden_state": h.numpy(), "mean": mean.numpy(), "mean_normalized": F.normalize(mean, p=2, dim=1).numpy(),
               "cls_normalized": F.normalize(h[:, 0], p=2, dim=1).numpy()}
        if out.pooler_output is not None:
            res["pooler_output"] = out.pooler_output.numpy()
    return res
