"""transformers.BertForQuestionAnswering as an independent numeric pin for span bundles (test infrastructure): a seeded
model with every parameter randomised, its parameters exported into a modelformat.bert_manifest(..., head="span") blob,
and its own fp64 forward as the reference. The same approach as torch_export.py for BertForSequenceClassification, for
the variant without a pooler whose last layer is the per-token qa_outputs Linear(hidden, 2)."""
from __future__ import annotations

import numpy as np

from torch_export import _rand_like


def hf_bert_qa(seed: int, hidden=768, layers=12, heads=12, inter=3072, vocab=30522, max_pos=512):
    """BertForQuestionAnswering with every parameter randomised (the default init zeroes all biases and sets LayerNorm to
    identity, which would leave those code paths unpinned). eval() mode, erf GELU."""
    import torch
    from transformers import BertConfig, BertForQuestionAnswering
    cfg = BertConfig(vocab_size=vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                     intermediate_size=inter, max_position_embeddings=max_pos, type_vocab_size=2, num_labels=2,
                     hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                     pad_token_id=0)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m = BertForQuestionAnswering(cfg)
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


def export_bert_qa(model, manifest: dict) -> np.ndarray:
    """Fill the blob of modelformat.bert_manifest(..., head="span") from a BertForQuestionAnswering: embeddings, fused
    Q|K|V projection, Linear weights transposed to [in, out], and qa_outputs as the last 1x1 conv (start | end)."""
    import torch
    bert = model.bert
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
    emb = bert.embeddings
    norm(o, emb.LayerNorm)
    put(o["word_offset"], emb.word_embeddings.weight)
    put(o["pos_offset"], emb.position_embeddings.weight)
    put(o["type_offset"], emb.token_type_embeddings.weight)
    for layer in bert.encoder.layer:
        att, so = layer.attention.self, layer.attention.output
        lin(next(ops), [att.query.weight, att.key.weight, att.value.weight], [att.query.bias, att.key.bias, att.value.bias])
        assert next(ops)["op"] == "attention"
        lin(next(ops), [so.dense.weight], [so.dense.bias])
        norm(next(ops), so.LayerNorm)
        lin(next(ops), [layer.intermediate.dense.weight], [layer.intermediate.dense.bias])
        lin(next(ops), [layer.output.dense.weight], [layer.output.dense.bias])
        norm(next(ops), layer.output.LayerNorm)
    o = next(ops)
    assert o["op"] == "conv" and o["dst"] == -2
    lin(o, [model.qa_outputs.weight], [model.qa_outputs.bias])
    assert next(ops, None) is None
    return blob


def bert_qa_reference(model, ids: np.ndarray, mask: np.ndarray, types: np.ndarray):
    """transformers' own BertForQuestionAnswering forward in fp64 with an explicit attention mask and segment ids:
    (start_logits [B, S], end_logits [B, S])."""
    import copy
    import torch
    m64 = copy.deepcopy(model).double()

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.int64))
    with torch.no_grad():
        out = m64(input_ids=t(ids), attention_mask=t(mask), token_type_ids=t(types))
    return out.start_logits.numpy(), out.end_logits.numpy()
