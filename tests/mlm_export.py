"""transformers.BertForMaskedLM as an independent numeric pin for fill-mask bundles (test infrastructure): a seeded model
with every parameter randomised, exported into a modelformat.bert_manifest(..., head="mlm") blob, and its own fp64
forward as the reference."""
from __future__ import annotations

import numpy as np

from torch_export import _rand_like


def hf_mlm_model(seed: int, hidden=768, layers=12, heads=12, inter=3072, vocab=30522, max_pos=512):
    """BertForMaskedLM with every parameter randomised (the default init zeroes all biases and sets LayerNorm to identity,
    which would leave those code paths unpinned). The decoder is tied to word_embeddings. eval() mode, erf GELU."""
    import torch
    from transformers import BertConfig, BertForMaskedLM
    cfg = BertConfig(vocab_size=vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                     intermediate_size=inter, max_position_embeddings=max_pos, type_vocab_size=2, hidden_act="gelu",
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12, pad_token_id=0)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m = BertForMaskedLM(cfg)
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


def export_mlm_model(model, manifest: dict) -> np.ndarray:
    """Fill the blob of modelformat.bert_manifest(..., head="mlm") from a BertForMaskedLM: the encoder as
    embed_export.export_bert_model writes it, then the prediction head: transform dense and LayerNorm, and the decoder as
    a transposed copy of word_embeddings [H, vocab] plus cls.predictions.bias, zero-padded to Vp columns."""
    import copy

    import embed_export as ee
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)
    ops = manifest["ops"]
    gi = next(i for i, o in enumerate(ops) if o["op"] == "mask_gather")
    enc = copy.deepcopy(manifest)
    enc["ops"] = enc["ops"][:gi]
    enc["ops"][-1]["dst"] = -2
    eb = ee.export_bert_model(model.bert, enc)                     # the encoder's tensors come first in the blob
    blob[:eb.size] = eb[:blob.size]

    def put(off, arr):
        a = np.ascontiguousarray(arr.detach().double().numpy(), np.float32).ravel()
        blob[off // 4: off // 4 + a.size] = a

    pred = model.cls.predictions
    dense, ln, dec = ops[gi + 1], ops[gi + 2], ops[gi + 3]
    assert dense["act"] == "gelu" and ln["op"] == "layernorm" and dec["dst"] == -2 and len(ops) == gi + 4
    put(dense["w_offset"], pred.transform.dense.weight.t().contiguous())
    put(dense["b_offset"], pred.transform.dense.bias)
    put(ln["w_offset"], pred.transform.LayerNorm.weight)
    put(ln["b_offset"], pred.transform.LayerNorm.bias)
    word = model.bert.embeddings.word_embeddings.weight.detach()   # [vocab, H]; the decoder is word^T
    V, H = word.shape
    vp = dec["cout"]
    w = np.zeros((H, vp), np.float32)
    w[:, :V] = word.t().double().numpy()
    b = np.zeros(vp, np.float32)
    b[:V] = pred.bias.detach().double().numpy()
    blob[dec["w_offset"] // 4: dec["w_offset"] // 4 + H * vp] = w.ravel()
    blob[dec["b_offset"] // 4: dec["b_offset"] // 4 + vp] = b
    return blob


def mlm_reference(model, ids: np.ndarray, mask=None, types=None) -> np.ndarray:
    """transformers' own BertForMaskedLM forward in fp64: prediction logits [B, S, vocab] at every position (the attention
    mask is ids != 0 without one)."""
    import copy

    import torch
    m64 = copy.deepcopy(model).double()

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.int64))
    am = t(mask) if mask is not None else (t(ids) != 0).long()
    with torch.no_grad():
        out = m64(input_ids=t(ids), attention_mask=am, token_type_ids=None if types is None else t(types))
    return out.logits.numpy()
