"""transformers.GPT2LMHeadModel as an independent numeric pin for next-token bundles (test infrastructure): a seeded model
from a config with every parameter randomised, exported into a modelformat.gpt2_manifest blob, and its own fp64 forward as
the reference."""
from __future__ import annotations

import numpy as np

from torch_export import _rand_like


def hf_gpt2_model(seed: int, hidden=768, layers=12, heads=12, vocab=50257, max_pos=1024):
    """GPT2LMHeadModel with every parameter randomised, LayerNorm and biases included (the default init zeroes the biases
    and sets LayerNorm to identity, which would leave those code paths unpinned). lm_head is tied to wte. eval() mode,
    tanh GELU (gelu_new), eager attention."""
    import torch
    from transformers import GPT2Config, GPT2LMHeadModel
    cfg = GPT2Config(vocab_size=vocab, n_positions=max_pos, n_embd=hidden, n_layer=layers, n_head=heads,
                     activation_function="gelu_new", resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0, layer_norm_epsilon=1e-5)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m = GPT2LMHeadModel(cfg)
    gen = torch.Generator().manual_seed(seed + 13)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith(("ln_1.weight", "ln_2.weight", "ln_f.weight")):
                p.copy_(_rand_like(p, gen, 0.1, 1.0))
            elif name.endswith("bias"):
                p.copy_(_rand_like(p, gen, 0.1))
            elif name.endswith(("wte.weight", "wpe.weight")):
                p.copy_(_rand_like(p, gen, 0.1))
            else:                                                   # Conv1D weights [in, out]
                p.copy_(_rand_like(p, gen, (1.0 / p.shape[0]) ** 0.5))
    return m.eval()


def export_gpt2_model(model, manifest: dict) -> np.ndarray:
    """Fill the blob of modelformat.gpt2_manifest from a GPT2LMHeadModel: wte and wpe, per block ln_1, c_attn, c_proj,
    ln_2, c_fc, c_proj (Conv1D weights are [in, out], the bundle's layout), ln_f, and the decoder as wte transposed
    [H, vocab] zero-padded to Vp columns with a zero bias."""
    blob = np.zeros(manifest["weights_bytes"] // 4, np.float32)

    def put(off, arr):
        a = np.ascontiguousarray(arr.detach().double().numpy(), np.float32).ravel()
        blob[off // 4: off // 4 + a.size] = a

    ops = manifest["ops"]
    tr = model.transformer
    emb = ops[0]
    put(emb["word_offset"], tr.wte.weight)
    put(emb["pos_offset"], tr.wpe.weight[:emb["max_pos"]])
    for i, blk in enumerate(tr.h):
        ln1, attn, _att, proj, ln2, fc, proj2 = ops[1 + 7 * i: 8 + 7 * i]
        for op, mod in ((ln1, blk.ln_1), (ln2, blk.ln_2), (attn, blk.attn.c_attn), (proj, blk.attn.c_proj), (fc, blk.mlp.c_fc),
                        (proj2, blk.mlp.c_proj)):
            put(op["w_offset"], mod.weight)
            put(op["b_offset"], mod.bias)
    _last, lnf, dec = ops[-3:]
    put(lnf["w_offset"], tr.ln_f.weight)
    put(lnf["b_offset"], tr.ln_f.bias)
    word = tr.wte.weight.detach()
    V, H = word.shape
    w = np.zeros((H, dec["cout"]), np.float32)
    w[:, :V] = word.t().double().numpy()
    blob[dec["w_offset"] // 4: dec["w_offset"] // 4 + w.size] = w.ravel()
    return blob


def gpt2_reference(model, ids: np.ndarray, mask=None, device="cpu", at=None) -> np.ndarray:
    """transformers' own GPT2LMHeadModel forward in fp64 on `device`: logits [B, S, vocab] at every position, or with
    at = positions [B] the [B, vocab] logits there, with its default position ids 0..S-1 whatever the padding."""
    import copy

    import torch
    m64 = copy.deepcopy(model).double().to(device)

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.int64)).to(device)
    with torch.no_grad():
        h = m64.transformer(input_ids=t(ids), attention_mask=None if mask is None else t(mask)).last_hidden_state
        if at is not None:
            h = h[torch.arange(h.shape[0], device=device), t(at)]
        return m64.lm_head(h).cpu().numpy()


def gpt2_inputs(B, S, vocab, seed):
    """{input_ids, attention_mask} int32 [B, S]: random ids in [0, vocab) (id 0 included: GPT-2's "!", not padding) and a
    padding pattern per row cycling through unpadded, right-padded and left-padded (padded ids 0)."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, vocab, (B, S)).astype(np.int32)
    mask = np.ones((B, S), np.int32)
    for r in range(B):
        n = int(rng.integers(1, S)) if S > 1 else 1
        if r % 3 == 1:
            mask[r, n:], ids[r, n:] = 0, 0
        elif r % 3 == 2:
            mask[r, :S - n], ids[r, :S - n] = 0, 0
    return {"input_ids": ids, "attention_mask": mask}
