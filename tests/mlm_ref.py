"""fp64 reference of fill-mask (masked-language-model) bundles, test infrastructure: the mask_gather op (which tokens are
[MASK] slots, in which order), the fill-mask head's top k (descending logit, ties to the lower id, as tf.math.top_k) with
softmax probabilities over the first `vocab` logits, and a whole-bundle forward that runs the encoder with
bert_pair_ref.pair_forward and the ops after the gather on the M slots."""
from __future__ import annotations

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def mask_gather_ref(hidden, ids, mask, mask_token_id, M):
    """positions [rows, M] int32 (-1: empty slot) and the gathered hidden states [rows, M, H] (zeros for empty slots).
    Token p is a candidate when ids[p] == mask_token_id and, with a mask, mask[p] != 0; slots fill in ascending p and
    candidates past the first M are not served."""
    rows, S = ids.shape
    H = hidden.shape[-1]
    pos = np.full((rows, M), -1, np.int32)
    gat = np.zeros((rows, M, H), hidden.dtype)
    for r in range(rows):
        cand = ids[r] == mask_token_id
        if mask is not None:
            cand &= mask[r] != 0
        p = np.nonzero(cand)[0][:M]
        pos[r, :len(p)] = p
        gat[r, :len(p)] = hidden[r, p]
    return pos, gat


def top_k_ref(logits, positions, vocab, k):
    """The fill-mask head on logits [rows, M, Vp] (only the first vocab columns count): ids [rows, M, k] by a stable argsort
    of the negated fp32 logits, probabilities [rows, M, k] from an fp64 softmax over the vocab logits, and the logits at
    those ids; an empty slot is (-1, 0, -FLT_MAX)."""
    rows, M = positions.shape
    lg = np.asarray(logits)[:, :, :vocab]
    ids = np.full((rows, M, k), -1, np.int32)
    probs = np.zeros((rows, M, k), np.float64)
    vals = np.full((rows, M, k), -FLT_MAX, np.float64)
    for r in range(rows):
        for s in range(M):
            if positions[r, s] < 0:
                continue
            x = lg[r, s]
            order = np.argsort(-x, kind="stable")[:k]
            x64 = x.astype(np.float64)
            e = np.exp(x64 - x64.max())
            ids[r, s] = order
            probs[r, s] = e[order] / e.sum()
            vals[r, s] = x64[order]
    return ids, probs, vals


def mlm_inputs(B, S, vocab, n_mask, seed, mask_token_id):
    """{input_ids, input_mask, segment_ids} int32 [B, S]: random ids in [mask_token_id + 1, vocab) (so no other token
    collides with [MASK]), a padded tail (mask 0, id 0) in odd rows, a second segment from the middle, and n_mask [MASK]
    tokens per row among the unpadded positions (positions 0 and S - 1 in row 0 when S allows). Row 1 also gets a [MASK]
    in its padded tail, which must not be served."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(mask_token_id + 1, vocab, (B, S)).astype(np.int32)
    mask = np.ones((B, S), np.int32)
    seg = np.zeros((B, S), np.int32)
    seg[:, S // 2:] = 1
    for r in range(B):
        live = S
        if r % 2 == 1 and S > 2:
            live = int(rng.integers(max(1, S // 2), S))
            ids[r, live:], mask[r, live:] = 0, 0
        n = min(n_mask, live)
        p = rng.choice(live, n, replace=False) if n else np.zeros(0, int)
        if r == 0 and n >= 2 and live == S:
            p[:2] = [0, S - 1]
            p = np.unique(p)
        ids[r, p] = mask_token_id
        if r == 1 and live < S:
            ids[r, S - 1] = mask_token_id                 # [MASK] under mask 0
    return {"input_ids": ids, "input_mask": mask, "segment_ids": seg}


def _truncated(man: dict, upto: int) -> dict:
    """The bundle's ops before index `upto`, the last of them answering: the encoder's [S, 1, H] hidden states."""
    import copy
    t = copy.deepcopy(man)
    t["ops"] = t["ops"][:upto]
    t["ops"][-1]["dst"] = -2
    t["signature"] = {k: v for k, v in t["signature"].items() if k != "outputs"}
    t["signature"]["output"] = "hidden"
    return t


def mlm_forward(man: dict, blob: np.ndarray, x, dtype=np.float64):
    """(positions [B, M] int32, logits [B, M, Vp]) of a fill-mask bundle in `dtype`. x as for bert_pair_ref.pair_forward:
    {name: int array [B, S]} for a bundle with signature.inputs, or the ids array of a single-input bundle."""
    import torch
    import torch.nn.functional as F

    import bert_pair_ref as pr
    from oracle import models
    td = torch.float64 if dtype == np.float64 else torch.float32
    gi = next(i for i, o in enumerate(man["ops"]) if o["op"] == "mask_gather")
    g = man["ops"][gi]
    S, H = g["h"], g["c"]
    hidden = pr.pair_forward(_truncated(man, gi), blob, x, dtype).reshape(-1, S, H)
    roles = {i["role"]: i["name"] for i in man["signature"].get("inputs", [])}
    ids = np.asarray(x[roles["ids"]] if roles else x).reshape(-1, S)
    mask = np.asarray(x[roles["mask"]]).reshape(-1, S) if "mask" in roles else None
    pos, gat = mask_gather_ref(hidden, ids, mask, g["mask_token_id"], g["slots"])

    def vec(off, n):
        return torch.from_numpy(blob[off // 4: off // 4 + n]).to(td)

    bufs = {g["dst"]: torch.from_numpy(gat).to(td)}
    for o in man["ops"][gi + 1:]:
        src = bufs[o["src"]]
        if o["op"] == "layernorm":
            y = models.layer_norm_ref(src, vec(o["w_offset"], o["c"]), vec(o["b_offset"], o["c"]), o.get("eps", 1e-12))
        elif o["op"] == "conv":
            y = src @ vec(o["w_offset"], o["c"] * o["cout"]).view(o["c"], o["cout"]) + vec(o["b_offset"], o["cout"])
            y = F.gelu(y) if o.get("act") == "gelu" else y
        else:
            raise ValueError(f"op {o['op']} is not part of a fill-mask head")
        bufs[o["dst"]] = y
    return pos, bufs[-2].numpy().astype(dtype)
