"""fp64 reference of the encoder head's outputs (test infrastructure), written from their definitions: from the last
hidden states h[rows, S, H] and the request's mask (or, without a mask input, the ids),

  sequence_output = h                                   cls_embedding  = h[:, 0]
  mean_embedding  = sum_p m[p] h[p] / max(sum_p m[p], 1e-9),  m[p] = mask[p] != 0 (no mask: ids[p] != 0)

and, with normalize, x / max(||x||_2, 1e-12) (torch.nn.functional.normalize). pooled_output is a copy of the pooler."""
from __future__ import annotations

import numpy as np


def token_mask(ids, mask=None) -> np.ndarray:
    """m[rows, S] as float64: the mask input's nonzero entries, or the nonzero ids when there is no mask input"""
    return (np.asarray(mask if mask is not None else ids) != 0).astype(np.float64)


def normalize(x, eps=1e-12) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), eps)


def mean_embedding(h, ids, mask=None, norm=False) -> np.ndarray:
    h = np.asarray(h, np.float64)
    m = token_mask(ids, mask)
    s = np.einsum("rs,rsh->rh", m, h)
    out = s / np.maximum(m.sum(axis=1, keepdims=True), 1e-9)
    return normalize(out) if norm else out


def cls_embedding(h, norm=False) -> np.ndarray:
    c = np.asarray(h, np.float64)[:, 0]
    return normalize(c) if norm else c


def embed_ref(h, ids, mask=None, normalize_cls=False, normalize_mean=False) -> dict:
    """{kind: fp64 array} of sequence_output, cls_embedding and mean_embedding"""
    return {"sequence_output": np.asarray(h, np.float64), "cls_embedding": cls_embedding(h, normalize_cls),
            "mean_embedding": mean_embedding(h, ids, mask, normalize_mean)}
