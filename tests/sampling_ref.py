"""fp64 reference of a sampling generate bundle's step (DESIGN §3): Philox4x32-10, the kept set of temperature, top-k and
top-p by its rank-order definition and by transformers' warpers, and the draw, with the flags that mark a draw whose
outcome could turn on fp32 rounding."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC 2011) of a counter of four and a key of two 32-bit words"""
    c0, c1, c2, c3 = (int(v) & MASK for v in ctr)
    k0, k1 = (int(v) & MASK for v in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
    return c0, c1, c2, c3


def uniform53(seed, t):
    """the step's u in [0, 1): 53 bits of Philox4x32-10 with key (uint32(seed), 0) and counter (t, 0, 0, 0), as an integer U
    (u = U * 2^-53)"""
    x = philox4x32_10((t, 0, 0, 0), (int(seed) & MASK, 0))
    return ((x[0] >> 5) << 26) | (x[1] >> 6)


def rank_order(z):
    """ids by logit descending, ties to the lower id"""
    z = np.asarray(z, np.float64)
    return np.lexsort((np.arange(len(z)), -z))


def kept_set(z, temperature=1.0, top_k=0, top_p=1.0):
    """(kept ids in rank order, their weights, ambiguous): the first top_k tokens in rank order (0: all), weighted
    exp((z - max z) / temperature), cut to the shortest prefix whose weight reaches top_p of theirs (1: no cut). Ambiguous
    when a top-k boundary logit is within 1e-6 relative of (and not equal to) a neighbour on the other side, or a prefix sum
    lies within 1e-5 W of top_p W."""
    z = np.asarray(z, np.float64)
    order = rank_order(z)
    ambiguous = False
    if 0 < top_k < len(z):
        a, b = z[order[top_k - 1]], z[order[top_k]]
        ambiguous |= a != b and abs(a - b) <= 1e-6 * max(abs(a), abs(b))
        order = order[:top_k]
    w = np.exp((z[order] - z.max()) / temperature)
    if top_p < 1.0:
        cs = np.cumsum(w)
        thr = top_p * cs[-1]
        n = int(np.argmax(cs >= thr)) + 1
        ambiguous |= bool(np.any(np.abs(cs - thr) <= 1e-5 * cs[-1]))
        order, w = order[:n], w[:n]
    return order, w, bool(ambiguous)


def warpers_kept(z, temperature=1.0, top_k=0, top_p=1.0):
    """the ids transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper chain leaves finite, in fp64"""
    import torch
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(np.asarray(z, np.float64))[None].clone()
    ids = torch.zeros((1, 1), dtype=torch.long)
    s = TemperatureLogitsWarper(temperature)(ids, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p)(ids, s)
    return np.nonzero(torch.isfinite(s[0]).numpy())[0]


def _pick(kept, w, U):
    """the first id of `kept`, ascending, whose running weight exceeds u * W, and whether u * W lies within 1e-5 W of either
    edge of its interval"""
    by_id = np.argsort(kept, kind="stable")
    ids, cs = kept[by_id], np.cumsum(w[by_id])
    W = cs[-1]
    target = U * 2.0 ** -53 * W
    i = int(np.argmax(cs > target)) if (cs > target).any() else len(ids) - 1
    lo = cs[i - 1] if i else 0.0
    return int(ids[i]), bool(abs(target - lo) <= 1e-5 * W or abs(cs[i] - target) <= 1e-5 * W)


def draw(z, seed, t, temperature=1.0, top_k=0, top_p=1.0):
    """(token, ambiguous): the first kept id, ascending, whose running weight exceeds u * W. Ambiguous when a top-k boundary
    logit is within 1e-6 relative of (and not equal to) a neighbour on the other side, when u * W lies within 1e-5 W of
    either edge of the chosen token's running-sum interval, or when a top-p cut anywhere the prefix sum is within 1e-5 W of
    top_p W would draw another token. top_k = 1 is the argmax."""
    z = np.asarray(z, np.float64)
    order = rank_order(z)
    ambiguous = False
    if 0 < top_k < len(z):
        a, b = z[order[top_k - 1]], z[order[top_k]]
        ambiguous |= a != b and abs(a - b) <= 1e-6 * max(abs(a), abs(b))
        order = order[:top_k]
    w = np.exp((z[order] - z.max()) / temperature)
    U = uniform53(seed, t)
    cuts = [len(order)]
    if top_p < 1.0:
        cs = np.cumsum(w)
        thr, tol = top_p * cs[-1], 1e-5 * cs[-1]
        first = lambda v: min(len(cs), int(np.argmax(cs >= v)) + 1 if (cs >= v).any() else len(cs))  # noqa: E731
        cuts = [first(thr), first(thr - tol), first(thr + tol)]
    g, edge = _pick(order[:cuts[0]], w[:cuts[0]], U)
    ambiguous |= edge or any(_pick(order[:c], w[:c], U)[0] != g for c in cuts[1:])
    return g, bool(ambiguous and top_k != 1)


def kept_probabilities(z, temperature=1.0, top_k=0, top_p=1.0):
    """{id: probability} of the kept distribution, fp64"""
    kept, w, _a = kept_set(z, temperature, top_k, top_p)
    return dict(zip(kept.tolist(), (w / w.sum()).tolist()))
