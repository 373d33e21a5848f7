"""-m gpu: the transformer kernels (X5) through their raw entries and through the server, against the fp64 reference of
oracle.models (attention_ref / layer_norm_ref, the functions graph_forward uses).  Tolerance 1e-4 relative to max(1,|ref|).

launch_attention picks its kernel from the sequence length S and the head width d: the tiled kernels for S <= 32 / 64 /
128 / 256 while their shared memory fits, the key-block (online softmax) kernel above that for d % 4 == 0 and d <= 128, the
row kernel for other widths while K and V of a head fit. The S values sit on both sides of every one of those boundaries."""
import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

pytestmark = pytest.mark.gpu
TOL = 1e-4
lib = t._lib.lib

SEQS = [13, 32, 33, 50, 64, 65, 128, 129, 188, 189, 200, 249, 250, 256, 257, 300, 367, 368, 384, 509, 512]


def _torch():
    import torch
    assert torch.cuda.is_available()
    return torch


def _err(got, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


def _ids(rng, bsz, S):
    """One sequence of each mask kind, then random ones: no [PAD]; a padded tail; every token [PAD] (all keys masked: the
    same -10000 on every score, so softmax over the raw scores); [PAD] at position 0 and a few inside."""
    ids = rng.integers(1, 1000, (bsz, S)).astype(np.int32)
    kinds = ["none", "tail", "all", "first"]
    for b in range(bsz):
        kind = kinds[b % 4]
        if kind == "tail":
            ids[b, max(1, (2 * S) // 3):] = 0
        elif kind == "all":
            ids[b] = 0
        elif kind == "first":
            ids[b, 0] = 0
            ids[b, rng.integers(0, S, max(1, S // 16))] = 0
    return ids


def _qkv(rng, bsz, S, H, score_std):
    """q and k scaled so that q.k / sqrt(d) has a standard deviation of score_std: the max subtraction and the key-block
    rescaling change the result at this spread."""
    qkv = rng.standard_normal((bsz, S, 3 * H))
    qkv[..., :2 * H] *= np.sqrt(score_std)
    return qkv.astype(np.float32)


def _attention(qkv, ids, H, heads, offset=0):
    """tfsc_k_attention twice into NaN-filled outputs; both launches must give the same bits. offset (floats) shifts
    qkv and ctx off 16-byte alignment."""
    torch = _torch()
    bsz, S, _ = qkv.shape
    qd = torch.empty(qkv.size + offset, device="cuda")
    qd[offset:] = torch.from_numpy(qkv.ravel()).cuda()
    idd = torch.from_numpy(ids).cuda() if ids is not None else None
    outs = []
    for _ in range(2):
        cd = torch.full((bsz * S * H + offset,), float("nan"), device="cuda")
        rc = lib.tfsc_k_attention(qd[offset:].data_ptr(), idd.data_ptr() if idd is not None else None, cd[offset:].data_ptr(),
                                  bsz, S, H, heads, None)
        if rc < 0:
            return rc
        torch.cuda.synchronize()
        outs.append(cd[offset:].cpu().numpy().reshape(bsz, S, H))
    assert np.array_equal(outs[0], outs[1], equal_nan=True), "two launches differ"
    return outs[0]


def _ref(qkv, ids, heads):
    import torch
    return models.attention_ref(torch.from_numpy(qkv).double(), None if ids is None else torch.from_numpy(ids), heads).numpy()


def _check(S, d, heads, bsz, score_std, seed, masked=True, offset=0):
    rng = np.random.default_rng(seed)
    H = d * heads
    qkv = _qkv(rng, bsz, S, H, score_std)
    ids = _ids(rng, bsz, S) if masked else None
    got = _attention(qkv, ids, H, heads, offset)
    assert not isinstance(got, int), f"tfsc_k_attention returned {got}: {lib.tfsc_last_error().decode()}"
    assert not np.isnan(got).any()
    err = _err(got, _ref(qkv, ids, heads))
    assert err <= TOL, err


@pytest.mark.parametrize("S", SEQS)
@pytest.mark.parametrize("d", [16, 64, 96, 128])
def test_attention_matches_fp64(S, d):
    heads = (1, 2, 12)[(SEQS.index(S) + d // 16) % 3]
    bsz = 4 if heads == 12 else 5
    _check(S, d, heads, bsz, 4.0, S * 131 + d)
    _check(S, d, heads, 2, 4.0, S * 131 + d + 1, masked=False)


@pytest.mark.parametrize("S,d", [(13, 64), (128, 64), (257, 32), (512, 64), (509, 128), (384, 96)])
def test_attention_peaked_scores(S, d):
    """scores with a spread near 30: softmax is close to one-hot and exp(m_old - m_new) underflows between key blocks"""
    _check(S, d, 2, 4, 30.0, S + d)


@pytest.mark.parametrize("S", [128, 384, 512])
def test_attention_bert_base_batch8(S):
    """BERT-base attention: batch 8, hidden 768, 12 heads (d = 64)"""
    _check(S, 64, 12, 8, 4.0, S)


@pytest.mark.parametrize("S,d,heads", [(13, 18, 2), (129, 18, 1), (300, 18, 2), (512, 18, 1), (13, 160, 1), (64, 160, 2),
                                       (151, 160, 1)])
def test_attention_row_kernel_head_widths(S, d, heads):
    """head widths the tiled kernels do not take (d % 4 != 0, d > 128) run on the row kernel"""
    _check(S, d, heads, 4, 4.0, S * 7 + d)


@pytest.mark.parametrize("S", [64, 256])
def test_attention_unaligned_buffers(S):
    """qkv / ctx off 16-byte alignment: the row kernel serves them while it fits"""
    _check(S, 64, 2, 3, 4.0, S, offset=1)


def test_attention_rejects_shapes_no_kernel_runs():
    torch = _torch()
    x = torch.zeros(4 * 1200 * 3 * 320, device="cuda")
    for S, H, heads, off in [(152, 160, 1, 0), (1110, 36, 2, 0), (512, 128, 2, 1), (64, 100, 3, 0), (0, 64, 1, 0)]:
        rc = lib.tfsc_k_attention(x[off:].data_ptr(), None, x[off:].data_ptr(), 2, S, H, heads, None)
        assert rc == t._lib.E_INVALID, (S, H, heads, off, rc)
    # the last size that fits the row kernel still runs
    assert not isinstance(_attention(np.zeros((1, 1109, 108), np.float32), None, 36, 2), int)


# ---- LayerNorm ----------------------------------------------------------------------------------------------------
def _layernorm(x, res, gamma, beta, eps):
    torch = _torch()
    tokens, H = x.shape
    xd, gd, bd = (torch.from_numpy(a).cuda() for a in (x, gamma, beta))
    rd = torch.from_numpy(res).cuda() if res is not None else None
    outs = []
    for _ in range(2):
        yd = torch.full((tokens, H), float("nan"), device="cuda")
        t._lib.check(lib.tfsc_k_layernorm(xd.data_ptr(), rd.data_ptr() if rd is not None else None, gd.data_ptr(), bd.data_ptr(),
                                          yd.data_ptr(), tokens, H, eps, None), "layernorm")
        torch.cuda.synchronize()
        outs.append(yd.cpu().numpy())
    assert np.array_equal(outs[0], outs[1], equal_nan=True), "two launches differ"
    return outs[0]


def _ln_ref(x, res, gamma, beta, eps):
    import torch
    v = torch.from_numpy(x).double() + (torch.from_numpy(res).double() if res is not None else 0)
    return models.layer_norm_ref(v, torch.from_numpy(gamma).double(), torch.from_numpy(beta).double(), eps).numpy()


@pytest.mark.parametrize("H", [64, 768, 1000, 1024, 4096, 12272])
@pytest.mark.parametrize("with_res", [False, True])
def test_layernorm_matches_fp64(H, with_res):
    rng = np.random.default_rng(H + with_res)
    tokens = 37
    x = rng.standard_normal((tokens, H)).astype(np.float32)
    res = rng.standard_normal((tokens, H)).astype(np.float32) if with_res else None
    gamma = (1 + 0.1 * rng.uniform(-1, 1, H)).astype(np.float32)
    beta = (0.1 * rng.uniform(-1, 1, H)).astype(np.float32)
    for eps in (1e-12, 1e-5):
        got = _layernorm(x, res, gamma, beta, eps)
        assert not np.isnan(got).any() and _err(got, _ln_ref(x, res, gamma, beta, eps)) <= TOL


@pytest.mark.parametrize("H", [64, 768, 1000, 1024, 4096])
def test_layernorm_large_mean_keeps_two_pass_variance(H):
    """rows 1e3 + N(0, 1): E[x^2] - E[x]^2 in fp32 would lose every digit of the variance"""
    rng = np.random.default_rng(H)
    x = (1e3 + rng.standard_normal((16, H))).astype(np.float32)
    gamma = (1 + 0.1 * rng.uniform(-1, 1, H)).astype(np.float32)
    beta = (0.1 * rng.uniform(-1, 1, H)).astype(np.float32)
    got = _layernorm(x, None, gamma, beta, 1e-12)
    assert _err(got, _ln_ref(x, None, gamma, beta, 1e-12)) <= TOL


def test_layernorm_rejects_rows_that_do_not_fit():
    torch = _torch()
    x = torch.zeros(2 * 12273, device="cuda")
    for H in (0, 12273):
        rc = lib.tfsc_k_layernorm(x.data_ptr(), None, x.data_ptr(), x.data_ptr(), x.data_ptr(), 2, H, 1e-12, None)
        assert rc == t._lib.E_INVALID, (H, rc)


# ---- through the server -------------------------------------------------------------------------------------------
def _server(man, count=4, arena=256 << 20):
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.template": "manifest",
           "modelProvider.synthetic.manifest": man, "modelProvider.synthetic.count": count, "gpu.devices": [0],
           "gpu.arenaBytes": arena, "serving.maxConcurrentModels": 4, "modelCache.size": 1 << 30, "gpu.maxBatch": 8}
    return t.Server(cfg)


@pytest.mark.parametrize("S", [384, 512])
def test_one_layer_bert_long_sequences_through_server(S):
    """S = 384 / 512 (the SQuAD lengths; max_pos defaults to 512) with 64-wide heads. Ids above the vocabulary and below 0
    are clamped for the embedding but are not [PAD], so they stay unmasked -- the oracle does the same."""
    _torch()
    vocab = 100
    args = dict(seq=S, hidden=128, layers=1, heads=2, inter=256, vocab=vocab, max_pos=512, labels=3)
    man = t.modelformat.bert_manifest(**args)
    oman = models.graph_manifest([S], models.bert_ops(**args), 4, ("input_ids", "logits"), "int32")
    rng = np.random.default_rng(S)
    ids = rng.integers(1, vocab, (4, S)).astype(np.int32)
    ids[0, 5], ids[0, 17], ids[2, 3] = vocab + 5, -3, -3
    ids[1, S // 2:] = 0
    ids[2, 0] = 0
    ids[3, 200:] = 0
    ids[3, 7] = vocab + 5
    with _server(man) as srv:
        y = srv.predict("m1", "1", ids)
    ref = models.graph_forward(oman, models.synth_graph_blob(oman, 1001), ids, np.float64)
    assert y.shape == (4, 3) and _err(y, ref) <= TOL


@pytest.mark.parametrize("inter", [385, 387])
def test_bert_with_odd_buffer_sizes_through_server(inter):
    """Buffer 1 holds qkv and the feed-forward intermediate, so it is S * max(3H, inter) floats per sequence. With S = 383 and
    an odd intermediate width, rows * that is not a multiple of 4 floats; the executor still places every scratch buffer on
    a 256-byte boundary, so the attention after it gets aligned qkv / ctx and the key-block kernel at any batch size."""
    _torch()
    args = dict(seq=383, hidden=128, layers=1, heads=2, inter=inter, vocab=100, max_pos=512, labels=3)
    man = t.modelformat.bert_manifest(**args)
    oman = models.graph_manifest([383], models.bert_ops(**args), 4, ("input_ids", "logits"), "int32")
    rng = np.random.default_rng(inter)
    blob = models.synth_graph_blob(oman, 1000)
    with _server(man) as srv:
        for bsz in (1, 3, 2):
            ids = rng.integers(1, 100, (bsz, 383)).astype(np.int32)
            ids[-1, 300:] = 0
            y = srv.predict("m0", "1", ids)
            ref = models.graph_forward(oman, blob, ids, np.float64)
            assert y.shape == (bsz, 3) and _err(y, ref) <= TOL, bsz


@pytest.mark.parametrize("hidden,heads,seq,what",[(320, 2, 384, "attention"), (36, 2, 1200, "attention"),
                                                   (12800, 100, 4, "LayerNorm")])
def test_loader_rejects_ops_no_kernel_runs(hidden, heads, seq, what):
    """a bundle whose attention or LayerNorm has no kernel fails when the manifest is read, with the reason, instead of
    paging in and answering every request with an internal error"""
    _torch()
    man = t.modelformat.bert_manifest(seq=seq, hidden=hidden, layers=1, heads=heads, inter=64, vocab=10, max_pos=seq, labels=2)
    with _server(man) as srv:
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("m0", "1", np.ones((1, seq), np.int32))
    assert e.value.code != t._lib.E_INTERNAL and f"no {what} kernel" in str(e.value), str(e.value)
