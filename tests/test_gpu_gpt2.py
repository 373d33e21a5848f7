"""-m gpu: GPT-2 next-token bundles. Causal attention against fp64 on both sides of every dispatch boundary and bit for bit
under changes past a query, the no-LayerNorm embedding and last_token bit for bit, the tanh GELU on both GEMM paths, the
next-token head against fp64 and bit for bit against the fill-mask head, a full-size seeded GPT-2 small through the
server against transformers fp64, every front-end, launch counts, programmatic-dependent-launch bit identity and the
forward hop between two ranks."""
import json
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import wire

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpt2_export as ge  # noqa: E402
import gpt2_ref as gr  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
K = 5
ALL = [{"name": "next_token_position", "kind": "next_token_position"}] + \
      [{"name": k, "kind": k, "k": K} for k in mf.NEXT_TOKEN_OUTPUT_KINDS[1:]]
NAMES = sorted(o["name"] for o in ALL)
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=512)
FLT_MAX = np.float32(np.finfo(np.float32).max)


def _ptr(x):
    return None if x is None else x.data_ptr()


# ------------------------------------------------------------------------------------- causal attention ----
def _attention(qkv, mask, heads, causal=True):
    import torch
    B, S, H3 = qkv.shape
    q = torch.from_numpy(np.ascontiguousarray(qkv, np.float32)).cuda()
    c = torch.full((B, S, H3 // 3), float("nan"), device="cuda")
    m = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, np.int32)).cuda()
    fn = lib.tfsc_k_attention_causal if causal else lib.tfsc_k_attention_mask
    t._lib.check(fn(_ptr(q), _ptr(m), S, _ptr(c), B, S, H3 // 3, heads, None), "attention_causal")
    torch.cuda.synchronize()
    return c.cpu().numpy()


def _masks(S):
    """rows: right-padded, left-padded, fully padded, unpadded"""
    m = np.ones((4, S), np.int32)
    n = max(1, S // 3)
    m[0, S - n:] = 0 if S > 1 else 1
    m[1, :S - n] = 0 if S > 1 else 1
    m[2] = 0
    return m


@pytest.mark.parametrize("d", [16, 64, 128])
@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 320, 511, 1024])
def test_causal_attention_matches_fp64(S, d):
    heads = 2
    rng = np.random.default_rng(S * 7 + d)
    for spread in (3.0, 30.0):
        # q . k / sqrt(d) of a few units or ~30: q and k entries of spread / d^(1/4)
        qkv = rng.standard_normal((4, S, 3 * heads * d)).astype(np.float32)
        qkv[..., :2 * heads * d] *= spread ** 0.5 / d ** 0.25 / 2
        for mask in (None, _masks(S)):
            got = _attention(qkv, mask, heads)
            ref = gr.causal_attention_ref(qkv.astype(np.float64), heads, mask)
            # padded queries of a partly padded row see only masked keys: their rows are not compared (the BERT -10000
            # rounds their scores in fp32); every other row is
            rows = np.ones((4, S), bool) if mask is None else (mask != 0) | (mask == 0).all(axis=1, keepdims=True)
            err = np.abs(got - ref)[rows].max()
            tol = 2e-5 * max(1.0, np.abs(ref).max())
            assert err <= tol, (spread, mask is None, err)


@pytest.mark.parametrize("S,i", [(200, 77), (1024, 600), (1024, 31)])
def test_causality_in_bits(S, i):
    """changing q, k and v of every position after i leaves the rows up to i bit-identical"""
    heads, d = 12, 64
    rng = np.random.default_rng(i)
    qkv = rng.standard_normal((2, S, 3 * heads * d)).astype(np.float32)
    mask = np.ones((2, S), np.int32)
    mask[1, S - 5:] = 0
    a = _attention(qkv, mask, heads)
    qkv[:, i + 1:] = rng.standard_normal(qkv[:, i + 1:].shape).astype(np.float32)
    b = _attention(qkv, mask, heads)
    assert a[:, :i + 1].tobytes() == b[:, :i + 1].tobytes()
    assert not np.array_equal(a[:, i + 1:], b[:, i + 1:])


def test_causal_attention_rejections():
    import torch
    q = torch.zeros(3 * 96 * 4 + 1, device="cuda")
    c = torch.zeros(96 * 4 + 1, device="cuda")
    E = t._lib.E_INVALID
    assert lib.tfsc_k_attention_causal(_ptr(q), None, 4, _ptr(c), 1, 4, 96, 16, None) == E          # d = 6
    assert lib.tfsc_k_attention_causal(_ptr(q[1:]), None, 4, _ptr(c), 1, 4, 96, 2, None) == E       # misaligned
    assert lib.tfsc_k_attention_causal(_ptr(q), _ptr(q), 3, _ptr(c), 1, 4, 96, 2, None) == E        # mask_stride < seq
    assert lib.tfsc_k_attention_causal(_ptr(q), None, 4, _ptr(c), 1, 4, 96, 2, None) == 0


# ------------------------------------------------------------------------------- embedding / last_token ----
@pytest.mark.parametrize("H,misalign", [(768, False), (768, True), (30, False)])
def test_embed_positions_bits(H, misalign):
    import torch
    B, S, V, P = 3, 37, 500, 64
    rng = np.random.default_rng(H)
    word = rng.standard_normal((V, H)).astype(np.float32)
    pos = rng.standard_normal((P, H)).astype(np.float32)
    ids = rng.integers(-3, V + 3, (B, S + 2)).astype(np.int32)                    # stride S + 2, ids out of range clamp
    off = 1 if misalign else 0
    wd = torch.from_numpy(np.concatenate([np.zeros(off, np.float32), word.ravel()])).cuda()
    pd = torch.from_numpy(pos).cuda()
    idd = torch.from_numpy(ids).cuda()
    y = torch.full((B * S * H,), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_embed_positions(_ptr(idd), S + 2, _ptr(wd[off:]), _ptr(pd), _ptr(y), B, S, H, V, None), "embed_positions")
    torch.cuda.synchronize()
    want = word[np.clip(ids[:, :S], 0, V - 1)] + pos[:S]
    assert y.cpu().numpy().reshape(B, S, H).tobytes() == want.tobytes()


@pytest.mark.parametrize("H,misalign", [(768, False), (768, True), (1, False)])
@pytest.mark.parametrize("S", [1, 300])
def test_last_token_bits(S, H, misalign):
    import torch
    rows = 7
    rng = np.random.default_rng(S + H)
    h = rng.standard_normal((rows, S, H)).astype(np.float32)
    mask = (rng.random((rows, S + 1)) < 0.5).astype(np.int32)
    mask[0] = 0                                                            # no attended token
    mask[1] = 1
    mask[2, :S] = 0
    mask[2, 0] = 1
    off = 1 if misalign else 0
    hd = torch.from_numpy(np.concatenate([np.zeros(off, np.float32), h.ravel()])).cuda()
    md = torch.from_numpy(mask).cuda()
    for m in (mask, None):
        pos = torch.full((rows,), 12345, dtype=torch.int32, device="cuda")
        gat = torch.full((rows * H + off,), float("nan"), device="cuda")
        t._lib.check(lib.tfsc_k_last_token(_ptr(hd[off:]), None if m is None else _ptr(md), S + 1, rows, S, H, _ptr(pos),
                                           _ptr(gat[off:]), None), "last_token")
        torch.cuda.synchronize()
        want_pos, want = gr.last_token_ref(h, None if m is None else mask[:, :S])
        assert np.array_equal(pos.cpu().numpy(), want_pos)
        assert gat[off:].cpu().numpy().reshape(rows, H).tobytes() == want.tobytes()


# ------------------------------------------------------------------------------------------- gelu_tanh ----
@pytest.mark.parametrize("M,tc", [(16, False), (128, True)])
def test_gelu_tanh_on_both_gemm_paths(M, tc):
    import torch
    N, Kd = 256, 128
    rng = np.random.default_rng(M)
    a = rng.standard_normal((M, Kd)).astype(np.float32)
    b = (rng.standard_normal((Kd, N)) / 4).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    ad, bd, biasd = (torch.from_numpy(v).cuda() for v in (a, b, bias))
    c = torch.full((M, N), float("nan"), device="cuda")
    fn = lib.tfsc_k_gemm_tc if tc else lib.tfsc_k_gemm
    t._lib.check(fn(_ptr(ad), _ptr(bd), _ptr(biasd), None, _ptr(c), M, N, Kd, Kd, 7, None), "gemm gelu_tanh")
    torch.cuda.synchronize()
    ref = gr.gelu_tanh(a.astype(np.float64) @ b + bias)
    assert np.abs(c.cpu().numpy() - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------ next-token head ----
def _head_logits(rows, vocab, vp, seed):
    """rows of vp logits: the first vocab random with ties among the largest, the padding columns 1e30 (never selected);
    row 1 has position -1"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, vp)).astype(np.float32)
    x[:, vocab:] = 1e30
    x[:, 7] = x[:, 3] = x[:, :vocab].max(axis=1) + 1                   # a tie for first place: the lower id wins
    pos = np.arange(rows, dtype=np.int32)
    if rows > 1:
        pos[1] = -1
    return x, pos


def _next_head(x, pos, vocab, k):
    import torch
    rows, vp = x.shape
    xd, pd = torch.from_numpy(x).cuda(), torch.from_numpy(pos).cuda()
    ids = torch.full((rows, k), 12345, dtype=torch.int32, device="cuda")
    pr = torch.full((rows, k), float("nan"), device="cuda")
    lg = torch.full((rows, k), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_next_token_head(_ptr(xd), vp, _ptr(pd), rows, vocab, k, _ptr(ids), _ptr(pr), _ptr(lg), None), "next_token_head")
    torch.cuda.synchronize()
    return ids.cpu().numpy(), pr.cpu().numpy(), lg.cpu().numpy()


@pytest.mark.parametrize("k", [1, 5, 32])
@pytest.mark.parametrize("vocab,vp", [(50257, 50272), (57344, 57344), (57343, 57344)])
def test_next_token_head_matches_fp64(vocab, vp, k):
    rows = 9
    x, pos = _head_logits(rows, vocab, vp, vocab + k)
    ids, pr, lg = _next_head(x, pos, vocab, k)
    rid, rp, rl = gr.top_k_ref(x, pos, vocab, k)
    assert np.array_equal(ids, rid) and (ids < vocab).all()
    assert ids[0, 0] == 3 and (k == 1 or ids[0, 1] == 7)
    assert np.array_equal(lg, rl.astype(np.float32))
    live = pos >= 0
    assert np.all(np.abs(pr[live] - rp[live]) <= 1e-5 * np.maximum(rp[live], 1e-30) + 1e-12)
    assert (pr[~live] == 0).all() and (lg[~live] == -FLT_MAX).all() and (ids[~live] == -1).all()


@pytest.mark.parametrize("vocab,vp", [(100, 128), (30522, 30528), (32768, 32768)])
def test_next_token_head_is_the_fill_mask_head(vocab, vp):
    import torch
    rows, k = 8, 5
    x, pos = _head_logits(rows, vocab, vp, vocab)
    ids, pr, lg = _next_head(x, pos, vocab, k)
    xd, pd = torch.from_numpy(x).cuda(), torch.from_numpy(pos).cuda()
    fi = torch.zeros((rows, k), dtype=torch.int32, device="cuda")
    fp, fl = torch.zeros((rows, k), device="cuda"), torch.zeros((rows, k), device="cuda")
    t._lib.check(lib.tfsc_k_fill_mask_head(_ptr(xd), vp, _ptr(pd), rows, 1, vocab, k, _ptr(fi), _ptr(fp), _ptr(fl), None), "fill_mask_head")
    torch.cuda.synchronize()
    assert ids.tobytes() == fi.cpu().numpy().tobytes() and pr.tobytes() == fp.cpu().numpy().tobytes()
    assert lg.tobytes() == fl.cpu().numpy().tobytes()


def test_next_token_head_rejections():
    import torch
    x = torch.zeros(57345, device="cuda")
    p = torch.zeros(1, dtype=torch.int32, device="cuda")
    y = torch.zeros(33, device="cuda")
    E = t._lib.E_INVALID
    assert lib.tfsc_k_next_token_head(_ptr(x), 57345, _ptr(p), 1, 57345, 1, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_next_token_head(_ptr(x), 100, _ptr(p), 1, 100, 33, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_next_token_head(_ptr(x), 99, _ptr(p), 1, 100, 5, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_next_token_head(_ptr(x), 100, None, 1, 100, 5, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_next_token_head(_ptr(x), 57344, _ptr(p), 1, 57344, 32, _ptr(y), None, None, None) == 0


# ------------------------------------------------------------------------------------------ served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 4 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 8 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _write_gpt2(tmp, seq, arch, seed, name="g", inputs=mf.GPT2_INPUTS, outputs=ALL, model=None):
    m = model or ge.hf_gpt2_model(seed, **arch)
    man = mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=outputs)
    mf.write_graph_bundle(os.path.join(str(tmp), name, "1"), man, ge.export_gpt2_model(m, man))
    return m


def _check_against_fp64(r, ref, pos, V):
    """positions exact, top-k logits within 1e-4 max(1, |ref|) of the fp64 logits at the returned ids, and the ids equal to
    the fp64 top k wherever the score gap exceeds the tolerance"""
    assert np.array_equal(r["next_token_position"], pos)
    rid, _rp, _rl = gr.top_k_ref(ref, pos, V, K)
    for i in range(len(pos)):
        ids = r["next_token_top_k_ids"][i]
        want = ref[i, ids]
        got = r["next_token_top_k_logits"][i].astype(np.float64)
        assert np.all(np.abs(got - want) <= 1e-4 * np.maximum(1.0, np.abs(want))), (i, np.abs(got - want).max())
        srt = np.sort(ref[i])[::-1][:K + 1]
        tol = 2e-4 * np.maximum(1.0, np.abs(srt))
        for j in range(K):
            if srt[j] - srt[j + 1] > tol[j] and (j == 0 or srt[j - 1] - srt[j] > tol[j]):
                assert ids[j] == rid[i, j], (i, j)
        p = r["next_token_top_k_probabilities"][i]
        assert (np.diff(p) <= 0).all() and 0 < p.sum() <= 1.0 + 1e-6


@pytest.mark.parametrize("S", [128, 1024])
def test_gpt2_small(S, tmp_path):
    import torch
    m = _write_gpt2(tmp_path, S, dict(max_pos=1024), 41)
    V = 50257
    x = ge.gpt2_inputs(8, S, V, seed=S)
    want_pos = np.array([max(np.nonzero(mk)[0]) for mk in x["attention_mask"]], np.int32)
    ref = ge.gpt2_reference(m, x["input_ids"], x["attention_mask"], device="cuda", at=want_pos)
    torch.cuda.empty_cache()
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (8, 3, 1):
            r = srv.predict("g", "1", {k: v[:bs] for k, v in x.items()}, outputs=NAMES)
            assert r["next_token_top_k_ids"].shape == (bs, K) and r["next_token_position"].shape == (bs,)
            _check_against_fp64(r, ref[:bs], want_pos[:bs], V)


def test_ids_only_bundle_attends_to_every_token(tmp_path):
    """without a mask input id 0 is a token like any other: position S - 1, every key visible"""
    S, B = 48, 5
    m = _write_gpt2(tmp_path, S, SMALL, 42, inputs=None)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], seed=1)["input_ids"]
    x[:, :4] = 0
    ref = ge.gpt2_reference(m, x, None, at=np.full(B, S - 1))
    with t.Server(_cfg(tmp_path)) as srv:
        r = srv.predict("g", "1", x, outputs=NAMES)
    _check_against_fp64(r, ref, np.full(B, S - 1, np.int32), SMALL["vocab"])


def test_empty_row(tmp_path):
    S = 16
    _write_gpt2(tmp_path, S, SMALL, 43)
    x = ge.gpt2_inputs(3, S, SMALL["vocab"], seed=2)
    x["attention_mask"][1] = 0
    with t.Server(_cfg(tmp_path)) as srv:
        r = srv.predict("g", "1", x, outputs=NAMES)
    assert r["next_token_position"][1] == -1 and (r["next_token_position"][[0, 2]] >= 0).all()
    assert (r["next_token_top_k_ids"][1] == -1).all() and (r["next_token_top_k_probabilities"][1] == 0).all()
    assert (r["next_token_top_k_logits"][1] == -FLT_MAX).all()


# ----------------------------------------------------------------------------------------- front-ends ----
def _session_run_request(name, feed, x, fetch):
    named = wire._ld(1, feed.encode()) + wire._ld(2, wire.encode_tensor(x))
    return wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())


def test_every_frontend_on_a_gpt2_bundle(tmp_path):
    import torch
    S, B = 32, 5
    _write_gpt2(tmp_path, S, SMALL, 73)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], seed=3)
    with t.Server(_cfg(tmp_path)) as srv:
        full = srv.predict("g", "1", x, outputs=NAMES)
        assert full["next_token_position"].shape == (B,) and full["next_token_position"].dtype == np.int32
        assert all(full[k].shape == (B, K) for k in NAMES if k != "next_token_position")
        assert full["next_token_top_k_ids"].dtype == np.int32 and full["next_token_top_k_probabilities"].dtype == np.float32
        sub = srv.predict("g", "1", x, outputs=["next_token_top_k_logits", "next_token_position"])
        assert list(sub) == ["next_token_top_k_logits", "next_token_position"]
        assert all(v.tobytes() == full[k].tobytes() for k, v in sub.items())
        one = srv.predict("g", "1", {k: v[0] for k, v in x.items()}, outputs=["next_token_position", "next_token_top_k_ids"])
        assert one["next_token_position"].shape == () and one["next_token_top_k_ids"].shape == (K,)
        assert one["next_token_position"] == full["next_token_position"][0]
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("g", "1", x, outputs=["nope"])
        assert "unknown output 'nope'" in str(e.value) and "'next_token_top_k_ids' (int32)" in str(e.value)
        tk = srv.predict_submit("g", "1", x, outputs=["next_token_top_k_ids", "next_token_position"])
        try:
            r = tk.wait(30.0)
        finally:
            tk.release()
        assert all(r[k].tobytes() == full[k].tobytes() for k in ("next_token_top_k_ids", "next_token_position"))
        # gRPC Predict: every output, or those output_filter names
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("g", 1, x)))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        assert outs["next_token_top_k_ids"].shape == (B, K) and outs["next_token_position"].shape == (B,)
        req = wire.encode_predict_request("g", 1, x, output_filter=["next_token_position"])
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(req))
        assert list(outs) == ["next_token_position"] and outs["next_token_position"].tobytes() == full["next_token_position"].tobytes()
        # REST, row and columnar
        st, b = srv.rest_handle("POST", "/v1/models/g/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        assert len(preds) == B and all(list(p) == NAMES for p in preds)
        for i, p in enumerate(preds):
            assert p["next_token_position"] == int(full["next_token_position"][i])
            assert np.array_equal(np.int32(p["next_token_top_k_ids"]), full["next_token_top_k_ids"][i])
            assert np.array_equal(np.float32(p["next_token_top_k_logits"]), full["next_token_top_k_logits"][i])
        st, b = srv.rest_handle("POST", "/v1/models/g/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES
        assert all(np.array_equal(np.asarray(cols[k], full[k].dtype), full[k]) for k in NAMES)
        # metadata
        st, b = srv.rest_handle("GET", "/v1/models/g/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {k: ("DT_FLOAT", ["-1", str(K)]) for k in NAMES}
        want["next_token_top_k_ids"] = ("DT_INT32", ["-1", str(K)])
        want["next_token_position"] = ("DT_INT32", ["-1"])
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        # SessionRun takes one feed, so it refuses a two-input bundle; Classify and Regress refuse it too
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(_session_run_request("g", "input_ids:0", x["input_ids"], "next_token_top_k_ids:0"))
        assert e.value.code == t._lib.E_INVALID and "'attention_mask'" in str(e.value)
        for verb in ("classify", "regress"):
            st, b = srv.rest_handle("POST", f"/v1/models/g/versions/1:{verb}", json.dumps({"examples": [{"x": 1.0}]}).encode())
            assert st == 400
        # tfsc_predict_device writes packed rows; split_packed_rows cuts them
        srv.ensure(0, "g", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(ALL, SMALL["vocab"]))
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.GPT2_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "g", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), ALL, SMALL["vocab"])
        for k in NAMES:
            assert dev[k].shape == full[k].shape and dev[k].tobytes() == full[k].tobytes(), k


@pytest.mark.parametrize("rows", [1, 8])
def test_launch_counts(tmp_path, rows):
    """one launch per op at these sizes: the embedding, seven per block, last_token, ln_f, the vocabulary projection (the
    weight-streaming dense kernel below 64 rows) and the head, besides the batch's input gather and output scatter"""
    S = 64
    arch = dict(SMALL)
    _write_gpt2(tmp_path, S, arch, 74)
    x = ge.gpt2_inputs(rows, S, arch["vocab"], seed=rows)
    with t.Server(_cfg(tmp_path)) as srv:
        srv.predict("g", "1", x, outputs=NAMES)
        s0 = srv.stats()
        srv.predict("g", "1", x, outputs=NAMES)
        s1 = srv.stats()
    assert s1["batches"] - s0["batches"] == 1
    assert s1["kernel_launches"] - s0["kernel_launches"] == 2 + 1 + 7 * arch["layers"] + 4


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_gpt2 as g
import gpt2_export as ge
tmp = sys.argv[2]
g._write_gpt2(tmp, 300, g.SMALL, 75)
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (1, 8):
        x = ge.gpt2_inputs(rows, 300, g.SMALL["vocab"], seed=rows)
        for k, v in srv.predict("g", "1", x, outputs=g.NAMES).items():
            out[f"{k}_r{rows}"] = v
np.savez(sys.argv[1], **out)
print("SAVED", len(out))
"""


def test_programmatic_dependent_launch_keeps_the_bits(tmp_path):
    res = {}
    for pdl in ("default", "0"):
        env = dict(os.environ, PYTHONPATH=ROOT)
        env.pop("TFSC_PDL", None)
        if pdl == "0":
            env["TFSC_PDL"] = "0"
        path, tmp = str(tmp_path / f"pdl_{pdl}.npz"), str(tmp_path / f"models_{pdl}")
        run = subprocess.run([sys.executable, "-c", PDL_SCRIPT, path, tmp], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
        assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]
        res[pdl] = dict(np.load(path))
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 2 * len(NAMES)
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key


# --------------------------------------------------------------------------------------- forward hop ----
N_MODELS = 4
HOP_S, HOP_ROWS = 64, 6


def _rank_cfg(rank, world, socks, base):
    members = [f"gpu{i}:0:0" for i in range(world)]
    return {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": base, "gpu.devices": [0],
            "gpu.arenaBytes": 256 << 20, "modelCache.size": 1 << 30, "serving.maxConcurrentModels": 16, "gpu.members": members,
            "gpu.localMembers": [members[rank]], "proxy.replicasPerModel": 1, "proxy.replicaPick": "first", "cluster.rank": rank,
            "cluster.endpoints": socks, "proxy.grpcTimeout": 60.0}


def _rank_main(rank, world, socks, base, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}}
        with t.Server(_rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = ge.gpt2_inputs(HOP_ROWS, HOP_S, SMALL["vocab"], seed=7)
            for j in range(N_MODELS):
                name = f"g{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=NAMES)
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, x)))
                res["grpc"][j] = dict(outs)
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict",
                                        json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
                res["rest"][j] = (st, b.decode())
            res["stats"] = srv.stats()
            barrier.wait(timeout=120)
        out.put(res)
    except BaseException as e:  # noqa: BLE001
        import traceback
        out.put({"rank": rank, "fatal": f"{e!r}\n{traceback.format_exc()}"})
        try:
            barrier.abort()
        except Exception:
            pass


def test_forward_hop_gpt2():
    import torch
    assert torch.cuda.is_available()
    world = 2
    base = tempfile.mkdtemp(prefix="tfscgpt2")
    for j in range(N_MODELS):
        _write_gpt2(base, HOP_S, SMALL, 80 + j, name=f"g{j}")
    socks = [os.path.join(base, f"r{r}.sock") for r in range(world)]
    ctx = mp.get_context("spawn")
    barrier, out = ctx.Barrier(world), ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, world, socks, base, barrier, out)) for r in range(world)]
    [p.start() for p in procs]
    results = {}
    deadline = time.time() + 600
    while len(results) < world and time.time() < deadline:
        try:
            r = out.get(timeout=5)
            results[r["rank"]] = r
        except Exception:
            if not any(p.is_alive() for p in procs):
                break
    [p.join(timeout=30) for p in procs]
    [p.kill() for p in procs if p.is_alive()]
    assert len(results) == world, f"ranks reported: {sorted(results)}"
    for r in results.values():
        assert "fatal" not in r, r.get("fatal")
    assert all(results[0]["owned"][j] != results[1]["owned"][j] for j in range(N_MODELS))
    for j in range(N_MODELS):
        owner = 0 if results[0]["owned"][j] else 1
        local, fwd = results[owner], results[1 - owner]
        assert sorted(local["y"][j]) == NAMES and local["y"][j]["next_token_top_k_ids"].shape == (HOP_ROWS, K)
        for k in NAMES:
            assert fwd["y"][j][k].shape == local["y"][j][k].shape and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
