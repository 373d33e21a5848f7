"""-m gpu: fill-mask (masked-language-model) outputs. The mask_gather and fill-mask head kernels against the fp64 reference
(the head bit for bit against the classification head), bert_small and BERT-base BertForMaskedLM bundles at S = 128 and
384 against transformers fp64, every front-end, launch counts, programmatic-dependent-launch bit identity and the forward
hop between two ranks."""
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
import embed_export as ee  # noqa: E402
import mlm_export as me  # noqa: E402
import mlm_ref as mr  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
K = 5
ALL = [{"name": "masked_positions", "kind": "masked_positions"}] + [{"name": k, "kind": k, "k": K} for k in mf.MLM_OUTPUT_KINDS[1:]]
NAMES = sorted(o["name"] for o in ALL)
SMALL = dict(hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=512)
MASK_SMALL, MASK_BASE = 4, 103
FLT_MAX = np.float32(np.finfo(np.float32).max)


def _ptr(x):
    return None if x is None else x.data_ptr()


# ------------------------------------------------------------------------------------------- gather ----
def _gather_rows(rows, S, H, M, seed, tok=7):
    """hidden [rows, S, H] and ids / mask [rows, S]. Rows cycle through: no [MASK]; more than M [MASK]s; [MASK] under
    mask 0; [MASK] at positions 0 and S - 1; a few random [MASK]s with a padded tail."""
    rng = np.random.default_rng(seed)
    h = rng.standard_normal((rows, S, H), dtype=np.float32)
    ids = rng.integers(tok + 1, 1000, (rows, S)).astype(np.int32)
    mask = np.ones((rows, S), np.int32)
    for r in range(rows):
        kind = r % 5
        if kind == 1:
            ids[r, rng.choice(S, min(S, M + 3), replace=False)] = tok
        elif kind == 2:
            p = rng.choice(S, min(S, M + 1), replace=False)
            ids[r, p] = tok
            mask[r, p[: (len(p) + 1) // 2]] = 0
        elif kind == 3:
            ids[r, 0] = ids[r, S - 1] = tok
        elif kind == 4:
            ids[r, rng.choice(S, max(1, min(S, M) // 2), replace=False)] = tok
            tail = int(rng.integers(0, S))
            mask[r, S - tail:] = 0
    return h, ids, mask


def _gather(h, ids, mask, S, H, M, tok=7, misalign=False):
    import torch
    rows = h.shape[0]
    off = 1 if misalign else 0
    hb = torch.empty(rows * S * H + off, device="cuda")
    hb[off:] = torch.from_numpy(h.reshape(-1)).cuda()
    di = torch.from_numpy(np.ascontiguousarray(ids)).cuda()
    dm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask)).cuda()
    pos = torch.full((rows, M), 12345, dtype=torch.int32, device="cuda")
    gb = torch.full((rows * M * H + off,), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_mask_gather(_ptr(hb[off:]), _ptr(di), _ptr(dm), S, rows, S, H, M, tok, _ptr(pos), _ptr(gb[off:]), None),
                 "mask_gather")
    torch.cuda.synchronize()
    return pos.cpu().numpy(), gb[off:].cpu().numpy().reshape(rows, M, H)


@pytest.mark.parametrize("H", [64, 768, 1024])
@pytest.mark.parametrize("S", [1, 17, 128, 512])
@pytest.mark.parametrize("rows", [1, 219])
def test_mask_gather_matches_reference(rows, S, H):
    if rows * S * H > 40_000_000:
        rows = 61                                      # the largest shapes keep the host arrays within memory
    for M in sorted({1, min(S, 20), S}):
        h, ids, mask = _gather_rows(rows, S, H, M, seed=rows * 31 + S * 7 + H + M)
        for m in (mask, None):
            pos, gat = _gather(h, ids, m, S, H, M)
            rp, rg = mr.mask_gather_ref(h, ids, m, 7, M)
            assert np.array_equal(pos, rp), (M, m is None)
            assert gat.tobytes() == rg.tobytes(), (M, m is None)
        if rows * S <= 128 * 219:
            pos2, gat2 = _gather(h, ids, mask, S, H, M, misalign=True)   # the scalar path: the same bits
            rp, rg = mr.mask_gather_ref(h, ids, mask, 7, M)
            assert np.array_equal(pos2, rp) and gat2.tobytes() == rg.tobytes()


def test_mask_gather_null_outputs_and_rejections():
    import torch
    rows, S, H, M = 3, 16, 64, 4
    h, ids, mask = _gather_rows(rows, S, H, M, seed=1)
    pos, gat = _gather(h, ids, mask, S, H, M)
    hd, di = torch.from_numpy(h).cuda(), torch.from_numpy(ids).cuda()
    p2 = torch.zeros(rows, M, dtype=torch.int32, device="cuda")
    assert lib.tfsc_k_mask_gather(None, _ptr(di), None, S, rows, S, H, M, 7, _ptr(p2), None, None) == 0  # positions alone
    torch.cuda.synchronize()
    assert np.array_equal(p2.cpu().numpy(), mr.mask_gather_ref(h, ids, None, 7, M)[0])
    E = t._lib.E_INVALID
    y = torch.zeros(rows, M, H, device="cuda")
    for S_, H_, M_ in ((0, 64, 1), (8193, 64, 1), (16, 0, 1), (16, 8193, 1), (16, 64, 0), (16, 64, 17)):
        assert lib.tfsc_k_mask_gather(_ptr(hd), _ptr(di), None, 16, rows, S_, H_, M_, 7, _ptr(p2), _ptr(y), None) == E, (S_, H_, M_)
    assert lib.tfsc_k_mask_gather(_ptr(hd), None, None, S, rows, S, H, M, 7, _ptr(p2), _ptr(y), None) == E
    assert lib.tfsc_k_mask_gather(_ptr(hd), _ptr(di), None, S - 1, rows, S, H, M, 7, _ptr(p2), _ptr(y), None) == E
    assert lib.tfsc_k_mask_gather(None, _ptr(di), None, S, rows, S, H, M, 7, _ptr(p2), _ptr(y), None) == E
    assert lib.tfsc_k_mask_gather(_ptr(hd), _ptr(di), None, S, -1, S, H, M, 7, _ptr(p2), _ptr(y), None) == E


# --------------------------------------------------------------------------------------------- head ----
def _head_logits(rows, M, vocab, vp, seed):
    """logits [rows * M, vp]: random rows with ties, a constant row, spreads of 1 and 80, and padding columns of 1e30
    that must never be selected"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows * M, vp)).astype(np.float32)
    for i in range(rows * M):
        kind = i % 4
        if kind == 1:
            x[i, :vocab] = np.round(x[i, :vocab] * 2) / 2          # many ties
        elif kind == 2:
            x[i, :vocab] = 0.25                                   # constant
        elif kind == 3:
            x[i, :vocab] *= 80
    x[:, vocab:] = 1e30
    return x


def _head(x, pos, rows, M, vocab, vp, k, want=(True, True, True)):
    import torch
    xd, pd = torch.from_numpy(x).cuda(), torch.from_numpy(np.ascontiguousarray(pos, np.int32)).cuda()
    outs = [torch.full((rows, M, k), 777, dtype=torch.int32, device="cuda") if want[0] else None,
            torch.full((rows, M, k), float("nan"), device="cuda") if want[1] else None,
            torch.full((rows, M, k), float("nan"), device="cuda") if want[2] else None]
    t._lib.check(lib.tfsc_k_fill_mask_head(_ptr(xd), vp, _ptr(pd), rows, M, vocab, k, *[_ptr(o) for o in outs], None), "fill_mask_head")
    torch.cuda.synchronize()
    return [None if o is None else o.cpu().numpy() for o in outs]


def _classify(x, vocab, k):
    import torch
    rows = x.shape[0]
    xd = torch.from_numpy(np.ascontiguousarray(x[:, :vocab])).cuda()
    idx = torch.empty(rows, k, dtype=torch.int32, device="cuda")
    pr = torch.empty(rows, k, device="cuda")
    t._lib.check(lib.tfsc_k_classify_head(_ptr(xd), rows, vocab, k, None, None, _ptr(idx), _ptr(pr), None), "classify_head")
    torch.cuda.synchronize()
    return idx.cpu().numpy(), pr.cpu().numpy()


@pytest.mark.parametrize("k", [1, 5, 32])
@pytest.mark.parametrize("vocab,vp", [(100, 128), (2048, 2048), (30522, 30528), (32768, 32768)])
@pytest.mark.parametrize("rows,M", [(1, 1), (8, 20), (13, 3)])
def test_fill_mask_head_matches_reference(rows, M, vocab, vp, k):
    x = _head_logits(rows, M, vocab, vp, seed=rows * 7 + M + vocab + k)
    rng = np.random.default_rng(vocab + k)
    pos = rng.integers(0, 50, (rows, M)).astype(np.int32)
    pos[rng.random((rows, M)) < 0.3] = -1
    ids, probs, lg = _head(x, pos, rows, M, vocab, vp, k)
    rid, rp, rl = mr.top_k_ref(x.reshape(rows, M, vp), pos, vocab, k)
    assert np.array_equal(ids, rid)
    live = pos >= 0
    assert np.all(np.abs(probs[live] - rp[live]) <= 1e-5 * rp[live] + 1e-37)
    assert np.array_equal(lg[live], rl[live].astype(np.float32))               # the logits at those ids, bit for bit
    assert (ids[~live] == -1).all() and (probs[~live] == 0).all() and (lg[~live] == -FLT_MAX).all()
    assert (ids[live] < vocab).all()                                          # the 1e30 padding columns are never selected
    # every filled slot: the classification head's ids and probabilities on its vocab logits, bit for bit
    ci, cp = _classify(x, vocab, k)
    ci, cp = ci.reshape(rows, M, k), cp.reshape(rows, M, k)
    assert np.array_equal(ids[live], ci[live]) and probs[live].tobytes() == cp[live].tobytes()


def test_fill_mask_head_null_outputs_and_rejections():
    import torch
    rows, M, vocab, vp = 4, 3, 1000, 1024
    x = _head_logits(rows, M, vocab, vp, seed=3)
    pos = np.array([[0, 5, -1]] * rows, np.int32)
    full = _head(x, pos, rows, M, vocab, vp, K)
    for bits in range(1, 8):
        want = tuple(bool(bits >> i & 1) for i in range(3))
        r = _head(x, pos, rows, M, vocab, vp, K, want)
        for a, b_, w in zip(r, full, want):
            assert (a is None) == (not w) and (a is None or a.tobytes() == b_.tobytes()), bits
    xd, pd = torch.from_numpy(x).cuda(), torch.from_numpy(pos).cuda()
    y = torch.zeros(rows, M, K, dtype=torch.int32, device="cuda")
    E = t._lib.E_INVALID
    for M_, V_, k_ in ((0, 1000, 5), (8193, 1000, 5), (3, 0, 1), (3, 32769, 5), (3, 1000, 0), (3, 1000, 33), (3, 4, 5)):
        assert lib.tfsc_k_fill_mask_head(_ptr(xd), vp, _ptr(pd), rows, M_, V_, k_, _ptr(y), None, None, None) == E, (M_, V_, k_)
    assert lib.tfsc_k_fill_mask_head(_ptr(xd), vp, None, rows, M, vocab, K, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_fill_mask_head(None, vp, _ptr(pd), rows, M, vocab, K, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_fill_mask_head(_ptr(xd), vocab - 1, _ptr(pd), rows, M, vocab, K, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_fill_mask_head(_ptr(xd), vp, _ptr(pd), -1, M, vocab, K, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_fill_mask_head(_ptr(xd), vp, _ptr(pd), 0, M, vocab, K, _ptr(y), None, None, None) == 0


# ------------------------------------------------------------------------------------ served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 6 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _write_mlm(tmp, seq, arch, seed, M, tok, name="ms", enc=None, model=None):
    """a fill-mask bundle `name` (every output, BERT_INPUTS) and, with enc, the encoder bundle of the same weights without a
    pooler answering sequence_output"""
    m = model or me.hf_mlm_model(seed, **arch)
    man = mf.bert_manifest(seq=seq, **arch, inputs=mf.BERT_INPUTS, outputs=ALL, head="mlm", slots=M, mask_token_id=tok)
    mf.write_graph_bundle(os.path.join(str(tmp), name, "1"), man, me.export_mlm_model(m, man))
    if enc:
        em = mf.bert_manifest(seq=seq, **arch, inputs=mf.BERT_INPUTS, outputs=[{"name": "sequence_output", "kind": "sequence_output"}],
                              head="encoder", pooler=False)
        mf.write_graph_bundle(os.path.join(str(tmp), enc, "1"), em, ee.export_bert_model(m.bert, em))
    return m


@pytest.mark.parametrize("M", [1, 20])
@pytest.mark.parametrize("S", [128, 384])
@pytest.mark.parametrize("kind", ["bert_small", "bert_base"])
def test_bert_fill_mask(kind, S, M, tmp_path):
    B = 8
    arch = dict(SMALL) if kind == "bert_small" else dict(max_pos=512)
    V = arch.get("vocab", 30522)
    tok = MASK_SMALL if kind == "bert_small" else MASK_BASE
    m = _write_mlm(tmp_path, S, arch, 41 + M + (kind == "bert_base"), M, tok)
    x = mr.mlm_inputs(B, S, V, M + 2, seed=S + M, mask_token_id=tok)
    ref = me.mlm_reference(m, x["input_ids"], x["input_mask"], x["segment_ids"])
    want_pos, _ = mr.mask_gather_ref(np.zeros((B, S, 1)), x["input_ids"], x["input_mask"], tok, M)
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (B, 3):
            xb = {k: v[:bs] for k, v in x.items()}
            r = srv.predict("ms", "1", xb, outputs=NAMES)
            pos = r["masked_positions"]
            assert pos.shape == (bs, M) and r["masked_top_k_ids"].shape == (bs, M, K)
            assert np.array_equal(pos, want_pos[:bs])
            live = pos >= 0
            assert live.any() and (live.all() or M > 1)
            refl = np.stack([ref[i, np.maximum(pos[i], 0)] for i in range(bs)])    # [bs, M, V] fp64 at the slots
            rid, _rp, _rl = mr.top_k_ref(refl, pos, V, K)
            got_l = r["masked_top_k_logits"].astype(np.float64)
            ids = r["masked_top_k_ids"]
            for i in range(bs):
                for s in range(M):
                    if not live[i, s]:
                        assert (ids[i, s] == -1).all() and (r["masked_top_k_probabilities"][i, s] == 0).all()
                        assert (r["masked_top_k_logits"][i, s] == -FLT_MAX).all()
                        continue
                    want = refl[i, s, ids[i, s]]
                    assert np.all(np.abs(got_l[i, s] - want) <= 1e-4 * np.maximum(1.0, np.abs(want))), (i, s)
                    # ids equal the fp64 top k wherever adjacent fp64 logits differ by more than the tolerance
                    srt = np.sort(refl[i, s])[::-1][:K + 1]
                    tol = 2e-4 * np.maximum(1.0, np.abs(srt))
                    for j in range(K):
                        if srt[j] - srt[j + 1] > tol[j] and (j == 0 or srt[j - 1] - srt[j] > tol[j]):
                            assert ids[i, s, j] == rid[i, s, j], (i, s, j)


# --------------------------------------------------------------------------------------- front-ends ----
def _session_run_request(name, feed, x, fetch):
    named = wire._ld(1, feed.encode()) + wire._ld(2, wire.encode_tensor(x))
    return wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())


def test_every_frontend_on_a_fill_mask_bundle(tmp_path):
    import torch
    S, B, M = 32, 5, 4
    _write_mlm(tmp_path, S, SMALL, 73, M, MASK_SMALL)
    x = mr.mlm_inputs(B, S, SMALL["vocab"], 3, seed=3, mask_token_id=MASK_SMALL)
    with t.Server(_cfg(tmp_path)) as srv:
        full = srv.predict("ms", "1", x, outputs=NAMES)
        assert full["masked_positions"].shape == (B, M) and full["masked_positions"].dtype == np.int32
        assert all(full[k].shape == (B, M, K) for k in NAMES if k != "masked_positions")
        assert full["masked_top_k_ids"].dtype == np.int32 and full["masked_top_k_probabilities"].dtype == np.float32
        sub = srv.predict("ms", "1", x, outputs=["masked_top_k_logits", "masked_positions"])
        assert list(sub) == ["masked_top_k_logits", "masked_positions"] and all(v.tobytes() == full[k].tobytes() for k, v in sub.items())
        one = srv.predict("ms", "1", {k: v[0] for k, v in x.items()}, outputs=["masked_positions", "masked_top_k_ids"])
        assert one["masked_positions"].shape == (M,) and one["masked_top_k_ids"].shape == (M, K)
        assert np.array_equal(one["masked_positions"], full["masked_positions"][0])
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("ms", "1", x, outputs=["nope"])
        assert "unknown output 'nope'" in str(e.value) and "'masked_top_k_ids' (int32)" in str(e.value)
        for r in (srv.predict_deadline("ms", "1", x, srv.now_ns() + 30_000_000_000, outputs=NAMES),
                  srv.predict_member(0, "ms", "1", x, outputs=NAMES)):
            assert all(r[k].tobytes() == full[k].tobytes() for k in NAMES)
        tk = srv.predict_submit("ms", "1", x, outputs=["masked_top_k_ids", "masked_positions"])
        try:
            r = tk.wait(30.0)
        finally:
            tk.release()
        assert all(r[k].tobytes() == full[k].tobytes() for k in ("masked_top_k_ids", "masked_positions"))
        # gRPC Predict: every output, or those output_filter names; the top-k outputs are [B, M, k]
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("ms", 1, x)))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        assert outs["masked_top_k_ids"].shape == (B, M, K) and outs["masked_positions"].shape == (B, M)
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("ms", 1, x, output_filter=["masked_top_k_ids"])))
        assert list(outs) == ["masked_top_k_ids"] and outs["masked_top_k_ids"].tobytes() == full["masked_top_k_ids"].tobytes()
        # REST, row and columnar: int32 and float rank-2 rows as nested lists; -FLT_MAX stays a finite JSON number
        st, b = srv.rest_handle("POST", "/v1/models/ms/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        assert len(preds) == B and all(list(p) == NAMES for p in preds)
        for i, p in enumerate(preds):
            assert np.array_equal(np.int32(p["masked_top_k_ids"]), full["masked_top_k_ids"][i])
            assert np.array_equal(np.int32(p["masked_positions"]), full["masked_positions"][i])
            assert np.array_equal(np.float32(p["masked_top_k_logits"]), full["masked_top_k_logits"][i])
        st, b = srv.rest_handle("POST", "/v1/models/ms/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES
        assert all(np.array_equal(np.asarray(cols[k], full[k].dtype), full[k]) for k in NAMES)
        # metadata
        st, b = srv.rest_handle("GET", "/v1/models/ms/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {k: ("DT_FLOAT", ["-1", str(M), str(K)]) for k in NAMES}
        want["masked_top_k_ids"] = ("DT_INT32", ["-1", str(M), str(K)])
        want["masked_positions"] = ("DT_INT32", ["-1", str(M)])
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        # SessionRun takes one feed, so it refuses a three-input bundle; Classify refuses it too
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(_session_run_request("ms", "input_ids:0", x["input_ids"], "masked_top_k_ids:0"))
        assert e.value.code == t._lib.E_INVALID and "'input_mask'" in str(e.value)
        st, b = srv.rest_handle("POST", "/v1/models/ms/versions/1:classify", json.dumps({"examples": [{"x": 1.0}]}).encode())
        assert st == 400
        st, b = srv.rest_handle("POST", "/v1/models/ms/versions/1:regress", json.dumps({"examples": [{"x": 1.0}]}).encode())
        assert st == 400
        # tfsc_predict_device writes packed rows; split_packed_rows cuts them, the top-k kinds as [B, M, k]
        srv.ensure(0, "ms", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(ALL, M))
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.BERT_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "ms", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), ALL, M)
        for k in NAMES:
            assert dev[k].shape == full[k].shape and dev[k].tobytes() == full[k].tobytes(), k


def test_served_positions_are_the_raw_gather(tmp_path):
    """The served positions are those of the raw gather on the hidden states of the encoder bundle of the same weights"""
    S, B, M = 64, 6, 5
    _write_mlm(tmp_path, S, SMALL, 77, M, MASK_SMALL, enc="enc")
    x = mr.mlm_inputs(B, S, SMALL["vocab"], 4, seed=9, mask_token_id=MASK_SMALL)
    with t.Server(_cfg(tmp_path)) as srv:
        r = srv.predict("ms", "1", x, outputs=NAMES)
        h = srv.predict("enc", "1", x, outputs=["sequence_output"])["sequence_output"]
    pos, gat = _gather(h, x["input_ids"], x["input_mask"], S, SMALL["hidden"], M, tok=MASK_SMALL)
    assert np.array_equal(pos, r["masked_positions"]) and (pos >= 0).any() and (pos < 0).any()
    assert np.isfinite(r["masked_top_k_logits"]).all() and (r["masked_top_k_ids"][pos < 0] == -1).all()


@pytest.mark.parametrize("B", [3, 30])
def test_unpadded_decoder(tmp_path, B):
    """A decoder that writes exactly `vocab` columns (not padded to a multiple of 32) stays on the GEMM path and answers
    what the padded bundle of the same weights answers: the same positions and ids, logits within the GEMMs' rounding"""
    S, M = 32, 2
    m = me.hf_mlm_model(78, **SMALL)
    for name, pad in (("pad", True), ("raw", False)):
        man = mf.bert_manifest(seq=S, **SMALL, inputs=mf.BERT_INPUTS, outputs=ALL, head="mlm", slots=M, mask_token_id=MASK_SMALL)
        if not pad:
            man["ops"][-1]["cout"] = SMALL["vocab"]                # 100 columns; the weights keep their offsets
        mf.write_graph_bundle(os.path.join(str(tmp_path), name, "1"), man, me.export_mlm_model(m, man))
    x = mr.mlm_inputs(B, S, SMALL["vocab"], 2, seed=4, mask_token_id=MASK_SMALL)
    with t.Server(_cfg(tmp_path, **{"gpu.maxBatch": 32})) as srv:
        a = srv.predict("pad", "1", x, outputs=NAMES)
        b = srv.predict("raw", "1", x, outputs=NAMES)
    assert np.array_equal(a["masked_positions"], b["masked_positions"]) and (a["masked_positions"] >= 0).any()
    live = a["masked_positions"] >= 0
    assert np.allclose(a["masked_top_k_logits"][live], b["masked_top_k_logits"][live], rtol=1e-5, atol=1e-5)
    assert np.allclose(a["masked_top_k_probabilities"][live], b["masked_top_k_probabilities"][live], rtol=1e-4, atol=1e-7)
    srt = np.sort(a["masked_top_k_logits"][live], axis=-1)
    if (np.diff(srt, axis=-1) > 1e-4).all():
        assert np.array_equal(a["masked_top_k_ids"], b["masked_top_k_ids"])


def test_positions_only_bundle(tmp_path):
    S, B, M = 32, 4, 3
    m = me.hf_mlm_model(79, **SMALL)
    man = mf.bert_manifest(seq=S, **SMALL, inputs=mf.BERT_INPUTS, outputs=[{"name": "where", "kind": "masked_positions"}],
                           head="mlm", slots=M, mask_token_id=MASK_SMALL)
    mf.write_graph_bundle(os.path.join(str(tmp_path), "mp", "1"), man, me.export_mlm_model(m, man))
    x = mr.mlm_inputs(B, S, SMALL["vocab"], 4, seed=2, mask_token_id=MASK_SMALL)
    with t.Server(_cfg(tmp_path)) as srv:
        r = srv.predict("mp", "1", x, outputs=["where"])
    want, _ = mr.mask_gather_ref(np.zeros((B, S, 1)), x["input_ids"], x["input_mask"], MASK_SMALL, M)
    assert np.array_equal(r["where"], want)


@pytest.mark.parametrize("rows", [1, 8, 13])
def test_launch_counts(tmp_path, rows):
    """A fill-mask bundle launches the encoder's kernels, then the gather, the transform dense, its LayerNorm and the
    vocabulary projection (one launch each at these sizes), then the head: four more than the encoder bundle of the same
    weights, whose sequence_output head is one launch"""
    S, M = 64, 3
    _write_mlm(tmp_path, S, SMALL, 74, M, MASK_SMALL, enc="enc")
    x = mr.mlm_inputs(rows, S, SMALL["vocab"], 2, seed=rows, mask_token_id=MASK_SMALL)
    with t.Server(_cfg(tmp_path, **{"gpu.maxBatch": 16})) as srv:
        srv.predict("enc", "1", x, outputs=["sequence_output"])
        srv.predict("ms", "1", x, outputs=NAMES)
        counts = {}
        for name, outs in (("enc", ["sequence_output"]), ("ms", NAMES)):
            s0 = srv.stats()
            srv.predict(name, "1", x, outputs=outs)
            s1 = srv.stats()
            counts[name] = (s1["kernel_launches"] - s0["kernel_launches"], s1["batches"] - s0["batches"])
        assert counts["enc"][1] == counts["ms"][1] == 1
        assert counts["ms"][0] == counts["enc"][0] + 4, (rows, counts)


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_mlm as g
import mlm_ref as mr
tmp = sys.argv[2]
g._write_mlm(tmp, 128, g.SMALL, 75, 20, g.MASK_SMALL)
g._write_mlm(tmp, 128, g.SMALL, 76, 1, g.MASK_SMALL, name="m1")
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (1, 8):
        for name in ("ms", "m1"):
            x = mr.mlm_inputs(rows, 128, g.SMALL["vocab"], 21, seed=rows, mask_token_id=g.MASK_SMALL)
            for k, v in srv.predict(name, "1", x, outputs=g.NAMES).items():
                out[f"{name}_{k}_r{rows}"] = v
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
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 2 * 2 * len(NAMES)
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key


# --------------------------------------------------------------------------------------- forward hop ----
N_MODELS = 4
HOP_S, HOP_ROWS, HOP_M = 128, 6, 8


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
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}, "ticket": {}}
        with t.Server(_rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = mr.mlm_inputs(HOP_ROWS, HOP_S, SMALL["vocab"], HOP_M + 1, seed=7, mask_token_id=MASK_SMALL)
            for j in range(N_MODELS):
                name = f"ms{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=NAMES)
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, x)))
                res["grpc"][j] = dict(outs)
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict",
                                        json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
                res["rest"][j] = (st, b.decode())
                tk = srv.predict_submit(name, "1", x, outputs=["masked_top_k_ids", "masked_positions"])
                try:
                    res["ticket"][j] = tk.wait(60.0)
                finally:
                    tk.release()
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


def test_forward_hop_fill_mask():
    import torch
    assert torch.cuda.is_available()
    world = 2
    base = tempfile.mkdtemp(prefix="tfscmlm")
    for j in range(N_MODELS):
        _write_mlm(base, HOP_S, SMALL, 80 + j, HOP_M, MASK_SMALL, name=f"ms{j}")
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
    assert any(results[0]["owned"]) and any(results[1]["owned"])
    for j in range(N_MODELS):
        owner = 0 if results[0]["owned"][j] else 1
        local, fwd = results[owner], results[1 - owner]
        assert sorted(local["y"][j]) == NAMES and local["y"][j]["masked_top_k_ids"].shape == (HOP_ROWS, HOP_M, K)
        for k in NAMES:
            assert fwd["y"][j][k].shape == local["y"][j][k].shape and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].shape == local["grpc"][j][k].shape
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
        for k in ("masked_top_k_ids", "masked_positions"):
            assert fwd["ticket"][j][k].tobytes() == local["ticket"][j][k].tobytes()
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
