"""-m gpu: question-answering span outputs. The span-head kernel against the brute-force reference, bert_small and
BERT-base BertForQuestionAnswering bundles at S = 384 next to the same weights served single-output, every front-end,
launch counts, programmatic-dependent-launch bit identity and the forward hop between two ranks."""
import copy
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
import span_ref as sr  # noqa: E402
import qa_export as qe  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
K, L, SEP = 20, 30, 3
SPANS = [{"name": n, "kind": n, "k": K, "max_answer_length": L, "sep_id": SEP} for n in ("span_starts", "span_ends", "span_scores")]
FULL = [{"name": "start_logits", "kind": "start_logits"}, {"name": "end_logits", "kind": "end_logits"}] + SPANS
NAMES = sorted(o["name"] for o in FULL)
SMALL = dict(hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=512)


def _ptr(x):
    return x.data_ptr()


# ------------------------------------------------------------------------------------------- kernel ----
def _rows(rows, S, seed):
    """logits [rows, S, 2] and ids / mask / types [rows, S]. Rows cycle through: normal logits, quantised logits (ties
    everywhere), a fully masked row, a row without a segment-1 token, and logits of spread 80."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, S, 2)).astype(np.float32)
    ids = rng.integers(1, 50, (rows, S)).astype(np.int32)
    mask = (rng.uniform(size=(rows, S)) < 0.9).astype(np.int32)
    types = np.zeros((rows, S), np.int32)
    for r in range(rows):
        cut = int(rng.integers(0, max(1, S // 2)))
        types[r, cut:] = 1
        ids[r, rng.integers(0, S, 2)] = SEP
        kind = r % 5
        if kind == 1:
            x[r] = np.round(rng.uniform(0, 3, (S, 2))) * 1.5
        elif kind == 2:
            mask[r] = 0
        elif kind == 3:
            types[r] = 0
        elif kind == 4:
            x[r] = rng.uniform(-40, 40, (S, 2))
    return x, ids, mask, types


def _launch(x, ids, mask, types, S, Lm, k, sep, with_logits=True):
    import torch
    rows = x.shape[0]
    dev = {n: torch.from_numpy(np.ascontiguousarray(a)).cuda() for n, a in (("x", x), ("ids", ids), ("mask", mask), ("types", types))
           if a is not None}
    st = torch.full((rows, S), float("nan"), device="cuda")
    en = torch.full((rows, S), float("nan"), device="cuda")
    s = torch.full((rows, k), -7, dtype=torch.int32, device="cuda")
    e = torch.full((rows, k), -7, dtype=torch.int32, device="cuda")
    v = torch.full((rows, k), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_span_head(_ptr(dev["x"]), _ptr(dev["ids"]), None if mask is None else _ptr(dev["mask"]),
                                      _ptr(dev["types"]), S, rows, S, Lm, k, sep, _ptr(st) if with_logits else None,
                                      _ptr(en) if with_logits else None, _ptr(s), _ptr(e), _ptr(v), None), "span_head")
    torch.cuda.synchronize()
    return st.cpu().numpy(), en.cpu().numpy(), s.cpu().numpy(), e.cpu().numpy(), v.cpu().numpy()


@pytest.mark.parametrize("k", [1, 5, 20, 32])
@pytest.mark.parametrize("Lsel", ["1", "30", "S"])
@pytest.mark.parametrize("S", [1, 7, 128, 384, 512])
@pytest.mark.parametrize("rows", [1, 37, 219])
def test_span_kernel_matches_reference(rows, S, Lsel, k):
    Lm = {"1": 1, "30": min(30, S), "S": S}[Lsel]
    x, ids, mask, types = _rows(rows, S, seed=rows * 7919 + S * 31 + Lm * 7 + k)
    use_mask = (S + k) % 2 == 0                       # half the cases derive the mask from the ids ([PAD] = 0)
    sep = SEP if k != 1 else -1
    m = mask if use_mask else None
    st, en, s, e, v = _launch(x, ids, m, types, S, Lm, k, sep)
    assert st.tobytes() == np.ascontiguousarray(x[..., 0]).tobytes() and en.tobytes() == np.ascontiguousarray(x[..., 1]).tobytes()
    el = sr.eligible(ids, m, types, None if sep < 0 else sep)
    rs, re_, rv = sr.span_ref(x[..., 0], x[..., 1], el, Lm, k)
    assert np.array_equal(s, rs) and np.array_equal(e, re_)
    assert v.view(np.int32).tolist() == rv.view(np.int32).tolist()
    # no passage, or a fully masked row (with a mask input): no candidate
    empty = [r for r in range(rows) if r % 5 == 3 or (use_mask and r % 5 == 2)]
    assert all((s[r] == -1).all() and (v[r] == -sr.FLT_MAX).all() for r in empty)
    # a second launch, into fresh NaN-filled buffers, gives the same bits
    again = _launch(x, ids, m, types, S, Lm, k, sep)
    assert all(a.tobytes() == b.tobytes() for a, b in zip((st, en, s, e, v), again))


def test_span_kernel_nan_logits_and_null_outputs():
    import torch
    rows, S, k = 6, 64, 8
    x, ids, mask, types = _rows(rows, S, seed=9)
    x[0, ::3, 0] = np.nan
    x[1] = np.nan
    x[2, 5, 1] = np.inf
    _st, _en, s, e, v = _launch(x, ids, mask, types, S, 16, k, SEP)
    rs, re_, rv = sr.span_ref(x[..., 0], x[..., 1], sr.eligible(ids, mask, types, SEP), 16, k)
    assert np.array_equal(s, rs) and np.array_equal(e, re_) and v.view(np.int32).tolist() == rv.view(np.int32).tolist()
    assert (s[1] == -1).all() and ((s >= -1) & (s < S)).all() and ((e >= -1) & (e < S)).all()
    # spans without logits, and logits without spans (no rounds: ids and types are not needed)
    _st, _en, s2, _e2, _v2 = _launch(x, ids, mask, types, S, 16, k, SEP, with_logits=False)
    assert np.array_equal(s2, s)
    xd = torch.from_numpy(x).cuda()
    st = torch.full((rows, S), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_span_head(_ptr(xd), None, None, None, 0, rows, S, 0, 0, -1, _ptr(st), None, None, None, None, None),
                 "span_head")
    torch.cuda.synchronize()
    assert st.cpu().numpy().tobytes() == np.ascontiguousarray(x[..., 0]).tobytes()


def test_span_kernel_rejections():
    import torch
    x = torch.zeros(4, 64, 2, device="cuda")
    ids = torch.ones(4, 64, dtype=torch.int32, device="cuda")
    y = torch.zeros(4, 64, dtype=torch.int32, device="cuda")
    for S, Lm, k in ((0, 1, 1), (4097, 1, 1), (64, 0, 5), (64, 65, 5), (64, 5, 0), (64, 5, 33)):
        assert lib.tfsc_k_span_head(_ptr(x), _ptr(ids), None, _ptr(ids), 64, 4, S, Lm, k, -1, None, None, _ptr(y), None, None,
                                    None) == t._lib.E_INVALID, (S, Lm, k)
    assert lib.tfsc_k_span_head(_ptr(x), None, None, _ptr(ids), 64, 4, 64, 5, 5, -1, None, None, _ptr(y), None, None, None) == t._lib.E_INVALID
    assert lib.tfsc_k_span_head(_ptr(x), _ptr(ids), None, None, 64, 4, 64, 5, 5, -1, None, None, _ptr(y), None, None, None) == t._lib.E_INVALID
    assert lib.tfsc_k_span_head(_ptr(x), _ptr(ids), None, _ptr(ids), 63, 4, 64, 5, 5, -1, None, None, _ptr(y), None, None, None) == t._lib.E_INVALID
    assert lib.tfsc_k_span_head(None, _ptr(ids), None, _ptr(ids), 64, 4, 64, 5, 5, -1, None, None, _ptr(y), None, None, None) == t._lib.E_INVALID
    assert lib.tfsc_k_span_head(_ptr(x), _ptr(ids), None, _ptr(ids), 64, 0, 64, 5, 5, -1, None, None, _ptr(y), None, None, None) == 0


# ------------------------------------------------------------------------------------ served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 6 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _write_qa(tmp, seq, arch, seed, outputs=FULL, single="q1", multi="qs"):
    m = qe.hf_bert_qa(seed, **arch)
    one = mf.bert_manifest(seq=seq, **arch, inputs=mf.BERT_INPUTS, head="span")
    blob = qe.export_bert_qa(m, one)
    mf.write_graph_bundle(os.path.join(str(tmp), single, "1"), one, blob)
    mf.write_graph_bundle(os.path.join(str(tmp), multi, "1"), mf.bert_manifest(seq=seq, **arch, inputs=mf.BERT_INPUTS,
                                                                                 outputs=outputs, head="span"), blob)
    return m


def _check_spans(r, x, k=K):
    """the spans are span_ref of the served logits, bit for bit"""
    el = sr.eligible(x["input_ids"], x["input_mask"], x["segment_ids"], SEP)
    rs, re_, rv = sr.span_ref(r["start_logits"], r["end_logits"], el, L, k)
    assert r["span_starts"].dtype == np.int32 and np.array_equal(r["span_starts"], rs)
    assert np.array_equal(r["span_ends"], re_) and r["span_scores"].view(np.int32).tolist() == rv.view(np.int32).tolist()


@pytest.mark.parametrize("kind", ["bert_small", "bert_base"])
def test_bert_qa_spans_at_384(kind, tmp_path):
    import torch
    S, B = 384, 8
    arch = dict(SMALL) if kind == "bert_small" else dict(max_pos=512)
    m = _write_qa(tmp_path, S, arch, 31 if kind == "bert_small" else 32)
    x = sr.qa_inputs(B, S, arch.get("vocab", 30522), seed=13, sep_id=SEP)
    m64 = copy.deepcopy(m).double().cuda()
    tt = {k: torch.from_numpy(np.ascontiguousarray(v, np.int64)).cuda() for k, v in x.items()}
    with torch.no_grad():
        o = m64(input_ids=tt["input_ids"], attention_mask=tt["input_mask"], token_type_ids=tt["segment_ids"])
    ref = {"start_logits": o.start_logits.cpu().numpy(), "end_logits": o.end_logits.cpu().numpy()}
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (B, 3):
            xb = {k: v[:bs] for k, v in x.items()}
            y1 = srv.predict("q1", "1", xb)
            assert y1.shape == (bs, S, 1, 2)
            r = srv.predict("qs", "1", xb, outputs=NAMES)
            assert r["start_logits"].shape == (bs, S) and r["span_scores"].shape == (bs, K)
            # the logits are the single-output bundle's, de-interleaved
            assert r["start_logits"].tobytes() == np.ascontiguousarray(y1[:, :, 0, 0]).tobytes()
            assert r["end_logits"].tobytes() == np.ascontiguousarray(y1[:, :, 0, 1]).tobytes()
            for name in ("start_logits", "end_logits"):
                rf = ref[name][:bs]
                err = np.max(np.abs(r[name] - rf) / np.maximum(1.0, np.abs(rf)))
                assert err <= 1e-4, (name, err)
            _check_spans(r, xb)
            # spans of the fp64 logits: the same wherever the score gap to the next candidate exceeds the tolerance
            el = sr.eligible(xb["input_ids"], xb["input_mask"], xb["segment_ids"], SEP)
            s64, e64, v64 = sr.span_ref(ref["start_logits"][:bs], ref["end_logits"][:bs], el, L, K + 1, dtype=np.float64)
            checked = 0
            for b in range(bs):
                for j in range(K):
                    tol = 4e-4 * max(1.0, abs(v64[b, j]))
                    if s64[b, j + 1] >= 0 and v64[b, j] - v64[b, j + 1] <= tol:
                        break
                    assert (r["span_starts"][b, j], r["span_ends"][b, j]) == (s64[b, j], e64[b, j]), (b, j)
                    checked += 1
            assert checked >= bs, checked


# --------------------------------------------------------------------------------------- front-ends ----
def _session_run_request(name, feed, x, fetch):
    named = wire._ld(1, feed.encode()) + wire._ld(2, wire.encode_tensor(x))
    return wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())


def test_every_frontend_on_a_span_bundle(tmp_path):
    import torch
    S, B = 64, 5
    _write_qa(tmp_path, S, SMALL, 33)
    x = sr.qa_inputs(B, S, SMALL["vocab"], seed=3, sep_id=SEP)
    with t.Server(_cfg(tmp_path)) as srv:
        full = srv.predict("qs", "1", x, outputs=NAMES)
        _check_spans(full, x)
        sub = srv.predict("qs", "1", x, outputs=["span_scores", "start_logits"])
        assert list(sub) == ["span_scores", "start_logits"] and all(v.tobytes() == full[k].tobytes() for k, v in sub.items())
        one = srv.predict("qs", "1", {k: v[0] for k, v in x.items()}, outputs=["span_starts", "end_logits"])
        assert one["span_starts"].shape == (K,) and one["end_logits"].shape == (S,)
        assert one["span_starts"].tobytes() == full["span_starts"][0].tobytes()
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("qs", "1", x, outputs=["nope"])
        assert "unknown output 'nope'" in str(e.value) and "'span_ends' (int32)" in str(e.value)
        for r in (srv.predict_deadline("qs", "1", x, srv.now_ns() + 30_000_000_000, outputs=NAMES),
                  srv.predict_member(0, "qs", "1", x, outputs=NAMES)):
            assert all(r[k].tobytes() == full[k].tobytes() for k in NAMES)
        tk = srv.predict_submit("qs", "1", x, outputs=["span_ends", "span_scores"])
        try:
            r = tk.wait(30.0)
        finally:
            tk.release()
        assert r["span_ends"].tobytes() == full["span_ends"].tobytes() and r["span_scores"].tobytes() == full["span_scores"].tobytes()
        # gRPC Predict: every output, or those output_filter names
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("qs", 1, x)))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("qs", 1, x, output_filter=["span_starts"])))
        assert list(outs) == ["span_starts"] and outs["span_starts"].tobytes() == full["span_starts"].tobytes()
        # REST, row and columnar: valid JSON, empty slots included
        st, b = srv.rest_handle("POST", "/v1/models/qs/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        assert len(preds) == B and all(list(p) == NAMES for p in preds)
        for i, p in enumerate(preds):
            assert p["span_starts"] == full["span_starts"][i].tolist() and p["span_ends"] == full["span_ends"][i].tolist()
            assert np.array_equal(np.float32(p["span_scores"]), full["span_scores"][i])
            assert np.array_equal(np.float32(p["start_logits"]), full["start_logits"][i])
        st, b = srv.rest_handle("POST", "/v1/models/qs/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES and cols["span_ends"] == full["span_ends"].tolist()
        assert np.array_equal(np.float32(cols["end_logits"]), full["end_logits"])
        # metadata
        st, b = srv.rest_handle("GET", "/v1/models/qs/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {"end_logits": ("DT_FLOAT", ["-1", str(S)]), "start_logits": ("DT_FLOAT", ["-1", str(S)]),
                "span_starts": ("DT_INT32", ["-1", str(K)]), "span_ends": ("DT_INT32", ["-1", str(K)]),
                "span_scores": ("DT_FLOAT", ["-1", str(K)])}
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        # SessionRun takes one feed, so it refuses a three-input bundle and names its inputs; Classify refuses it too
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(_session_run_request("qs", "input_ids:0", x["input_ids"], "span_starts:0"))
        assert e.value.code == t._lib.E_INVALID and "'input_mask'" in str(e.value) and "'segment_ids'" in str(e.value)
        st, b = srv.rest_handle("POST", "/v1/models/qs/versions/1:classify", json.dumps({"examples": [{"x": 1.0}]}).encode())
        assert st == 400
        # tfsc_predict_device writes packed rows; packed_output_layout splits them
        srv.ensure(0, "qs", 1)
        layout = mf.packed_output_layout(FULL, S)
        width = sum(w for _n, _o, w, _d in layout)
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.BERT_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "qs", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), FULL, S)
        for k in NAMES:
            assert dev[k].tobytes() == full[k].tobytes(), k


def test_launch_counts(tmp_path):
    """A span bundle launches exactly one kernel more per batch than the same weights with one output"""
    S = 64
    _write_qa(tmp_path, S, SMALL, 34)
    for rows in (1, 8):
        x = sr.qa_inputs(rows, S, SMALL["vocab"], seed=rows, sep_id=SEP)
        with t.Server(_cfg(tmp_path)) as srv:
            srv.predict("q1", "1", x)
            srv.predict("qs", "1", x, outputs=["span_starts"])
            counts = {}
            for name in ("q1", "qs"):
                s0 = srv.stats()
                srv.predict(name, "1", x, outputs=None if name == "q1" else ["span_starts"])
                s1 = srv.stats()
                counts[name] = (s1["kernel_launches"] - s0["kernel_launches"], s1["batches"] - s0["batches"])
            assert counts["q1"][1] == counts["qs"][1] >= 1
            assert counts["qs"][0] == counts["q1"][0] + counts["qs"][1], (rows, counts)


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_spans as g
import span_ref as sr
tmp = sys.argv[2]
g._write_qa(tmp, 384, g.SMALL, 35)
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (1, 8):
        x = sr.qa_inputs(rows, 384, g.SMALL["vocab"], seed=rows, sep_id=g.SEP)
        for k, v in srv.predict("qs", "1", x, outputs=g.NAMES).items():
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


def _rank_cfg(rank, world, socks, base):
    members = [f"gpu{i}:0:0" for i in range(world)]
    return {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": base, "gpu.devices": [0],
            "gpu.arenaBytes": 256 << 20, "modelCache.size": 1 << 30, "serving.maxConcurrentModels": 16, "gpu.members": members,
            "gpu.localMembers": [members[rank]], "proxy.replicasPerModel": 1, "proxy.replicaPick": "first", "cluster.rank": rank,
            "cluster.endpoints": socks, "cluster.slotBytes": 1 << 20, "cluster.windowSlots": 8, "proxy.grpcTimeout": 60.0}


def _rank_main(rank, world, socks, base, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}, "ticket": {}}
        with t.Server(_rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = sr.qa_inputs(3, 32, SMALL["vocab"], seed=7, sep_id=SEP)
            for j in range(N_MODELS):
                name = f"qs{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=NAMES)
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, x)))
                res["grpc"][j] = dict(outs)
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict",
                                        json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
                res["rest"][j] = (st, b.decode())
                tk = srv.predict_submit(name, "1", x, outputs=["span_scores", "span_starts"])
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


def test_forward_hop_spans():
    import torch
    assert torch.cuda.is_available()
    world = 2
    base = tempfile.mkdtemp(prefix="tfscqa")
    for j in range(N_MODELS):
        _write_qa(base, 32, SMALL, 40 + j, single=f"q1_{j}", multi=f"qs{j}")
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
    x = sr.qa_inputs(3, 32, SMALL["vocab"], seed=7, sep_id=SEP)
    for j in range(N_MODELS):
        owner = 0 if results[0]["owned"][j] else 1
        local, fwd = results[owner], results[1 - owner]
        assert sorted(local["y"][j]) == NAMES
        _check_spans(local["y"][j], x)
        for k in NAMES:
            assert fwd["y"][j][k].dtype == local["y"][j][k].dtype and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
        for k in ("span_scores", "span_starts"):
            assert fwd["ticket"][j][k].tobytes() == local["ticket"][j][k].tobytes()
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
