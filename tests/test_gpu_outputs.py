"""-m gpu: multi-output signatures (signature.outputs). The classification-head kernel against fp64, ResNet-50 and BERT
bundles with logits / probabilities / classes / top-5 next to their single-output bundles, every front-end on a
multi-output MLP, launch counts, programmatic-dependent-launch bit identity and the forward hop between two ranks."""
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

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_bert_pair_golden as pg  # noqa: E402
import torch_export as te  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
K = 5
FULL = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"},
        {"name": "classes", "kind": "classes"}, {"name": "top_k_classes", "kind": "top_k_classes", "k": K},
        {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": K}]
NAMES = sorted(o["name"] for o in FULL)   # packed order
MLP_DIMS = [512, 1024, 1000]


def _ptr(x):
    return x.data_ptr()


def _softmax64(x):
    x = np.asarray(x, np.float64)
    e = np.exp(x - x.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def _topk_ref(logits, k):
    """tf.math.top_k on the fp32 logits: descending, ties to the lower index"""
    return np.argsort(-np.asarray(logits, np.float32), axis=-1, kind="stable")[..., :k]


def _check_head(logits, r, k=K):
    """classes / top-k exact against `logits`, top-k probabilities the same bits as probabilities[index]"""
    idx = _topk_ref(logits, k)
    assert r["top_k_classes"].dtype == np.int32 and np.array_equal(r["top_k_classes"], idx)
    assert r["classes"].dtype == np.int64 and np.array_equal(r["classes"], idx[..., 0])
    tp = np.take_along_axis(r["probabilities"], idx.astype(np.int64), axis=-1)
    assert tp.view(np.int32).tolist() == r["top_k_probabilities"].view(np.int32).tolist()


# ------------------------------------------------------------------------------------------- kernel ----
def _logits(rows, n, seed):
    """rows cycle through: spread 1, spread 80, exact ties (few distinct values), a constant row"""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, n), np.float32)
    for r in range(rows):
        kind = (r + n) % 4
        off = rng.standard_normal() * 10
        if kind == 0:
            x[r] = off + rng.uniform(-0.5, 0.5, n)
        elif kind == 1:
            x[r] = off + rng.uniform(-40, 40, n)
        elif kind == 2:
            x[r] = np.round(rng.uniform(0, 4, n)) * 2.5 - 3          # five distinct values: ties everywhere
        else:
            x[r] = 3.25                                                # uniform probabilities, class 0
    return x


@pytest.mark.parametrize("k", [1, 5, 32])
@pytest.mark.parametrize("n", [2, 3, 13, 1000, 1001, 9216, 30522, 32768])
@pytest.mark.parametrize("rows", [1, 3, 8, 64, 128, 219])
def test_head_kernel_matches_fp64(rows, n, k):
    import torch
    k = min(k, n)
    x = _logits(rows, n, seed=rows * 100003 + n * 7 + k)
    xd = torch.from_numpy(x).cuda()
    probs = torch.full((rows, n), float("nan"), device="cuda")
    classes = torch.full((rows,), -7, dtype=torch.int64, device="cuda")
    idx = torch.full((rows, k), -7, dtype=torch.int32, device="cuda")
    tprob = torch.full((rows, k), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_classify_head(_ptr(xd), rows, n, k, _ptr(probs), _ptr(classes), _ptr(idx), _ptr(tprob), None),
                 "classify_head")
    torch.cuda.synchronize()
    p, p64 = probs.cpu().numpy(), _softmax64(x)
    assert np.all(np.abs(p - p64) <= 1e-5 * p64 + 1e-37), float(np.nanmax(np.abs(p - p64) / (p64 + 1e-37)))
    assert np.all(np.abs(p.astype(np.float64).sum(axis=1) - 1.0) <= 1e-5)
    const = [r for r in range(rows) if (r + n) % 4 == 3]
    assert all(np.all(p[r] == p[r][0]) for r in const)
    _check_head(x, {"probabilities": p, "classes": classes.cpu().numpy(), "top_k_classes": idx.cpu().numpy(),
                    "top_k_probabilities": tprob.cpu().numpy()}, k)
    assert all(classes.cpu().numpy()[r] == 0 for r in const)


def test_head_kernel_with_null_outputs():
    import torch
    rows, n, k = 5, 1001, 7
    x = torch.from_numpy(_logits(rows, n, 3)).cuda()
    ref_cls = torch.full((rows,), -7, dtype=torch.int64, device="cuda")
    t._lib.check(lib.tfsc_k_classify_head(_ptr(x), rows, n, k, None, _ptr(ref_cls), None, None, None), "classify_head")
    idx = torch.full((rows, k), -7, dtype=torch.int32, device="cuda")
    t._lib.check(lib.tfsc_k_classify_head(_ptr(x), rows, n, k, None, None, _ptr(idx), None, None), "classify_head")
    torch.cuda.synchronize()
    assert np.array_equal(ref_cls.cpu().numpy(), _topk_ref(x.cpu().numpy(), 1)[:, 0])
    assert np.array_equal(idx.cpu().numpy(), _topk_ref(x.cpu().numpy(), k))


def test_head_kernel_rejections():
    import torch
    x = torch.zeros(4, 64, device="cuda")
    y = torch.zeros(4, 64, device="cuda")
    for n, k in ((0, 1), (-3, 1), (32769, 1), (64, 0), (64, -1), (10, 11), (64, 33)):
        assert lib.tfsc_k_classify_head(_ptr(x), 4, n, k, _ptr(y), None, None, None, None) == t._lib.E_INVALID, (n, k)
    assert lib.tfsc_k_classify_head(None, 4, 64, 5, _ptr(y), None, None, None, None) == t._lib.E_INVALID
    assert lib.tfsc_k_classify_head(_ptr(x), -1, 64, 5, _ptr(y), None, None, None, None) == t._lib.E_INVALID
    assert lib.tfsc_k_classify_head(_ptr(x), 0, 64, 5, _ptr(y), None, None, None, None) == 0


# ------------------------------------------------------------------------------------ served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 6 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _served(srv, single, multi, x, ref64):
    y1 = srv.predict(single, "1", x)
    r = srv.predict(multi, "1", x, outputs=NAMES)
    assert sorted(r) == NAMES
    assert r["logits"].tobytes() == y1.tobytes()
    assert r["probabilities"].shape == y1.shape and r["top_k_classes"].shape == y1.shape[:-1] + (K,)
    assert np.max(np.abs(r["probabilities"] - _softmax64(ref64))) <= 1e-4
    _check_head(r["logits"], r)
    return r


def test_resnet50_multi_output(tmp_path):
    m = te.torchvision_resnet(5)
    single, multi = mf.resnet50_manifest(), mf.resnet50_manifest(outputs=FULL)
    blob = te.export_resnet(m, single)
    mf.write_graph_bundle(str(tmp_path / "r1" / "1"), single, blob)
    mf.write_graph_bundle(str(tmp_path / "r5" / "1"), multi, blob)
    x = np.random.default_rng(1).standard_normal((4, 224, 224, 3)).astype(np.float32)
    ref = te.resnet_reference(m, x)
    with t.Server(_cfg(tmp_path)) as srv:
        _served(srv, "r1", "r5", x, ref)
        _served(srv, "r1", "r5", x[:1], ref[:1])


@pytest.mark.parametrize("kind", ["bert_small", "bert_base"])
def test_bert_three_inputs_multi_output(kind, tmp_path):
    import copy
    import torch
    arch = dict(hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=512) if kind == "bert_small" else dict(max_pos=512)
    arch["labels"] = 6
    S = 128
    m = te.hf_bert(4 if kind == "bert_small" else 3, **arch)
    single = mf.bert_manifest(seq=S, **arch, inputs=mf.BERT_INPUTS)
    multi = mf.bert_manifest(seq=S, **arch, inputs=mf.BERT_INPUTS, outputs=FULL)
    blob = te.export_bert(m, single)
    mf.write_graph_bundle(str(tmp_path / "b1" / "1"), single, blob)
    mf.write_graph_bundle(str(tmp_path / "b5" / "1"), multi, blob)
    x = pg.pair_inputs(8, S, arch.get("vocab", 30522), seed=11)
    m64 = copy.deepcopy(m).double().cuda()
    tt = {k: torch.from_numpy(np.ascontiguousarray(v, np.int64)).cuda() for k, v in x.items()}
    with torch.no_grad():
        ref = m64(input_ids=tt["input_ids"], attention_mask=tt["input_mask"], token_type_ids=tt["segment_ids"]).logits.cpu().numpy()
    with t.Server(_cfg(tmp_path)) as srv:
        _served(srv, "b1", "b5", x, ref)
        _served(srv, "b1", "b5", {k: v[:3] for k, v in x.items()}, ref[:3])


# --------------------------------------------------------------------------------------- front-ends ----
def _write_mlp(tmp, name, outputs, dims=MLP_DIMS, seed=0):
    rng = np.random.default_rng(seed)
    ws = [(rng.standard_normal((a, b)) / np.sqrt(a)).astype(np.float32) for a, b in zip(dims[:-1], dims[1:])]
    bs = [(rng.standard_normal(b) * 0.1).astype(np.float32) for b in dims[1:]]
    mf.write_mlp_bundle(os.path.join(str(tmp), name, "1"), ws, bs, outputs=outputs)


def _session_run_request(name, feed, x, fetch):
    named = wire._ld(1, feed.encode()) + wire._ld(2, wire.encode_tensor(x))
    return wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())


def _session_run_tensor(resp):
    for f, _wt, v in wire._fields(resp):
        if f == 1:
            for f2, _w2, v2 in wire._fields(bytes(v)):
                if f2 == 2:
                    return wire.decode_tensor(bytes(v2))
    raise AssertionError("no tensor in SessionRunResponse")


def test_every_frontend_on_a_multi_output_mlp(tmp_path):
    import torch
    _write_mlp(tmp_path, "one", None)
    _write_mlp(tmp_path, "multi", FULL)
    x = np.random.default_rng(2).standard_normal((5, MLP_DIMS[0])).astype(np.float32)
    with t.Server(_cfg(tmp_path)) as srv:
        y1 = srv.predict("one", "1", x)
        full = srv.predict("multi", "1", x, outputs=NAMES)
        assert full["logits"].tobytes() == y1.tobytes()
        assert np.max(np.abs(full["probabilities"] - _softmax64(y1))) <= 1e-5
        _check_head(y1, full)
        assert full["classes"].shape == (5,) and full["top_k_probabilities"].shape == (5, K)
        # C ABI: any subset, any order, the same bits
        sub = srv.predict("multi", "1", x, outputs=["top_k_classes", "probabilities", "classes"])
        assert list(sub) == ["top_k_classes", "probabilities", "classes"]
        for k, v in sub.items():
            assert v.dtype == full[k].dtype and v.tobytes() == full[k].tobytes(), k
        # one row as a 1-D input: classes is a scalar, probabilities [N]
        one = srv.predict("multi", "1", x[0], outputs=["classes", "probabilities"])
        assert one["classes"].shape == () and one["classes"] == full["classes"][0]
        assert one["probabilities"].tobytes() == full["probabilities"][0].tobytes()
        # errors name the outputs; nothing is launched for them
        launches = srv.stats()["kernel_launches"]
        for outs, why in ((None, "every out[i].name must name one of"), (["nope"], "unknown output 'nope'"),
                          (["classes", "logits", "classes"], "'classes' is requested twice")):
            with pytest.raises(t._lib.TfscError) as e:
                srv.predict("multi", "1", x, outputs=outs)
            assert e.value.code == t._lib.E_INVALID and why in str(e.value), str(e.value)
            assert "'classes' (int64), 'logits' (float), 'probabilities' (float), 'top_k_classes' (int32)" in str(e.value)
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("multi", "1", x, outputs=["probabilities"], out_capacity_elems=100)
        assert e.value.code == t._lib.E_BUFFER
        assert srv.stats()["kernel_launches"] == launches
        # deadline, member and asynchronous tickets
        for r in (srv.predict_deadline("multi", "1", x, srv.now_ns() + 30_000_000_000, outputs=NAMES),
                  srv.predict_member(0, "multi", "1", x, outputs=NAMES)):
            assert all(r[k].tobytes() == full[k].tobytes() for k in NAMES)
        tk = srv.predict_submit("multi", "1", x, outputs=["classes", "top_k_probabilities"])
        try:
            r = tk.wait(30.0)
        finally:
            tk.release()
        assert r["classes"].tobytes() == full["classes"].tobytes() and r["top_k_probabilities"].tobytes() == full["top_k_probabilities"].tobytes()
        # gRPC Predict: no filter = every output in sorted order; a filter selects; unknown / duplicate aliases are refused
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("multi", 1, {"x": x})))
        assert list(outs) == NAMES
        for k in NAMES:
            assert outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes(), k
        resp = srv.grpc_predict(wire.encode_predict_request("multi", 1, {"x": x}, output_filter=["top_k_classes", "classes"]))
        _spec, outs = wire.decode_predict_response(resp)
        assert list(outs) == ["classes", "top_k_classes"] and outs["top_k_classes"].tobytes() == full["top_k_classes"].tobytes()
        for filt, why in ((["classes", "scores"], "output tensor alias not found in signature: scores Outputs expected to be in the set "
                                                  "{classes,logits,probabilities,top_k_classes,top_k_probabilities}."),
                          (["logits", "logits"], "duplicate output tensor alias: logits")):
            with pytest.raises(t._lib.TfscError) as e:
                srv.grpc_predict(wire.encode_predict_request("multi", 1, {"x": x}, output_filter=filt))
            assert e.value.code == t._lib.E_INVALID and why in str(e.value), str(e.value)
        # a single-output bundle keeps ignoring output_filter
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("one", 1, {"x": x}, output_filter=["zz"])))
        assert list(outs) == ["y"] and outs["y"].tobytes() == y1.tobytes()
        # REST, row and columnar
        st, b = srv.rest_handle("POST", "/v1/models/multi/versions/1:predict", json.dumps({"instances": x.tolist()}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        assert len(preds) == 5 and all(list(p) == NAMES for p in preds)
        for i, p in enumerate(preds):
            assert p["classes"] == int(full["classes"][i]) and isinstance(p["classes"], int)
            assert p["top_k_classes"] == full["top_k_classes"][i].tolist()
            assert np.array_equal(np.float32(p["probabilities"]), full["probabilities"][i])
            assert np.array_equal(np.float32(p["logits"]), full["logits"][i])
        st, b = srv.rest_handle("POST", "/v1/models/multi/versions/1:predict", json.dumps({"inputs": {"x": x.tolist()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES and cols["classes"] == full["classes"].tolist()
        assert cols["top_k_classes"] == full["top_k_classes"].tolist()
        assert np.array_equal(np.float32(cols["top_k_probabilities"]), full["top_k_probabilities"])
        # metadata: every output with its dtype and shape
        st, b = srv.rest_handle("GET", "/v1/models/multi/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {"classes": ("DT_INT64", ["-1"]), "logits": ("DT_FLOAT", ["-1", "1000"]), "probabilities": ("DT_FLOAT", ["-1", "1000"]),
                "top_k_classes": ("DT_INT32", ["-1", str(K)]), "top_k_probabilities": ("DT_FLOAT", ["-1", str(K)])}
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        # SessionRun: the fetch names any one output
        for fetch in ("classes:0", "probabilities", "top_k_classes:0"):
            tsr = _session_run_tensor(srv.grpc_session_run(_session_run_request("multi", "x:0", x, fetch)))
            key = fetch.split(":")[0]
            assert tsr.dtype == full[key].dtype and tsr.tobytes() == full[key].tobytes(), fetch
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(_session_run_request("multi", "x:0", x, "y:0"))
        assert e.value.code == t._lib.E_INVALID and "'top_k_classes' (int32)" in str(e.value)
        # Classify / Regress refuse a multi-output model and name its outputs
        st, b = srv.rest_handle("POST", "/v1/models/multi/versions/1:classify", json.dumps({"examples": [{"x": 1.0}]}).encode())
        assert st == 400 and "'top_k_probabilities' (float)" in json.loads(b)["error"]
        # tfsc_predict_device writes packed rows; packed_output_layout splits them
        srv.ensure(0, "multi", 1)
        layout = mf.packed_output_layout(FULL, MLP_DIMS[-1])
        width = sum(w for _n, _o, w, _d in layout)
        xd = torch.from_numpy(x).cuda()
        yd = torch.full((5, width), float("nan"), device="cuda")
        srv.predict_device(0, "multi", 1, _ptr(xd), 5, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), FULL, MLP_DIMS[-1])
        for k in NAMES:
            assert dev[k].tobytes() == full[k].tobytes(), k


def test_launch_counts(tmp_path):
    """A multi-output bundle launches exactly one kernel more per batch than the same weights with one output"""
    _write_mlp(tmp_path, "one", None)
    _write_mlp(tmp_path, "multi", FULL)
    with t.Server(_cfg(tmp_path)) as srv:
        for rows in (1, 8, 64):
            x = np.random.default_rng(rows).standard_normal((rows, MLP_DIMS[0])).astype(np.float32)
            srv.predict("one", "1", x)
            srv.predict("multi", "1", x, outputs=["classes"])   # both resident, caches warm
            counts = {}
            for name in ("one", "multi"):
                s0 = srv.stats()
                srv.predict(name, "1", x, outputs=None if name == "one" else ["classes"])
                s1 = srv.stats()
                counts[name] = (s1["kernel_launches"] - s0["kernel_launches"], s1["batches"] - s0["batches"])
            assert counts["one"][1] == counts["multi"][1] >= 1
            assert counts["multi"][0] == counts["one"][0] + counts["multi"][1], (rows, counts)


PDL_SCRIPT = r"""
import sys
import numpy as np, torch
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_outputs as g
tmp = sys.argv[2]
g._write_mlp(tmp, "multi", g.FULL)
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (8, 64):
        x = np.random.default_rng(rows).standard_normal((rows, g.MLP_DIMS[0])).astype(np.float32)
        for k, v in srv.predict("multi", "1", x, outputs=g.NAMES).items():
            out[f"{k}_r{rows}"] = v
        srv.ensure(0, "multi", 1)
        xd = torch.from_numpy(x).cuda()
        yd = torch.full((rows, 1000 + 1000 + 2 + 5 + 5), float("nan"), device="cuda")
        for _ in range(3):   # back to back on one stream: the head follows the last PDL dense pass
            srv.predict_device(0, "multi", 1, xd.data_ptr(), rows, yd.data_ptr(), 0)
        srv.sync(0)
        out[f"device_r{rows}"] = yd.cpu().numpy()
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
    assert sorted(res["default"]) == sorted(res["0"])
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key
        if key.startswith("device"):
            assert not np.isnan(y).any()


# --------------------------------------------------------------------------------------- forward hop ----
N_MODELS = 6


def _outs(j):
    """every third model declares probabilities, classes and top-k classes only"""
    return FULL if j % 3 else FULL[1:4]


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
            x = np.random.default_rng(7).standard_normal((3, 64)).astype(np.float32)
            for j in range(N_MODELS):
                name = f"m{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=[o["name"] for o in _outs(j)])
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, {"x": x})))
                res["grpc"][j] = {k: v for k, v in outs.items()}
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict", json.dumps({"instances": x.tolist()}).encode())
                res["rest"][j] = (st, b.decode())
                tk = srv.predict_submit(name, "1", x, outputs=["top_k_classes", "classes"])
                try:
                    res["ticket"][j] = tk.wait(60.0)
                finally:
                    tk.release()
            try:
                jr = next(j for j in range(N_MODELS) if not res["owned"][j])
                srv.predict(f"m{jr}", "1", x, outputs=["nope"])
                res["remote_error"] = None
            except t._lib.TfscError as e:
                res["remote_error"] = (e.code, str(e))
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


def test_forward_hop_multi_output():
    import torch
    assert torch.cuda.is_available()
    world = 2
    base = tempfile.mkdtemp(prefix="tfscmo")
    for j in range(N_MODELS):
        _write_mlp(base, f"m{j}", _outs(j), dims=[64, 96, 40 + j], seed=j)
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
        names = sorted(o["name"] for o in _outs(j))
        assert sorted(local["y"][j]) == names
        for k in names:
            assert fwd["y"][j][k].dtype == local["y"][j][k].dtype and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert list(local["grpc"][j]) == names == list(fwd["grpc"][j])
        for k in names:
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
        for k in ("top_k_classes", "classes"):
            assert fwd["ticket"][j][k].tobytes() == local["ticket"][j][k].tobytes()
    for r in results.values():
        code, msg = r["remote_error"]
        assert code == t._lib.E_INVALID and "unknown output 'nope'" in msg
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
