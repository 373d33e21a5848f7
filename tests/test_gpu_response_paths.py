"""-m gpu: every Predict front-end answers with the values, dtype and shape of the synchronous tfsc_predict, for the
response shapes that the other suites do not take through every front-end: an affine bundle, a single-output graph
whose output has rank 3, and bundles that declare exactly one output (float, then int32)."""
import json

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import wire

pytestmark = pytest.mark.gpu
mf = t.modelformat


def _cfg(tmp):
    return {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
            "gpu.arenaBytes": 256 << 20, "serving.maxConcurrentModels": 8, "modelCache.size": 1 << 30, "gpu.maxBatch": 8}


def _write_mlp(tmp, name, outputs, dims=(16, 32, 10)):
    rng = np.random.default_rng(3)
    ws = [(rng.standard_normal((a, b)) / np.sqrt(a)).astype(np.float32) for a, b in zip(dims[:-1], dims[1:])]
    bs = [(rng.standard_normal(b) * 0.1).astype(np.float32) for b in dims[1:]]
    mf.write_mlp_bundle(str(tmp / name / "1"), ws, bs, outputs=outputs)


def _same(got, want, what):
    got = np.asarray(got)
    assert got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes(), what


def _session_run(srv, name, x, fetch):
    named = wire._ld(1, b"x:0") + wire._ld(2, wire.encode_tensor(x))
    req = wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())
    for f, _wt, v in wire._fields(srv.grpc_session_run(req)):
        if f == 1:
            for f2, _w2, v2 in wire._fields(bytes(v)):
                if f2 == 2:
                    return wire.decode_tensor(bytes(v2))
    raise AssertionError("no tensor in SessionRunResponse")


def _grpc(srv, name, x, key):
    _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, {"x": x})))
    assert list(outs) == [key]
    return outs[key]


def _submit(srv, name, x, **kw):
    tk = srv.predict_submit(name, "1", x, **kw)
    try:
        return tk.wait(30.0)
    finally:
        tk.release()


def _rest(srv, name, body):
    st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict", json.dumps(body).encode())
    assert st == 200, b
    return json.loads(b)


def test_affine_bundle_through_every_frontend(tmp_path):
    mf.write_affine_bundle(str(tmp_path / "aff" / "1"), 0.5, 2.0)
    x = np.arange(6, dtype=np.float32).reshape(2, 3) - 2.5
    with t.Server(_cfg(tmp_path)) as srv:
        y = srv.predict("aff", "1", x)
        assert y.shape == (2, 3) and np.array_equal(y, x * 0.5 + 2.0)
        _same(_submit(srv, "aff", x), y, "predict_submit")
        _same(_grpc(srv, "aff", x, "y"), y, "gRPC Predict")
        _same(_session_run(srv, "aff", x, "y:0"), y, "SessionRun")


def test_rank3_graph_output_through_every_frontend(tmp_path):
    man = mf._graph_manifest([8, 8, 4], [mf._conv(-1, -2, 8, 4, 6, k=3)], 1)
    mf.write_graph_bundle(str(tmp_path / "g" / "1"), man, np.random.default_rng(4).standard_normal(man["weights_bytes"] // 4))
    x = np.random.default_rng(5).standard_normal((2, 8, 8, 4)).astype(np.float32)
    with t.Server(_cfg(tmp_path)) as srv:
        y = srv.predict("g", "1", x)
        assert y.shape == (2, 8, 8, 6)
        _same(srv.predict_deadline("g", "1", x, srv.now_ns() + 30_000_000_000), y, "predict_deadline")
        _same(srv.predict_member(0, "g", "1", x), y, "predict_member")
        _same(_submit(srv, "g", x), y, "predict_submit")
        _same(_grpc(srv, "g", x, "y"), y, "gRPC Predict")
        _same(_session_run(srv, "g", x, "y:0"), y, "SessionRun")
        _same(np.float32(_rest(srv, "g", {"instances": x.tolist()})["predictions"]), y, "REST row")
        _same(np.float32(_rest(srv, "g", {"inputs": x.tolist()})["outputs"]), y, "REST columnar")


def test_one_declared_float_output_through_grpc_and_session_run(tmp_path):
    _write_mlp(tmp_path, "p", [{"name": "probabilities", "kind": "probabilities"}])
    x = np.random.default_rng(6).standard_normal((5, 16)).astype(np.float32)
    with t.Server(_cfg(tmp_path)) as srv:
        y = srv.predict("p", "1", x, outputs=["probabilities"])["probabilities"]
        assert y.shape == (5, 10) and y.dtype == np.float32
        _same(_submit(srv, "p", x, outputs=["probabilities"])["probabilities"], y, "predict_submit")
        _same(_grpc(srv, "p", x, "probabilities"), y, "gRPC Predict")
        _same(_session_run(srv, "p", x, "probabilities:0"), y, "SessionRun")


def test_one_declared_int32_output_through_rest(tmp_path):
    _write_mlp(tmp_path, "k", [{"name": "top_k_classes", "kind": "top_k_classes", "k": 3}])
    x = np.random.default_rng(7).standard_normal((5, 16)).astype(np.float32)
    with t.Server(_cfg(tmp_path)) as srv:
        y = srv.predict("k", "1", x, outputs=["top_k_classes"])["top_k_classes"]
        assert y.shape == (5, 3) and y.dtype == np.int32
        preds = _rest(srv, "k", {"instances": x.tolist()})["predictions"]
        assert all(list(p) == ["top_k_classes"] for p in preds)
        _same(np.int32([p["top_k_classes"] for p in preds]), y, "REST row")
        cols = _rest(srv, "k", {"inputs": {"x": x.tolist()}})["outputs"]
        assert list(cols) == ["top_k_classes"]
        _same(np.int32(cols["top_k_classes"]), y, "REST columnar")
        _same(_grpc(srv, "k", x, "top_k_classes"), y, "gRPC Predict")
        _same(_session_run(srv, "k", x, "top_k_classes:0"), y, "SessionRun")
