"""-m gpu: parity of the CUDA path (through the C ABI) with the oracle.  fp32 tolerance 1e-4
(north_star); routing / residency outcomes bit-exact."""
import base64
import ctypes as C
import json
import os
import threading

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import cachemanager as ocm
from oracle import models, wire
from oracle.lrucache import Model as OModel
from oracle.lrucache import ModelIdentifier as OId
from tools.traces import zipf_trace

pytestmark = pytest.mark.gpu
TOL = 1e-4  # north_star: fp32 outputs within 1e-4


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device; there is no CPU fallback"
    return torch


def _close(got, ref64, tol=TOL):
    """|gpu - fp64 oracle| <= tol * max(1, |ref|)"""
    got = np.asarray(got, np.float64)
    scale = np.maximum(1.0, np.abs(ref64))
    return float(np.max(np.abs(got - ref64) / scale))


# ---- X1 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 4096, 1 << 20, (1 << 20) + 3])
def test_k_affine(n):
    torch = _torch()
    x = torch.randn(n + 1, device="cuda")[1:] if n % 2 else torch.randn(n, device="cuda")  # odd n: unaligned view
    y = torch.empty_like(x)
    ab = torch.tensor([0.5, 2.0], device="cuda")
    t._lib.check(t._lib.lib.tfsc_k_affine(x.data_ptr(), y.data_ptr(), n, ab.data_ptr(), ab.data_ptr() + 4, None))
    torch.cuda.synchronize()
    ref = np.float32(0.5) * x.cpu().numpy() + np.float32(2.0)
    np.testing.assert_allclose(y.cpu().numpy(), ref, rtol=1e-6, atol=1e-6)


# ---- X2 -------------------------------------------------------------------------------------
def _dense(x, w, b, relu, variant=None):
    torch = _torch()
    rows, k = x.shape
    n = w.shape[1]
    ws_bytes = t._lib.lib.tfsc_k_dense_workspace(rows, k, n)
    ws = torch.zeros(ws_bytes // 4 + 64, device="cuda")
    xd, wd, bd = (torch.from_numpy(a).cuda() for a in (x, w, b))
    yd = torch.full((rows, n), float("nan"), device="cuda")
    for _ in range(2):  # twice: the split-K arrival counters must self-reset
        yd.fill_(float("nan"))
        if variant is None:
            t._lib.check(t._lib.lib.tfsc_k_dense(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), yd.data_ptr(), rows, k, n,
                                                  1 if relu else 0, ws.data_ptr(), ws_bytes, None))
        else:
            t._lib.check(t._lib.lib.tfsc_k_dense_variant(variant, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), yd.data_ptr(), rows,
                                                          k, n, 1 if relu else 0, ws.data_ptr(), ws_bytes, None))
        torch.cuda.synchronize()
    return yd.cpu().numpy()


@pytest.mark.parametrize("rows", [1, 2, 3, 4, 5, 7, 8, 9, 16, 19, 65, 72, 73, 128, 219])
@pytest.mark.parametrize("k,n", [(64, 64), (100, 512), (577, 1032), (1024, 520), (9216, 1024), (33, 8), (5000, 4096)])
def test_k_dense_matches_oracle(rows, k, n):
    """above 64 rows tfsc_k_dense runs several passes back to back on one split-K workspace: 219 rows = tensor-core passes
    of 64, 64, 64, 27; 65 / 72 rows = one of 64 and a <= 8-row pass; 73 = 64 + 9"""
    rng = np.random.default_rng(rows * 7919 + k + n)
    x = rng.standard_normal((rows, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    for relu in (False, True):
        got = _dense(x, w, b, relu)
        ref = x.astype(np.float64) @ w.astype(np.float64) + b
        if relu:
            ref = np.maximum(ref, 0)
        assert not np.isnan(got).any()
        assert _close(got, ref) <= TOL


@pytest.mark.parametrize("variant", [1, 2, 4])   # LDG stream, bulk-copy (TMA) ring with 8 / 4 k-lanes
@pytest.mark.parametrize("rows", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("k,n", [(64, 8), (100, 520), (777, 1032), (4096, 4096), (20000, 64)])
def test_k_dense_variants_match_oracle(variant, rows, k, n):
    rng = np.random.default_rng(variant * 31 + rows * 7919 + k + n)
    x = rng.standard_normal((rows, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    for relu in (False, True):
        got = _dense(x, w, b, relu, variant)
        ref = x.astype(np.float64) @ w.astype(np.float64) + b
        if relu:
            ref = np.maximum(ref, 0)
        assert not np.isnan(got).any()
        assert _close(got, ref) <= TOL


@pytest.mark.parametrize("k,n", [(7, 10), (64, 3), (129, 1001), (16, 12)])
def test_k_dense_generic_shapes(k, n):
    rng = np.random.default_rng(k * n)
    x = rng.standard_normal((3, k)).astype(np.float32)
    w = rng.standard_normal((k, n)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    got = _dense(x, w, b, True)
    ref = np.maximum(x.astype(np.float64) @ w + b, 0)
    assert _close(got, ref) <= TOL


def test_k_dense_is_deterministic_and_linear():
    rng = np.random.default_rng(5)
    k, n = 9216, 9216
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = np.zeros(n, np.float32)
    x = rng.standard_normal((8, k)).astype(np.float32)
    y1, y2 = _dense(x, w, b, False), _dense(x, w, b, False)
    assert np.array_equal(y1, y2)  # fixed-order split-K reduction: bit-reproducible
    ya = _dense(x[:4], w, b, False)
    # rows are independent: a 4-row launch equals the first 4 rows of the 8-row launch up to the
    # template's accumulation order (same order by construction)
    np.testing.assert_allclose(ya, y1[:4], rtol=1e-5, atol=1e-5)
    ref = x.astype(np.float64) @ w.astype(np.float64)
    assert _close(y1, ref) <= TOL
    # linearity at full size: f(2x) = 2 f(x) exactly in fp32 (power-of-two scaling)
    assert np.array_equal(_dense(2 * x, w, b, False), 2 * y1)


# ---- server: synthetic provider + predict -------------------------------------------------------
DIMS = [128, 264, 72, 16]


def _cfg(**kw):
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": DIMS,
           "modelProvider.synthetic.count": 64, "gpu.devices": [0], "gpu.arenaBytes": 8 << 20,
           "modelCache.size": 1 << 30, "serving.maxConcurrentModels": 4, "proxy.seed": 1, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _oracle_mlp(j, x, dims=DIMS, dtype=np.float64):
    man, blob = models.synth_mlp_blob(dims, seed=1000 + j)
    return models.forward(man, blob, x, dtype)


def test_predict_matches_oracle_and_counts():
    _torch()
    rng = np.random.default_rng(1)
    with t.Server(_cfg()) as srv:
        for j, rows in [(0, 1), (5, 3), (0, 8), (9, 13), (5, 1)]:
            x = rng.standard_normal((rows, DIMS[0])).astype(np.float32)
            y = srv.predict(f"m{j}", "1", x)
            assert y.shape == (rows, DIMS[-1])
            assert _close(y, _oracle_mlp(j, x)) <= TOL
        st = srv.stats()
        assert (st["cache_total"], st["cache_hits_total"], st["cache_misses_total"]) == (5, 2, 3)
        assert st["h2d_weight_bytes"] == 3 * models.mlp_manifest(DIMS)["weights_bytes"]
        assert st["kernel_launches"] > 0
        # 1-D input is a single row; output drops the batch dim like TF
        x1 = rng.standard_normal(DIMS[0]).astype(np.float32)
        assert srv.predict("m0", "1", x1).shape == (DIMS[-1],)


def test_predict_errors():
    _torch()
    with t.Server(_cfg()) as srv:
        x = np.zeros((1, DIMS[0]), np.float32)
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("m999", "1", x)          # provider: No matching model found
        assert e.value.code == t._lib.E_NOT_FOUND
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("m1", "abc", x)           # strconv.ParseInt fails (cachemanager.go:297)
        assert e.value.code == t._lib.E_INVALID
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("m1", "1", np.zeros((1, DIMS[0] + 1), np.float32))
        assert e.value.code == t._lib.E_INVALID
        assert srv.status(0, "never", 1) == t._lib.E_NOT_FOUND   # servingcontroller.go:137


def test_residency_machine_matches_oracle_trace(golden):
    """Same Zipf trace through the product and the oracle: outcome per request, counters, host
    tier order and HBM-resident set must be identical (bit-exact control path)."""
    _torch()
    size = models.mlp_manifest(DIMS)["weights_bytes"]

    class Prov:
        def model_size(self, name, ver):
            return size

        def load_model(self, name, ver):
            return OModel(OId(name, ver), f"{name}/{ver}", size)

    names = {t._lib.FETCH_HIT: "hit", t._lib.FETCH_RELOAD: "reload", t._lib.FETCH_MISS: "miss"}
    for case in golden("trace_golden.json"):
        cfg = _cfg(**{"modelCache.size": case["cache_models"] * size, "serving.maxConcurrentModels": case["max_concurrent"],
                      "gpu.arenaBytes": 64 << 20})
        orc = ocm.CacheManager(Prov(), case["cache_models"] * size, case["max_concurrent"])
        with t.Server(cfg) as srv:
            for step, j in enumerate(case["trace"]):
                got = names[srv.ensure(0, f"m{j}", 1)]
                want = orc.fetch_model(OId(f"m{j}", 1))
                assert got == want == case["outcomes"][step], (case["seed"], step, j, got, want)
            st = srv.stats()
            assert (st["cache_total"], st["cache_hits_total"], st["cache_misses_total"]) == (orc.total, orc.hits, orc.misses)
            assert (orc.hits, orc.misses) == (case["hits"], case["misses"])
            assert [n for n, _v, _b in srv.host_models(0)] == [m.identifier.model_name for m in orc.local_cache.list_models()]
            res = srv.resident(0)
            assert [n for n, _v, _b, _s in res] == [m.identifier.model_name for m in orc.resident_prefix()]
            assert all(s == t._lib.STATE_AVAILABLE for *_x, s in res)
            # evicted models report END, like an unloaded TF-Serving servable
            resident = {n for n, *_ in res}
            seen = {f"m{j}" for j in case["trace"]}
            for n in seen - resident:
                assert srv.status(0, n, 1) == t._lib.STATE_END


def test_arena_byte_budget_bounds_resident_set():
    _torch()
    size = models.mlp_manifest(DIMS)["weights_bytes"]
    arena = 3 * ((size + 1023) // 1024 * 1024) + 512
    with t.Server(_cfg(**{"gpu.arenaBytes": arena, "serving.maxConcurrentModels": 100})) as srv:
        rng = np.random.default_rng(3)
        for j in [1, 2, 3, 4, 5, 1, 2]:
            x = rng.standard_normal((2, DIMS[0])).astype(np.float32)
            assert _close(srv.predict(f"m{j}", "1", x), _oracle_mlp(j, x)) <= TOL
        st = srv.stats()
        assert st["resident_models"] == 3 and st["arena_bytes_used"] <= arena
        assert st["evictions_hbm"] >= 2
        assert [n for n, *_ in srv.resident(0)] == ["m2", "m1", "m5"]


def test_concurrent_predicts_are_batched_and_correct():
    _torch()
    rng = np.random.default_rng(11)
    jobs = [(int(rng.integers(0, 6)), rng.standard_normal((int(rng.integers(1, 4)), DIMS[0])).astype(np.float32))
            for _ in range(96)]
    out = [None] * len(jobs)
    with t.Server(_cfg(**{"serving.maxConcurrentModels": 3, "gpu.arenaBytes": 4 << 20})) as srv:
        def work(lo, hi):
            for i in range(lo, hi):
                out[i] = srv.predict(f"m{jobs[i][0]}", "1", jobs[i][1])
        ths = [threading.Thread(target=work, args=(i * 8, (i + 1) * 8)) for i in range(12)]
        [th.start() for th in ths]
        [th.join() for th in ths]
        st = srv.stats()
    for (j, x), y in zip(jobs, out):
        assert _close(y, _oracle_mlp(j, x)) <= TOL
    assert st["batched_rows"] == sum(x.shape[0] for _j, x in jobs)
    assert st["batches"] <= len(jobs)


# ---- wire-level entry points --------------------------------------------------------------------
def test_grpc_predict_wire_roundtrip(golden):
    _torch()
    rng = np.random.default_rng(2)
    with t.Server(_cfg()) as srv:
        for use_content in (True, False):
            x = rng.standard_normal((4, DIMS[0])).astype(np.float32)
            req = wire.encode_predict_request("m3", 1, {"x": x}, use_content=use_content)
            spec, outs = wire.decode_predict_response(srv.grpc_predict(req))
            assert spec == ("m3", 1, "serving_default")
            assert outs["y"].shape == (4, DIMS[-1]) and _close(outs["y"], _oracle_mlp(3, x)) <= TOL
        # wrong input key / wrong dtype / unknown model map to gRPC codes
        bad = wire.encode_predict_request("m3", 1, {"nope": np.zeros((1, DIMS[0]), np.float32)})
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_predict(bad)
        assert e.value.code == t._lib.E_INVALID
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_predict(wire.encode_predict_request("m3", 1, {"x": np.zeros((1, DIMS[0]), np.int32)}))
        assert e.value.code == t._lib.E_INVALID
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_predict(wire.encode_predict_request("zzz", 1, {"x": np.zeros((1, DIMS[0]), np.float32)}))
        assert e.value.code == t._lib.E_NOT_FOUND
        st = srv.stats()
        assert st["proxy_requests_grpc"] == 5 and st["proxy_failures_grpc"] == 3


def test_disk_provider_serves_tensorflow_savedmodel_trees(tmp_path):
    """SURVEY 8f-1: a model repository of TensorFlow SavedModel directories (saved_model.pb + variables/), as
    TF-Serving would load them, served without conversion step: the disk provider imports graph + variables on the fly.
    half_plus_two graph shape (y = a*x + b, deploy/docker-compose/readme.md:40-42) and a Keras-style dense MLP."""
    _torch()
    from savedmodel_fixtures import _mlp_fixture, write_bundle, write_saved_model
    repo = tmp_path
    d = repo / "saved_model_half_plus_two_cpu" / "00000123"
    os.makedirs(d)
    write_bundle(str(d / "variables" / "variables"), {"a": np.array(0.5, np.float32), "b": np.array(2.0, np.float32)})
    write_saved_model(str(d / "saved_model.pb"),
                      [("x", "Placeholder", []), ("a", "VariableV2", []), ("a/read", "Identity", ["a"]), ("b", "VariableV2", []),
                       ("b/read", "Identity", ["b"]), ("Mul", "Mul", ["a/read", "x"]), ("y", "Add", ["Mul", "b/read"])],
                      ("x", "x:0", "y", "y:0"))
    tensors = _mlp_fixture(repo / "mlp" / "7", np.random.default_rng(21), (48, 64, 16))
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(repo), "modelCache.size": 1 << 20,
           "serving.maxConcurrentModels": 2, "gpu.devices": [0], "gpu.arenaBytes": 1 << 20}
    with t.Server(cfg) as srv:
        st, body = srv.rest_handle("POST", "/v1/models/saved_model_half_plus_two_cpu/versions/00000123:predict",
                                   b'{"instances": [1.0, 2.0, 5.0]}')
        assert st == 200 and json.loads(body) == {"predictions": [2.5, 3.0, 4.5]}
        x = np.random.default_rng(22).standard_normal((5, 48)).astype(np.float32)
        y = srv.predict("mlp", "7", x)
        h = np.maximum(x.astype(np.float64) @ tensors["dense/kernel"] + tensors["dense/bias"], 0)
        ref = h @ tensors["dense_1/kernel"] + tensors["dense_1/bias"]
        assert y.shape == (5, 16) and _close(y, ref) <= TOL


def test_half_plus_two_rest_and_grpc_known_answer(tmp_path, golden):
    """The only end-to-end known answer in the reference (deploy/docker-compose/readme.md:25-42),
    through the disk provider, REST and gRPC, version directory 00000123."""
    _torch()
    repo = str(tmp_path)
    t.modelformat.write_affine_bundle(os.path.join(repo, "saved_model_half_plus_two_cpu", "00000123"), 0.5, 2.0)
    t.modelformat.write_affine_bundle(os.path.join(repo, "half_plus_two", "123"), 0.5, 2.0)
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": repo, "modelCache.size": 30000,
           "serving.maxConcurrentModels": 2, "gpu.devices": [0], "gpu.arenaBytes": 1 << 20}
    with t.Server(cfg) as srv:
        base = "/v1/models/saved_model_half_plus_two_cpu/versions/00000123"
        st, body = srv.rest_handle("POST", base + ":predict", b'{"instances": [1.0, 2.0, 5.0]}')
        assert st == 200 and json.loads(body) == {"predictions": [2.5, 3.0, 4.5]}
        assert body == b'{\n    "predictions": [2.5, 3.0, 4.5\n    ]\n}'
        st, body = srv.rest_handle("GET", base)
        assert st == 200 and json.loads(body) == {"model_version_status": [
            {"version": "123", "state": "AVAILABLE", "status": {"error_code": "OK", "error_message": ""}}]}
        st, body = srv.rest_handle("POST", base + ":predict", b'{"inputs": [[1.0, 2.0], [5.0, 7.0]]}')
        assert st == 200 and json.loads(body) == {"outputs": [[2.5, 3.0], [4.5, 5.5]]}
        assert srv.rest_handle("GET", "/v1/thisisabadrequest/foobar/versions/42") == (404, b'{"Status":"Error","Message":"Not found"}\n')
        assert srv.rest_handle("GET", "/v1/models/foobar")[0] == 400
        assert srv.rest_handle("POST", "/v1/models/nope/versions/1:predict", b'{"instances": [1.0]}')[0] == 404
        st, body = srv.rest_handle("GET", base + "/metadata")
        assert st == 200 and json.loads(body)["model_spec"]["version"] == "123"
        g = golden("wire_golden.json")
        req = base64.b64decode(g["requests"][1]["request_b64"])   # serialized by the reference's own schema
        resp = srv.grpc_predict(req)
        spec, outs = wire.decode_predict_response(resp)
        assert spec == ("half_plus_two", 123, "serving_default") and outs["y"].tolist() == [2.5, 3.0, 4.5]
        # byte-identical to what python-protobuf emits from the reference's schema for this response
        assert resp == base64.b64decode(g["response"]["response_b64"])


def test_disk_provider_mlp_bundle(tmp_path):
    _torch()
    rng = np.random.default_rng(4)
    dims = [40, 56, 24]
    ws = [(rng.standard_normal((dims[i], dims[i + 1])) / 6).astype(np.float32) for i in range(2)]
    bs = [rng.standard_normal(dims[i + 1]).astype(np.float32) for i in range(2)]
    t.modelformat.write_mlp_bundle(os.path.join(str(tmp_path), "tenant", "000000042"), ws, bs)
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp_path),
           "gpu.devices": [0], "gpu.arenaBytes": 1 << 20}
    with t.Server(cfg) as srv:
        x = rng.standard_normal((5, 40)).astype(np.float32)
        y = srv.predict("tenant", "42", x)
        man, blob = models.load_bundle(os.path.join(str(tmp_path), "tenant", "000000042"))
        assert _close(y, models.forward(man, blob, x, np.float64)) <= TOL


def test_full_size_tenant_model_matches_oracle():
    """BASELINE configs[2] model (9216->9216->9216->9216, 1 019 326 464 B of weights): the oracle's
    numpy fp32/fp64 forward finishes in seconds, so compare directly at full size."""
    _torch()
    dims = [9216, 9216, 9216, 9216]
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": dims, "modelProvider.synthetic.count": 8,
           "gpu.devices": [0], "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 2, "modelCache.size": 4 << 30}
    rng = np.random.default_rng(9)
    x = rng.standard_normal((8, dims[0])).astype(np.float32)
    with t.Server(cfg) as srv:
        y = srv.predict("m3", "1", x)
        y1 = srv.predict("m3", "1", x[:1])
        st = srv.stats()
    assert st["h2d_weight_bytes"] == 1019326464  # 254 831 616 fp32 params (BASELINE.md)
    ref = _oracle_mlp(3, x, dims, np.float64)
    assert y.shape == (8, 9216) and _close(y, ref) <= TOL
    assert _close(y1, ref[:1]) <= TOL


@pytest.mark.parametrize("rows", [219, 70])
def test_full_size_tenant_model_device_batches_match_oracle(rows):
    """bench.py's value path: one model group of a step in one tfsc_predict_device call. With Zipf(1) over 60 models and
    1024 requests the hottest group is ~219 rows (tensor-core passes 64, 64, 64, 27 per layer, programmatic dependent launch
    between them); 70 rows end in a tensor-core pass followed by a cluster-kernel pass."""
    torch = _torch()
    dims = [9216, 9216, 9216, 9216]
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": dims, "modelProvider.synthetic.count": 8,
           "gpu.devices": [0], "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 2, "modelCache.size": 4 << 30}
    x = np.random.default_rng(rows).standard_normal((rows, dims[0])).astype(np.float32)
    stream = torch.cuda.Stream()
    with t.Server(cfg) as srv:
        srv.ensure(0, "m5", 1)
        xd = torch.from_numpy(x).cuda()
        outs = []
        for _ in range(2):
            yd = torch.full((rows, dims[-1]), float("nan"), device="cuda")
            torch.cuda.synchronize()
            srv.predict_device(0, "m5", 1, xd.data_ptr(), rows, yd.data_ptr(), stream.cuda_stream)
            stream.synchronize()
            outs.append(yd.cpu().numpy())
    assert np.array_equal(outs[0], outs[1])
    ref = _oracle_mlp(5, x, dims, np.float64)
    assert outs[0].shape == ref.shape and not np.isnan(outs[0]).any() and _close(outs[0], ref) <= TOL
