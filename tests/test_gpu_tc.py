"""-m gpu: X3, the wgmma 3xTF32 dense path (tfsc_k_dense_tc) vs the fp64 oracle; tolerance
1e-4 (north_star) although the split keeps it near 1e-5."""
import ctypes as C

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _run(x, w, b, relu, fn="tfsc_k_dense_tc"):
    import torch
    assert torch.cuda.is_available()
    lib = t._lib.lib
    f = getattr(lib, fn)
    f.restype = C.c_int
    f.argtypes = [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p, C.c_size_t, C.c_void_p]
    rows, k = x.shape
    n = w.shape[1]
    wsb = lib.tfsc_k_dense_workspace(rows, k, n)
    ws = torch.zeros(wsb // 4 + 64, device="cuda")
    xd, wd, bd = (torch.from_numpy(a).cuda() for a in (x, w, b))
    yd = torch.empty(rows, n, device="cuda")
    for _ in range(2):  # arrival counters self-reset
        yd.fill_(float("nan"))
        t._lib.check(f(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), yd.data_ptr(), rows, k, n, 1 if relu else 0,
                       ws.data_ptr(), wsb, None), fn)
        torch.cuda.synchronize()
    return yd.cpu().numpy()


def _err(got, ref):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


@pytest.mark.parametrize("rows", [1, 9, 16, 17, 31, 32, 33, 48, 63, 64])
@pytest.mark.parametrize("k,n", [(32, 32), (128, 256), (36, 64), (1000, 512), (2048, 800), (9216, 1024), (4100, 9216)])
def test_dense_tc_matches_oracle(rows, k, n):
    rng = np.random.default_rng(rows * 1009 + k + n)
    x = rng.standard_normal((rows, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    for relu in (False, True):
        got = _run(x, w, b, relu)
        ref = x.astype(np.float64) @ w.astype(np.float64) + b
        if relu:
            ref = np.maximum(ref, 0)
        assert not np.isnan(got).any()
        assert _err(got, ref) <= TOL


def test_dense_tc_beats_plain_tf32_accuracy_and_is_deterministic():
    rng = np.random.default_rng(3)
    k = n = 9216
    x = rng.standard_normal((64, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = np.zeros(n, np.float32)
    y1, y2 = _run(x, w, b, False), _run(x, w, b, False)
    assert np.array_equal(y1, y2)
    ref = x.astype(np.float64) @ w.astype(np.float64)
    e = _err(y1, ref)
    assert e <= 5e-5, e      # single-pass TF32 would sit near 5e-4 at K=9216
    # dispatcher: > 8 rows go to the tensor-core path, results agree with the SIMT path within tolerance
    y3 = _run(x, w, b, False, fn="tfsc_k_dense")
    assert _err(y3, ref) <= TOL and np.max(np.abs(y3 - y1)) <= 1e-4


def test_dense_tc_rejects_unsupported_shapes():
    import torch
    lib = t._lib.lib
    lib.tfsc_k_dense_tc.restype = C.c_int
    lib.tfsc_k_dense_tc.argtypes = [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p, C.c_size_t, C.c_void_p]
    x = torch.zeros(4, 64, device="cuda")
    w = torch.zeros(64, 40, device="cuda")
    assert lib.tfsc_k_dense_tc(x.data_ptr(), w.data_ptr(), w.data_ptr(), w.data_ptr(), 4, 64, 40, 0, None, 0, None) == t._lib.E_INVALID


def test_full_size_tenant_model_64_rows_through_server():
    """3 chained tensor-core layers (configs[2] model) against the fp64 oracle."""
    import torch
    assert torch.cuda.is_available()
    dims = [9216, 9216, 9216, 9216]
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": dims, "modelProvider.synthetic.count": 8,
           "gpu.devices": [0], "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 2, "modelCache.size": 4 << 30,
           "gpu.maxBatch": 64}
    rng = np.random.default_rng(10)
    x = rng.standard_normal((50, dims[0])).astype(np.float32)
    with t.Server(cfg) as srv:
        y = srv.predict("m5", "1", x)
    man, blob = models.synth_mlp_blob(dims, seed=1005)
    ref = models.forward(man, blob, x, np.float64)
    assert y.shape == (50, 9216) and _err(y, ref) <= TOL
