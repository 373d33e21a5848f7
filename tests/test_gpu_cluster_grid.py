"""-m gpu: the one-wave grid of the <= 8-row cluster-pair kernel (strip width sized from the co-resident cluster count,
clusters looping over several strips when N needs more) against the fp64 oracle (tolerance 1e-4, north_star)."""
import ctypes as C

import numpy as np
import pytest

import tfservingcache_b200 as t

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _data(rows, k, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    return x, w, b


def _run(x, w, b, relu, fn, variant=None):
    """Two back-to-back calls (arrival counters self-reset); returns y and the kernel launches of the second call."""
    import torch
    assert torch.cuda.is_available()
    lib = t._lib.lib
    rows, k = x.shape
    n = w.shape[1]
    wsb = lib.tfsc_k_dense_workspace(rows, k, n)
    ws = torch.zeros(wsb // 4 + 64, device="cuda")
    xd, wd, bd = (torch.from_numpy(a).cuda() for a in (x, w, b))
    yd = torch.empty(rows, n, device="cuda")
    launches = 0
    for _ in range(2):
        yd.fill_(float("nan"))
        before = lib.tfsc_kernel_launches()
        args = (xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), yd.data_ptr(), rows, k, n, 1 if relu else 0, ws.data_ptr(), wsb, None)
        if variant is None:
            t._lib.check(getattr(lib, fn)(*args), fn)
        else:
            t._lib.check(lib.tfsc_k_dense_variant(variant, *args), fn)
        torch.cuda.synchronize()
        launches = lib.tfsc_kernel_launches() - before
    return yd.cpu().numpy(), launches


def _ref(x, w, b, relu):
    ref = x.astype(np.float64) @ w.astype(np.float64) + b
    return np.maximum(ref, 0) if relu else ref


def _err(got, ref):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


def test_cluster_grid_is_one_wave():
    lib = t._lib.lib
    for rows in (1, 2, 4, 8):
        for n in (1000, 4100, 9216, 9232, 20000):
            a, s = C.c_int(), C.c_int()
            t._lib.check(lib.tfsc_k_dense_cluster_grid(rows, n, C.byref(a), C.byref(s)))
            assert a.value >= 1
            assert s.value % 16 == 0 and 16 <= s.value <= 144
            # a strip per cluster where the widest strip allows it
            assert (n + s.value - 1) // s.value <= a.value or s.value == 144


@pytest.mark.parametrize("rows", [1, 3, 8])
@pytest.mark.parametrize("k,n", [(512, 1000), (1000, 4100), (9216, 9216 + 16), (256, 20000)])
def test_cluster_kernel_uneven_strips_matches_oracle(rows, k, n):
    x, w, b = _data(rows, k, n, rows * 7 + k + n)
    for relu in (False, True):
        got, launches = _run(x, w, b, relu, "tfsc_k_dense", variant=5)
        assert launches == 1
        assert not np.isnan(got).any()
        assert _err(got, _ref(x, w, b, relu)) <= TOL
