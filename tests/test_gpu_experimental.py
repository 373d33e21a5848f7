"""-m gpu: the dense-kernel variants and their programmatic-dependent-launch switch, each in its own process (TFSC_PDL /
TFSC_DENSE_VARIANT are read once per process). The cluster-pair kernel + PDL is the default for <= 8 rows; the other
variants stay selectable for A/B runs, so they stay under test."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PDL_SCRIPT = r"""
import os
import numpy as np, torch
import tfservingcache_b200 as t
lib = t._lib.lib
VARIANTS = tuple(int(v) for v in os.environ.get('TFSC_TEST_VARIANTS', '1,2,4').split(','))
rng = np.random.default_rng(0)
worst = 0.0
for (K, N) in [(64, 8), (100, 520), (128, 64), (132, 260), (780, 1032), (2048 + 64, 512), (4096, 4096), (9216, 9216)]:
    for rows in (1, 3, 8):
        x = torch.randn(rows, K, device="cuda"); w = torch.randn(K, N, device="cuda") / K ** 0.5; b = torch.randn(N, device="cuda")
        ws_bytes = lib.tfsc_k_dense_workspace(rows, K, N); ws = torch.zeros(ws_bytes // 4 + 64, device="cuda")
        ref = (x.double() @ w.double() + b.double()).clamp_min(0)
        for variant in VARIANTS:
            y = torch.full((rows, N), float("nan"), device="cuda")
            # back-to-back launches on one stream: with TFSC_PDL=1 each pass may start under the tail of the previous one
            for _ in range(6):
                t._lib.check(lib.tfsc_k_dense_variant(variant, x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), rows, K, N, 1,
                                                      ws.data_ptr(), ws_bytes, None))
            torch.cuda.synchronize()
            worst = max(worst, (y.double() - ref).abs().max().item())
# a 3-layer MLP through the server: layer l+1 reads layer l's output, the dependency PDL must keep
from oracle import models
dims = [512, 1024, 1024, 64]
cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": dims, "modelProvider.synthetic.count": 4,
       "gpu.devices": [0], "gpu.arenaBytes": 64 << 20, "modelCache.size": 1 << 30}
with t.Server(cfg) as srv:
    for j in range(4):
        x = rng.standard_normal((5, dims[0])).astype(np.float32)
        for _ in range(3):
            y = srv.predict(f"m{j}", "1", x)
        man, blob = models.synth_mlp_blob(dims, seed=1000 + j)
        worst = max(worst, float(np.max(np.abs(y - models.forward(man, blob, x, np.float64)))))
print("WORST", worst)
assert worst < 2e-4, worst
"""


@pytest.mark.parametrize("variant_env", ["0", "2", "4"])
def test_programmatic_dependent_launch_keeps_results(variant_env):
    env = dict(os.environ, TFSC_PDL="1", TFSC_DENSE_VARIANT=variant_env, PYTHONPATH=ROOT)
    run = subprocess.run([sys.executable, "-c", PDL_SCRIPT], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]
    assert "WORST" in run.stdout


@pytest.mark.parametrize("pdl", ["0", "1"])
def test_cluster_pair_dense_kernel(pdl):
    """tfsc_k_dense_variant 5 (csrc/dense_cluster.cu): 2-CTA clusters, K halves meet in distributed shared memory."""
    env = dict(os.environ, TFSC_PDL=pdl, TFSC_DENSE_VARIANT="5", TFSC_TEST_VARIANTS="5", PYTHONPATH=ROOT)
    run = subprocess.run([sys.executable, "-c", PDL_SCRIPT], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]
    assert "WORST" in run.stdout


BATCH_SCRIPT = r"""
import sys
import numpy as np, torch
import tfservingcache_b200 as t
lib = t._lib.lib
out = {}
rng = np.random.default_rng(0)
for (K, N) in [(1024, 520), (4096, 4096), (9216, 9216)]:
    w = torch.from_numpy((rng.standard_normal((K, N)) / K ** 0.5).astype(np.float32)).cuda()
    b = torch.from_numpy(rng.standard_normal(N).astype(np.float32)).cuda()
    for rows in (65, 72, 73, 128, 219):
        x = torch.from_numpy(rng.standard_normal((rows, K)).astype(np.float32)).cuda()
        ws_bytes = lib.tfsc_k_dense_workspace(rows, K, N); ws = torch.zeros(ws_bytes // 4 + 64, device="cuda")
        y = torch.full((rows, N), float("nan"), device="cuda")
        for _ in range(3):   # back to back on one stream and one workspace
            t._lib.check(lib.tfsc_k_dense(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), rows, K, N, 1, ws.data_ptr(),
                                          ws_bytes, None))
        torch.cuda.synchronize()
        out[f"k{K}_n{N}_r{rows}"] = y.cpu().numpy()
dims = [9216, 9216, 9216, 9216]
cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": dims, "modelProvider.synthetic.count": 2,
       "gpu.devices": [0], "gpu.arenaBytes": 3 << 30, "modelCache.size": 4 << 30}
stream = torch.cuda.Stream()
with t.Server(cfg) as srv:
    srv.ensure(0, "m1", 1)
    x = torch.from_numpy(rng.standard_normal((219, dims[0])).astype(np.float32)).cuda()
    ys = {r: torch.full((r, dims[-1]), float("nan"), device="cuda") for r in (219, 70)}
    for r, y in ys.items():   # the two groups back to back on one stream, as a bench step issues them
        srv.predict_device(0, "m1", 1, x.data_ptr(), r, y.data_ptr(), stream.cuda_stream)
    stream.synchronize()
    for r, y in ys.items():
        out[f"model_r{r}"] = y.cpu().numpy()
np.savez(sys.argv[1], **out)
print("SAVED", len(out))
"""


def test_programmatic_dependent_launch_is_bit_identical_above_64_rows(tmp_path):
    """Batches above 64 rows run as several dense passes back to back, each allowed to start under the previous one's
    tail (PDL, on by default). PDL does not change the summation order, so TFSC_PDL=0 must give the same bits: a
    difference means a pass read x, the workspace or its counters before the previous pass was done with them."""
    import numpy as np
    res = {}
    for pdl in ("default", "0"):
        env = dict(os.environ, PYTHONPATH=ROOT)
        env.pop("TFSC_PDL", None)
        env.pop("TFSC_DENSE_VARIANT", None)
        if pdl == "0":
            env["TFSC_PDL"] = "0"
        path = str(tmp_path / f"pdl_{pdl}.npz")
        run = subprocess.run([sys.executable, "-c", BATCH_SCRIPT, path], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
        assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]
        res[pdl] = dict(np.load(path))
    assert sorted(res["default"]) == sorted(res["0"])
    for key, y in res["default"].items():
        assert not np.isnan(y).any(), key
        assert np.array_equal(y, res["0"][key]), key
