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
