"""Numeric parity pinned on INDEPENDENT implementations (VERDICT r1 'next' #1): torchvision's ResNet-50 and transformers'
BERT-base define the two model families of BASELINE configs[1] / configs[3]; their own fp64 forward is the reference,
their parameters are exported into the bundle format (tests/torch_export.py), and both the CPU oracle (here, not gpu) and
the GPU executor (-m gpu) must reproduce it within north_star's 1e-4. Committed numbers: tests/golden/model_torch_golden.json
(tests/golden/make_model_golden.py), required bit-for-bit-ish (1e-9) when the library versions match the recorded ones."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_model_golden as mg  # noqa: E402
import torch_export as te  # noqa: E402
import tfservingcache_b200 as t  # noqa: E402
from oracle import models  # noqa: E402

TOL = 1e-4


def _err(got, ref):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


def _versions_match(g):
    import torch
    import torchvision
    import transformers
    have = {"torch": torch.__version__, "torchvision": torchvision.__version__, "transformers": transformers.__version__}
    return have == g["versions"]


def _case(name, golden):
    g = golden("model_torch_golden.json")
    c = mg.CASES[name]
    m, x, ref = (mg.resnet_case if name.startswith("resnet") else mg.bert_case)(c)
    if _versions_match(g):   # the committed fixture: same seeds, same libraries -> same numbers
        want = np.array(g["cases"][name]["logits"]).reshape(g["cases"][name]["shape"])
        assert np.max(np.abs(ref - want)) <= 1e-9
    return c, m, x, ref


def _manifest(name, c):
    if name.startswith("resnet"):
        return t.modelformat.resnet50_manifest(image=c.get("image", 224), classes=c.get("classes", 1000), blocks=tuple(c.get("blocks", (3, 4, 6, 3))))
    kw = {k: c[k] for k in ("seq", "hidden", "layers", "heads", "inter", "vocab", "max_pos", "labels") if k in c}
    return t.modelformat.bert_manifest(**kw)


def _oracle_manifest(name, c):
    """the oracle's OWN restatement of the topology (oracle/models.py), not the product manifest"""
    if name == "resnet50":
        return models.graph_manifest([224, 224, 3], models.resnet50_ops())
    if name.startswith("bert"):
        kw = {k: c[k] for k in ("seq", "hidden", "layers", "heads", "inter", "vocab", "max_pos", "labels") if k in c}
        return models.graph_manifest([kw.get("seq", 128)], models.bert_ops(**kw), 4, ("input_ids", "logits"), "int32")
    return None   # resnet_small uses a block layout the oracle's fixed ResNet-50 restatement does not produce


@pytest.mark.parametrize("name", ["resnet50", "resnet_small", "bert_base", "bert_small"])
def test_oracle_matches_torchvision_and_transformers(name, golden):
    c, m, x, ref = _case(name, golden)
    man = _manifest(name, c)
    blob = (te.export_resnet if name.startswith("resnet") else te.export_bert)(m, man)
    oman = _oracle_manifest(name, c)
    if oman is not None:   # offsets of the two independent manifests must agree before one blob can serve both
        assert oman["weights_bytes"] == man["weights_bytes"]
        assert [(o["op"], o.get("w_offset")) for o in oman["ops"]] == [(o["op"], o.get("w_offset")) for o in man["ops"]]
    y = models.graph_forward(oman or man, blob, x, np.float64)
    assert y.shape == ref.shape and _err(y, ref) <= 1e-6     # fp64 forward; only the fp32 rounding of the folded weights differs
    y32 = models.graph_forward(oman or man, blob, x, np.float32)
    assert _err(y32, ref) <= TOL


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["resnet_small", "resnet50", "bert_small", "bert_base"])
def test_executor_matches_torchvision_and_transformers(name, golden, tmp_path):
    """The GPU graph executor on bundles exported from the defining libraries, served from disk through the public
    predict path (disk provider -> pinned host -> HBM arena -> kernels)."""
    import torch
    assert torch.cuda.is_available()
    c, m, x, ref = _case(name, golden)
    man = _manifest(name, c)
    blob = (te.export_resnet if name.startswith("resnet") else te.export_bert)(m, man)
    t.modelformat.write_graph_bundle(str(tmp_path / name / "1"), man, blob)
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp_path), "gpu.devices": [0],
           "gpu.arenaBytes": 1 << 30, "serving.maxConcurrentModels": 2, "modelCache.size": 2 << 30, "gpu.maxBatch": 8}
    with t.Server(cfg) as srv:
        y = srv.predict(name, "1", x)
        assert y.shape == ref.shape and _err(y, ref) <= TOL
        if x.shape[0] > 1:   # one row at a time takes different kernels (batch-1 GEMM shapes): same answers
            y1 = srv.predict(name, "1", x[:1])
            assert _err(y1, ref[:1]) <= TOL
        assert srv.stats()["kernel_launches"] > 0
