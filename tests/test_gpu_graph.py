"""-m gpu: X4 -- conv-net building blocks and the graph executor (ResNet-50 bundle) vs the oracle
(torch-CPU fp64 functional conv2d / max_pool2d on the same blob).  Tolerance 1e-4 relative to max(1,|ref|)."""
import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

pytestmark = pytest.mark.gpu
TOL = 1e-4
lib = t._lib.lib


def _torch():
    import torch
    assert torch.cuda.is_available()
    return torch


def _err(got, ref):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


@pytest.mark.parametrize("m,n,k,lda", [(1, 8, 4, 4), (49, 64, 147, 148), (200, 100, 37, 37), (128, 64, 16, 16), (300, 1000, 2048, 2048),
                                        (3136, 256, 64, 64), (130, 66, 18, 20)])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_k_gemm(m, n, k, lda, act):
    torch = _torch()
    rng = np.random.default_rng(m * 7 + n + k + act)
    a = rng.standard_normal((m, lda)).astype(np.float32)
    b = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float32)
    ad, bd, biasd, rd = (torch.from_numpy(v).cuda() for v in (a, b, bias, r))
    cd = torch.full((m, n), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_gemm(ad.data_ptr(), bd.data_ptr(), biasd.data_ptr(), rd.data_ptr(), cd.data_ptr(), m, n, k, lda, act, None))
    torch.cuda.synchronize()
    ref = a[:, :k].astype(np.float64) @ b.astype(np.float64) + bias + r
    if act == 1:
        ref = np.maximum(ref, 0)
    elif act == 2:
        ref = torch.nn.functional.gelu(torch.from_numpy(ref)).numpy()
    assert _err(cd.cpu().numpy(), ref) <= TOL


@pytest.mark.parametrize("m,n,k,lda", [(128, 128, 32, 32), (64, 64, 64, 64), (300, 256, 96, 96), (3136, 64, 147, 148), (1024, 768, 768, 768),
                                        (1000, 3072, 768, 768), (512, 768, 3072, 3072), (6272, 128, 1152, 1152), (130, 96, 40, 44)])
@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_k_gemm_tc_matches_oracle(m, n, k, lda, act):
    """wgmma 3xTF32 GEMM (gemm_tc.cu) vs fp64; bias + residual + activation fused in the epilogue."""
    torch = _torch()
    rng = np.random.default_rng(m + n + k + act)
    a = rng.standard_normal((m, lda)).astype(np.float32)
    b = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float32)
    ad, bd, biasd, rd = (torch.from_numpy(v).cuda() for v in (a, b, bias, r))
    cd = torch.full((m, n), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_gemm_tc(ad.data_ptr(), bd.data_ptr(), biasd.data_ptr(), rd.data_ptr(), cd.data_ptr(), m, n, k, lda, act, None), "gemm_tc")
    torch.cuda.synchronize()
    ref = a[:, :k].astype(np.float64) @ b.astype(np.float64) + bias + r
    if act == 1:
        ref = np.maximum(ref, 0)
    elif act == 2:
        ref = torch.nn.functional.gelu(torch.from_numpy(ref)).numpy()
    elif act == 3:
        ref = np.tanh(ref)
    got = cd.cpu().numpy()
    assert not np.isnan(got).any() and _err(got, ref) <= TOL


def test_k_gemm_tc_rejects_unsupported_shapes():
    torch = _torch()
    x = torch.zeros(64, 64, device="cuda")
    assert lib.tfsc_k_gemm_tc(x.data_ptr(), x.data_ptr(), None, None, x.data_ptr(), 32, 64, 64, 64, 0, None) == t._lib.E_INVALID   # M < 64
    assert lib.tfsc_k_gemm_tc(x.data_ptr(), x.data_ptr(), None, None, x.data_ptr(), 64, 40, 64, 64, 0, None) == t._lib.E_INVALID   # N % 32


@pytest.mark.parametrize("h,c,kh,stride,pad,cout", [(16, 3, 7, 2, 3, 8), (14, 16, 3, 1, 1, 24), (14, 16, 3, 2, 1, 24), (9, 5, 1, 2, 0, 7)])
def test_conv_as_im2col_gemm_matches_torch(h, c, kh, stride, pad, cout):
    torch = _torch()
    rng = np.random.default_rng(h + c + kh)
    bsz = 3
    x = rng.standard_normal((bsz, h, h, c)).astype(np.float32)
    w = (rng.standard_normal((kh, kh, c, cout)) / np.sqrt(kh * kh * c)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    oh = (h + 2 * pad - kh) // stride + 1
    kk = kh * kh * c
    ldc = (kk + 3) // 4 * 4
    xd, wd, bd = (torch.from_numpy(v).cuda() for v in (x, w, b))
    col = torch.full((bsz * oh * oh, ldc), float("nan"), device="cuda")
    y = torch.empty(bsz * oh * oh, cout, device="cuda")
    t._lib.check(lib.tfsc_k_im2col(xd.data_ptr(), col.data_ptr(), bsz, h, h, c, kh, kh, stride, pad, ldc, None))
    t._lib.check(lib.tfsc_k_gemm(col.data_ptr(), wd.data_ptr(), bd.data_ptr(), None, y.data_ptr(), bsz * oh * oh, cout, kk, ldc, 1, None))
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.conv2d(torch.from_numpy(x).double().permute(0, 3, 1, 2),
                                                torch.from_numpy(w).double().permute(3, 2, 0, 1),
                                                torch.from_numpy(b).double(), stride=stride, padding=pad)).permute(0, 2, 3, 1).numpy()
    assert _err(y.cpu().numpy().reshape(bsz, oh, oh, cout), ref) <= TOL


@pytest.mark.parametrize("h,c,kh,stride,pad,cout,bsz", [(14, 64, 3, 1, 1, 64, 3), (14, 32, 3, 2, 1, 96, 5), (9, 64, 1, 2, 0, 128, 4),
                                                         (28, 128, 3, 1, 1, 128, 2), (7, 512, 3, 1, 1, 512, 8), (56, 64, 3, 1, 1, 64, 1),
                                                         (12, 96, 5, 1, 2, 160, 2), (15, 64, 3, 2, 1, 64, 3)])
@pytest.mark.parametrize("act,with_res", [(1, True), (0, False)])
def test_implicit_gemm_conv_matches_torch(h, c, kh, stride, pad, cout, bsz, act, with_res):
    """X4: conv as implicit GEMM -- the A tiles come from TMA im2col tensor maps over the NHWC activations (padding = TMA
    zero fill, stride = traversal stride), wgmma 3xTF32, bias / residual / ReLU in the epilogue. vs torch conv2d fp64."""
    torch = _torch()
    rng = np.random.default_rng(h * 31 + c + kh + stride)
    x = rng.standard_normal((bsz, h, h, c)).astype(np.float32)
    w = (rng.standard_normal((kh, kh, c, cout)) / np.sqrt(kh * kh * c)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    oh = (h + 2 * pad - kh) // stride + 1
    r = rng.standard_normal((bsz, oh, oh, cout)).astype(np.float32)
    xd, wd, bd, rd = (torch.from_numpy(v).cuda() for v in (x, w, b, r))
    y = torch.full((bsz, oh, oh, cout), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_conv_tc(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), rd.data_ptr() if with_res else None, y.data_ptr(),
                                    bsz, h, h, c, kh, kh, stride, pad, cout, act, None), "conv_tc")
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double().permute(0, 3, 1, 2), torch.from_numpy(w).double().permute(3, 2, 0, 1),
                                     torch.from_numpy(b).double(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    if with_res:
        ref = ref + torch.from_numpy(r).double()
    if act == 1:
        ref = torch.relu(ref)
    got = y.cpu().numpy()
    assert not np.isnan(got).any() and _err(got, ref.numpy()) <= TOL


def test_pools_match_torch():
    torch = _torch()
    x = torch.randn(2, 13, 13, 10)
    xd = x.cuda()
    y = torch.empty(2, 7, 7, 10, device="cuda")
    t._lib.check(lib.tfsc_k_maxpool(xd.data_ptr(), y.data_ptr(), 2, 13, 13, 10, 3, 3, 2, 1, None))
    ref = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(y.cpu(), ref)
    a = torch.empty(2, 10, device="cuda")
    t._lib.check(lib.tfsc_k_avgpool(xd.data_ptr(), a.data_ptr(), 2, 169, 10, None))
    assert torch.allclose(a.cpu(), x.mean(dim=(1, 2)), atol=1e-6)


def _server(man, count=8, arena=1 << 30, **kw):
    cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.template": "manifest",
           "modelProvider.synthetic.manifest": man, "modelProvider.synthetic.count": count, "gpu.devices": [0],
           "gpu.arenaBytes": arena, "serving.maxConcurrentModels": 4, "modelCache.size": 4 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return t.Server(cfg)


def test_small_resnet_through_server_matches_oracle():
    _torch()
    man = t.modelformat.resnet50_manifest(image=64, classes=10)
    oman = models.graph_manifest([64, 64, 3], models.resnet50_ops(64, 10))
    rng = np.random.default_rng(0)
    with _server(man, arena=256 << 20) as srv:
        for j, bsz in [(0, 1), (3, 5), (0, 2)]:
            x = rng.random((bsz, 64, 64, 3)).astype(np.float32)
            y = srv.predict(f"m{j}", "1", x)
            ref = models.graph_forward(oman, models.synth_graph_blob(oman, 1000 + j), x, np.float64)
            assert y.shape == (bsz, 10) and _err(y, ref) <= TOL
        st = srv.stats()
        assert st["cache_misses_total"] == 2 and st["cache_hits_total"] == 1


def test_resnet50_full_size_matches_oracle_and_rest():
    """BASELINE configs[1] model: ResNet-50, 224x224x3, 25.5 M parameters (102 MB)."""
    _torch()
    import json
    man = t.modelformat.resnet50_manifest()
    assert man["weights_bytes"] == models.graph_manifest([224, 224, 3], models.resnet50_ops())["weights_bytes"] == 102121984
    oman = models.graph_manifest([224, 224, 3], models.resnet50_ops())
    x = np.random.default_rng(1).random((2, 224, 224, 3)).astype(np.float32)
    with _server(man) as srv:
        y = srv.predict("m1", "1", x)
        st = srv.stats()
    ref = models.graph_forward(oman, models.synth_graph_blob(oman, 1001), x, np.float64)
    assert y.shape == (2, 1000) and _err(y, ref) <= TOL
    assert st["h2d_weight_bytes"] == 102121984


# ---- X5: transformer ops / BERT bundle -------------------------------------------------------------------
def test_small_bert_through_server_grpc_and_rest_matches_oracle():
    _torch()
    import json
    from oracle import wire
    args = dict(seq=16, hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=32, labels=3)
    man = t.modelformat.bert_manifest(**args)
    oman = models.graph_manifest([16], models.bert_ops(**args), 4, ("input_ids", "logits"), "int32")
    rng = np.random.default_rng(0)
    with _server(man, arena=64 << 20) as srv:
        for j, bsz in [(1, 1), (2, 4)]:
            ids = rng.integers(1, 100, (bsz, 16)).astype(np.int32)
            ids[-1, 9:] = 0                                   # [PAD] tail -> masked keys
            y = srv.predict(f"m{j}", "1", ids)
            ref = models.graph_forward(oman, models.synth_graph_blob(oman, 1000 + j), ids, np.float64)
            assert y.shape == (bsz, 3) and _err(y, ref) <= TOL
        # float ids are a signature error; gRPC int_val and tensor_content both work; REST resolves ints from JSON
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("m1", "1", ids.astype(np.float32))
        assert e.value.code == t._lib.E_INVALID
        ref = models.graph_forward(oman, models.synth_graph_blob(oman, 1001), ids, np.float64)
        for use_content in (True, False):
            req = wire.encode_predict_request("m1", 1, {"input_ids": ids}, use_content=use_content)
            _spec, outs = wire.decode_predict_response(srv.grpc_predict(req))
            assert _err(outs["logits"], ref) <= TOL
        st, body = srv.rest_handle("POST", "/v1/models/m1/versions/1:predict", json.dumps({"instances": ids.tolist()}).encode())
        assert st == 200 and _err(np.array(json.loads(body)["predictions"]), ref) <= TOL


def test_bert_base_full_size_matches_oracle():
    """BASELINE configs[3] model: BERT-base (L12/H768/A12, vocab 30522, 109.5 M parameters = 438 MB), batch 8 x 128."""
    _torch()
    man = t.modelformat.bert_manifest()
    oman = models.graph_manifest([128], models.bert_ops(), 4, ("input_ids", "logits"), "int32")
    assert man["weights_bytes"] == oman["weights_bytes"] == 437935360
    rng = np.random.default_rng(2)
    ids = rng.integers(1, 30522, (8, 128)).astype(np.int32)
    ids[3, 100:] = 0
    ids[7, 5:] = 0
    with _server(man, arena=1 << 30, count=4) as srv:
        y = srv.predict("m2", "1", ids)
    ref = models.graph_forward(oman, models.synth_graph_blob(oman, 1002), ids, np.float64)
    assert y.shape == (8, 2) and _err(y, ref) <= TOL


@pytest.mark.parametrize("splits", ["2", "8"])
def test_cluster_split_k_paths_of_the_graph_gemm(splits):
    """The cluster split-K fold (DSMEM) is only chosen for small tile grids; force it for every GEMM / implicit conv case of
    this file (TFSC_GEMM_SPLITK is read once per process, hence the subprocess)."""
    import os
    import subprocess
    import sys
    if os.environ.get("TFSC_GEMM_SPLITK"):
        pytest.skip("already inside the forced-split run")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, TFSC_GEMM_SPLITK=splits)
    run = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-k",
                          "gemm_tc_matches or implicit_gemm or small_resnet or small_bert"], capture_output=True, text=True, timeout=900,
                         env=env, cwd=root)
    assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]
