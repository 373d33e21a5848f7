"""-m gpu: MobileNetV2 and EfficientNet. The depthwise_conv and channel_scale kernels against fp64 / fp32 numpy (batch and
path bit identity, refusals at the limits), relu6 / silu / sigmoid in every GEMM epilogue, full-size MobileNetV2 and
EfficientNet-B0 through the server against torchvision fp64, the front-ends, launch counts, programmatic-dependent-launch
bit identity and the forward hop between two ranks."""
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
import convnet_export as ce  # noqa: E402
import convnet_ref as cr  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
E = t._lib.E_INVALID
K = 5
ALL = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"}, {"name": "classes", "kind": "classes"},
       {"name": "top_k_classes", "kind": "top_k_classes", "k": K}, {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": K}]
NAMES = sorted(o["name"] for o in ALL)
ACTS = [0, 1, 4, 5, 6]


def _torch():
    import torch
    assert torch.cuda.is_available()
    return torch


def _ptr(x):
    return None if x is None else x.data_ptr()


def _err(got, ref):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


# ------------------------------------------------------------------------------------- depthwise_conv ----
def _dw(torch, xd, wd, bd, B, H, C, k, s, p, act, x_off=0, y_off=0):
    """launch on x / y shifted by x_off / y_off floats (a misaligned shift selects the scalar path); returns y [B, OH, OW, C]"""
    oh = (H + 2 * p - k) // s + 1
    n = B * oh * oh * C
    yb = torch.full((n + 4,), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_depthwise_conv(xd.data_ptr() + 4 * x_off, _ptr(wd), _ptr(bd), yb.data_ptr() + 4 * y_off, B, H, H, C, k, k, s, p,
                                           act, None), "depthwise_conv")
    torch.cuda.synchronize()
    return yb[y_off:y_off + n].cpu().numpy().reshape(B, oh, oh, C)


def _cases(k, s):
    """(pad, H, C, batch) over pad 0..k/2, H in {1, 7, 14, 56, 112, 113}, C in {1, 3, 4, 5, 32, 144, 1152}: the batch is the
    largest of 64 / 8 / 1 that keeps the case within 2^22 input values"""
    for p in range(k // 2 + 1):
        for H in (1, 7, 14, 56, 112, 113):
            if H + 2 * p < k:
                continue
            for C in (1, 3, 4, 5, 32, 144, 1152):
                if H * H * C > 113 * 113 * 32:
                    continue
                yield p, H, C, next(b for b in (64, 8, 1) if b == 1 or b * H * H * C <= 1 << 22)


@pytest.mark.parametrize("k", [1, 3, 5, 7])
@pytest.mark.parametrize("s", [1, 2])
def test_depthwise_conv_matches_fp64(k, s):
    torch = _torch()
    rng = np.random.default_rng(k * 10 + s)
    for n, (p, H, C, B) in enumerate(_cases(k, s)):
        act = ACTS[n % len(ACTS)]
        x = rng.standard_normal((B, H, H, C), dtype=np.float32)
        w = (rng.standard_normal((k, k, C)) / k).astype(np.float32)
        b = rng.standard_normal(C).astype(np.float32)
        xb = torch.zeros(x.size + 4, device="cuda")
        xb[:x.size] = torch.from_numpy(x.ravel()).cuda()
        wd, bd = torch.from_numpy(w).cuda(), torch.from_numpy(b).cuda()
        y = _dw(torch, xb, wd, bd, B, H, C, k, s, p, act)
        ref = cr.depthwise_conv(x, w, b, s, p, cr.ACTS[act])
        assert _err(y, ref) <= 1e-5, (p, H, C, B, act)
        # a row's bits do not depend on the batch
        for r in {0, B - 1}:
            one = _dw(torch, xb, wd, bd, 1, H, C, k, s, p, act, x_off=r * H * H * C)
            assert one.tobytes() == y[r:r + 1].tobytes(), (p, H, C, B, act, r)
        # nor on the path: a one-float shift of x and y makes them misaligned, which selects the scalar kernel
        if C % 4 == 0 and B * H * H * C <= 1 << 20:
            xs = torch.zeros(x.size + 4, device="cuda")
            xs[1:1 + x.size] = xb[:x.size]
            assert _dw(torch, xs, wd, bd, B, H, C, k, s, p, act, x_off=1, y_off=1).tobytes() == y.tobytes(), (p, H, C, B, act)


def test_depthwise_conv_refusals():
    torch = _torch()
    x = torch.zeros(64 * 64 * 8, device="cuda")
    ok = (x, x, x, x, 2, 8, 8, 8, 3, 3, 1, 1, 0)

    def call(*a):
        return lib.tfsc_k_depthwise_conv(*[_ptr(v) if hasattr(v, "data_ptr") else v for v in a], None)
    assert call(*ok) == 0
    assert call(x, x, x, x, 2, 8, 8, 8, 7, 7, 2, 3, 6) == 0                            # at the limits
    assert call(x, x, x, x, 0, 8, 8, 8, 3, 3, 1, 1, 0) == 0                            # an empty batch
    for kh, kw, s, p, h in ((8, 3, 1, 1, 8), (3, 8, 1, 1, 8), (3, 3, 3, 1, 8), (3, 3, 0, 1, 8), (3, 3, 1, 2, 8), (7, 7, 1, 4, 8),
                            (5, 5, 1, 0, 4), (0, 3, 1, 0, 8), (3, 3, 1, -1, 8)):
        assert call(x, x, x, x, 2, h, h, 8, kh, kw, s, p, 0) == E, (kh, kw, s, p, h)
    for act in (2, 3, 7, -1):
        assert call(x, x, x, x, 2, 8, 8, 8, 3, 3, 1, 1, act) == E, act
    for i in range(4):
        a = list(ok)
        a[i] = None
        assert call(*a) == E, i
    assert call(x, x, x, x, -1, 8, 8, 8, 3, 3, 1, 1, 0) == E
    assert call(x, x, x, x, 2, 8, 8, 0, 3, 3, 1, 1, 0) == E
    assert call(x, x, x, x, 1, 65536, 65536, 1, 3, 3, 1, 1, 0) == E                     # h * w * c >= 2^31


# -------------------------------------------------------------------------------------- channel_scale ----
@pytest.mark.parametrize("B,HW,C", [(1, 1, 1), (3, 49, 5), (8, 196, 96), (64, 49, 1152), (2, 12544, 32), (5, 7, 4)])
def test_channel_scale_is_the_fp32_product(B, HW, C):
    torch = _torch()
    rng = np.random.default_rng(B + HW + C)
    x = rng.standard_normal((B, HW, C), dtype=np.float32)
    g = rng.random((B, C), dtype=np.float32)
    want = (x * g[:, None, :]).tobytes()
    for shift in (0, 1):                                                                 # 1: misaligned, the scalar path
        xd = torch.zeros(x.size + 4, device="cuda")
        xd[shift:shift + x.size] = torch.from_numpy(x.ravel()).cuda()
        gd = torch.from_numpy(g).cuda()
        yd = torch.full((x.size + 4,), float("nan"), device="cuda")
        t._lib.check(lib.tfsc_k_channel_scale(xd.data_ptr() + 4 * shift, _ptr(gd), yd.data_ptr() + 4 * shift, B, HW, C, None))
        torch.cuda.synchronize()
        assert yd[shift:shift + x.size].cpu().numpy().tobytes() == want, shift
    assert lib.tfsc_k_channel_scale(_ptr(xd), None, _ptr(yd), B, HW, C, None) == E
    assert lib.tfsc_k_channel_scale(_ptr(xd), _ptr(gd), _ptr(yd), B, 0, C, None) == E
    assert lib.tfsc_k_channel_scale(_ptr(xd), _ptr(gd), _ptr(yd), -1, HW, C, None) == E


# -------------------------------------------------------------------------- new activations in the GEMMs ----
def _act64(v, act):
    return cr.act(v, {4: "relu6", 5: "silu", 6: "sigmoid"}[act])


@pytest.mark.parametrize("m,n,k", [(1, 8, 4), (8, 24, 96), (33, 1000, 1280), (200, 100, 37), (130, 66, 18), (128, 128, 64), (300, 256, 96)])
@pytest.mark.parametrize("act", [4, 5, 6])
@pytest.mark.parametrize("res", [False, True])
def test_new_activations_in_the_gemms(m, n, k, act, res):
    """tfsc_k_gemm (the SIMT kernel below 64 rows or for n % 32 != 0, the tensor cores otherwise) and tfsc_k_gemm_tc"""
    torch = _torch()
    rng = np.random.default_rng(m + n + k + act)
    a = rng.standard_normal((m, k)).astype(np.float32)
    b = (rng.standard_normal((k, n)) * 3 / np.sqrt(k)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float32)
    ad, bd, biasd, rd = (torch.from_numpy(v).cuda() for v in (a, b, bias, r))
    ref = _act64(a.astype(np.float64) @ b + bias + (r if res else 0), act)
    entries = [lib.tfsc_k_gemm] + ([lib.tfsc_k_gemm_tc] if m >= 64 and n >= 64 and n % 32 == 0 and k >= 32 else [])
    for fn in entries:
        cd = torch.full((m, n), float("nan"), device="cuda")
        t._lib.check(fn(_ptr(ad), _ptr(bd), _ptr(biasd), _ptr(rd) if res else None, _ptr(cd), m, n, k, k, act, None))
        torch.cuda.synchronize()
        got = cd.cpu().numpy()
        assert not np.isnan(got).any() and _err(got, ref) <= 1e-4, fn.__name__


@pytest.mark.parametrize("h,c,kh,stride,pad,cout,bsz", [(14, 32, 3, 1, 1, 64, 2), (12, 64, 5, 2, 2, 96, 3), (9, 32, 1, 2, 0, 128, 4)])
@pytest.mark.parametrize("act", [4, 5, 6])
@pytest.mark.parametrize("res", [False, True])
def test_new_activations_in_the_implicit_gemm_conv(h, c, kh, stride, pad, cout, bsz, act, res):
    torch = _torch()
    rng = np.random.default_rng(h * 31 + c + kh + act)
    x = rng.standard_normal((bsz, h, h, c)).astype(np.float32)
    w = (rng.standard_normal((kh, kh, c, cout)) * 3 / np.sqrt(kh * kh * c)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    oh = (h + 2 * pad - kh) // stride + 1
    r = rng.standard_normal((bsz, oh, oh, cout)).astype(np.float32)
    xd, wd, bd, rd = (torch.from_numpy(v).cuda() for v in (x, w, b, r))
    y = torch.full((bsz, oh, oh, cout), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_conv_tc(_ptr(xd), _ptr(wd), _ptr(bd), _ptr(rd) if res else None, _ptr(y), bsz, h, h, c, kh, kh, stride, pad,
                                    cout, act, None), "conv_tc")
    torch.cuda.synchronize()
    ref = cr.conv(x, w, b, stride, pad, {4: "relu6", 5: "silu", 6: "sigmoid"}[act], r if res else None)
    got = y.cpu().numpy()
    assert not np.isnan(got).any() and _err(got, ref) <= 1e-4


# ------------------------------------------------------------------------------------- served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 2 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 4 << 30, "gpu.maxBatch": 64}
    cfg.update(kw)
    return cfg


def _model(net, seed, image=224, classes=1000, width=1.0, depth=1.0):
    if net == "mobilenet_v2":
        return ce.torchvision_mobilenet_v2(seed, width, classes), lambda outputs: mf.mobilenet_v2_manifest(image, classes, width, outputs)
    return ce.torchvision_efficientnet(seed, width, depth, classes), lambda outputs: mf.efficientnet_manifest(image, classes, width, depth, outputs)


def _write(tmp, net, seed, names=("one", "all"), **kw):
    """the bundle `names[0]` with the single logits output and `names[1]` with every classification output, same weights"""
    m, man = _model(net, seed, **kw)
    for name, outs in zip(names, (None, ALL)):
        mm = man(outs)
        mf.write_graph_bundle(os.path.join(str(tmp), name, "1"), mm, ce.export_convnet(m, mm))
    return m


@pytest.mark.parametrize("net", ["mobilenet_v2", "efficientnet"])
def test_full_size_through_the_server(net, tmp_path):
    m = _write(tmp_path, net, 21 if net == "mobilenet_v2" else 22)
    x = ce.images(33, 224, 5)
    ref = ce.reference(m, x)
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (1, 8, 33):
            y = srv.predict("one", "1", x[:bs])
            assert y.shape == (bs, 1000) and _err(y, ref[:bs]) <= 1e-4, (net, bs, _err(y, ref[:bs]))
            r = srv.predict("all", "1", x[:bs], outputs=NAMES)
            assert r["logits"].tobytes() == y.tobytes()
            assert np.array_equal(r["classes"], r["top_k_classes"][:, 0].astype(np.int64))
            for i in range(bs):
                srt = np.sort(ref[i])[::-1][:K + 1]
                rid = np.argsort(-ref[i], kind="stable")[:K]
                tol = 2e-4 * np.maximum(1.0, np.abs(srt))
                for j in range(K):        # ids equal fp64's wherever the neighbouring fp64 logits are further apart than the tolerance
                    if srt[j] - srt[j + 1] > tol[j] and (j == 0 or srt[j - 1] - srt[j] > tol[j]):
                        assert r["top_k_classes"][i, j] == rid[j], (net, bs, i, j)


def _session_run_request(name, feed, x, fetch):
    named = wire._ld(1, feed.encode()) + wire._ld(2, wire.encode_tensor(x))
    return wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())


@pytest.mark.parametrize("net", ["mobilenet_v2", "efficientnet"])
def test_every_frontend(net, tmp_path):
    torch = _torch()
    B, C = 5, 10
    kw = dict(image=64, classes=C, width=0.35 if net == "mobilenet_v2" else 0.5, depth=0.5)
    m = _write(tmp_path, net, 31, **kw)
    x = ce.images(B, 64, 6)
    ref = ce.reference(m, x)
    with t.Server(_cfg(tmp_path)) as srv:
        y = srv.predict("one", "1", x)
        full = srv.predict("all", "1", x, outputs=NAMES)
        assert _err(y, ref) <= 1e-4 and full["logits"].tobytes() == y.tobytes()
        assert full["classes"].dtype == np.int64 and full["top_k_classes"].dtype == np.int32 and full["top_k_classes"].shape == (B, K)
        # gRPC Predict, every output and a filter
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("all", 1, {"x": x})))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("all", 1, {"x": x}, output_filter=["classes"])))
        assert list(outs) == ["classes"] and outs["classes"].tobytes() == full["classes"].tobytes()
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("one", 1, {"x": x})))
        assert list(outs) == ["y"] and outs["y"].tobytes() == y.tobytes()
        # REST, row and columnar
        st, b = srv.rest_handle("POST", "/v1/models/all/versions/1:predict", json.dumps({"instances": x.tolist()}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        assert len(preds) == B and all(list(p) == NAMES for p in preds)
        for i, p in enumerate(preds):
            assert p["classes"] == int(full["classes"][i]) and p["top_k_classes"] == full["top_k_classes"][i].tolist()
            assert np.array_equal(np.float32(p["logits"]), full["logits"][i])
        st, b = srv.rest_handle("POST", "/v1/models/all/versions/1:predict", json.dumps({"inputs": {"x": x.tolist()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES and cols["classes"] == full["classes"].tolist()
        assert np.array_equal(np.float32(cols["probabilities"]), full["probabilities"])
        st, b = srv.rest_handle("POST", "/v1/models/one/versions/1:predict", json.dumps({"instances": x.tolist()}).encode())
        assert st == 200 and np.array_equal(np.float32(json.loads(b)["predictions"]), y)
        # metadata
        st, b = srv.rest_handle("GET", "/v1/models/all/versions/1/metadata")
        sd = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]
        want = {"classes": ("DT_INT64", ["-1"]), "logits": ("DT_FLOAT", ["-1", str(C)]), "probabilities": ("DT_FLOAT", ["-1", str(C)]),
                "top_k_classes": ("DT_INT32", ["-1", str(K)]), "top_k_probabilities": ("DT_FLOAT", ["-1", str(K)])}
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sd["outputs"].items()} == want
        assert [d["size"] for d in sd["inputs"]["x"]["tensor_shape"]["dim"]] == ["-1", str(64 * 64 * 3)]
        # tfsc_predict_device writes packed rows
        srv.ensure(0, "all", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(ALL, C))
        xd = torch.from_numpy(x).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "all", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), ALL, C)
        assert all(dev[k].tobytes() == full[k].tobytes() for k in NAMES)


@pytest.mark.parametrize("net", ["mobilenet_v2", "efficientnet"])
@pytest.mark.parametrize("rows", [1, 8])
def test_launch_counts(net, rows, tmp_path):
    """one launch per op, one more for the stem conv's patch matrix (3 input channels: no implicit GEMM), the batch's gather
    and scatter copies, and the head's one when outputs are declared"""
    _write(tmp_path, net, 41, image=64, classes=10, width=0.5, depth=0.5)
    man = _model(net, 41, image=64, classes=10, width=0.5, depth=0.5)[1](None)
    x = ce.images(rows, 64, rows)
    with t.Server(_cfg(tmp_path)) as srv:
        srv.predict("one", "1", x)
        srv.predict("all", "1", x, outputs=["classes"])
        counts = {}
        for name, outs in (("one", None), ("all", ["classes"])):
            s0 = srv.stats()
            srv.predict(name, "1", x, outputs=outs)
            s1 = srv.stats()
            counts[name] = (s1["kernel_launches"] - s0["kernel_launches"], s1["batches"] - s0["batches"])
    assert counts["one"] == (len(man["ops"]) + 3, 1) and counts["all"] == (len(man["ops"]) + 4, 1), counts


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_convnets as g
import convnet_export as ce
tmp = sys.argv[2]
g._write(tmp, "mobilenet_v2", 51, names=("m1", "ma"), image=96, classes=100, width=0.5)
g._write(tmp, "efficientnet", 52, names=("e1", "ea"), image=96, classes=100, width=0.5, depth=0.5)
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (1, 8, 64):
        x = ce.images(rows, 96, rows)
        for name in ("m1", "e1"):
            out[f"{name}_r{rows}"] = srv.predict(name, "1", x)
        for name in ("ma", "ea"):
            for k, v in srv.predict(name, "1", x, outputs=g.NAMES).items():
                out[f"{name}_{k}_r{rows}"] = v
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
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 3 * 2 * (1 + len(NAMES))
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key


# --------------------------------------------------------------------------------------- forward hop ----
N_MODELS = 4
HOP_ROWS, HOP_IMAGE = 6, 64


def _rank_cfg(rank, world, socks, base):
    members = [f"gpu{i}:0:0" for i in range(world)]
    return {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": base, "gpu.devices": [0],
            "gpu.arenaBytes": 256 << 20, "modelCache.size": 1 << 30, "serving.maxConcurrentModels": 16, "gpu.members": members,
            "gpu.localMembers": [members[rank]], "proxy.replicasPerModel": 1, "proxy.replicaPick": "first", "cluster.rank": rank,
            "cluster.endpoints": socks, "proxy.grpcTimeout": 60.0}


def _rank_main(rank, world, socks, base, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}}
        with t.Server(_rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = ce.images(HOP_ROWS, HOP_IMAGE, 7)
            for j in range(N_MODELS):
                name = f"c{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=NAMES)
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, {"x": x})))
                res["grpc"][j] = dict(outs)
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict", json.dumps({"instances": x.tolist()}).encode())
                res["rest"][j] = (st, b.decode())
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


def test_forward_hop():
    _torch()
    world = 2
    base = tempfile.mkdtemp(prefix="tfscconv")
    for j in range(N_MODELS):
        net = "mobilenet_v2" if j % 2 == 0 else "efficientnet"
        m, man = _model(net, 60 + j, image=HOP_IMAGE, classes=10, width=0.5, depth=0.5)
        mm = man(ALL)
        mf.write_graph_bundle(os.path.join(base, f"c{j}", "1"), mm, ce.export_convnet(m, mm))
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
        assert sorted(local["y"][j]) == NAMES and local["y"][j]["top_k_classes"].shape == (HOP_ROWS, K)
        for k in NAMES:
            assert fwd["y"][j][k].shape == local["y"][j][k].shape and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
