"""-m gpu: Swin Transformer. The window_attention kernel against fp64 (shapes of every Swin-T stage and of Swin-B at 384 px,
every kind of shift, batch and path bit identity, refusals), the patch_merge kernel bit for bit against numpy, full-size
swin_t through the server against torchvision fp64, the classification outputs through every front-end, launch counts,
programmatic-dependent-launch bit identity and the forward hop between two ranks."""
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
import swin_export as se  # noqa: E402
import swin_ref as sr  # noqa: E402
from test_gpu_convnets import _cfg, _err, _ptr, _rank_cfg  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
E = t._lib.E_INVALID
K = 5
ALL = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"}, {"name": "classes", "kind": "classes"},
       {"name": "top_k_classes", "kind": "top_k_classes", "k": K}, {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": K}]
NAMES = sorted(o["name"] for o in ALL)
SMALL = dict(embed_dim=32, depths=(2, 2), heads=(1, 2))     # 56 px: stages of 14 x 14 and 7 x 7 tokens


def _torch():
    import torch
    assert torch.cuda.is_available()
    return torch


# ------------------------------------------------------------------------------------------ window_attention ----
def _wa(torch, qd, bd, B, H, W, C, heads, ws, shift, q_off=0, y_off=0):
    """launch on qkv / ctx shifted by q_off / y_off floats (a misaligned shift selects the scalar path); returns [B, H, W, C]"""
    n = B * H * W * C
    yb = torch.full((n + 4,), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_window_attention(qd.data_ptr() + 4 * q_off, _ptr(bd), yb.data_ptr() + 4 * y_off, B, H, W, C, heads, ws, shift,
                                             None), "window_attention")
    torch.cuda.synchronize()
    return yb[y_off:y_off + n].cpu().numpy().reshape(B, H, W, C)


# (H, W, window, heads, head width): Swin-T's four stages, a non-square map, Swin-B's third stage at 384 px, and head widths
# other than 32 (16, 64, and 13 and 6, which only the scalar path takes)
SHAPES = [(56, 56, 7, 3, 32), (28, 28, 7, 6, 32), (14, 14, 7, 12, 32), (7, 7, 7, 24, 32), (14, 28, 7, 1, 32), (24, 24, 12, 16, 32),
          (14, 14, 7, 2, 16), (7, 14, 7, 2, 64), (12, 12, 12, 3, 13), (8, 8, 4, 5, 6)]


@pytest.mark.parametrize("H,W,ws,heads,d", SHAPES)
@pytest.mark.parametrize("spread", [1.0, 5.5])
def test_window_attention_matches_fp64(H, W, ws, heads, d, spread):
    """q and k of scale `spread`: scores spread over a few units (1.0) and over ~30 (5.5), plus a N(0, 1) bias"""
    torch = _torch()
    C, N = heads * d, ws * ws
    for n, shift in enumerate(sorted({0, 1, ws // 2, ws - 1})):
        B = (1, 3, 8)[n % 3]
        rng = np.random.default_rng(H * 1000 + W * 10 + shift + int(spread * 10))
        qkv = rng.standard_normal((B, H, W, 3 * C)).astype(np.float32)
        qkv[..., :2 * C] *= spread
        bias = rng.standard_normal((heads, N, N)).astype(np.float32)
        qd = torch.zeros(qkv.size + 4, device="cuda")
        qd[:qkv.size] = torch.from_numpy(qkv.ravel()).cuda()
        bd = torch.from_numpy(bias).cuda()
        y = _wa(torch, qd, bd, B, H, W, C, heads, ws, shift)
        ref = sr.window_attention(qkv, bias, heads, ws, shift)
        err = _err(y, ref)
        assert not np.isnan(y).any() and err <= 1e-4, (H, W, ws, heads, d, shift, B, err)
        # a window's bits do not depend on the batch
        for r in {0, B - 1}:
            one = _wa(torch, qd, bd, 1, H, W, C, heads, ws, shift, q_off=r * H * W * 3 * C)
            assert one.tobytes() == y[r:r + 1].tobytes(), (H, W, ws, heads, d, shift, B, r)
        # nor on the path: a one-float shift of qkv makes it misaligned, which selects the scalar loads
        if d % 4 == 0:
            qs = torch.zeros(qkv.size + 4, device="cuda")
            qs[1:1 + qkv.size] = qd[:qkv.size]
            assert _wa(torch, qs, bd, B, H, W, C, heads, ws, shift, q_off=1, y_off=1).tobytes() == y.tobytes(), (H, W, ws, shift)


def test_window_attention_refusals():
    torch = _torch()
    x = torch.zeros(3 * 24 * 24 * 96, device="cuda")
    ok = (x, x, x, 2, 14, 14, 64, 2, 7, 3)

    def call(*a):
        return lib.tfsc_k_window_attention(*[_ptr(v) if hasattr(v, "data_ptr") else v for v in a], None)
    assert call(*ok) == 0
    assert call(x, x, x, 0, 14, 14, 64, 2, 7, 3) == 0                                  # an empty batch
    assert call(x, x, x, 1, 12, 12, 78, 2, 12, 11) == 0                                # d = 39 at window 12: 48400 bytes
    for h, w, c, heads, ws, s in ((15, 14, 64, 2, 7, 0), (14, 15, 64, 2, 7, 0), (14, 14, 64, 2, 7, 7), (14, 14, 64, 2, 7, -1),
                                  (14, 14, 64, 3, 7, 0), (14, 14, 64, 0, 7, 0), (14, 14, 64, 2, 0, 0), (17, 17, 16, 1, 17, 0),
                                  (7, 7, 130, 2, 7, 0), (12, 12, 80, 2, 12, 0), (0, 14, 64, 2, 7, 0)):
        assert call(x, x, x, 2, h, w, c, heads, ws, s) == E, (h, w, c, heads, ws, s)
    for i in range(3):
        a = list(ok)
        a[i] = None
        assert call(*a) == E, i
    assert call(x, x, x, -1, 14, 14, 64, 2, 7, 3) == E
    assert call(x, x, x, 1, 65536, 65536, 1, 1, 1, 0) == E                               # h * w * 3c >= 2^31


# ------------------------------------------------------------------------------------------------ patch_merge ----
@pytest.mark.parametrize("B,H,W,C", [(1, 56, 56, 96), (3, 28, 28, 192), (8, 14, 14, 384), (2, 2, 2, 1), (3, 4, 6, 3), (5, 8, 8, 5),
                                     (64, 14, 14, 96)])
def test_patch_merge_is_the_numpy_gather(B, H, W, C):
    torch = _torch()
    x = np.random.default_rng(B + H + C).standard_normal((B, H, W, C), dtype=np.float32)
    want = sr.patch_merge(x).astype(np.float32).tobytes()
    for shift in (0, 1):                                                                 # 1: misaligned, the scalar path
        xd = torch.zeros(x.size + 4, device="cuda")
        xd[shift:shift + x.size] = torch.from_numpy(x.ravel()).cuda()
        yd = torch.full((x.size + 4,), float("nan"), device="cuda")
        t._lib.check(lib.tfsc_k_patch_merge(xd.data_ptr() + 4 * shift, yd.data_ptr() + 4 * shift, B, H, W, C, None), "patch_merge")
        torch.cuda.synchronize()
        assert yd[shift:shift + x.size].cpu().numpy().tobytes() == want, shift
    assert lib.tfsc_k_patch_merge(_ptr(xd), None, B, H, W, C, None) == E
    assert lib.tfsc_k_patch_merge(_ptr(xd), _ptr(yd), -1, H, W, C, None) == E
    assert lib.tfsc_k_patch_merge(_ptr(xd), _ptr(yd), B, H + 1, W, C, None) == E
    assert lib.tfsc_k_patch_merge(_ptr(xd), _ptr(yd), B, H, W + 1, C, None) == E
    assert lib.tfsc_k_patch_merge(_ptr(xd), _ptr(yd), B, H, W, 0, None) == E
    assert lib.tfsc_k_patch_merge(_ptr(xd), _ptr(yd), 0, H, W, C, None) == 0


# ------------------------------------------------------------------------------------------------ served models ----
def _write(tmp, seed, names=("one", "all"), image=224, classes=1000, **kw):
    """the bundle `names[0]` with the single logits output and `names[1]` with every classification output, same weights"""
    m = se.torchvision_swin(seed, classes=classes, **kw)
    for name, outs in zip(names, (None, ALL)):
        man = mf.swin_manifest(image=image, classes=classes, outputs=outs, **kw)
        mf.write_graph_bundle(os.path.join(str(tmp), name, "1"), man, se.export_swin(m, man))
    return m


def test_swin_t_through_the_server(tmp_path):
    m = _write(tmp_path, 21)
    x = se.images(8, 224, 5)
    ref = se.reference(m, x)
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (1, 3, 8):
            y = srv.predict("one", "1", x[:bs])
            err = _err(y, ref[:bs])
            assert y.shape == (bs, 1000) and err <= 1e-4, (bs, err)
            r = srv.predict("all", "1", x[:bs], outputs=NAMES)
            assert r["logits"].tobytes() == y.tobytes()
            assert np.array_equal(r["classes"], r["top_k_classes"][:, 0].astype(np.int64))
            for i in range(bs):
                srt = np.sort(ref[i])[::-1][:K + 1]
                rid = np.argsort(-ref[i], kind="stable")[:K]
                tol = 2e-4 * np.maximum(1.0, np.abs(srt))
                for j in range(K):        # ids equal fp64's wherever the neighbouring fp64 logits are further apart than the tolerance
                    if srt[j] - srt[j + 1] > tol[j] and (j == 0 or srt[j - 1] - srt[j] > tol[j]):
                        assert r["top_k_classes"][i, j] == rid[j], (bs, i, j)


def test_every_frontend(tmp_path):
    torch = _torch()
    B, C = 5, 10
    m = _write(tmp_path, 31, image=56, classes=C, **SMALL)
    x = se.images(B, 56, 6)
    ref = se.reference(m, x)
    with t.Server(_cfg(tmp_path)) as srv:
        y = srv.predict("one", "1", x)
        full = srv.predict("all", "1", x, outputs=NAMES)
        assert _err(y, ref) <= 1e-4 and full["logits"].tobytes() == y.tobytes()
        assert full["classes"].dtype == np.int64 and full["top_k_classes"].dtype == np.int32 and full["top_k_classes"].shape == (B, K)
        assert np.allclose(full["probabilities"].sum(axis=1), 1.0, atol=1e-5)
        # the async C ABI
        assert all(v.tobytes() == full[k].tobytes() for k, v in srv.predict_submit("all", "1", x, outputs=NAMES).wait().items())
        assert srv.predict_submit("one", "1", x).wait().tobytes() == y.tobytes()
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
        # metadata
        st, b = srv.rest_handle("GET", "/v1/models/all/versions/1/metadata")
        sd = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]
        want = {"classes": ("DT_INT64", ["-1"]), "logits": ("DT_FLOAT", ["-1", str(C)]), "probabilities": ("DT_FLOAT", ["-1", str(C)]),
                "top_k_classes": ("DT_INT32", ["-1", str(K)]), "top_k_probabilities": ("DT_FLOAT", ["-1", str(K)])}
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sd["outputs"].items()} == want
        assert [d["size"] for d in sd["inputs"]["x"]["tensor_shape"]["dim"]] == ["-1", str(56 * 56 * 3)]
        # tfsc_predict_device writes packed rows
        srv.ensure(0, "all", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(ALL, C))
        xd = torch.from_numpy(x).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "all", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), ALL, C)
        assert all(dev[k].tobytes() == full[k].tobytes() for k in NAMES)


@pytest.mark.parametrize("rows", [1, 8])
def test_launch_counts(rows, tmp_path):
    """one launch per op, one more for the stem conv's patch matrix (3 input channels: no implicit GEMM), the batch's gather
    and scatter copies, and the head's one when outputs are declared"""
    _write(tmp_path, 41, image=56, classes=10, **SMALL)
    man = mf.swin_manifest(image=56, classes=10, **SMALL)
    x = se.images(rows, 56, rows)
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
import test_gpu_swin as g
import swin_export as se
tmp = sys.argv[2]
g._write(tmp, 51, names=("s1", "sa"), image=112, classes=100, embed_dim=32, depths=(2, 2, 2), heads=(1, 2, 4))
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (1, 8, 64):
        x = se.images(rows, 112, rows)
        out[f"s1_r{rows}"] = srv.predict("s1", "1", x)
        for k, v in srv.predict("sa", "1", x, outputs=g.NAMES).items():
            out[f"sa_{k}_r{rows}"] = v
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
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 3 * (1 + len(NAMES))
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key


# --------------------------------------------------------------------------------------------------- forward hop ----
N_MODELS = 4
HOP_ROWS, HOP_IMAGE = 6, 56


def _rank_main(rank, world, socks, base, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}}
        with t.Server(_rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = se.images(HOP_ROWS, HOP_IMAGE, 7)
            for j in range(N_MODELS):
                name = f"s{j}"
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
    base = tempfile.mkdtemp(prefix="tfscswin")
    for j in range(N_MODELS):
        m = se.torchvision_swin(60 + j, classes=10, **SMALL)
        man = mf.swin_manifest(image=HOP_IMAGE, classes=10, outputs=ALL, **SMALL)
        mf.write_graph_bundle(os.path.join(base, f"s{j}", "1"), man, se.export_swin(m, man))
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
