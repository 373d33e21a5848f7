"""-m gpu: BERT bundles with three inputs (input_ids, input_mask, segment_ids). The raw attention-mask and embedding
kernels against fp64, bert_small / bert_base exported from transformers and served from disk through every front-end, the
single-input bundle against the same bundle with three inputs, request and manifest rejections, and the forward hop."""
import copy
import json
import multiprocessing as mp
import os
import sys
import tempfile
import time

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models, wire

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_bert_pair_golden as pg  # noqa: E402
import torch_export as te  # noqa: E402

import bert_pair_ref as pr  # noqa: E402

pytestmark = pytest.mark.gpu
INPUTS = t.modelformat.BERT_INPUTS
NAMES = ["input_ids", "input_mask", "segment_ids"]   # byte-wise sorted = packed order
SMALL = dict(hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=512, labels=3)
BASE = dict(max_pos=512)
lib = t._lib.lib


def _err(got, ref):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


def _ptr(x):
    return x.data_ptr()


# ------------------------------------------------------------------------------------------- kernels ----
@pytest.mark.parametrize("d", [18, 64, 128])
@pytest.mark.parametrize("S", [13, 32, 64, 128, 256, 384, 512])
def test_attention_mask_kernel_matches_fp64(S, d):
    import torch
    heads, B = 2, 4
    H = heads * d
    g = torch.Generator().manual_seed(S * 1000 + d)
    qkv = torch.randn(B, S, 3 * H, generator=g, dtype=torch.float32)
    ids = torch.randint(1, 50, (B, S), generator=g, dtype=torch.int32)
    ids[0, S // 3:] = 0                                     # the ids say [PAD]: the mask disagrees below
    mask = (torch.rand(B, S, generator=g) > 0.3).to(torch.int32)
    mask[0] = 1                                             # row 0: every key attended although its ids say [PAD]
    mask[1] = 0                                             # row 1: fully masked
    mask[2, : S // 2] = 0                                   # row 2: real tokens masked out
    # the mask sits in the middle third of a [B, 3S] buffer whose other columns hold the bit pattern of NaN
    buf = torch.full((B, 3 * S), 0x7FC00000, dtype=torch.int32)
    buf[:, S:2 * S] = mask
    qd, bd = qkv.cuda(), buf.cuda()
    ctx = torch.full((B, S, H), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_attention_mask(_ptr(qd), _ptr(bd) + S * 4, 3 * S, _ptr(ctx), B, S, H, heads, None), "attention_mask")
    torch.cuda.synchronize()
    ref = pr.attention_mask_ref(qkv.double(), mask, heads)
    assert _err(ctx.cpu().numpy(), ref.numpy()) <= 1e-4
    # (ids, S) through the new entry gives the bits of tfsc_k_attention
    idd = ids.cuda()
    a = torch.full((B, S, H), float("nan"), device="cuda")
    b = torch.full((B, S, H), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_attention(_ptr(qd), _ptr(idd), _ptr(a), B, S, H, heads, None), "attention")
    t._lib.check(lib.tfsc_k_attention_mask(_ptr(qd), _ptr(idd), S, _ptr(b), B, S, H, heads, None), "attention_mask")
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    # a stride below seq is refused
    assert lib.tfsc_k_attention_mask(_ptr(qd), _ptr(bd), S - 1, _ptr(ctx), B, S, H, heads, None) == t._lib.E_INVALID


def _embed_ref(ids, types, word, pos, typ, gamma, beta, eps):
    import torch
    S = ids.shape[1]
    seg = typ[types.clamp(0, 1).long()] if types is not None else typ[0]
    v = word[ids.clamp(0, word.shape[0] - 1).long()] + pos[:S] + seg
    return models.layer_norm_ref(v, gamma, beta, eps)


@pytest.mark.parametrize("S,Hd", [(13, 64), (128, 768), (384, 96)])
def test_embed_kernel_types_and_stride(S, Hd):
    import torch
    B, V, eps = 3, 97, 1e-12
    g = torch.Generator().manual_seed(S + Hd)
    word, pos, typ = (torch.randn(n, Hd, generator=g) * 0.05 for n in (V, 512, 2))
    gamma, beta = torch.randn(Hd, generator=g) * 0.1 + 1, torch.randn(Hd, generator=g) * 0.1
    ids = torch.randint(-5, V + 5, (B, S), generator=g, dtype=torch.int32)     # out-of-range ids are clamped
    types = torch.randint(0, 2, (B, S), generator=g, dtype=torch.int32)
    types[0, :4] = torch.tensor([-3, 5, 2, -1], dtype=torch.int32)           # out-of-range types are clamped
    packed = torch.cat([ids, torch.zeros_like(ids), types], dim=1).contiguous()   # [B, 3S]: ids | (mask) | types
    dev = {k: v.cuda() for k, v in dict(word=word, pos=pos, typ=typ, gamma=gamma, beta=beta, packed=packed, ids=ids.contiguous()).items()}

    def run(idp, typp, stride):
        y = torch.full((B * S, Hd), float("nan"), device="cuda")
        t._lib.check(lib.tfsc_k_embed(idp, typp, stride, _ptr(dev["word"]), _ptr(dev["pos"]), _ptr(dev["typ"]), _ptr(dev["gamma"]),
                                      _ptr(dev["beta"]), _ptr(y), B, S, Hd, V, eps, None), "embed")
        torch.cuda.synchronize()
        return y.cpu()

    p = _ptr(dev["packed"])
    y = run(p, p + 2 * S * 4, 3 * S)
    ref = _embed_ref(ids, types, word.double(), pos.double(), typ.double(), gamma.double(), beta.double(), eps).reshape(B * S, Hd)
    assert _err(y.numpy(), ref.numpy()) <= 1e-4
    # types = NULL is segment 0, the single-input embedding: the same bits at stride S and inside the packed row
    y_single = run(_ptr(dev["ids"]), None, S)
    assert torch.equal(run(p, None, 3 * S).view(torch.int32), y_single.view(torch.int32))
    ref0 = _embed_ref(ids, None, word.double(), pos.double(), typ.double(), gamma.double(), beta.double(), eps).reshape(B * S, Hd)
    assert _err(y_single.numpy(), ref0.numpy()) <= 1e-4
    assert lib.tfsc_k_embed(p, None, S - 1, _ptr(dev["word"]), _ptr(dev["pos"]), _ptr(dev["typ"]), _ptr(dev["gamma"]),
                            _ptr(dev["beta"]), p, B, S, Hd, V, eps, None) == t._lib.E_INVALID


# ------------------------------------------------------------------------------------ served models ----
_MODELS = {}


def _model(kind):
    if kind not in _MODELS:
        _MODELS[kind] = te.hf_bert(4 if kind == "bert_small" else 3, **(SMALL if kind == "bert_small" else BASE))
    return _MODELS[kind]


def _reference(model, x):
    """transformers' forward in fp64 (on the GPU: the same fp64 arithmetic, in a fraction of the CPU time)"""
    import torch
    m64 = copy.deepcopy(model).double().cuda()
    tt = {k: torch.from_numpy(np.ascontiguousarray(v, np.int64)).cuda() for k, v in x.items()}
    with torch.no_grad():
        return m64(input_ids=tt["input_ids"], attention_mask=tt["input_mask"], token_type_ids=tt["segment_ids"]).logits.cpu().numpy()


def _write(tmp, name, kind, S, inputs):
    arch = dict(SMALL if kind == "bert_small" else BASE, seq=S)
    man = t.modelformat.bert_manifest(**arch, inputs=inputs)
    blob = te.export_bert(_model(kind), man)
    t.modelformat.write_graph_bundle(os.path.join(tmp, name, "1"), man, blob)
    return man, blob


def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 2 << 30, "serving.maxConcurrentModels": 4, "modelCache.size": 4 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _rest(srv, name, body):
    st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict", json.dumps(body).encode())
    return st, json.loads(b)


@pytest.mark.parametrize("kind", ["bert_small", "bert_base"])
@pytest.mark.parametrize("S", [128, 384])
def test_three_input_bert_matches_transformers(kind, S, tmp_path):
    vocab = SMALL["vocab"] if kind == "bert_small" else 30522
    x = pg.pair_inputs(8, S, vocab, seed=S + len(kind))
    ref = _reference(_model(kind), x)
    _write(str(tmp_path), kind, kind, S, INPUTS)
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (8, 3, 1):
            xb = {k: v[:bs] for k, v in x.items()}
            assert _err(srv.predict(kind, "1", xb), ref[:bs]) <= 1e-4, bs
        xb = {k: v[:3] for k, v in x.items()}
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(kind, 1, xb)))
        assert _err(outs["logits"], ref[:3]) <= 1e-4
        st, body = _rest(srv, kind, {"instances": [{k: xb[k][i].tolist() for k in reversed(NAMES)} for i in range(3)]})
        assert st == 200 and _err(body["predictions"], ref[:3]) <= 1e-4
        st, body = _rest(srv, kind, {"inputs": {k: xb[k].tolist() for k in NAMES}})
        assert st == 200 and _err(body["outputs"], ref[:3]) <= 1e-4


def test_single_input_bundle_and_three_inputs_give_the_same_bits(tmp_path):
    """mask = ids != 0 and segment 0 is what a single-input bundle derives: the logits must be bit-identical."""
    S = 128
    _write(str(tmp_path), "one", "bert_base", S, None)
    _write(str(tmp_path), "three", "bert_base", S, INPUTS)
    ids = np.random.default_rng(9).integers(1, 30522, (8, S)).astype(np.int32)
    ids[5, 70:] = 0
    ids[7, 3] = 0
    x3 = {"input_ids": ids, "input_mask": (ids != 0).astype(np.int32), "segment_ids": np.zeros_like(ids)}
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (8, 3):
            y1 = srv.predict("one", "1", ids[:bs])
            y3 = srv.predict("three", "1", {k: v[:bs] for k, v in x3.items()})
            assert y1.tobytes() == y3.tobytes(), bs


def test_request_rejections_name_the_inputs_and_launch_nothing(tmp_path):
    S = 16
    _write(str(tmp_path), "b3", "bert_small", S, INPUTS)
    x = pg.pair_inputs(2, S, SMALL["vocab"], seed=1)
    with t.Server(_cfg(tmp_path)) as srv:
        srv.predict("b3", "1", x)   # resident
        launches = srv.stats()["kernel_launches"]
        ids = x["input_ids"]
        bad = {
            "missing": {k: x[k] for k in ("input_ids", "segment_ids")},
            "extra": dict(x, token_type_ids=x["segment_ids"]),
            "misnamed": {"input_ids": ids, "attention_mask": x["input_mask"], "segment_ids": x["segment_ids"]},
            "batch": dict(x, input_mask=x["input_mask"][:1]),
            "row_size": {"input_ids": np.zeros((2, S + 1), np.int32), "input_mask": np.zeros((2, S - 1), np.int32),
                         "segment_ids": np.zeros((2, S), np.int32)},
            "float": dict(x, input_mask=x["input_mask"].astype(np.float32)),
            "single": ids,
        }
        for why, req in bad.items():
            with pytest.raises(t._lib.TfscError) as e:
                srv.predict("b3", "1", req)
            assert e.value.code == t._lib.E_INVALID and "'input_ids', 'input_mask', 'segment_ids'" in str(e.value), (why, str(e.value))
            if isinstance(req, dict) and why != "float":
                with pytest.raises(t._lib.TfscError) as e:
                    srv.grpc_predict(wire.encode_predict_request("b3", 1, req))
                assert e.value.code == t._lib.E_INVALID and "input_mask" in str(e.value), why
                n = min(v.shape[0] for v in req.values())
                st, body = _rest(srv, "b3", {"inputs": {k: v.tolist() for k, v in req.items()}})
                assert st == 400 and "segment_ids" in body["error"], (why, body)
                if why != "batch":
                    st, body = _rest(srv, "b3", {"instances": [{k: v[i].tolist() for k, v in req.items()} for i in range(n)]})
                    assert st == 400 and "segment_ids" in body["error"], (why, body)
        with pytest.raises(t._lib.TfscError) as e:   # gRPC float tensor
            srv.grpc_predict(wire.encode_predict_request("b3", 1, bad["float"]))
        assert e.value.code == t._lib.E_INVALID
        st, body = _rest(srv, "b3", {"instances": ids.tolist()})   # single-input REST body to a three-input model
        assert st == 400 and "input_mask" in body["error"]
        assert srv.stats()["kernel_launches"] == launches
        assert [r[0] for r in srv.resident(0)] == ["b3"]
        # Classify / Regress serve single-input models only: the refusal names the inputs
        st, body = srv.rest_handle("POST", "/v1/models/b3/versions/1:classify", json.dumps({"examples": [{"x": 1.0}]}).encode())
        assert st == 400 and "'input_ids', 'input_mask', 'segment_ids'" in json.loads(body)["error"]
        # a multi-key body to a single-input model stays a 400 and names its input
        _write(str(tmp_path), "b1", "bert_small", S, None)
        st, body = _rest(srv, "b1", {"inputs": {k: x[k].tolist() for k in NAMES}})
        assert st == 400 and "'input_ids'" in body["error"]


def test_submit_member_and_metadata(tmp_path):
    S = 16
    _write(str(tmp_path), "b3", "bert_small", S, INPUTS)
    x = pg.pair_inputs(3, S, SMALL["vocab"], seed=2)
    ref = _reference(_model("bert_small"), x)
    with t.Server(_cfg(tmp_path)) as srv:
        tk = srv.predict_submit("b3", "1", x)
        try:
            assert _err(tk.wait(30.0), ref) <= 1e-4
        finally:
            tk.release()
        assert _err(srv.predict_member(0, "b3", "1", x), ref) <= 1e-4
        assert _err(srv.predict_deadline("b3", "1", x, srv.now_ns() + 30_000_000_000), ref) <= 1e-4
        st, body = srv.rest_handle("GET", "/v1/models/b3/versions/1/metadata")
        sig = json.loads(body)["metadata"]["signature_def"]["signature_def"]["serving_default"]
        assert st == 200 and sorted(sig["inputs"]) == NAMES
        for k in NAMES:
            info = sig["inputs"][k]
            assert info["dtype"] == "DT_INT32" and [d["size"] for d in info["tensor_shape"]["dim"]] == ["-1", str(S)]


BAD_MANIFESTS = {
    "unknown role": lambda s: s.update(inputs=[{"name": "a", "role": "ids"}, {"name": "b", "role": "position_ids"}]),
    "duplicate role": lambda s: s.update(inputs=[{"name": "a", "role": "ids"}, {"name": "b", "role": "ids"}]),
    "duplicate name": lambda s: s.update(inputs=[{"name": "a", "role": "ids"}, {"name": "a", "role": "mask"}]),
    "no input has the role 'ids'": lambda s: s.update(inputs=[{"name": "a", "role": "mask"}]),
    "mutually exclusive": lambda s: s.update(input="input_ids"),
}


@pytest.mark.parametrize("why", list(BAD_MANIFESTS) + ["first op is 'embed'", "input_dtype int32"])
def test_loader_refuses_bad_inputs_manifests(why, tmp_path):
    man = t.modelformat.bert_manifest(seq=16, **SMALL, inputs=INPUTS)
    blob = np.zeros(man["weights_bytes"] // 4, np.float32)
    if why in BAD_MANIFESTS:
        BAD_MANIFESTS[why](man["signature"])
    elif why == "input_dtype int32":
        man["input_dtype"] = "float32"
    else:   # an MLP bundle cannot declare several inputs
        mlp = t.modelformat.write_mlp_bundle(str(tmp_path / "scratch" / "1"), [np.zeros((16, 4), np.float32)], [np.zeros(4, np.float32)])
        man = dict(mlp, signature={"inputs": INPUTS, "output": "y"})
        blob = np.zeros(man["weights_bytes"] // 4, np.float32)
    t.modelformat.write_graph_bundle(str(tmp_path / "bad" / "1"), man, blob)
    with t.Server(_cfg(tmp_path)) as srv:
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("bad", "1", pg.pair_inputs(1, 16, 100, seed=0))
        assert why in str(e.value), str(e.value)


# --------------------------------------------------------------------------------------- forward hop ----
N_FWD = 6


def _fwd_rank(rank, base, socks, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        members = ["gpu0:0:0", "gpu1:0:0"]
        cfg = _cfg(base, **{"gpu.arenaBytes": 256 << 20, "gpu.members": members, "gpu.localMembers": [members[rank]],
                            "proxy.replicasPerModel": 1, "proxy.replicaPick": "first", "cluster.rank": rank,
                            "cluster.endpoints": socks, "cluster.slotBytes": 1 << 16, "cluster.windowSlots": 8,
                            "proxy.grpcTimeout": 30.0})
        x = pg.pair_inputs(3, 16, SMALL["vocab"], seed=4)
        res = {"rank": rank}
        with t.Server(cfg) as srv:
            barrier.wait(timeout=120)
            srv.fwd_peer_window(1 - rank)
            owned = [srv.route(f"f{j}", "1")[0][0] >= 0 for j in range(N_FWD)]
            res["owned"] = owned
            res["y"] = {j: srv.predict(f"f{j}", "1", x) for j in range(N_FWD)}   # local and forwarded
            barrier.wait(timeout=120)
            res["launches0"] = srv.stats()["kernel_launches"]
            barrier.wait(timeout=120)
            if rank == 0:   # a layout the owner's manifest refuses (a misnamed input), sent to a model of rank 1
                j = next(j for j in range(N_FWD) if not owned[j])
                try:
                    srv.predict(f"f{j}", "1", {"input_ids": x["input_ids"], "attention_mask": x["input_mask"],
                                                "segment_ids": x["segment_ids"]})
                    res["bad"] = None
                except t._lib.TfscError as e:
                    res["bad"] = (e.code, str(e))
            barrier.wait(timeout=120)
            res["launches1"] = srv.stats()["kernel_launches"]
            res["fwd"] = srv.stats()["fwd_in_requests"]
            barrier.wait(timeout=120)
        out.put(res)
    except BaseException as e:  # noqa: BLE001
        import traceback
        out.put({"rank": rank, "fatal": f"{e!r}\n{traceback.format_exc()}"})
        try:
            barrier.abort()
        except Exception:
            pass


def test_forward_hop_packs_three_inputs(tmp_path):
    man, blob = _write(str(tmp_path), "f0", "bert_small", 16, INPUTS)
    for j in range(1, N_FWD):
        t.modelformat.write_graph_bundle(str(tmp_path / f"f{j}" / "1"), man, blob)
    sock_dir = tempfile.mkdtemp(prefix="tfscbi")
    socks = [os.path.join(sock_dir, f"r{r}.sock") for r in range(2)]
    ctx = mp.get_context("spawn")
    barrier, out = ctx.Barrier(2), ctx.Queue()
    procs = [ctx.Process(target=_fwd_rank, args=(r, str(tmp_path), socks, barrier, out)) for r in range(2)]
    [p.start() for p in procs]
    results, deadline = {}, time.time() + 300
    while len(results) < 2 and time.time() < deadline:
        try:
            r = out.get(timeout=5)
            results[r["rank"]] = r
        except Exception:
            if not any(p.is_alive() for p in procs):
                break
    [p.join(timeout=30) for p in procs]
    [p.kill() for p in procs if p.is_alive()]
    assert len(results) == 2 and all("fatal" not in r for r in results.values()), results
    r0, r1 = results[0], results[1]
    assert any(r0["owned"]) and not all(r0["owned"])
    x = pg.pair_inputs(3, 16, SMALL["vocab"], seed=4)
    ref = _reference(_model("bert_small"), x)
    for j in range(N_FWD):   # a request that enters at the non-owner rank gets the bits of one that enters at the owner
        assert r0["y"][j].tobytes() == r1["y"][j].tobytes(), j
        assert _err(r0["y"][j], ref) <= 1e-4, j
    code, msg = r0["bad"]
    assert code == t._lib.E_INVALID and "'input_ids', 'input_mask', 'segment_ids'" in msg
    assert r1["launches1"] == r1["launches0"] and r1["fwd"] > 0   # the owner rejected it without a launch
