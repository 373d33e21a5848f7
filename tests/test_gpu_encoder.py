"""-m gpu: encoder (embedding) outputs. The encoder-head kernel against the fp64 reference, bert_small and BERT-base
BertModel bundles with and without a pooler at S = 128 and 384 against transformers fp64, every front-end, launch counts,
programmatic-dependent-launch bit identity and the forward hop between two ranks."""
import copy
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
import embed_export as ee  # noqa: E402
import embed_ref as er  # noqa: E402
import span_ref as sr  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
ALL = [{"name": k, "kind": k} for k in mf.ENCODER_OUTPUT_KINDS]
NAMES = sorted(o["name"] for o in ALL)
SMALL = dict(hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=512)
SEP = 3


def _ptr(x):
    return None if x is None else x.data_ptr()


# ------------------------------------------------------------------------------------------- kernel ----
def _rows(rows, S, H, seed):
    """hidden [rows, S, H] fp32 and ids / mask [rows, S]. Rows cycle through: a padded tail, a fully masked row, [PAD]
    (id 0) at position 0 with its mask set, values of magnitude 10^3, and no padding at all."""
    rng = np.random.default_rng(seed)
    h = rng.standard_normal((rows, S, H), dtype=np.float32)
    ids = rng.integers(1, 50, (rows, S)).astype(np.int32)
    mask = np.ones((rows, S), np.int32)
    for r in range(rows):
        kind = r % 5
        tail = int(rng.integers(0, S)) if S > 1 else 0
        if kind == 0:
            mask[r, S - tail:], ids[r, S - tail:] = 0, 0
        elif kind == 1:
            mask[r], ids[r] = 0, 0
        elif kind == 2:
            ids[r, 0] = 0
            mask[r, S - tail:], ids[r, S - tail:] = 0, 0
        elif kind == 3:
            h[r] *= np.float32(1000.0)
    return h, ids, mask


def _launch(h, ids, mask, S, H, norm_cls=False, norm_mean=False, pooled=None, want=(True, True, True, True), misalign=False):
    """tfsc_k_encoder_head on device copies; outputs not wanted are NULL. misalign: the hidden states and sequence_output
    start one float past a 16-byte boundary (the scalar path)."""
    import torch
    rows = h.shape[0]
    off = 1 if misalign else 0
    hb = torch.empty(rows * S * H + off, device="cuda")
    hb[off:] = torch.from_numpy(h.reshape(-1)).cuda()
    hd = hb[off:]
    dev_ids = torch.from_numpy(np.ascontiguousarray(ids)).cuda()
    dev_mask = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask)).cuda()
    pd = None if pooled is None else torch.from_numpy(np.ascontiguousarray(pooled)).cuda()
    sb = torch.full((rows * S * H + off,), float("nan"), device="cuda")
    outs = [sb[off:] if want[0] else None] + [torch.full((rows, H), float("nan"), device="cuda") if w else None for w in want[1:]]
    if pooled is None:
        outs[1] = None
    t._lib.check(lib.tfsc_k_encoder_head(_ptr(hd), _ptr(pd), _ptr(dev_ids), _ptr(dev_mask), S, rows, S, H, int(norm_cls),
                                         int(norm_mean), *[_ptr(o) for o in outs], None), "encoder_head")
    torch.cuda.synchronize()
    res = [None if o is None else o.cpu().numpy() for o in outs]
    if res[0] is not None:
        res[0] = res[0].reshape(rows, S, H)
    return dict(zip(("sequence_output", "pooled_output", "cls_embedding", "mean_embedding"), res))


def _close(got, ref, scale, tol):
    err = np.max(np.abs(got.astype(np.float64) - ref) / np.maximum(1.0, scale)) if got.size else 0.0
    assert err <= tol, err


@pytest.mark.parametrize("H", [64, 384, 768, 1024])
@pytest.mark.parametrize("S", [1, 16, 17, 128, 129, 384, 512])
@pytest.mark.parametrize("rows", [1, 219])
def test_encoder_kernel_matches_reference(rows, S, H):
    if rows * S * H > 40_000_000:
        rows = 61                                      # the largest shapes keep the host reference within memory
    h, ids, mask = _rows(rows, S, H, seed=rows * 7919 + S * 31 + H)
    use_mask = (S + H // 64 + rows) % 2 == 0           # half the cases: no mask input, ids != 0
    m = mask if use_mask else None
    for norm in (False, True):
        r = _launch(h, ids, m, S, H, norm_cls=norm, norm_mean=norm)
        ref = er.embed_ref(h, ids, m, normalize_cls=norm, normalize_mean=norm)
        assert r["sequence_output"].tobytes() == h.tobytes()
        if norm:
            _close(r["cls_embedding"], ref["cls_embedding"], 1.0, 2e-6)
            _close(r["mean_embedding"], ref["mean_embedding"], 1.0, 2e-6)
        else:
            assert r["cls_embedding"].tobytes() == np.ascontiguousarray(h[:, 0]).tobytes()
            scale = np.abs(h).max(axis=(1, 2), keepdims=False)[:, None]
            _close(r["mean_embedding"], ref["mean_embedding"], scale, 2e-5)
        live = er.token_mask(ids, m).sum(axis=1)
        assert (r["mean_embedding"][live == 0] == 0).all()       # fully masked rows: a zero vector, normalised or not
        # each row's bits are those of a batch of one, and of the scalar path on a misaligned layout
        for i in sorted({0, rows // 2, rows - 1}):
            one = _launch(h[i:i + 1], ids[i:i + 1], None if m is None else m[i:i + 1], S, H, norm, norm)
            assert all(one[k].tobytes() == r[k][i:i + 1].tobytes() for k in ("sequence_output", "cls_embedding", "mean_embedding"))
        if rows <= 61 or S * H <= 128 * 384:
            mis = _launch(h, ids, m, S, H, norm, norm, misalign=True)
            assert all(mis[k].tobytes() == r[k].tobytes() for k in ("sequence_output", "cls_embedding", "mean_embedding"))


def test_encoder_kernel_null_outputs_and_pooled():
    rows, S, H = 9, 40, 128
    h, ids, mask = _rows(rows, S, H, seed=5)
    pooled = np.random.default_rng(6).standard_normal((rows, H), dtype=np.float32)
    full = _launch(h, ids, mask, S, H, norm_mean=True, pooled=pooled)
    assert full["pooled_output"].tobytes() == pooled.tobytes()
    for bits in range(16):
        want = tuple(bool(bits >> i & 1) for i in range(4))
        r = _launch(h, ids, mask, S, H, norm_mean=True, pooled=pooled, want=want)
        for k, w in zip(("sequence_output", "pooled_output", "cls_embedding", "mean_embedding"), want):
            assert (r[k] is None) == (not w) and (r[k] is None or r[k].tobytes() == full[k].tobytes()), (bits, k)


def test_encoder_kernel_rejections():
    import torch
    h = torch.zeros(4, 64, 64, device="cuda")
    ids = torch.ones(4, 64, dtype=torch.int32, device="cuda")
    y = torch.zeros(4, 64, device="cuda")
    E = t._lib.E_INVALID
    for S, H in ((0, 64), (8193, 64), (64, 0), (64, 8193)):
        assert lib.tfsc_k_encoder_head(_ptr(h), None, _ptr(ids), None, 64, 4, S, H, 0, 0, None, None, _ptr(y), None, None) == E, (S, H)
    assert lib.tfsc_k_encoder_head(_ptr(h), None, _ptr(ids), None, 64, -1, 64, 64, 0, 0, None, None, _ptr(y), None, None) == E
    assert lib.tfsc_k_encoder_head(None, None, _ptr(ids), None, 64, 4, 64, 64, 0, 0, None, None, _ptr(y), None, None) == E
    assert lib.tfsc_k_encoder_head(_ptr(h), None, _ptr(ids), None, 64, 4, 64, 64, 0, 0, None, _ptr(y), None, None, None) == E
    assert lib.tfsc_k_encoder_head(_ptr(h), None, None, None, 64, 4, 64, 64, 0, 0, None, None, None, _ptr(y), None) == E
    assert lib.tfsc_k_encoder_head(_ptr(h), None, _ptr(ids), None, 63, 4, 64, 64, 0, 0, None, None, None, _ptr(y), None) == E
    assert lib.tfsc_k_encoder_head(_ptr(h), None, _ptr(ids), None, 64, 0, 64, 64, 0, 0, None, None, None, _ptr(y), None) == 0
    # cls_embedding alone needs neither ids nor a stride
    assert lib.tfsc_k_encoder_head(_ptr(h), None, None, None, 0, 4, 64, 64, 0, 0, None, None, _ptr(y), None, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(y, h[:, 0])


# ------------------------------------------------------------------------------------ served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 3 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 6 << 30, "gpu.maxBatch": 8}
    cfg.update(kw)
    return cfg


def _outputs(pooler, norm_mean):
    outs = [dict(o) for o in ALL if pooler or o["kind"] != "pooled_output"]
    for o in outs:
        if o["kind"] == "mean_embedding" and norm_mean:
            o["normalize"] = True
    return outs


def _write_enc(tmp, seq, arch, seed, pooler=True, norm_mean=False, single="e1", multi="es"):
    m = ee.hf_bert_model(seed, pooler=pooler, **arch)
    one = mf.bert_manifest(seq=seq, **arch, inputs=mf.BERT_INPUTS, head="encoder", pooler=pooler)
    blob = ee.export_bert_model(m, one)
    mf.write_graph_bundle(os.path.join(str(tmp), single, "1"), one, blob)
    mf.write_graph_bundle(os.path.join(str(tmp), multi, "1"),
                          mf.bert_manifest(seq=seq, **arch, inputs=mf.BERT_INPUTS, outputs=_outputs(pooler, norm_mean),
                                           head="encoder", pooler=pooler), blob)
    return m


@pytest.mark.parametrize("pooler", [True, False])
@pytest.mark.parametrize("S", [128, 384])
@pytest.mark.parametrize("kind", ["bert_small", "bert_base"])
def test_bert_embeddings(kind, S, pooler, tmp_path):
    import torch
    B = 8
    arch = dict(SMALL) if kind == "bert_small" else dict(max_pos=512)
    H = arch.get("hidden", 768)
    norm_mean = not pooler                           # sentence-embedding checkpoints: no pooler, normalised mean
    m = _write_enc(tmp_path, S, arch, (71 if kind == "bert_small" else 72) + pooler, pooler, norm_mean)
    x = sr.qa_inputs(B, S, arch.get("vocab", 30522), seed=17, sep_id=SEP)
    m64 = copy.deepcopy(m).double().cuda()
    tt = {k: torch.from_numpy(np.ascontiguousarray(v, np.int64)).cuda() for k, v in x.items()}
    with torch.no_grad():
        o = m64(input_ids=tt["input_ids"], attention_mask=tt["input_mask"], token_type_ids=tt["segment_ids"])
    h64 = o.last_hidden_state.cpu().numpy()
    names = sorted(o_["name"] for o_ in _outputs(pooler, norm_mean))
    with t.Server(_cfg(tmp_path)) as srv:
        for bs in (B, 3):
            xb = {k: v[:bs] for k, v in x.items()}
            r = srv.predict("es", "1", xb, outputs=names)
            assert r["sequence_output"].shape == (bs, S, H) and r["cls_embedding"].shape == (bs, H)
            _close(r["sequence_output"], h64[:bs], np.abs(h64[:bs]), 1e-4)
            assert r["cls_embedding"].tobytes() == np.ascontiguousarray(r["sequence_output"][:, 0]).tobytes()
            mean64 = er.mean_embedding(h64[:bs], xb["input_ids"], xb["input_mask"], norm=norm_mean)
            _close(r["mean_embedding"], mean64, np.abs(mean64), 1e-4)
            # the served mean is the raw kernel on the served hidden states, bit for bit
            raw = _launch(r["sequence_output"], xb["input_ids"], xb["input_mask"], S, H, norm_mean=norm_mean)
            assert raw["mean_embedding"].tobytes() == r["mean_embedding"].tobytes()
            y1 = srv.predict("e1", "1", xb, out_capacity_elems=bs * S * H)
            if pooler:
                _close(r["pooled_output"], o.pooler_output.cpu().numpy()[:bs], np.abs(o.pooler_output.cpu().numpy()[:bs]), 1e-4)
                assert y1.shape == (bs, H) and r["pooled_output"].tobytes() == y1.tobytes()
            else:
                assert y1.shape == (bs, S, 1, H) and r["sequence_output"].tobytes() == y1.tobytes()


# --------------------------------------------------------------------------------------- front-ends ----
def _session_run_request(name, feed, x, fetch):
    named = wire._ld(1, feed.encode()) + wire._ld(2, wire.encode_tensor(x))
    return wire._ld(1, wire.encode_model_spec(name, 1)) + wire._ld(2, named) + wire._ld(3, fetch.encode())


def test_every_frontend_on_an_encoder_bundle(tmp_path):
    import torch
    S, B, H = 32, 5, SMALL["hidden"]
    _write_enc(tmp_path, S, SMALL, 73)
    x = sr.qa_inputs(B, S, SMALL["vocab"], seed=3, sep_id=SEP)
    with t.Server(_cfg(tmp_path)) as srv:
        full = srv.predict("es", "1", x, outputs=NAMES)
        assert full["sequence_output"].shape == (B, S, H) and all(full[k].shape == (B, H) for k in NAMES if k != "sequence_output")
        sub = srv.predict("es", "1", x, outputs=["mean_embedding", "sequence_output"])
        assert list(sub) == ["mean_embedding", "sequence_output"] and all(v.tobytes() == full[k].tobytes() for k, v in sub.items())
        # one example without a batch dimension: the outputs of a batch of one (the encoder's GEMMs tile by batch size, so
        # its hidden states need not have the bits of the same row in a batch of five)
        one = srv.predict("es", "1", {k: v[0] for k, v in x.items()}, outputs=["sequence_output", "pooled_output"])
        assert one["sequence_output"].shape == (S, H) and one["pooled_output"].shape == (H,)
        b1 = srv.predict("es", "1", {k: v[:1] for k, v in x.items()}, outputs=NAMES)
        assert one["sequence_output"].tobytes() == b1["sequence_output"].tobytes() and one["pooled_output"].tobytes() == b1["pooled_output"].tobytes()
        _close(one["sequence_output"], full["sequence_output"][0].astype(np.float64), np.abs(full["sequence_output"][0]), 1e-5)
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("es", "1", x, outputs=["nope"])
        assert "unknown output 'nope'" in str(e.value) and "'sequence_output' (float)" in str(e.value)
        for r in (srv.predict_deadline("es", "1", x, srv.now_ns() + 30_000_000_000, outputs=NAMES),
                  srv.predict_member(0, "es", "1", x, outputs=NAMES)):
            assert all(r[k].tobytes() == full[k].tobytes() for k in NAMES)
        tk = srv.predict_submit("es", "1", x, outputs=["sequence_output", "cls_embedding"])
        try:
            r = tk.wait(30.0)
        finally:
            tk.release()
        assert r["sequence_output"].tobytes() == full["sequence_output"].tobytes() and r["cls_embedding"].tobytes() == full["cls_embedding"].tobytes()
        # gRPC Predict: every output, or those output_filter names; sequence_output is [B, S, H]
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("es", 1, x)))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        assert outs["sequence_output"].shape == (B, S, H)
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("es", 1, x, output_filter=["sequence_output"])))
        assert list(outs) == ["sequence_output"] and outs["sequence_output"].shape == (B, S, H)
        assert outs["sequence_output"].tobytes() == full["sequence_output"].tobytes()
        # REST, row and columnar: nested lists for the rank-2 output
        st, b = srv.rest_handle("POST", "/v1/models/es/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        assert len(preds) == B and all(list(p) == NAMES for p in preds)
        for i, p in enumerate(preds):
            assert np.array_equal(np.float32(p["sequence_output"]), full["sequence_output"][i])
            assert np.array_equal(np.float32(p["mean_embedding"]), full["mean_embedding"][i])
        st, b = srv.rest_handle("POST", "/v1/models/es/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES
        assert all(np.array_equal(np.float32(cols[k]), full[k]) for k in NAMES)
        # metadata
        st, b = srv.rest_handle("GET", "/v1/models/es/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {k: ("DT_FLOAT", ["-1", str(H)]) for k in NAMES}
        want["sequence_output"] = ("DT_FLOAT", ["-1", str(S), str(H)])
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        # SessionRun takes one feed, so it refuses a three-input bundle and names its inputs; Classify refuses it too
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(_session_run_request("es", "input_ids:0", x["input_ids"], "mean_embedding:0"))
        assert e.value.code == t._lib.E_INVALID and "'input_mask'" in str(e.value) and "'segment_ids'" in str(e.value)
        st, b = srv.rest_handle("POST", "/v1/models/es/versions/1:classify", json.dumps({"examples": [{"x": 1.0}]}).encode())
        assert st == 400
        # tfsc_predict_device writes packed rows; split_packed_rows cuts them, sequence_output as [B, S, H]
        srv.ensure(0, "es", 1)
        layout = mf.packed_output_layout(ALL, H, S)
        width = sum(w for _n, _o, w, _d in layout)
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.BERT_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "es", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), ALL, H, S)
        for k in NAMES:
            assert dev[k].shape == full[k].shape and dev[k].tobytes() == full[k].tobytes(), k


@pytest.mark.parametrize("pooler", [True, False])
def test_launch_counts(tmp_path, pooler):
    """An encoder bundle launches exactly one kernel more per batch than the same weights with one output"""
    S = 64
    _write_enc(tmp_path, S, SMALL, 74, pooler=pooler)
    names = [o["name"] for o in _outputs(pooler, False)]
    for rows in (1, 8):
        x = sr.qa_inputs(rows, S, SMALL["vocab"], seed=rows, sep_id=SEP)
        with t.Server(_cfg(tmp_path)) as srv:
            srv.predict("e1", "1", x)
            srv.predict("es", "1", x, outputs=names)
            counts = {}
            for name in ("e1", "es"):
                s0 = srv.stats()
                srv.predict(name, "1", x, outputs=None if name == "e1" else names)
                s1 = srv.stats()
                counts[name] = (s1["kernel_launches"] - s0["kernel_launches"], s1["batches"] - s0["batches"])
            assert counts["e1"][1] == counts["es"][1] >= 1
            assert counts["es"][0] == counts["e1"][0] + counts["es"][1], (rows, counts)


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_encoder as g
import span_ref as sr
tmp = sys.argv[2]
g._write_enc(tmp, 384, g.SMALL, 75)
g._write_enc(tmp, 128, g.SMALL, 76, pooler=False, norm_mean=True, single="n1", multi="ns")
out = {}
with t.Server(g._cfg(tmp)) as srv:
    for rows in (1, 8):
        for name, S in (("es", 384), ("ns", 128)):
            x = sr.qa_inputs(rows, S, g.SMALL["vocab"], seed=rows, sep_id=g.SEP)
            names = g.NAMES if name == "es" else [n for n in g.NAMES if n != "pooled_output"]
            for k, v in srv.predict(name, "1", x, outputs=names).items():
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
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 2 * (2 * len(NAMES) - 1)
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key


# --------------------------------------------------------------------------------------- forward hop ----
N_MODELS = 4
HOP_S, HOP_ROWS = 128, 6          # 6 rows of sequence_output [128, 64]: 197 KB, more than half the default slot


def _rank_cfg(rank, world, socks, base):
    members = [f"gpu{i}:0:0" for i in range(world)]
    return {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": base, "gpu.devices": [0],
            "gpu.arenaBytes": 256 << 20, "modelCache.size": 1 << 30, "serving.maxConcurrentModels": 16, "gpu.members": members,
            "gpu.localMembers": [members[rank]], "proxy.replicasPerModel": 1, "proxy.replicaPick": "first", "cluster.rank": rank,
            "cluster.endpoints": socks, "cluster.slotBytes": 4 << 20, "cluster.windowSlots": 8, "proxy.grpcTimeout": 60.0}


def _rank_main(rank, world, socks, base, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}, "ticket": {}}
        with t.Server(_rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = sr.qa_inputs(HOP_ROWS, HOP_S, SMALL["vocab"], seed=7, sep_id=SEP)
            for j in range(N_MODELS):
                name = f"es{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=NAMES)
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, x)))
                res["grpc"][j] = dict(outs)
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict",
                                        json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
                res["rest"][j] = (st, b.decode())
                tk = srv.predict_submit(name, "1", x, outputs=["sequence_output", "mean_embedding"])
                try:
                    res["ticket"][j] = tk.wait(60.0)
                finally:
                    tk.release()
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


def test_forward_hop_embeddings():
    import torch
    assert torch.cuda.is_available()
    world = 2
    base = tempfile.mkdtemp(prefix="tfscenc")
    for j in range(N_MODELS):
        _write_enc(base, HOP_S, SMALL, 80 + j, single=f"e1_{j}", multi=f"es{j}")
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
        assert sorted(local["y"][j]) == NAMES and local["y"][j]["sequence_output"].shape == (HOP_ROWS, HOP_S, SMALL["hidden"])
        for k in NAMES:
            assert fwd["y"][j][k].shape == local["y"][j][k].shape and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].shape == local["grpc"][j][k].shape
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
        for k in ("sequence_output", "mean_embedding"):
            assert fwd["ticket"][j][k].tobytes() == local["ticket"][j][k].tobytes()
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
