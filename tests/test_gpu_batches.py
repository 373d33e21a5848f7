"""-m gpu: the batch sizes a small request never reaches. The batch size picks the kernels (Node::run_model and the
launchers): below 64 rows a plain classifier Dense runs on launch_dense, from 64 on launch_gemm runs it (gemm_tc for
N % 32 == 0, else the SIMT gemm_f32); BERT's pooler (act 3, lda = S*H) runs on gemm_f32 below 64 rows and on gemm_tc,
whose A map then strides S*H*4 bytes, from 64 on; gemm_tc's tile width and split-K and the implicit-GEMM conv's
M >= 64 rule all follow M = B*OH*OW.

* the raw kernels past CUDA's 65,535 cap on gridDim.y: the launchers split such a batch on the host;
* every served family at 63, 64, 65 and 128 rows against fp64, full-size ResNet-50 and BERT-base at 64;
* full-size image nets at 668 rows (the last batch whose 112 x 112 stem GEMM fits one grid) and 700 rows (past it);
* requests coalesced into one batch give the bits of the same rows sent as one request.
Tolerance 1e-4 relative to max(1, |ref|), as the rest of the suite."""
import copy
import os
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import models

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import convnet_export as ce  # noqa: E402
import embed_ref as er  # noqa: E402
import make_bert_pair_golden as pg  # noqa: E402
import mlm_export as me  # noqa: E402
import mlm_ref as mr  # noqa: E402
import span_ref as sr  # noqa: E402
import swin_export as se  # noqa: E402
import test_gpu_attention as ga  # noqa: E402
import test_gpu_encoder as genc  # noqa: E402
import test_gpu_mlm as gm  # noqa: E402
import test_gpu_outputs as go  # noqa: E402
import test_gpu_spans as gs  # noqa: E402
import torch_export as te  # noqa: E402

pytestmark = pytest.mark.gpu
lib = t._lib.lib
mf = t.modelformat
TOL = 1e-4
K = go.K
CLASSIFY, CLASSIFY_NAMES = go.FULL, go.NAMES
SMALL = dict(hidden=64, layers=2, heads=4, inter=128, vocab=100, max_pos=512)
SWIN_SMALL = dict(embed_dim=32, depths=(2, 2), heads=(1, 2))
S = 128                            # BERT sequence length of the served cases
GRID_Y = 65535                     # CUDA's cap on gridDim.y
CHUNK_ROWS = GRID_Y * 128          # rows of one gemm_tc / gemm_f32 launch (128-row tiles along y)


def _torch():
    import torch
    assert torch.cuda.is_available()
    return torch


def _ptr(x):
    return None if x is None else x.data_ptr()


def _err(got, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))))


# ---------------------------------------------------------------------------- kernels past the grid limit ----
def _boundary_rows(M, seed):
    """every row of the first tile, of the tiles on both sides of the first launch boundary and of the last tile, plus 256
    random rows"""
    rng = np.random.default_rng(seed)
    idx = np.concatenate([np.arange(0, 128), np.arange(CHUNK_ROWS - 128, CHUNK_ROWS + 128), np.arange(M - 128, M),
                          rng.integers(0, M, 256)])
    return np.unique(idx)


def _gemm_past_the_limit(fn, n, lda, act, seed):
    """C = act(A[:, :64] B + bias + A) over M = 65,535 * 128 + 300 rows; R aliases A (n == lda), so the residual's chunk
    offset is checked without another 2 GB"""
    torch = _torch()
    M, k = CHUNK_ROWS + 300, 64
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, lda, device="cuda", generator=g)
    b = torch.randn(k, n, device="cuda", generator=g) / 8
    bias = torch.randn(n, device="cuda", generator=g)
    c = torch.full((M, n), float("nan"), device="cuda")
    t._lib.check(fn(_ptr(a), _ptr(b), _ptr(bias), _ptr(a), _ptr(c), M, n, k, lda, act, None), fn.__name__)
    torch.cuda.synchronize()
    idx = torch.from_numpy(_boundary_rows(M, seed)).cuda()
    a64 = a[idx].double().cpu().numpy()
    got = c[idx].cpu().numpy()
    ref = a64[:, :k] @ b.double().cpu().numpy() + bias.double().cpu().numpy() + a64
    if act == 1:
        ref = np.maximum(ref, 0)
    del a, c
    torch.cuda.empty_cache()
    assert not np.isnan(got).any() and _err(got, ref) <= TOL, _err(got, ref)


def test_k_gemm_tc_past_the_grid_limit():
    _gemm_past_the_limit(lib.tfsc_k_gemm_tc, 64, 64, 0, 1)


def test_k_gemm_past_the_grid_limit():
    """n = 72 (n % 32 != 0) keeps tfsc_k_gemm on the SIMT gemm_f32 kernel; at n = 64 it would take gemm_tc, as above"""
    _gemm_past_the_limit(lib.tfsc_k_gemm, 72, 72, 1, 2)


@pytest.mark.parametrize("with_res", [False, True])
def test_k_conv_tc_past_the_grid_limit(with_res):
    """670 images of 112 x 112 x 32 -> 64, 3 x 3, pad 1: 670 * 12,544 output pixels need more than 65,535 row tiles, so
    the conv runs as 668 images and then 2; images 0, 667 | 668 and 669 against fp64 conv2d of those images alone"""
    torch = _torch()
    B, H, C, N = 670, 112, 32, 64
    g = torch.Generator(device="cuda").manual_seed(3 + with_res)
    x = torch.randn(B, H, H, C, device="cuda", generator=g)
    w = torch.randn(3, 3, C, N, device="cuda", generator=g) / np.sqrt(9 * C)
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(B, H, H, N, device="cuda", generator=g) if with_res else None
    y = torch.full((B, H, H, N), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_conv_tc(_ptr(x), _ptr(w), _ptr(b), _ptr(r), _ptr(y), B, H, H, C, 3, 3, 1, 1, N, 1, None), "conv_tc")
    torch.cuda.synchronize()
    pick = [0, 667, 668, 669]
    ref = torch.nn.functional.conv2d(x[pick].double().permute(0, 3, 1, 2), w.double().permute(3, 2, 0, 1), b.double(), padding=1)
    ref = ref.permute(0, 2, 3, 1)
    if with_res:
        ref = ref + r[pick].double()
    ref = torch.relu(ref).cpu().numpy()
    got = y[pick].cpu().numpy()
    del x, r, y
    torch.cuda.empty_cache()
    assert not np.isnan(got).any() and _err(got, ref) <= TOL, _err(got, ref)


@pytest.mark.parametrize("seq,check", [(13, None), (300, [0, 1, 2, 3, 4094, 4095, 4096, 4097, 4099])])
def test_k_attention_past_the_grid_limit(seq, check):
    """4,100 sequences x 16 heads = 65,600 (sequence, head) CTAs along y: the launcher runs 4,095 sequences and then 5.
    S = 13 takes the tiled kernel (the whole output is compared), S = 300 the key-block kernel (sequences on both sides
    of the split, every mask kind of ga._ids among them)."""
    torch = _torch()
    B, heads, d = 4100, 16, 4
    H = heads * d
    rng = np.random.default_rng(seq)
    g = torch.Generator(device="cuda").manual_seed(seq)
    qkv = torch.randn(B, seq, 3 * H, device="cuda", generator=g)
    qkv[..., :2 * H] *= 2.0                           # scores with a standard deviation of 4, as test_gpu_attention
    ids = ga._ids(rng, B, seq)
    idd = torch.from_numpy(ids).cuda()
    ctx = torch.full((B, seq, H), float("nan"), device="cuda")
    t._lib.check(lib.tfsc_k_attention(_ptr(qkv), _ptr(idd), _ptr(ctx), B, seq, H, heads, None), "attention")
    torch.cuda.synchronize()
    pick = list(range(B)) if check is None else check
    got = ctx[pick].cpu().numpy()
    ref = models.attention_ref(qkv[pick].double().cpu(), torch.from_numpy(ids[pick]), heads).numpy()
    del qkv, ctx
    torch.cuda.empty_cache()
    assert not np.isnan(got).any() and _err(got, ref) <= TOL, _err(got, ref)


# ---------------------------------------------------------------------------------------- served models ----
def _cfg(tmp, **kw):
    cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": str(tmp), "gpu.devices": [0],
           "gpu.arenaBytes": 1 << 30, "serving.maxConcurrentModels": 16, "modelCache.size": 4 << 30, "gpu.maxBatch": 128}
    cfg.update(kw)
    return cfg


def _vision64(m, x):
    """a torchvision model's own forward in fp64 on the GPU, NHWC fp32 input"""
    torch = _torch()
    m64 = copy.deepcopy(m).double().cuda()
    with torch.no_grad():
        return m64(torch.from_numpy(np.ascontiguousarray(x)).cuda().double().permute(0, 3, 1, 2)).cpu().numpy()


def _bert64(m, x):
    """a transformers model's own forward in fp64 on the GPU with explicit attention mask and segment ids"""
    torch = _torch()
    m64 = copy.deepcopy(m).double().cuda()
    tt = {k: torch.from_numpy(np.ascontiguousarray(v, np.int64)).cuda() for k, v in x.items()}
    with torch.no_grad():
        return m64(input_ids=tt["input_ids"], attention_mask=tt["input_mask"], token_type_ids=tt["segment_ids"])


def _topk_vs_fp64(ids, ref, tag):
    """top-k ids equal fp64's wherever the neighbouring fp64 logits are further apart than 2e-4"""
    for i in range(ref.shape[0]):
        srt = np.sort(ref[i])[::-1][:K + 1]
        rid = np.argsort(-ref[i], kind="stable")[:K]
        tol = 2e-4 * np.maximum(1.0, np.abs(srt))
        for j in range(K):
            if srt[j] - srt[j + 1] > tol[j] and (j == 0 or srt[j - 1] - srt[j] > tol[j]):
                assert ids[i, j] == rid[j], (tag, i, j)


def _check_classified(r, ref, tag):
    assert sorted(r) == CLASSIFY_NAMES and r["logits"].shape == ref.shape
    assert _err(r["logits"], ref) <= TOL, (tag, _err(r["logits"], ref))
    assert np.max(np.abs(r["probabilities"] - go._softmax64(ref))) <= TOL, tag
    go._check_head(r["logits"], r)                    # classes / top-k exact on the served logits
    _topk_vs_fp64(r["top_k_classes"], ref, tag)


def _check_spans(r, x, ref, tag):
    for name in ("start_logits", "end_logits"):
        assert _err(r[name], ref[name]) <= TOL, (tag, name, _err(r[name], ref[name]))
    gs._check_spans(r, x)                             # the spans of the served logits, bit for bit
    el = sr.eligible(x["input_ids"], x["input_mask"], x["segment_ids"], gs.SEP)
    s64, e64, v64 = sr.span_ref(ref["start_logits"], ref["end_logits"], el, gs.L, gs.K + 1, dtype=np.float64)
    for b in range(len(s64)):                         # and of the fp64 logits, wherever the score gap exceeds the tolerance
        for j in range(gs.K):
            if s64[b, j + 1] >= 0 and v64[b, j] - v64[b, j + 1] <= 4e-4 * max(1.0, abs(v64[b, j])):
                break
            assert (r["span_starts"][b, j], r["span_ends"][b, j]) == (s64[b, j], e64[b, j]), (tag, b, j)


def _check_embeddings(r, x, ref, tag):
    h64, p64 = ref
    genc._close(r["sequence_output"], h64, np.abs(h64), TOL)
    assert r["cls_embedding"].tobytes() == np.ascontiguousarray(r["sequence_output"][:, 0]).tobytes(), tag
    mean64 = er.mean_embedding(h64, x["input_ids"], x["input_mask"])
    genc._close(r["mean_embedding"], mean64, np.abs(mean64), TOL)
    genc._close(r["pooled_output"], p64, np.abs(p64), TOL)


def _check_fill_mask(r, x, ref, tag):
    tok, M, V = gm.MASK_SMALL, MLM_SLOTS, SMALL["vocab"]
    bs = len(x["input_ids"])
    want_pos, _ = mr.mask_gather_ref(np.zeros((bs, S, 1)), x["input_ids"], x["input_mask"], tok, M)
    pos = r["masked_positions"]
    assert np.array_equal(pos, want_pos) and (pos >= 0).any(), tag
    refl = np.stack([ref[i, np.maximum(pos[i], 0)] for i in range(bs)])
    rid, _rp, _rl = mr.top_k_ref(refl, pos, V, gm.K)
    ids = r["masked_top_k_ids"]
    for i in range(bs):
        for s in range(M):
            if pos[i, s] < 0:
                assert (ids[i, s] == -1).all(), (tag, i, s)
                continue
            want = refl[i, s, ids[i, s]]
            assert np.all(np.abs(r["masked_top_k_logits"][i, s].astype(np.float64) - want) <= TOL * np.maximum(1.0, np.abs(want))), (tag, i, s)
            srt = np.sort(refl[i, s])[::-1][:gm.K + 1]
            tol = 2e-4 * np.maximum(1.0, np.abs(srt))
            for j in range(gm.K):
                if srt[j] - srt[j + 1] > tol[j] and (j == 0 or srt[j - 1] - srt[j] > tol[j]):
                    assert ids[i, s, j] == rid[i, s, j], (tag, i, s, j)


MLM_SLOTS = 3


class Family:
    """one served bundle: its name, its outputs, seeded inputs of any batch, the fp64 reference of them and the check"""

    def __init__(self, name, outputs, inputs, reference, check):
        self.name, self.outputs, self.inputs, self.reference, self.check = name, outputs, inputs, reference, check


def _write_families(tmp):
    """One bundle per family. Routes at 63 | 64+ rows (run_model): the convnet / Swin classifiers (Dense, act 0, N = 10)
    launch_dense | gemm_f32 (N % 32 != 0); their conv / 1x1 GEMMs are on gemm_tc at every batch here (M = B*OH*OW >= 64)
    with pick_bn and split-K following M. BERT: QKV / FFN GEMMs gemm_tc at every batch (M = B*S); the pooler (act 3,
    lda = S*H) gemm_f32 | gemm_tc (N = H = 64); the classifier (N = 6) launch_dense | gemm_f32; the QA projection and the
    fill-mask decoder are 1x1 convs over B*S (resp. B*slots) rows."""
    fams = {}
    vision = {
        "resnet": (te.torchvision_resnet(61, classes=10), lambda: mf.resnet50_manifest(image=64, classes=10),
                   lambda outs: mf.resnet50_manifest(image=64, classes=10, outputs=outs), 64),
        "mobilenet_v2": (ce.torchvision_mobilenet_v2(62, 0.35, 10), None,
                         lambda outs: mf.mobilenet_v2_manifest(64, 10, 0.35, outs), 64),
        "efficientnet": (ce.torchvision_efficientnet(63, 0.5, 0.5, 10), None,
                         lambda outs: mf.efficientnet_manifest(64, 10, 0.5, 0.5, outs), 64),
        "swin": (se.torchvision_swin(64, classes=10, **SWIN_SMALL), None,
                 lambda outs: mf.swin_manifest(image=56, classes=10, outputs=outs, **SWIN_SMALL), 56),
    }
    for fam, (m, single, man, image) in vision.items():
        mm = man(CLASSIFY)
        if fam == "resnet":
            blob = te.export_resnet(m, single())
        elif fam == "swin":
            blob = se.export_swin(m, mm)
        else:
            blob = ce.export_convnet(m, mm)
        mf.write_graph_bundle(os.path.join(str(tmp), fam, "1"), mm, blob)
        fams[fam] = Family(fam, CLASSIFY_NAMES, lambda B, seed, image=image: ce.images(B, image, seed),
                           lambda x, m=m: _vision64(m, x), lambda r, x, ref, tag: _check_classified(r, ref, tag))
    arch = dict(SMALL, labels=6)
    m = te.hf_bert(65, **arch)
    blob = te.export_bert(m, mf.bert_manifest(seq=S, **arch, inputs=mf.BERT_INPUTS))
    mf.write_graph_bundle(os.path.join(str(tmp), "bert", "1"), mf.bert_manifest(seq=S, **arch, inputs=mf.BERT_INPUTS, outputs=CLASSIFY), blob)
    fams["bert"] = Family("bert", CLASSIFY_NAMES, lambda B, seed: pg.pair_inputs(B, S, SMALL["vocab"], seed=seed),
                          lambda x, m=m: _bert64(m, x).logits.cpu().numpy(), lambda r, x, ref, tag: _check_classified(r, ref, tag))
    m = gs._write_qa(tmp, S, SMALL, 66, single="bert_qa1", multi="bert_qa")
    fams["bert_qa"] = Family("bert_qa", gs.NAMES, lambda B, seed: sr.qa_inputs(B, S, SMALL["vocab"], seed=seed, sep_id=gs.SEP),
                             lambda x, m=m: {k: getattr(_bert64(m, x), k).cpu().numpy() for k in ("start_logits", "end_logits")},
                             _check_spans)
    m = genc._write_enc(tmp, S, SMALL, 67, pooler=True, single="bert_embed1", multi="bert_embed")
    fams["bert_embed"] = Family("bert_embed", sorted(o["name"] for o in genc._outputs(True, False)),
                                lambda B, seed: sr.qa_inputs(B, S, SMALL["vocab"], seed=seed, sep_id=genc.SEP),
                                lambda x, m=m: tuple(v.cpu().numpy() for v in (lambda o: (o.last_hidden_state, o.pooler_output))(_bert64(m, x))),
                                _check_embeddings)
    m = gm._write_mlm(tmp, S, SMALL, 68, MLM_SLOTS, gm.MASK_SMALL, name="bert_mlm")
    fams["bert_mlm"] = Family("bert_mlm", gm.NAMES,
                              lambda B, seed: mr.mlm_inputs(B, S, SMALL["vocab"], MLM_SLOTS + 2, seed=seed, mask_token_id=gm.MASK_SMALL),
                              lambda x, m=m: me.mlm_reference(m, x["input_ids"], x["input_mask"], x["segment_ids"]), _check_fill_mask)
    return fams


@pytest.fixture(scope="module")
def families(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("families")
    return tmp, _write_families(tmp)


def _rows(x, lo, hi):
    return {k: v[lo:hi] for k, v in x.items()} if isinstance(x, dict) else x[lo:hi]


FAMILIES = ["resnet", "mobilenet_v2", "efficientnet", "swin", "bert", "bert_qa", "bert_embed", "bert_mlm"]


@pytest.mark.parametrize("fam", FAMILIES)
def test_route_boundaries_against_fp64(families, fam):
    """one request of 63, 64, 65 and 128 rows (gpu.maxBatch 128): both sides of the 64-row route switch and a two-tile M"""
    tmp, fams = families
    f = fams[fam]
    x = f.inputs(128, 7)
    ref = f.reference(x)
    with t.Server(_cfg(tmp)) as srv:
        for B in (63, 64, 65, 128):
            xb = _rows(x, 0, B)
            r = srv.predict(f.name, "1", xb, outputs=f.outputs)
            refb = tuple(v[:B] for v in ref) if isinstance(ref, tuple) else \
                {k: v[:B] for k, v in ref.items()} if isinstance(ref, dict) else ref[:B]
            f.check(r, xb, refb, (fam, B))


@pytest.mark.parametrize("kind", ["resnet50", "bert_base"])
def test_full_size_at_64_rows(kind, tmp_path):
    """the bench's extra models at 64 rows. ResNet-50: the classifier (N = 1000) leaves launch_dense for gemm_f32, the
    stem GEMM and every conv stay on gemm_tc. BERT-base: the pooler (N = 768, lda = 128*768) moves from gemm_f32 to gemm_tc
    with its strided A map, the classifier (N = 6) from launch_dense to gemm_f32."""
    if kind == "resnet50":
        m = te.torchvision_resnet(5)
        blob = te.export_resnet(m, mf.resnet50_manifest())
        mf.write_graph_bundle(str(tmp_path / "m" / "1"), mf.resnet50_manifest(outputs=CLASSIFY), blob)
        x = ce.images(64, 224, 8)
        ref = _vision64(m, x)
    else:
        arch = dict(max_pos=512, labels=6)
        m = te.hf_bert(3, **arch)
        blob = te.export_bert(m, mf.bert_manifest(seq=S, **arch, inputs=mf.BERT_INPUTS))
        mf.write_graph_bundle(str(tmp_path / "m" / "1"), mf.bert_manifest(seq=S, **arch, inputs=mf.BERT_INPUTS, outputs=CLASSIFY), blob)
        x = pg.pair_inputs(64, S, 30522, seed=9)
        ref = _bert64(m, x).logits.cpu().numpy()
    with t.Server(_cfg(tmp_path, **{"gpu.arenaBytes": 2 << 30})) as srv:
        _check_classified(srv.predict("m", "1", x, outputs=CLASSIFY_NAMES), ref, kind)


# ------------------------------------------------------------------------------------------ large requests ----
def _device_used_bytes():
    free, total = _torch().cuda.mem_get_info()
    return total - free


@pytest.mark.parametrize("net", ["resnet50", "mobilenet_v2", "efficientnet"])
def test_large_requests(net, tmp_path):
    """668 rows: the last batch whose 112 x 112 stem GEMM (and MobileNet's 1 x 1 convs at 112 x 112) fits 65,535 row tiles;
    700 rows: past it, split by the launchers. Sampled rows against fp64 of those images alone; MobileNetV2's 700 rows
    also through tfsc_predict_device (the per-stream scratch), bit for bit the Predict's. Device memory in use, whole
    device (H100 80GB HBM3, 700 W power limit): ResNet-50 at 700 rows 19.4 GiB, MobileNetV2 with both scratches 31.5 GiB,
    the most this file needs."""
    torch = _torch()
    if net == "resnet50":
        m = te.torchvision_resnet(11)
        man = mf.resnet50_manifest()
        blob = te.export_resnet(m, man)
    elif net == "mobilenet_v2":
        m = ce.torchvision_mobilenet_v2(12)
        man = mf.mobilenet_v2_manifest()
        blob = ce.export_convnet(m, man)
    else:
        m = ce.torchvision_efficientnet(13)
        man = mf.efficientnet_manifest()
        blob = ce.export_convnet(m, man)
    mf.write_graph_bundle(str(tmp_path / "m" / "1"), man, blob)
    x = ce.images(700, 224, 14)
    rng = np.random.default_rng(15)
    # one slot: a batch's scratch (~15 GB for ResNet-50 at 700 rows) is allocated once
    with t.Server(_cfg(tmp_path, **{"gpu.arenaBytes": 512 << 20, "gpu.maxBatch": 64, "gpu.stagingSlots": 1})) as srv:
        for rows in (668, 700):
            y = srv.predict("m", "1", x[:rows])
            print(f"{net} {rows} rows: device memory in use {_device_used_bytes() / 2**30:.2f} GiB")
            pick = sorted({0, 1, rows - 1, 667, 668 if rows > 668 else 0} | set(rng.integers(0, rows, 8).tolist()))
            ref = _vision64(m, x[pick])
            assert y.shape == (rows, 1000) and _err(y[pick], ref) <= TOL, (net, rows, _err(y[pick], ref))
        if net == "mobilenet_v2":
            srv.ensure(0, "m", 1)
            xd = torch.from_numpy(x).cuda()
            yd = torch.full((700, 1000), float("nan"), device="cuda")
            srv.predict_device(0, "m", 1, _ptr(xd), 700, _ptr(yd), 0)
            srv.sync(0)
            print(f"{net} 700 rows + predict_device: device memory in use {_device_used_bytes() / 2**30:.2f} GiB")
            assert yd.cpu().numpy().tobytes() == y.tobytes()


# ------------------------------------------------------------------------------------------------ coalescing ----
COALESCED = ["bert", "bert_qa", "bert_embed", "bert_mlm", "mobilenet_v2", "swin"]
TICK_US = 3_000_000                 # a partial batch waits 3 s for more rows: far longer than submitting a few tickets


def _bits(r):
    return {k: (v.dtype.str, v.shape, v.tobytes()) for k, v in r.items()}


def _slice_bits(r, lo, hi):
    return {k: (v.dtype.str, v[lo:hi].shape, np.ascontiguousarray(v[lo:hi]).tobytes()) for k, v in r.items()}


def _coalesce(srv, f, x, sizes, expired_at=None):
    """submit tickets of `sizes` rows in order from this thread (and, before ticket `expired_at`, one whose deadline has
    passed); returns each ticket's outputs, the stats deltas and the expired ticket's error code"""
    st0 = srv.stats()
    tickets, lo, code = [], 0, None
    for i, n in enumerate(sizes):
        if i == expired_at:
            dead = srv.predict_submit(f.name, "1", _rows(x, 0, 4), deadline_ns=max(1, srv.now_ns() - 1), outputs=f.outputs)
        tickets.append(srv.predict_submit(f.name, "1", _rows(x, lo, lo + n), outputs=f.outputs))
        lo += n
    if expired_at is not None:
        with pytest.raises(t._lib.TfscError) as e:
            dead.wait(30.0)
        code = e.value.code
        dead.release()
    outs = [tk.wait(30.0) for tk in tickets]
    [tk.release() for tk in tickets]
    st1 = srv.stats()
    return outs, st1["batches"] - st0["batches"], st1["batched_rows"] - st0["batched_rows"], code


@pytest.mark.parametrize("case", ["40+24", "1+62", "5+5", "3+20+3", "40+expired+24"])
def test_coalesced_requests_give_the_bits_of_one_request(families, case):
    """gpu.maxBatch is the rows of the batch the tickets should form, so the batcher holds a partial batch until they are
    all queued and serves them in arrival order. Each ticket's outputs are its slice of one request of the batch's rows."""
    tmp, fams = families
    sizes = [int(s) for s in case.replace("+expired", "").split("+")]
    expired_at = 1 if "expired" in case else None
    if case == "5+5":                    # two batches of 5: each is a 5-row request
        max_batch, batches = 8, [[0], [1]]
    elif case == "3+20+3":               # the 20-row ticket does not fit a batch of 8 next to a 3: it runs alone
        max_batch, batches = 8, [[0], [1], [2]]
    else:
        max_batch, batches = sum(sizes), [list(range(len(sizes)))]
    with t.Server(_cfg(tmp, **{"gpu.maxBatch": max_batch, "gpu.tickMicros": TICK_US})) as srv, \
            t.Server(_cfg(tmp, **{"gpu.maxBatch": 128})) as one:
        for fam in COALESCED:
            f = fams[fam]
            x = f.inputs(sum(sizes), 21)
            srv.predict(f.name, "1", _rows(x, 0, max_batch), outputs=f.outputs)     # resident; a full batch does not wait
            outs, n_batches, n_rows, code = _coalesce(srv, f, x, sizes, expired_at)
            assert (n_batches, n_rows) == (len(batches), sum(sizes)), (fam, case, n_batches, n_rows)
            if expired_at is not None:
                assert code == t._lib.E_TIMEOUT, (fam, code)
            starts = np.cumsum([0] + sizes)
            for group in batches:
                lo, hi = starts[group[0]], starts[group[-1] + 1]
                whole = one.predict(f.name, "1", _rows(x, lo, hi), outputs=f.outputs)
                for i in group:
                    want = _slice_bits(whole, starts[i] - lo, starts[i + 1] - lo)
                    assert _bits(outs[i]) == want, (fam, case, i)
