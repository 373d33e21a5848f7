"""-m gpu: GPT-2 generate bundles. Decode attention against fp64 on both sides of every key-block boundary and bit for bit
(the appended slot, batch independence, the scalar path, hidden and masked keys), the select step against fp64 and bit for
bit against tfsc_k_embed_positions, a full-size seeded GPT-2 small through the server teacher-forced against transformers
fp64, every front-end, coalesced batches, launch counts, programmatic-dependent-launch bit identity and the forward hop."""
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
import gpt2_export as ge  # noqa: E402
import gpt2_ref as gr  # noqa: E402
import test_gpu_gpt2 as g2  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
SMALL = g2.SMALL
N = 6


def _outs(n=N, eos=None):
    return [dict({"name": k, "kind": k, "max_new_tokens": n}, **({} if eos is None else {"eos_token_id": eos}))
            for k in mf.GENERATE_OUTPUT_KINDS]


NAMES = sorted(mf.GENERATE_OUTPUT_KINDS)


def _ptr(x):
    return None if x is None else x.data_ptr()


def _cuda(a, dtype=np.float32, off=0):
    """a device copy of `a`, starting `off` elements into its allocation (off = 1: not 16-byte aligned)"""
    import torch
    flat = np.concatenate([np.zeros(off, dtype), np.ascontiguousarray(a, dtype).ravel()])
    return torch.from_numpy(flat).cuda()[off:]


# ------------------------------------------------------------------------------------- decode attention ----
def _decode_case(L, d, heads, spread, seed):
    """Four rows over one launch of L = S + t + 1 keys: unpadded, right-padded, left-padded and fully padded prompts of S
    tokens. Returns the full per-row sequences' qkv [4, L, 3H], the prompt mask [4, S], pos [4], S and t."""
    rng = np.random.default_rng(seed)
    H = heads * d
    t_ = (L - 1) // 2
    S = L - 1 - t_
    qkv = rng.standard_normal((4, L, 3 * H)).astype(np.float32)
    qkv[..., :2 * H] *= spread ** 0.5 / d ** 0.25 / 2
    mask = np.ones((4, S), np.int32)
    n = max(1, S // 3)
    if S > 1:
        mask[1, S - n:] = 0
        mask[2, :n] = 0
    mask[3] = 0
    pos = np.array([max(np.nonzero(m)[0]) if m.any() else -1 for m in mask], np.int32)
    return qkv, mask, pos, S, t_


def _decode(qkv_full, mask, pos, S, t_, heads, T=None, use_mask=True, off=0, kc_fill=None):
    """runs tfsc_k_decode_attention for every row's query at slot q = pos + 1 + t, with the cache holding keys 0..q-1 (and
    kc_fill, if given, in every slot the query does not see). Returns ctx [rows, H], kc, vc [rows, T, H]"""
    import torch
    B, L, H3 = qkv_full.shape
    H = H3 // 3
    T = T or S + t_ + 1
    kc = np.full((B, T, H), np.nan, np.float32) if kc_fill is None else kc_fill[0].copy()
    vc = np.full((B, T, H), np.nan, np.float32) if kc_fill is None else kc_fill[1].copy()
    step = np.zeros((B, 3 * H), np.float32)
    for b in range(B):
        q = pos[b] + 1 + t_
        kc[b, :q] = qkv_full[b, :q, H:2 * H]
        vc[b, :q] = qkv_full[b, :q, 2 * H:]
        step[b] = qkv_full[b, q]
    qd, kd, vd = _cuda(step, off=off), _cuda(kc, off=off), _cuda(vc, off=off)
    pd, md = _cuda(pos, np.int32), _cuda(mask, np.int32)
    ctx = torch.full((B * H,), float("nan"), device="cuda")
    wb = lib.tfsc_k_decode_attention_work_bytes(B, S + t_ + 1, H, heads)
    work = torch.zeros(wb // 4 + 1, dtype=torch.int32, device="cuda")
    t._lib.check(lib.tfsc_k_decode_attention(_ptr(qd), _ptr(kd), _ptr(vd), _ptr(pd), t_, _ptr(md) if use_mask else None, S, S, T,
                                             _ptr(ctx), B, H, heads, _ptr(work), wb, None), "decode_attention")
    torch.cuda.synchronize()
    assert not work[:B * heads].any()                                          # the counters are left zero
    return ctx.cpu().numpy().reshape(B, H), kd.cpu().numpy().reshape(B, T, H), vd.cpu().numpy().reshape(B, T, H)


def _decode_ref(qkv_full, mask, pos, t_, heads, use_mask=True):
    B, _L, H3 = qkv_full.shape
    out = np.zeros((B, H3 // 3))
    for b in range(B):
        q = pos[b] + 1 + t_
        m = np.ones(q + 1, np.int32)
        if use_mask and pos[b] >= 0:
            m[:pos[b] + 1] = mask[b, :pos[b] + 1]
        out[b] = gr.causal_attention_ref(qkv_full[b:b + 1, :q + 1].astype(np.float64), heads, m[None])[0, q]
    return out


@pytest.mark.parametrize("d", [4, 16, 64, 128])
@pytest.mark.parametrize("L", [2, 3, 63, 64, 65, 66, 127, 128, 129, 130, 513, 1023, 1024, 1025, 2049])
def test_decode_attention_matches_fp64(L, d):
    """at L = 2049 the right- and fully padded rows' queries sit 16 blocks before the launch's last key block; at d = 4 that
    is farther than the CTA's staged keys reach, so a block past the query must touch nothing"""
    heads = 2
    for spread in (3.0, 30.0):
        qkv, mask, pos, S, t_ = _decode_case(L, d, heads, spread, L * 7 + d)
        for use_mask in (True, False):
            ctx, kc, vc = _decode(qkv, mask, pos, S, t_, heads, use_mask=use_mask)
            ref = _decode_ref(qkv, mask, pos, t_, heads, use_mask)
            err = np.abs(ctx - ref).max()
            assert err <= 2e-5 * max(1.0, np.abs(ref).max()), (spread, use_mask, err)
            H = heads * d
            for b in range(4):                                         # the appended slot: a bit-exact copy of k and v
                q = pos[b] + 1 + t_
                assert kc[b, q].tobytes() == qkv[b, q, H:2 * H].tobytes() and vc[b, q].tobytes() == qkv[b, q, 2 * H:].tobytes()


@pytest.mark.parametrize("d", [4, 64])
def test_decode_attention_single_key(d):
    """L = 1: a row with no attended prompt token at the first step sees its own key alone, weight 1: ctx is v, bit for bit"""
    heads, rows = 2, 3
    rng = np.random.default_rng(d)
    qkv = rng.standard_normal((rows, 1, 3 * heads * d)).astype(np.float32)
    mask = np.zeros((rows, 1), np.int32)
    pos = np.full(rows, -1, np.int32)
    ctx, kc, vc = _decode(qkv, mask, pos, 1, 0, heads)
    H = heads * d
    assert ctx.tobytes() == qkv[:, 0, 2 * H:].tobytes()
    assert kc[:, 0].tobytes() == qkv[:, 0, H:2 * H].tobytes() and vc[:, 0].tobytes() == qkv[:, 0, 2 * H:].tobytes()


def test_decode_attention_bits():
    """batch 1 vs batch 8, the scalar path, and keys the query does not see (past it, or masked prompt keys) changed"""
    heads, d, L = 12, 64, 1000
    qkv, mask, pos, S, t_ = _decode_case(L, d, heads, 3.0, 5)
    qkv8 = np.concatenate([qkv, qkv[::-1]])
    mask8, pos8 = np.concatenate([mask, mask[::-1]]), np.concatenate([pos, pos[::-1]])
    c8, _k, _v = _decode(qkv8, mask8, pos8, S, t_, heads)
    for b in range(4):
        c1, _k, _v = _decode(qkv[b:b + 1], mask[b:b + 1], pos[b:b + 1], S, t_, heads)
        assert c1.tobytes() == c8[b:b + 1].tobytes(), b
    cs, _k, _v = _decode(qkv8, mask8, pos8, S, t_, heads, off=1)
    assert cs.tobytes() == c8.tobytes()
    # a larger T and garbage in every slot the query does not read, and new values for the masked (left-padding) keys
    rng = np.random.default_rng(1)
    T = S + t_ + 40
    H = heads * d
    fill = (rng.standard_normal((8, T, H)).astype(np.float32) * 50, rng.standard_normal((8, T, H)).astype(np.float32) * 50)
    q2 = qkv8.copy()
    for b in range(8):
        hid = np.nonzero(mask8[b, :pos8[b] + 1] == 0)[0]
        q2[b, hid, H:] = rng.standard_normal((len(hid), 2 * H)).astype(np.float32)
    cg, _k, _v = _decode(q2, mask8, pos8, S, t_, heads, T=T, kc_fill=fill)
    assert cg.tobytes() == c8.tobytes()


def test_decode_attention_rejections():
    import torch
    z = torch.zeros(1 << 16, device="cuda")
    p = torch.zeros(4, dtype=torch.int32, device="cuda")
    E = t._lib.E_INVALID
    wb = lib.tfsc_k_decode_attention_work_bytes(1, 8, 64, 4)
    work = torch.zeros(wb // 4, dtype=torch.int32, device="cuda")
    args = lambda S, t_, T, H, heads, w=wb: (_ptr(z), _ptr(z), _ptr(z), _ptr(p), t_, None, S, S, T, _ptr(z), 1, H, heads, _ptr(work), w, None)  # noqa: E731
    assert lib.tfsc_k_decode_attention(*args(4, 3, 8, 64, 4)) == 0
    assert lib.tfsc_k_decode_attention(*args(4, 3, 7, 64, 4)) == E                 # S + t + 1 > T
    assert lib.tfsc_k_decode_attention(*args(4, 3, 8, 72, 12)) == E                # d = 6
    assert lib.tfsc_k_decode_attention(*args(4, 3, 8, 64, 4, wb - 4)) == E         # work too small
    assert lib.tfsc_k_decode_attention_work_bytes(1, 16385, 64, 4) == -1


# ------------------------------------------------------------------------------------------- select step ----
def _select(x, pos, vocab, t_, last, eos, done, word, ptab, off=0):
    import torch
    rows, vp = x.shape
    n = t_ + 2
    ids = torch.full((rows, n), 12345, dtype=torch.int32, device="cuda")
    lp = torch.full((rows, n), float("nan"), device="cuda")
    ln = torch.full((rows,), 777, dtype=torch.int32, device="cuda")
    H = word.shape[1]
    y = torch.full((rows * H + off,), float("nan"), device="cuda")
    xd, pd, dd = _cuda(x), _cuda(pos, np.int32), _cuda(done, np.int32)
    wd, td = _cuda(word, off=off), _cuda(ptab, off=off)
    t._lib.check(lib.tfsc_k_generate_select(_ptr(xd), vp, vocab, _ptr(pd), t_, int(last), eos, _ptr(dd), _ptr(ids), n, _ptr(lp), n,
                                            _ptr(ln), 1, _ptr(wd), _ptr(td), _ptr(y[off:]), rows, H, None), "generate_select")
    torch.cuda.synchronize()
    return ids.cpu().numpy()[:, t_], lp.cpu().numpy()[:, t_], ln.cpu().numpy(), dd.cpu().numpy(), y[off:].cpu().numpy().reshape(rows, H)


@pytest.mark.parametrize("vocab,vp", [(50257, 50272), (57344, 57344), (100, 128)])
@pytest.mark.parametrize("misalign", [False, True])
def test_select_matches_fp64(vocab, vp, misalign):
    import torch
    rows, H, P = 9, 768 if not misalign else 30, 64
    rng = np.random.default_rng(vocab)
    x, pos = g2._head_logits(rows, vocab, vp, vocab)                    # ties for first place, padding 1e30, row 1 empty
    x[2] = 0.5                                                          # a constant row
    x[3, :vocab] = rng.standard_normal(vocab).astype(np.float32) * 30
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((P, H)).astype(np.float32)
    pos = pos % (P // 2)
    pos[1] = -1
    ids, lp, ln, done, y = _select(x, pos, vocab, 0, False, -1, np.full(rows, 9, np.int32), word, ptab, off=int(misalign))
    want = np.argsort(-x[:, :vocab], axis=1, kind="stable")[:, 0]
    live = pos >= 0
    assert np.array_equal(ids[live], want[live]) and ids[1] == -1 and ids[0] == 3 and ids[2] == 0
    x64 = x[:, :vocab].astype(np.float64)
    ref = x64[np.arange(rows), want] - (x64.max(1) + np.log(np.exp(x64 - x64.max(1, keepdims=True)).sum(1)))
    assert np.all(np.abs(lp[live] - ref[live]) <= 1e-6 * np.maximum(1.0, np.abs(ref[live])))
    assert lp[1] == 0 and ln.tolist() == [1 if v else 0 for v in live] and done.tolist() == [0 if v else 1 for v in live]
    # the next step's input, for an empty row too: the bits tfsc_k_embed_positions gives for the argmax at position pos + 1
    gd = _cuda(want[:, None], np.int32)
    e = torch.full((rows * H,), float("nan"), device="cuda")
    wd = _cuda(word)
    for r in range(rows):
        tab = _cuda(ptab[pos[r] + 1:pos[r] + 2])
        t._lib.check(lib.tfsc_k_embed_positions(_ptr(gd[r:r + 1]), 1, _ptr(wd), _ptr(tab), _ptr(e[r * H:(r + 1) * H]), 1, 1, H,
                                                vocab, None), "embed_positions")
    torch.cuda.synchronize()
    assert y.tobytes() == e.cpu().numpy().reshape(rows, H).tobytes()


def test_select_eos_and_done():
    rows, vocab, H, P = 4, 50, 8, 32
    rng = np.random.default_rng(3)
    x = rng.standard_normal((rows, 64)).astype(np.float32)
    x[:, vocab:] = 1e30
    eos = int(np.argmax(x[0, :vocab]))
    word, ptab = rng.standard_normal((vocab, H)).astype(np.float32), rng.standard_normal((P, H)).astype(np.float32)
    pos = np.array([3, 5, -1, 2], np.int32)
    done = np.array([0, 1, 0, 0], np.int32)                              # row 1 ended earlier
    ids, lp, ln, dn, _y = _select(x, pos, vocab, 4, False, eos, done, word, ptab)
    assert ids[0] == eos and ln[0] == 5 and dn[0] == 1                   # EOS is emitted and counted, then the row is done
    assert ids[1] == -1 and lp[1] == 0 and ln[1] == 777 and dn[1] == 1   # a done row keeps its length
    assert ids[2] == np.argmax(x[2, :vocab]) and ln[2] == 5              # after t = 0 only the done flag counts
    _ids, _lp, ln, dn, _y = _select(x, pos, vocab, 0, True, eos, np.zeros(rows, np.int32), word, ptab)
    assert ln[2] == 0 and dn[2] == 1 and _ids[2] == -1


# ------------------------------------------------------------------------------------------ served models ----
def _write(tmp, seq, arch, seed, name="g", outputs=None, model=None, inputs=mf.GPT2_INPUTS):
    m = model or ge.hf_gpt2_model(seed, **arch)
    man = mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=_outs() if outputs is None else outputs)
    mf.write_graph_bundle(os.path.join(str(tmp), name, "1"), man, ge.export_gpt2_model(m, man))
    return m


def _teacher_forced(model, x, r, device="cuda"):
    """transformers fp64 logits [N, vocab] that predict each generated token of row `r` from the prompt and the tokens
    before it: a right-padded row alone with its attended prompt, any other row with its mask and default positions"""
    mask = x["attention_mask"][r]
    p = int(np.nonzero(mask)[0].max())
    n = len(r_ids := x["gen"][r])
    right = mask[0] == 1 and not mask.all()
    prompt, pm = (x["input_ids"][r, :p + 1], mask[:p + 1]) if right else (x["input_ids"][r], mask)
    seq = np.concatenate([prompt, np.maximum(r_ids[:n - 1], 0)])[None]
    sm = np.concatenate([pm, np.ones(n - 1, np.int32)])[None]
    at = len(prompt) - 1 + np.arange(n)
    full = ge.gpt2_reference(model, seq, sm, device=device)
    return full[0, at]


def _check_teacher_forced(model, x, r_out, V):
    for r in range(len(x["input_ids"])):
        ids, lp, n = r_out["generated_ids"][r], r_out["generated_log_probs"][r], r_out["generated_length"][r]
        assert n == len(ids) and (ids >= 0).all() and (ids < V).all()
        ref = _teacher_forced(model, dict(x, gen=r_out["generated_ids"]), r)[:, :V]
        lse = ref.max(1) + np.log(np.exp(ref - ref.max(1, keepdims=True)).sum(1))
        want_lp = ref[np.arange(len(ids)), ids] - lse
        assert np.all(np.abs(lp - want_lp) <= 1e-4 * np.maximum(1.0, np.abs(want_lp))), (r, np.abs(lp - want_lp).max())
        srt = np.sort(ref, axis=1)[:, ::-1]
        clear = srt[:, 0] - srt[:, 1] > 2e-4 * np.maximum(1.0, np.abs(srt[:, 0]))
        assert np.array_equal(ids[clear], np.argmax(ref, axis=1)[clear]), r


@pytest.mark.parametrize("S", [128, 992])
def test_gpt2_small_generates(S, tmp_path):
    import torch
    n, V = 32, 50257
    m = _write(tmp_path, S, dict(max_pos=1024), 41, outputs=_outs(n))
    _write(tmp_path, S, dict(max_pos=1024), 41, name="nt", model=m, outputs=[{"name": "ids", "kind": "next_token_top_k_ids", "k": 1}])
    x = ge.gpt2_inputs(8, S, V, seed=S)
    torch.cuda.empty_cache()
    full = None
    with t.Server(g2._cfg(tmp_path)) as srv:
        for bs in (8, 3, 1):
            xb = {k: v[:bs] for k, v in x.items()}
            r = srv.predict("g", "1", xb, outputs=NAMES)
            assert r["generated_ids"].shape == (bs, n) and r["generated_length"].shape == (bs,)
            nt = srv.predict("nt", "1", xb, outputs=["ids"])
            assert r["generated_ids"][:, 0].tobytes() == nt["ids"][:, 0].tobytes()
            _check_teacher_forced(m, xb, r, V)
            full = full if bs < 8 else r
        # an EOS the model emits mid-sequence: the row stops there, counted, and pads with -1 and 0
        eos = int(full["generated_ids"][0, n // 2])
        first = list(full["generated_ids"][0]).index(eos)
        _write(tmp_path, S, dict(max_pos=1024), 41, name="e", model=m, outputs=_outs(n, eos=eos))
        r = srv.predict("e", "1", x, outputs=NAMES)
    for b in range(8):
        ids = list(full["generated_ids"][b])
        k = ids.index(eos) + 1 if eos in ids else n
        assert r["generated_length"][b] == k and r["generated_ids"][b, :k].tobytes() == full["generated_ids"][b, :k].tobytes()
        assert (r["generated_ids"][b, k:] == -1).all() and (r["generated_log_probs"][b, k:] == 0).all()
        assert r["generated_log_probs"][b, :k].tobytes() == full["generated_log_probs"][b, :k].tobytes()
    assert r["generated_length"][0] == first + 1


def test_empty_row_and_ids_only(tmp_path):
    S = 16
    _write(tmp_path, S, SMALL, 43)
    _write(tmp_path, S, SMALL, 43, name="i", inputs=None)
    x = ge.gpt2_inputs(3, S, SMALL["vocab"], seed=2)
    x["attention_mask"][1] = 0
    with t.Server(g2._cfg(tmp_path)) as srv:
        r = srv.predict("g", "1", x, outputs=NAMES)
        ri = srv.predict("i", "1", x["input_ids"], outputs=NAMES)
    assert r["generated_length"].tolist() == [N, 0, N]
    assert (r["generated_ids"][1] == -1).all() and (r["generated_log_probs"][1] == 0).all()
    assert (ri["generated_length"] == N).all() and (ri["generated_ids"] >= 0).all()


# ----------------------------------------------------------------------------------------- front-ends ----
def test_every_frontend_on_a_generate_bundle(tmp_path):
    import torch
    S, B = 32, 5
    _write(tmp_path, S, SMALL, 73)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], seed=3)
    with t.Server(g2._cfg(tmp_path)) as srv:
        full = srv.predict("g", "1", x, outputs=NAMES)
        assert full["generated_length"].dtype == np.int32 and full["generated_ids"].dtype == np.int32
        assert full["generated_log_probs"].dtype == np.float32 and full["generated_log_probs"].shape == (B, N)
        sub = srv.predict("g", "1", x, outputs=["generated_log_probs", "generated_length"])
        assert list(sub) == ["generated_log_probs", "generated_length"] and all(v.tobytes() == full[k].tobytes() for k, v in sub.items())
        one = srv.predict("g", "1", {k: v[0] for k, v in x.items()}, outputs=["generated_length", "generated_ids"])
        assert one["generated_length"].shape == () and one["generated_ids"].shape == (N,)
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("g", 1, x)))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        req = wire.encode_predict_request("g", 1, x, output_filter=["generated_ids"])
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(req))
        assert list(outs) == ["generated_ids"] and outs["generated_ids"].tobytes() == full["generated_ids"].tobytes()
        st, b = srv.rest_handle("POST", "/v1/models/g/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        for i, p in enumerate(preds):
            assert list(p) == NAMES and p["generated_length"] == int(full["generated_length"][i])
            assert np.array_equal(np.int32(p["generated_ids"]), full["generated_ids"][i])
            assert np.array_equal(np.float32(p["generated_log_probs"]), full["generated_log_probs"][i])
        st, b = srv.rest_handle("POST", "/v1/models/g/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES and all(np.array_equal(np.asarray(cols[k], full[k].dtype), full[k]) for k in NAMES)
        st, b = srv.rest_handle("GET", "/v1/models/g/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {"generated_ids": ("DT_INT32", ["-1", str(N)]), "generated_log_probs": ("DT_FLOAT", ["-1", str(N)]),
                "generated_length": ("DT_INT32", ["-1"])}
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(g2._session_run_request("g", "input_ids:0", x["input_ids"], "generated_ids:0"))
        assert e.value.code == t._lib.E_INVALID and "'attention_mask'" in str(e.value)
        for verb in ("classify", "regress"):
            st, b = srv.rest_handle("POST", f"/v1/models/g/versions/1:{verb}", json.dumps({"examples": [{"x": 1.0}]}).encode())
            assert st == 400
        srv.ensure(0, "g", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(_outs(), SMALL["vocab"]))
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.GPT2_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "g", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), _outs(), SMALL["vocab"])
        for k in NAMES:
            assert dev[k].shape == full[k].shape and dev[k].tobytes() == full[k].tobytes(), k


def test_coalesced_requests_give_the_bits_of_one_request(tmp_path):
    S, sizes = 40, [2, 3]
    _write(tmp_path, S, SMALL, 76)
    x = ge.gpt2_inputs(sum(sizes), S, SMALL["vocab"], seed=8)
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": sum(sizes), "gpu.tickMicros": 3_000_000})) as srv, \
            t.Server(g2._cfg(tmp_path)) as one:
        srv.predict("g", "1", x, outputs=NAMES)
        st0 = srv.stats()
        tk = [srv.predict_submit("g", "1", {k: v[lo:lo + n] for k, v in x.items()}, outputs=NAMES)
              for lo, n in ((0, sizes[0]), (sizes[0], sizes[1]))]
        outs = [k.wait(30.0) for k in tk]
        [k.release() for k in tk]
        assert srv.stats()["batches"] - st0["batches"] == 1
        whole = one.predict("g", "1", x, outputs=NAMES)
    for (lo, n), r in zip(((0, sizes[0]), (sizes[0], sizes[1])), outs):
        assert all(r[k].tobytes() == np.ascontiguousarray(whole[k][lo:lo + n]).tobytes() for k in NAMES)


@pytest.mark.parametrize("rows", [1, 8])
def test_launch_counts(tmp_path, rows):
    """the next-token graph's launches with the select step for the head, one cache write per attention op, and N - 1
    decode steps of one launch per decoder op, last_token, ln_f, the vocabulary projection and the select step; besides
    the batch's input gather and output scatter"""
    S, L = 64, SMALL["layers"]
    _write(tmp_path, S, SMALL, 74)
    x = ge.gpt2_inputs(rows, S, SMALL["vocab"], seed=rows)
    with t.Server(g2._cfg(tmp_path)) as srv:
        srv.predict("g", "1", x, outputs=NAMES)
        s0 = srv.stats()
        srv.predict("g", "1", x, outputs=NAMES)
        s1 = srv.stats()
    prefill = 1 + 7 * L + L + 4
    assert s1["kernel_launches"] - s0["kernel_launches"] == 2 + prefill + (N - 1) * (7 * L + 4)


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_generate as g
import gpt2_export as ge
tmp = sys.argv[2]
g._write(tmp, 300, g.SMALL, 75)
out = {}
with t.Server(g.g2._cfg(tmp)) as srv:
    for rows in (1, 8):
        x = ge.gpt2_inputs(rows, 300, g.SMALL["vocab"], seed=rows)
        for k, v in srv.predict("g", "1", x, outputs=g.NAMES).items():
            out[f"{k}_r{rows}"] = v
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
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 2 * len(NAMES)
    for key, y in res["default"].items():
        assert y.tobytes() == res["0"][key].tobytes(), key


# --------------------------------------------------------------------------------------- forward hop ----
N_MODELS, HOP_S, HOP_ROWS = 4, 48, 6


def _rank_main(rank, world, socks, base, barrier, out):
    try:
        import torch
        torch.cuda.set_device(0)
        res = {"rank": rank, "owned": [], "y": {}, "grpc": {}, "rest": {}}
        with t.Server(g2._rank_cfg(rank, world, socks, base)) as srv:
            barrier.wait(timeout=120)
            x = ge.gpt2_inputs(HOP_ROWS, HOP_S, SMALL["vocab"], seed=7)
            for j in range(N_MODELS):
                name = f"g{j}"
                res["owned"].append(srv.route(name, "1")[0][0] >= 0)
                res["y"][j] = srv.predict(name, "1", x, outputs=NAMES)
                _s, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request(name, 1, x)))
                res["grpc"][j] = dict(outs)
                st, b = srv.rest_handle("POST", f"/v1/models/{name}/versions/1:predict",
                                        json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
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


def test_forward_hop_generate():
    world = 2
    base = tempfile.mkdtemp(prefix="tfscgen")
    for j in range(N_MODELS):
        _write(base, HOP_S, SMALL, 80 + j, name=f"g{j}")
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
    for j in range(N_MODELS):
        owner = 0 if results[0]["owned"][j] else 1
        local, fwd = results[owner], results[1 - owner]
        assert sorted(local["y"][j]) == NAMES and local["y"][j]["generated_ids"].shape == (HOP_ROWS, N)
        for k in NAMES:
            assert fwd["y"][j][k].shape == local["y"][j][k].shape and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
