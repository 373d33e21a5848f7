"""-m gpu: GPT-2 score bundles. tfsc_k_token_score against fp64 at a 100-token, GPT-2's and the widest vocabulary with
poisoned padding columns, ties and constant rows, every padding pattern, out-of-range ids and chunks that start and end
mid-row; its log-probabilities bit for bit tfsc_k_generate_select's, rank 0 exactly at the next-token head's top-1, a row
alone as in its batch; tfsc_k_score_head against numpy. Through the server: seeded GPT-2 small at S = 7, 128 and 1,024 over
1-128 rows (every projection route) and GPT-2 medium against transformers fp64, the scores of a greedy generation against
its generated_log_probs, every front-end, coalescing, TFSC_PDL=0, two chunks of very different logits, launch counts, the
forward hop and a 128 x 1,024 request."""
import json
import math
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import pytest

import tfservingcache_b200 as t
from oracle import wire

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpt2_export as ge  # noqa: E402
import score_ref as sr  # noqa: E402
import test_gpu_generate as gg  # noqa: E402
import test_gpu_gpt2 as g2  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
SMALL = g2.SMALL
ALL = [{"name": k, "kind": k} for k in mf.SCORE_OUTPUT_KINDS]
NAMES = sorted(mf.SCORE_OUTPUT_KINDS)
V = 50257
_ptr, _cuda = gg._ptr, gg._cuda


# ----------------------------------------------------------------------------------------------- the kernels ----
def _token_score(logits, ld, ids, mask, vocab, chunks=None, fill=np.nan):
    """tfsc_k_token_score over the [rows, S] batch of ids / mask (mask None: every position), logits [rows * S, ld], in
    launches of `chunks` token rows (default: one). Returns log_probs [rows, S] and ranks [rows, S] (unwritten slots keep
    `fill` and -7)."""
    import torch
    rows, S = ids.shape
    xd = _cuda(logits)
    idd, md = _cuda(ids, np.int32), None if mask is None else _cuda(mask, np.int32)
    lp = torch.full((rows * S,), float(fill), device="cuda")
    rk = torch.full((rows * S,), -7, dtype=torch.int32, device="cuda")
    first = 0
    for n in chunks or [rows * S]:
        t._lib.check(lib.tfsc_k_token_score(_ptr(xd[first * ld:]), ld, first, n, _ptr(idd), _ptr(md), S, rows, S, vocab, _ptr(lp),
                                            _ptr(rk), None), "token_score")
        first += n
    assert first == rows * S
    torch.cuda.synchronize()
    return lp.cpu().numpy().reshape(rows, S), rk.cpu().numpy().reshape(rows, S)


def _batch(vocab, ld, seed, S=9):
    """logits [6 * S, ld] with tied maxima, a constant row and large values, padding columns poisoned with NaN, +Inf and
    1e30 in turn; ids with out-of-range values; masks unpadded, left-padded, right-padded, holed, fully masked, one token"""
    rng = np.random.default_rng(seed)
    rows = 6
    x = (rng.standard_normal((rows * S, ld)) * 4).astype(np.float32)
    x[:, vocab:] = np.array([np.nan, np.inf, 1e30], np.float32)[np.arange(rows * S) % 3][:, None]
    x[::4, 3] = x[::4, min(7, vocab - 1)] = x[::4, :vocab].max(axis=1) + 1   # ties for first place
    x[5] = 0.5                                                                # a constant row
    x[6, :vocab] *= 30
    x[7, :vocab] = np.round(x[7, :vocab])                                     # many ties at every rank
    ids = rng.integers(0, vocab, (rows, S)).astype(np.int32)
    ids[0, 1], ids[0, 2], ids[3, 4] = -5, vocab + 3, 10 ** 9                  # clamped as the embedding clamps
    ids[0, 5] = ids[0, 6] = 3                      # at 5 a tie for first place (the lower id), at 6 the constant row
    mask = np.ones((rows, S), np.int32)
    mask[1, :4] = 0
    mask[2, 5:] = 0
    mask[3, [1, 2, 6]] = 0
    mask[4] = 0
    mask[5] = 0
    mask[5, 3] = 1
    return x, ids, mask


def _check_scores(lp, rk, x, ids, mask, vocab, fill):
    rows, S = ids.shape
    lg = x.reshape(rows, S, -1)
    want_lp, want_rk, _s, _c = sr.score(lg, ids, mask, vocab)
    scored = want_rk >= 0
    assert scored.sum() > 10
    err = np.abs(lp[scored] - want_lp[scored]) / np.maximum(1.0, np.abs(want_lp[scored]))
    assert err.max() <= 2e-6, err.max()
    assert np.array_equal(rk[scored], want_rk[scored])
    assert (rk[~scored] == -7).all() and (np.isnan(lp[~scored]) if np.isnan(fill) else lp[~scored] == fill).all()


@pytest.mark.parametrize("vocab,ld", [(100, 131), (50257, 50272), (57344, 57376)])
@pytest.mark.parametrize("chunks", [None, [5, 13, 20, 16], [1] * 54])
def test_token_score_matches_fp64(vocab, ld, chunks):
    x, ids, mask = _batch(vocab, ld, vocab + len(chunks or []))
    lp, rk = _token_score(x, ld, ids, mask, vocab, chunks)
    _check_scores(lp, rk, x, ids, mask, vocab, np.nan)
    assert rk[0, 5] == 0 and rk[0, 6] == 3 and rk[0, 1] == sr.rank(x[0, :vocab], 0) and rk[0, 2] == sr.rank(x[1, :vocab], vocab - 1)
    assert (rk[4] == -7).all() and (rk[5] == -7).all()                       # no token, one token: nothing scored
    # no mask: every position but 0 is scored from the one before it
    lp, rk = _token_score(x, ld, ids, None, vocab, chunks)
    _check_scores(lp, rk, x, ids, None, vocab, np.nan)
    assert (rk[:, 0] == -7).all() and (rk[:, 1:] >= 0).all()


def test_log_probs_are_the_select_steps_and_rank_0_is_the_top_1():
    """two tokens per row: position 0's logits score the id at position 1. Where that id is the argmax, the log-probability
    has the bits tfsc_k_generate_select writes; rank 0 exactly where it is tfsc_k_next_token_head's top-1"""
    for vocab, vp in ((50257, 50272), (57344, 57344), (100, 128)):
        rows = 9
        x, pos = g2._head_logits(rows, vocab, vp, vocab)                 # ties for first place, padding 1e30
        x[2] = 0.5
        pos[:] = 0
        top1 = g2._next_head(x, pos, vocab, 1)[0][:, 0]
        ids = np.zeros((rows, 2), np.int32)
        ids[:, 1] = top1
        ids[[1, 4], 1] = (top1[[1, 4]] + 1) % vocab                          # not the top-1
        logits = np.zeros((rows * 2, vp), np.float32)
        logits[0::2] = x
        logits[1::2] = np.nan                                                # position 1 predicts nothing here
        lp, rk = _token_score(logits, vp, ids, None, vocab)
        assert np.array_equal(rk[:, 1] == 0, ids[:, 1] == top1), (vocab, rk[:, 1])
        word = np.zeros((vocab, 4), np.float32)
        _g, sel_lp, _ln, _d, _y = gg._select(x, np.zeros(rows, np.int32), vocab, 0, True, -1, np.zeros(rows, np.int32), word,
                                            np.zeros((4, 4), np.float32))
        same = ids[:, 1] == top1
        assert lp[same, 1].tobytes() == sel_lp[same].tobytes(), vocab


def test_a_row_alone_keeps_its_bits():
    vocab, ld, S = 50257, 50272, 9
    x, ids, mask = _batch(vocab, ld, 5, S)
    lp, rk = _token_score(x, ld, ids, mask, vocab, [7, 30, 17])
    for r in range(len(ids)):
        lp1, rk1 = _token_score(x[r * S:(r + 1) * S], ld, ids[r:r + 1], mask[r:r + 1], vocab)
        assert lp1[0].tobytes() == lp[r].tobytes() and rk1[0].tobytes() == rk[r].tobytes(), r


def _score_head(lp, rk, mask, lds=None):
    import torch
    rows, S = lp.shape
    lpd, rkd = _cuda(lp), _cuda(rk, np.int32)
    md = None if mask is None else _cuda(mask, np.int32)
    o_lp = torch.full((rows, S), float("nan"), device="cuda")
    o_rk = torch.full((rows, S), 99, dtype=torch.int32, device="cuda")
    o_sum = torch.full((rows,), float("nan"), device="cuda")
    o_n = torch.full((rows,), 99, dtype=torch.int32, device="cuda")
    t._lib.check(lib.tfsc_k_score_head(_ptr(lpd), _ptr(rkd), _ptr(md), S, rows, S, _ptr(o_lp), S, _ptr(o_rk), S, _ptr(o_sum), 1,
                                       _ptr(o_n), 1, None), "score_head")
    torch.cuda.synchronize()
    return o_lp.cpu().numpy(), o_rk.cpu().numpy(), o_sum.cpu().numpy(), o_n.cpu().numpy()


@pytest.mark.parametrize("S", [9, 1, 1024, 3000])
def test_score_head_matches_numpy(S):
    rng = np.random.default_rng(S)
    rows = 6
    lp = (-rng.random((rows, S)) * 20).astype(np.float32)
    rk = rng.integers(0, 50000, (rows, S)).astype(np.int32)
    mask = (rng.random((rows, S)) < 0.8).astype(np.int32)
    mask[1] = 0
    mask[2] = 1
    mask[3, :] = 0
    mask[3, S // 2] = 1
    for m in (mask, None):
        pairs = [sr.scored_pairs(None if m is None else m[r], S) for r in range(rows)]
        scored = np.zeros((rows, S), bool)
        for r, pr in enumerate(pairs):
            scored[r, [s for _p, s in pr]] = True
        src_lp = np.where(scored, lp, np.nan).astype(np.float32)          # unscored slots hold NaN: never read
        src_rk = np.where(scored, rk, -99).astype(np.int32)
        o_lp, o_rk, o_sum, o_n = _score_head(src_lp, src_rk, m)
        assert np.array_equal(o_lp, np.where(scored, lp, 0).astype(np.float32))
        assert np.array_equal(o_rk, np.where(scored, rk, -1))
        assert np.array_equal(o_n, scored.sum(axis=1))
        for r in range(rows):
            exact = math.fsum(lp[r, scored[r]].astype(np.float64))
            assert abs(o_sum[r] - exact) <= abs(np.spacing(np.float32(exact))), r
            assert (o_sum[r] == 0) == (not scored[r].any())


def test_rejections():
    import torch
    z, zo = torch.zeros(1 << 16, device="cuda"), torch.zeros(1 << 16, device="cuda")
    i, io = torch.zeros(1 << 12, dtype=torch.int32, device="cuda"), torch.zeros(1 << 12, dtype=torch.int32, device="cuda")
    E = t._lib.E_INVALID
    p, q, po, qo = _ptr(z), _ptr(i), _ptr(zo), _ptr(io)
    assert lib.tfsc_k_token_score(p, 100, 0, 4, q, None, 8, 1, 8, 100, po, qo, None) == 0
    assert lib.tfsc_k_token_score(p, 99, 0, 4, q, None, 8, 1, 8, 100, p, q, None) == E           # ld < vocab
    assert lib.tfsc_k_token_score(p, 100, 6, 4, q, None, 8, 1, 8, 100, p, q, None) == E           # past rows * S
    assert lib.tfsc_k_token_score(p, 100, 0, 4, q, None, 7, 1, 8, 100, p, q, None) == E           # stride < S
    assert lib.tfsc_k_token_score(p, 57345, 0, 1, q, None, 8, 1, 8, 57345, p, q, None) == E       # vocab
    assert lib.tfsc_k_token_score(p, 100, 0, 1, None, None, 8, 1, 8, 100, p, q, None) == E
    assert lib.tfsc_k_token_score(p, 100, 0, 0, q, None, 8, 1, 8, 100, p, q, None) == 0           # nothing to do
    assert lib.tfsc_k_score_head(p, q, None, 8, 1, 8, po, 8, qo, 8, po, 1, qo, 1, None) == 0
    assert lib.tfsc_k_score_head(p, q, None, 7, 1, 8, p, 8, q, 8, p, 1, q, 1, None) == E
    assert lib.tfsc_k_score_head(None, q, None, 8, 1, 8, p, 8, None, 8, None, 1, None, 1, None) == E
    assert lib.tfsc_k_score_head(p, q, None, 8 << 12, 1, 16385, p, 8, q, 8, p, 1, q, 1, None) == E
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ served models ----
def _cfg(tmp, **kw):
    return g2._cfg(tmp, **dict({"gpu.arenaBytes": 8 << 30, "gpu.maxBatch": 128}, **kw))


def _write(tmp, seq, arch, seed, name="s", outputs=ALL, model=None, inputs=mf.GPT2_INPUTS):
    m = model or ge.hf_gpt2_model(seed, **arch)
    man = mf.gpt2_manifest(seq=seq, **arch, inputs=inputs, outputs=outputs)
    mf.write_graph_bundle(os.path.join(str(tmp), name, "1"), man, ge.export_gpt2_model(m, man))
    return m


def _reference(m64, ids, mask, vocab, tol=1e-4, batch=4):
    """transformers fp64 (m64: the model in fp64 on the GPU) at every scored position: log-probabilities [B, S] (0
    elsewhere), rank bounds lo / hi [B, S] (the counts of ids above the target with the log-probabilities' tolerance,
    tol * max(1, |log-probability|), taken against, then for it), the top-1 / top-2 margin at the predicting position,
    and the scored mask"""
    import torch
    B, S = ids.shape
    lp, lo, hi, margin = np.zeros((B, S)), np.full((B, S), -1), np.full((B, S), -1), np.zeros((B, S))
    scored = np.zeros((B, S), bool)
    for b0 in range(0, B, batch):
        ib = torch.from_numpy(ids[b0:b0 + batch].astype(np.int64)).cuda()
        mb = torch.from_numpy(mask[b0:b0 + batch].astype(np.int64)).cuda()
        with torch.no_grad():
            z = m64.lm_head(m64.transformer(input_ids=ib, attention_mask=mb).last_hidden_state)[..., :vocab]
            for j in range(len(ib)):
                r = b0 + j
                pairs = sr.scored_pairs(mask[r], S)
                if not pairs:
                    continue
                P = torch.tensor([p for p, _s in pairs], device="cuda")
                Ss = np.array([s for _p, s in pairs])
                tgt = torch.from_numpy(np.clip(ids[r, Ss], 0, vocab - 1).astype(np.int64)).cuda()
                zz = z[j, P]
                zt = zz.gather(1, tgt[:, None])
                lpt = zt[:, 0] - torch.logsumexp(zz, 1)
                tl = tol * torch.clamp(lpt.abs(), min=1.0)[:, None]
                lp[r, Ss] = lpt.cpu().numpy()
                lo[r, Ss] = (zz > zt + tl).sum(1).cpu().numpy()
                hi[r, Ss] = ((zz >= zt - tl).sum(1) - 1).cpu().numpy()
                top2 = zz.topk(2, dim=1).values
                margin[r, Ss] = (top2[:, 0] - top2[:, 1]).cpu().numpy()
                scored[r, Ss] = True
            del z
    return SimpleNamespace(lp=lp, lo=lo, hi=hi, margin=margin, scored=scored)


def _check_against_fp64(r, ref):
    scored = ref.scored
    assert np.array_equal(r["token_count"], scored.sum(axis=1))
    lp, rk = r["token_log_probs"], r["token_ranks"]
    assert (lp[~scored] == 0).all() and (rk[~scored] == -1).all()
    err = np.abs(lp[scored] - ref.lp[scored]) / np.maximum(1.0, np.abs(ref.lp[scored]))
    assert err.max() <= 1e-4, err.max()
    assert (rk[scored] >= ref.lo[scored]).all() and (rk[scored] <= ref.hi[scored]).all()
    for b in range(len(lp)):
        exact = math.fsum(lp[b, scored[b]].astype(np.float64))
        assert abs(r["token_log_prob_sum"][b] - exact) <= abs(np.spacing(np.float32(exact))), b
        bound = 1e-4 * np.maximum(1.0, np.abs(ref.lp[b, scored[b]])).sum()
        assert abs(r["token_log_prob_sum"][b] - ref.lp[b, scored[b]].sum()) <= bound, b


def _holed(x, seed):
    """gpt2_inputs' unpadded / right / left rows, every fourth row with holes in its mask as well"""
    rng = np.random.default_rng(seed)
    for r in range(3, len(x["attention_mask"]), 4):
        S = x["attention_mask"].shape[1]
        x["attention_mask"][r, rng.integers(0, S, max(1, S // 10))] = 0
    return x


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    import copy

    import torch
    tmp = tmp_path_factory.mktemp("score_small")
    m = ge.hf_gpt2_model(29, max_pos=1024)
    for S in (7, 128, 1024):
        _write(tmp, S, dict(max_pos=1024), 29, name=f"s{S}", model=m)
    m64 = copy.deepcopy(m).double().cuda()
    torch.cuda.empty_cache()
    with t.Server(_cfg(tmp)) as srv:
        yield SimpleNamespace(tmp=tmp, model=m, m64=m64, srv=srv)


@pytest.mark.parametrize("S,B", [(7, 1), (7, 5), (128, 1), (128, 8), (128, 65), (128, 128), (1024, 1), (1024, 8), (1024, 65),
                                 (1024, 128)])
def test_gpt2_small_against_fp64(small, S, B):
    """1-128 rows of 7, 128 and 1,024 tokens: chunks of 7 and 35 token rows (the <= 8 and 9-63 routes), 128 and 1,024
    (the GEMM), and 65 x 1,024 in 65 chunks"""
    import torch
    x = _holed(ge.gpt2_inputs(B, S, V, seed=S + B), S + B)
    mem0 = torch.cuda.mem_get_info()
    r = small.srv.predict(f"s{S}", "1", x, outputs=NAMES)
    free, total = torch.cuda.mem_get_info()
    if B * S == 128 * 1024:
        print(f"\n128 x 1024 score request: {(total - min(free, mem0[0])) / 2 ** 30:.1f} GiB of device memory in use, whole device")
    assert r["token_log_probs"].shape == (B, S) and r["token_count"].shape == (B,)
    _check_against_fp64(r, _reference(small.m64, x["input_ids"], x["attention_mask"], V))


def test_gpt2_medium_against_fp64(tmp_path):
    import copy

    import torch
    S, B = 128, 9
    m = _write(tmp_path, S, dict(hidden=1024, layers=24, heads=16, max_pos=1024), 31, name="med")
    x = _holed(ge.gpt2_inputs(B, S, V, seed=3), 3)
    with t.Server(_cfg(tmp_path)) as srv:
        r = srv.predict("med", "1", x, outputs=NAMES)
    m64 = copy.deepcopy(m).double().cuda()
    _check_against_fp64(r, _reference(m64, x["input_ids"], x["attention_mask"], V))
    del m64
    torch.cuda.empty_cache()


def test_scores_of_a_generation_are_its_log_probs(small):
    """a greedy bundle (prompt 128, N = 32) and a score bundle of S = 160 from the same model: the prompt and the generated
    ids, scored, give generated_log_probs at the generated positions, and rank 0 wherever fp64's top-1 is clear"""
    S, N, B = 128, 32, 6
    gg._write(small.tmp, S, dict(max_pos=1024), 29, name="gen_g", model=small.model, outputs=gg._outs(N))
    _write(small.tmp, S + N, dict(max_pos=1024), 29, name="gen_s", model=small.model)
    x = ge.gpt2_inputs(B, S, V, seed=11)
    srv = small.srv
    g = srv.predict("gen_g", "1", x, outputs=gg.NAMES)
    ids = np.zeros((B, S + N), np.int32)
    mask = np.zeros((B, S + N), np.int32)
    at = []
    for r in range(B):
        p = int(np.nonzero(x["attention_mask"][r])[0].max())
        ids[r, :p + 1], mask[r, :p + 1] = x["input_ids"][r, :p + 1], x["attention_mask"][r, :p + 1]
        ids[r, p + 1:p + 1 + N], mask[r, p + 1:p + 1 + N] = g["generated_ids"][r], 1
        at.append(p + 1 + np.arange(N))
    sc = srv.predict("gen_s", "1", {"input_ids": ids, "attention_mask": mask}, outputs=NAMES)
    ref = _reference(small.m64, ids, mask, V)
    clear = 0
    for r in range(B):
        lp, want = sc["token_log_probs"][r, at[r]], g["generated_log_probs"][r]
        assert np.all(np.abs(lp - want) <= 1e-4 * np.maximum(1.0, np.abs(want))), (r, np.abs(lp - want).max())
        c = ref.margin[r, at[r]] > 1e-4
        assert (sc["token_ranks"][r, at[r]][c] == 0).all(), r
        clear += c.sum()
    assert clear > B * N // 2


def test_every_frontend_on_a_score_bundle(tmp_path):
    import torch
    S, B = 32, 5
    _write(tmp_path, S, SMALL, 73)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], seed=3)
    with t.Server(g2._cfg(tmp_path)) as srv:
        full = srv.predict("s", "1", x, outputs=NAMES)
        assert full["token_log_probs"].shape == (B, S) and full["token_log_probs"].dtype == np.float32
        assert full["token_ranks"].dtype == np.int32 and full["token_count"].shape == (B,) and full["token_count"].dtype == np.int32
        assert full["token_log_prob_sum"].shape == (B,) and full["token_log_prob_sum"].dtype == np.float32
        sub = srv.predict("s", "1", x, outputs=["token_count", "token_log_probs"])
        assert list(sub) == ["token_count", "token_log_probs"] and all(v.tobytes() == full[k].tobytes() for k, v in sub.items())
        one = srv.predict("s", "1", {k: v[0] for k, v in x.items()}, outputs=NAMES)
        assert one["token_count"].shape == () and one["token_ranks"].shape == (S,)
        row = srv.predict("s", "1", {k: v[:1] for k, v in x.items()}, outputs=NAMES)   # the same 32 tokens, the same route
        assert all(one[k].tobytes() == row[k][0].tobytes() for k in NAMES)
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("s", "1", x, outputs=["nope"])
        assert "unknown output 'nope'" in str(e.value) and "'token_ranks' (int32)" in str(e.value)
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("s", 1, x)))
        assert list(outs) == NAMES and all(outs[k].dtype == full[k].dtype and outs[k].tobytes() == full[k].tobytes() for k in NAMES)
        req = wire.encode_predict_request("s", 1, x, output_filter=["token_log_prob_sum"])
        _spec, outs = wire.decode_predict_response(srv.grpc_predict(req))
        assert list(outs) == ["token_log_prob_sum"] and outs["token_log_prob_sum"].tobytes() == full["token_log_prob_sum"].tobytes()
        st, b = srv.rest_handle("POST", "/v1/models/s/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        preds = json.loads(b)["predictions"]
        for i, p in enumerate(preds):
            assert list(p) == NAMES and p["token_count"] == int(full["token_count"][i])
            assert np.array_equal(np.float32(p["token_log_probs"]), full["token_log_probs"][i])
            assert np.array_equal(np.int32(p["token_ranks"]), full["token_ranks"][i])
            assert np.float32(p["token_log_prob_sum"]) == full["token_log_prob_sum"][i]
        st, b = srv.rest_handle("POST", "/v1/models/s/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and list(cols) == NAMES
        assert all(np.array_equal(np.asarray(cols[k], full[k].dtype), full[k]) for k in NAMES)
        st, b = srv.rest_handle("GET", "/v1/models/s/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["outputs"]
        want = {"token_log_probs": ("DT_FLOAT", ["-1", str(S)]), "token_ranks": ("DT_INT32", ["-1", str(S)]),
                "token_log_prob_sum": ("DT_FLOAT", ["-1"]), "token_count": ("DT_INT32", ["-1"])}
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == want
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(g2._session_run_request("s", "input_ids:0", x["input_ids"], "token_ranks:0"))
        assert e.value.code == t._lib.E_INVALID
        for verb in ("classify", "regress"):
            st, b = srv.rest_handle("POST", f"/v1/models/s/versions/1:{verb}", json.dumps({"examples": [{"x": 1.0}]}).encode())
            assert st == 400
        srv.ensure(0, "s", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(ALL, S))
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.GPT2_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "s", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), ALL, S)
        assert all(dev[k].shape == full[k].shape and dev[k].tobytes() == full[k].tobytes() for k in NAMES)


def test_coalesced_requests_give_the_bits_of_one_request(tmp_path):
    """two requests coalesced into one batch, whose chunks start mid-row, answer each request's rows as one request of
    the same rows does"""
    S = 300
    _write(tmp_path, S, SMALL, 75)
    x = ge.gpt2_inputs(9, S, SMALL["vocab"], seed=5)
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": 9, "gpu.tickMicros": 3_000_000})) as srv:
        joint = srv.predict("s", "1", x, outputs=NAMES)
        st0 = srv.stats()
        parts = ((0, 4), (4, 5))
        tk = [srv.predict_submit("s", "1", {k: v[lo:lo + n] for k, v in x.items()}, outputs=NAMES) for lo, n in parts]
        outs = [k.wait(30.0) for k in tk]
        [k.release() for k in tk]
        assert srv.stats()["batches"] - st0["batches"] == 1
    for (lo, n), r in zip(parts, outs):
        assert all(r[k].tobytes() == np.ascontiguousarray(joint[k][lo:lo + n]).tobytes() for k in NAMES)


def test_two_chunks_of_different_logits(tmp_path):
    """2 x 1,024 tokens are two chunks of 1,024 token rows: a row of one repeated id and a random row. Each chunk's scores
    are those of its row launched alone (the same projection of 1,024 rows), so no score kernel read logits the next
    chunk's projection wrote"""
    S = 1024
    _write(tmp_path, S, dict(max_pos=1024), 33, name="s")
    rng = np.random.default_rng(1)
    ids = np.stack([np.full(S, 464, np.int32), rng.integers(0, V, S).astype(np.int32)])
    x = {"input_ids": ids, "attention_mask": np.ones((2, S), np.int32)}
    with t.Server(_cfg(tmp_path)) as srv:
        both = [srv.predict("s", "1", x, outputs=NAMES) for _ in range(3)]
        alone = [srv.predict("s", "1", {k: v[i:i + 1] for k, v in x.items()}, outputs=NAMES) for i in range(2)]
    assert np.abs(both[0]["token_log_probs"][0] - both[0]["token_log_probs"][1]).max() > 1
    for r in both:
        for i in range(2):
            assert all(r[k][i:i + 1].tobytes() == alone[i][k].tobytes() for k in NAMES), i


@pytest.mark.parametrize("rows", [1, 9])
def test_launch_counts(tmp_path, rows):
    """the next-token bundle's trunk, then ln_f over every token, a projection and a score kernel per chunk of 1,024 token
    rows, and one head: the next-token bundle's count (last_token, ln_f, one projection, its head) plus 2 per chunk past
    the first"""
    S = 128
    m = _write(tmp_path, S, SMALL, 74)
    g2._write_gpt2(tmp_path, S, SMALL, 74, name="nt", model=m)
    x = ge.gpt2_inputs(rows, S, SMALL["vocab"], seed=rows)
    counts = {}
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": 16})) as srv:
        for name, outs in (("s", NAMES), ("nt", g2.NAMES)):
            srv.predict(name, "1", x, outputs=outs)
            s0 = srv.stats()
            srv.predict(name, "1", x, outputs=outs)
            counts[name] = srv.stats()["kernel_launches"] - s0["kernel_launches"]
    chunks = -(-rows * S // 1024)
    assert counts["s"] - counts["nt"] == 2 * chunks - 2, (counts, chunks)


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_score as s
import gpt2_export as ge
tmp = sys.argv[2]
s._write(tmp, 512, dict(s.SMALL, max_pos=512), 76)
out = {}
with t.Server(s.g2._cfg(tmp, **{"gpu.maxBatch": 9})) as srv:
    for rows in (1, 9):
        x = s._holed(ge.gpt2_inputs(rows, 512, s.SMALL["vocab"], rows), rows)
        for k, v in srv.predict("s", "1", x, outputs=s.NAMES).items():
            out[f"{k}_r{rows}"] = v
np.savez(sys.argv[1], **out)
"""


def test_programmatic_dependent_launch_keeps_the_bits(tmp_path):
    """9 x 512 tokens are five chunks: their projections and score kernels overlap under PDL, not their bytes"""
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
                name = f"s{j}"
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


def test_forward_hop_score():
    world = 2
    base = tempfile.mkdtemp(prefix="tfscscore")
    for j in range(N_MODELS):
        _write(base, HOP_S, SMALL, 80 + j, name=f"s{j}")
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
        for k in NAMES:
            assert fwd["y"][j][k].shape == local["y"][j][k].shape and fwd["y"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
            assert fwd["grpc"][j][k].tobytes() == local["grpc"][j][k].tobytes() == local["y"][j][k].tobytes(), (j, k)
        assert fwd["rest"][j] == local["rest"][j] and local["rest"][j][0] == 200
    for r in results.values():
        assert r["stats"]["fwd_out_requests"] > 0 and r["stats"]["fwd_in_requests"] > 0
