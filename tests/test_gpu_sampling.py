"""-m gpu: GPT-2 sampling generate bundles. tfsc_k_generate_sample against the fp64 reference sampler (sampling_ref) at
GPT-2's and the widest vocabulary, its log-probabilities and next-step input bit for bit against tfsc_k_generate_select,
top_k = 1 as the greedy step, a chi-square test of 32768 draws of one row per config, and through the server: seeded GPT-2
small teacher-forced against transformers fp64, batch and coalescing independence, repeatability, every front-end, the
forward hop, programmatic dependent launch and launch counts."""
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
import sampling_ref as sr  # noqa: E402
import test_gpu_generate as gg  # noqa: E402
import test_gpu_gpt2 as g2  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = t._lib.lib
mf = t.modelformat
SMALL = g2.SMALL
N = 6
NAMES = gg.NAMES
_ptr, _cuda = gg._ptr, gg._cuda


def _outs(n=N, eos=None, **fields):
    return [dict(o, **fields) for o in gg._outs(n, eos)]


# ----------------------------------------------------------------------------------------------- the kernel ----
def _step(fn, x, pos, vocab, t_, done, word, ptab, seeds=None, cfg=None, off=0, last=False, eos=-1):
    """one launch of tfsc_k_generate_select (fn = "select") or tfsc_k_generate_sample with cfg = (temperature, top_k, top_p)
    and seeds; returns ids[:, t], log_probs[:, t], length, done and y"""
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
    common = (_ptr(xd), vp, vocab, _ptr(pd), t_, int(last), eos, _ptr(dd), _ptr(ids), n, _ptr(lp), n, _ptr(ln), 1, _ptr(wd), _ptr(td),
              _ptr(y[off:]), rows, H)
    if fn == "select":
        t._lib.check(lib.tfsc_k_generate_select(*common, None), "generate_select")
    else:
        sd = _cuda(np.asarray(seeds, np.int32), np.int32)
        t._lib.check(lib.tfsc_k_generate_sample(*common, _ptr(sd), 1, *cfg, None), "generate_sample")
    torch.cuda.synchronize()
    return (ids.cpu().numpy()[:, t_], lp.cpu().numpy()[:, t_], ln.cpu().numpy(), dd.cpu().numpy(),
            y[off:].cpu().numpy().reshape(rows, H))


def _rows(rows, vocab, vp, seed):
    """_head_logits' rows (ties for first place, 1e30 padding, row 1 with no attended token) with a constant row, rows of
    spread 8..32, rows with many exact ties and rows with NaN / +inf past the vocabulary"""
    rng = np.random.default_rng(seed)
    x, pos = g2._head_logits(rows, vocab, vp, seed)
    x[:2, :vocab] *= 8                                                    # keeps the tie for first place
    x[2] = 0.5
    for r in range(3, rows):
        x[r, :vocab] = rng.standard_normal(vocab).astype(np.float32) * (8 + (r % 7) * 4)
        if r % 5 == 0:
            x[r, :vocab] = np.round(x[r, :vocab])                         # many exact ties
        if r % 3 == 0 and vp > vocab:
            x[r, vocab:] = np.nan if r % 2 else np.inf
    pos = pos % 24
    pos[1] = -1
    return x, pos


CONFIGS = [(1.0, 0, 1.0), (0.5, 40, 1.0), (1.7, 0, 0.9), (1.0, 40, 0.5), (0.5, 0, 0.5), (1.7, -1, 1.0), (1.0, -1, 0.9),
           (0.5, 1, 0.9), (1.7, 40, 0.9)]


@pytest.mark.parametrize("vocab,vp", [(50257, 50272), (57344, 57344), (100, 128)])
@pytest.mark.parametrize("misalign", [False, True])
def test_sample_matches_reference(vocab, vp, misalign):
    rows, H, P = 96, 768 if not misalign else 30, 64
    x, pos = _rows(rows, vocab, vp, vocab + misalign)
    rng = np.random.default_rng(vocab)
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((P, H)).astype(np.float32)
    t_ = 3
    done = np.where(np.arange(rows) % 11 == 4, 1, 0).astype(np.int32)  # a few rows ended earlier
    sel = _step("select", x, pos, vocab, t_, done, word, ptab, off=int(misalign))
    L = -sel[1].astype(np.float32)                                        # log(sum) of each row: the argmax has logit m
    m = x[:, :vocab].max(1)
    seeds = rng.integers(-2 ** 31, 2 ** 31, rows).astype(np.int32)
    total = amb = 0
    live = done == 0
    for temperature, top_k, top_p in CONFIGS:
        k = vocab if top_k < 0 else top_k
        ids, lp, ln, dn, y = _step("sample", x, pos, vocab, t_, done, word, ptab, seeds, (temperature, k, top_p), off=int(misalign))
        assert np.array_equal(ln, sel[2]) and np.array_equal(dn, sel[3])
        assert (ids[~live] == -1).all() and (lp[~live] == 0).all()
        for r in np.nonzero(live)[0]:
            g = ids[r]
            assert 0 <= g < vocab, (r, g)
            want, a = sr.draw(x[r, :vocab], seeds[r], t_, temperature, k, top_p)
            assert a or g == want, (temperature, k, top_p, r, g, want)
            if r != 2:  # the constant row: every weight is 1 / vocab of W, so most draws lie within 1e-5 W of an edge
                total += 1
                amb += a
            exp_lp = np.float32(np.float32(x[r, g]) - m[r]) - L[r]
            assert lp[r].tobytes() == np.float32(exp_lp).tobytes(), (r, lp[r], exp_lp)
            assert y[r].tobytes() == (word[g] + ptab[pos[r] + 1 + t_]).astype(np.float32).tobytes(), r
        for r in (0, 5, 30):                                               # a row alone: its bits in the batch
            one = _step("sample", x[r:r + 1], pos[r:r + 1], vocab, t_, done[r:r + 1], word, ptab, seeds[r:r + 1], (temperature, k, top_p),
                        off=int(misalign))
            for a_, b_ in zip(one, (ids, lp, ln, dn, y)):
                assert a_.tobytes() == b_[r:r + 1].tobytes(), r
        if k == 1:                                                         # top_k = 1: the select step's bits
            for a_, b_ in zip((ids, lp, ln, dn, y), sel):
                assert a_.tobytes() == b_.tobytes()
    assert amb <= 0.01 * total, (amb, total)


def test_sample_rejections():
    import torch
    z = torch.zeros(1 << 16, device="cuda")
    p = torch.zeros(4, dtype=torch.int32, device="cuda")
    E = t._lib.E_INVALID

    def call(vocab=100, temperature=1.0, top_k=0, top_p=1.0, seeds=True, stride=1):
        return lib.tfsc_k_generate_sample(_ptr(z), 128, vocab, _ptr(p), 0, 1, -1, _ptr(p), None, 0, None, 0, None, 0, None, None, None,
                                          1, 8, _ptr(p) if seeds else None, stride, temperature, top_k, top_p, None)
    assert call() == 0 and call(top_k=100) == 0 and call(top_p=1e-6) == 0
    for kw in (dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=float("inf")), dict(temperature=float("nan")),
               dict(temperature=1e-39),
               dict(top_k=101), dict(top_k=-1), dict(top_p=0.0), dict(top_p=1.5), dict(seeds=False), dict(stride=0),
               dict(vocab=57345)):
        assert call(**kw) == E, kw
    torch.cuda.synchronize()


DIST = [(1.0, 0, 1.0), (0.7, 50, 1.0), (1.3, 0, 0.9), (1.0, 200, 0.95), (0.5, 20, 0.5), (2.0, 0, 0.3)]


def test_distribution_chi_square():
    """one designed row replicated over 32768 rows with seeds 0..32767, one launch per config: no draw outside the kept set,
    and the counts fit the fp64 kept distribution (the seeds are fixed, so the verdict is too)"""
    from scipy import stats
    vocab, vp, rows, H = 1000, 1024, 32768, 4
    rng = np.random.default_rng(11)
    z = np.sort(rng.standard_normal(vocab) * 2.5)[::-1].astype(np.float32)
    z = z[rng.permutation(vocab)]
    z[[17, 400]] = z.max()                                                # a tie for first place
    x = np.tile(np.concatenate([z, np.full(vp - vocab, np.nan, np.float32)]), (rows, 1))
    pos = np.zeros(rows, np.int32)
    word = np.zeros((vocab, H), np.float32)
    ptab = np.zeros((4, H), np.float32)
    for temperature, top_k, top_p in DIST:
        ids, _lp, _ln, _dn, _y = _step("sample", x, pos, vocab, 0, np.zeros(rows, np.int32), word, ptab, np.arange(rows), (temperature, top_k, top_p),
                                       last=True)
        probs = sr.kept_probabilities(z, temperature, top_k, top_p)
        assert set(np.unique(ids).tolist()) <= set(probs), (temperature, top_k, top_p)
        keys = sorted(probs, key=lambda i: -probs[i])
        expct = np.array([probs[i] * rows for i in keys])
        obs = np.array([(ids == i).sum() for i in keys], np.float64)
        big = expct >= 5                                                  # pool the small bins
        o, e = list(obs[big]), list(expct[big])
        if (~big).any():
            o.append(obs[~big].sum())
            e.append(expct[~big].sum())
        pval = stats.chisquare(o, np.array(e) * sum(o) / sum(e)).pvalue if len(o) > 1 else 1.0
        assert pval > 1e-3, (temperature, top_k, top_p, pval)


# ------------------------------------------------------------------------------------------ served models ----
def _write(tmp, seq, arch, seed, name="s", outputs=None, model=None, inputs=mf.GPT2_SAMPLING_INPUTS):
    return gg._write(tmp, seq, arch, seed, name=name, outputs=_outs(top_k=40) if outputs is None else outputs, model=model,
                     inputs=inputs)


def _inputs(B, S, vocab, seed, seeds=None):
    x = ge.gpt2_inputs(B, S, vocab, seed=seed)
    x["seed"] = (np.arange(B, dtype=np.int32) * 7919 + seed if seeds is None else np.asarray(seeds, np.int32)).reshape(B, 1)
    return x


def _check_sampled(model, x, r, V, cfg):
    """teacher-forced against transformers fp64: log-probs within 1e-4, every token in the reference's kept set, and every
    non-ambiguous step the reference's draw on the fp64 logits"""
    temperature, top_k, top_p = cfg
    amb = total = 0
    for b in range(len(x["input_ids"])):
        ids, lp, n = r["generated_ids"][b], r["generated_log_probs"][b], r["generated_length"][b]
        assert n == len(ids) and (ids >= 0).all() and (ids < V).all()
        ref = gg._teacher_forced(model, dict(x, gen=r["generated_ids"]), b)[:, :V]
        lse = ref.max(1) + np.log(np.exp(ref - ref.max(1, keepdims=True)).sum(1))
        want_lp = ref[np.arange(len(ids)), ids] - lse
        assert np.all(np.abs(lp - want_lp) <= 1e-4 * np.maximum(1.0, np.abs(want_lp))), (b, np.abs(lp - want_lp).max())
        for s in range(len(ids)):
            kept, _w, _a = sr.kept_set(ref[s], temperature, top_k, top_p)
            assert ids[s] in set(kept.tolist()), (b, s)
            want, a = sr.draw(ref[s], x["seed"][b, 0], s, temperature, top_k, top_p)
            # fp32 logits differ from fp64 ones by ~1e-5: a boundary or draw edge that close is not the kernel's to decide
            a = a or (ids[s] != want and _near(ref[s], temperature, top_k, top_p, x["seed"][b, 0], s))
            total += 1
            amb += a
            assert a or ids[s] == want, (b, s, ids[s], want)
    # a seeded GPT-2 is nearly uniform over its vocabulary, so many draws sit within 1e-5 W of an edge: most must not
    assert amb <= 0.5 * total, (amb, total)


def _near(z, temperature, top_k, top_p, seed, s):
    """whether moving each logit by up to 2e-4 max(1, |z|) could change the draw: the draws at the two extremes disagree"""
    d = 2e-4 * np.maximum(1.0, np.abs(z))
    ks, _w, _a = sr.kept_set(z, temperature, top_k, top_p)
    out = set()
    for sign in (1, -1):
        zz = z.copy()
        zz[ks] += sign * d[ks]
        out.add(sr.draw(zz, seed, s, temperature, top_k, top_p)[0])
        zz = z.copy()
        zz[ks] -= sign * d[ks]
        zz[ks[:1]] += sign * d[ks[:1]] * 2
        out.add(sr.draw(zz, seed, s, temperature, top_k, top_p)[0])
    return len(out) > 1


E2E = [(0.8, 40, 1.0), (1.0, 0, 0.9), (1.3, 200, 0.95)]


@pytest.mark.parametrize("S", [128, 992])
def test_gpt2_small_samples(S, tmp_path):
    import torch
    n, V = 32, 50257
    m = _write(tmp_path, S, dict(max_pos=1024), 41, name="s0", outputs=_outs(n, temperature=E2E[0][0], top_k=E2E[0][1]))
    for i, (temperature, top_k, top_p) in enumerate(E2E[1:], 1):
        fields = dict(temperature=temperature, top_p=top_p, **({"top_k": top_k} if top_k else {}))
        _write(tmp_path, S, dict(max_pos=1024), 41, name=f"s{i}", model=m, outputs=_outs(n, **fields))
    _write(tmp_path, S, dict(max_pos=1024), 41, name="k1", model=m, outputs=_outs(n, temperature=1.3, top_k=1, top_p=0.5))
    _write(tmp_path, S, dict(max_pos=1024), 41, name="g", model=m, outputs=gg._outs(n), inputs=mf.GPT2_INPUTS)
    _write(tmp_path, S, dict(max_pos=1024), 41, name="ids", model=m, inputs=[{"name": "input_ids", "role": "ids"}, {"name": "seed", "role": "seed"}],
           outputs=_outs(n, temperature=1.0, top_p=0.9))
    x = _inputs(8, S, V, S)
    torch.cuda.empty_cache()
    with t.Server(g2._cfg(tmp_path)) as srv:
        for i, cfg in enumerate(E2E):
            r = srv.predict(f"s{i}", "1", x, outputs=NAMES)
            _check_sampled(m, x, r, V, cfg)
            again = srv.predict(f"s{i}", "1", x, outputs=NAMES)
            assert all(again[k].tobytes() == r[k].tobytes() for k in NAMES)            # the same seeds: the same bits
            other = srv.predict(f"s{i}", "1", dict(x, seed=x["seed"] + 1), outputs=NAMES)
            assert sum(not np.array_equal(other["generated_ids"][b], r["generated_ids"][b]) for b in range(8)) >= 6
        greedy = srv.predict("g", "1", {k: v for k, v in x.items() if k != "seed"}, outputs=NAMES)
        k1 = srv.predict("k1", "1", x, outputs=NAMES)
        assert all(k1[k].tobytes() == greedy[k].tobytes() for k in NAMES)              # top_k = 1 is greedy
        # ids and seed only: every position attended, as the ids-only greedy bundle
        xi = {"input_ids": x["input_ids"], "seed": x["seed"]}
        ri = srv.predict("ids", "1", xi, outputs=NAMES)
        _check_sampled(m, dict(xi, attention_mask=np.ones_like(x["input_ids"])), ri, V, E2E[1])
        # an EOS the bundle draws mid-sequence: the row stops there, counted, and pads with -1 and 0
        full = srv.predict("s1", "1", x, outputs=NAMES)
        eos = int(full["generated_ids"][0, n // 2])
        _write(tmp_path, S, dict(max_pos=1024), 41, name="e", model=m, outputs=_outs(n, eos=eos, temperature=1.0, top_p=0.9))
        r = srv.predict("e", "1", x, outputs=NAMES)
    for b in range(8):
        ids = list(full["generated_ids"][b])
        k = ids.index(eos) + 1 if eos in ids else n
        assert r["generated_length"][b] == k and r["generated_ids"][b, :k].tobytes() == full["generated_ids"][b, :k].tobytes()
        assert (r["generated_ids"][b, k:] == -1).all() and (r["generated_log_probs"][b, k:] == 0).all()


def test_rows_do_not_depend_on_their_batch(tmp_path):
    """at any position of a 64-row request beside other seeds, and coalesced requests as one request of the same rows: the
    same bits. (The decoder's dense layers route by batch size, so a row's logits, not its draw, may differ between a 1-row
    and a 64-row request; the draw's own batch independence is tested on the kernel.)"""
    S = 40
    _write(tmp_path, S, SMALL, 77, outputs=_outs(temperature=1.2, top_k=50, top_p=0.95))
    x = _inputs(64, S, SMALL["vocab"], 5)
    x["seed"][:8] = 4242                                                  # the same prompt and seed twice: the same tokens
    x["input_ids"][1], x["attention_mask"][1] = x["input_ids"][0], x["attention_mask"][0]
    sizes = [3, 5]
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": 64})) as srv:
        whole = srv.predict("s", "1", x, outputs=NAMES)
        assert whole["generated_ids"][0].tobytes() == whole["generated_ids"][1].tobytes()
        perm = np.random.default_rng(0).permutation(64)
        shuffled = srv.predict("s", "1", {k: v[perm] for k, v in x.items()}, outputs=NAMES)
        assert all(shuffled[k].tobytes() == np.ascontiguousarray(whole[k][perm]).tobytes() for k in NAMES)
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": sum(sizes), "gpu.tickMicros": 3_000_000})) as srv:
        joint = srv.predict("s", "1", {k: v[:sum(sizes)] for k, v in x.items()}, outputs=NAMES)
        st0 = srv.stats()
        parts = ((0, sizes[0]), (sizes[0], sizes[1]))
        tk = [srv.predict_submit("s", "1", {k: v[lo:lo + n] for k, v in x.items()}, outputs=NAMES) for lo, n in parts]
        outs = [k.wait(30.0) for k in tk]
        [k.release() for k in tk]
        assert srv.stats()["batches"] - st0["batches"] == 1
    for (lo, n), r in zip(parts, outs):                                   # the bits of one request of the same rows
        assert all(r[k].tobytes() == np.ascontiguousarray(joint[k][lo:lo + n]).tobytes() for k in NAMES)


# ----------------------------------------------------------------------------------------- front-ends ----
def test_every_frontend_on_a_sampling_bundle(tmp_path):
    import torch
    S, B = 32, 5
    outs = _outs(temperature=0.9, top_p=0.9)
    _write(tmp_path, S, SMALL, 73, outputs=outs)
    x = _inputs(B, S, SMALL["vocab"], 3)
    with t.Server(g2._cfg(tmp_path)) as srv:
        full = srv.predict("s", "1", x, outputs=NAMES)
        one = srv.predict("s", "1", {k: v[0] for k, v in x.items()}, outputs=NAMES)
        assert one["generated_ids"].shape == (N,) and one["generated_ids"].tobytes() == full["generated_ids"][0].tobytes()
        _spec, g = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("s", 1, x)))
        assert list(g) == NAMES and all(g[k].tobytes() == full[k].tobytes() for k in NAMES)
        st, b = srv.rest_handle("POST", "/v1/models/s/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        for i, p in enumerate(json.loads(b)["predictions"]):
            assert np.array_equal(np.int32(p["generated_ids"]), full["generated_ids"][i])
            assert np.array_equal(np.float32(p["generated_log_probs"]), full["generated_log_probs"][i])
        st, b = srv.rest_handle("POST", "/v1/models/s/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and all(np.array_equal(np.asarray(cols[k], full[k].dtype), full[k]) for k in NAMES)
        st, b = srv.rest_handle("GET", "/v1/models/s/versions/1/metadata")
        sig = json.loads(b)["metadata"]["signature_def"]["signature_def"]["serving_default"]["inputs"]
        assert st == 200 and {k: (v["dtype"], [d["size"] for d in v["tensor_shape"]["dim"]]) for k, v in sig.items()} == {
            "input_ids": ("DT_INT32", ["-1", str(S)]), "attention_mask": ("DT_INT32", ["-1", str(S)]), "seed": ("DT_INT32", ["-1", "1"])}
        # the layout messages: the seed is one value per row, the other inputs S
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("s", "1", dict(x, seed=np.zeros((B, 2), np.int32)), outputs=NAMES)
        assert ("input 'seed' has 2 values per row, not 1; model expects inputs 'attention_mask', 'input_ids', 'seed', DT_INT32"
                f" [batch, {S}] each, 'seed' DT_INT32 [batch, 1]") in str(e.value)
        with pytest.raises(t._lib.TfscError) as e:
            srv.predict("s", "1", {k: v for k, v in x.items() if k != "seed"}, outputs=NAMES)
        assert "input 'seed' is missing" in str(e.value)
        with pytest.raises(t._lib.TfscError) as e:
            srv.grpc_session_run(g2._session_run_request("s", "input_ids:0", x["input_ids"], "generated_ids:0"))
        assert e.value.code == t._lib.E_INVALID
        for verb in ("classify", "regress"):
            st, b = srv.rest_handle("POST", f"/v1/models/s/versions/1:{verb}", json.dumps({"examples": [{"x": 1.0}]}).encode())
            assert st == 400
        srv.ensure(0, "s", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, SMALL["vocab"]))
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.GPT2_SAMPLING_INPUTS)], axis=1)
        assert packed.shape == (B, 2 * S + 1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "s", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), outs, SMALL["vocab"])
        assert all(dev[k].tobytes() == full[k].tobytes() for k in NAMES)


@pytest.mark.parametrize("rows", [1, 8])
def test_launch_counts_equal_the_greedy_bundle(tmp_path, rows):
    S = 64
    m = _write(tmp_path, S, SMALL, 74, outputs=_outs(top_k=20, top_p=0.9))
    _write(tmp_path, S, SMALL, 74, name="g", model=m, outputs=gg._outs(), inputs=mf.GPT2_INPUTS)
    x = _inputs(rows, S, SMALL["vocab"], rows)
    counts = []
    with t.Server(g2._cfg(tmp_path)) as srv:
        for name, xx in (("s", x), ("g", {k: v for k, v in x.items() if k != "seed"})):
            srv.predict(name, "1", xx, outputs=NAMES)
            s0 = srv.stats()
            srv.predict(name, "1", xx, outputs=NAMES)
            counts.append(srv.stats()["kernel_launches"] - s0["kernel_launches"])
    assert counts[0] == counts[1], counts


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_sampling as s
tmp = sys.argv[2]
s._write(tmp, 300, s.SMALL, 75, outputs=s._outs(temperature=1.1, top_k=30, top_p=0.9))
out = {}
with t.Server(s.g2._cfg(tmp)) as srv:
    for rows in (1, 8):
        for k, v in srv.predict("s", "1", s._inputs(rows, 300, s.SMALL["vocab"], rows), outputs=s.NAMES).items():
            out[f"{k}_r{rows}"] = v
np.savez(sys.argv[1], **out)
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
            x = _inputs(HOP_ROWS, HOP_S, SMALL["vocab"], 7)
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


def test_forward_hop_sampling():
    world = 2
    base = tempfile.mkdtemp(prefix="tfscsample")
    for j in range(N_MODELS):
        _write(base, HOP_S, SMALL, 80 + j, name=f"s{j}", outputs=_outs(temperature=0.9 + 0.1 * j, top_k=50, top_p=0.9))
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
