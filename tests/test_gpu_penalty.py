"""-m gpu: GPT-2 processing generate bundles (repetition_penalty, no_repeat_ngram_size, min_new_tokens).
tfsc_k_generate_process against the reference (penalty_ref) over chained steps at GPT-2's, the widest and a 100-token
vocabulary, greedy and sampled, on the vector and scalar paths, with unpadded, left-, right- and fully padded prompts, done
rows, out-of-range prompt ids and an all-banned row; its log-probabilities and next-step input bit for bit against
tfsc_k_generate_select's formula; a row alone as in its batch; p = 1 as the select and sample steps. Through the server:
seeded GPT-2 small teacher-forced against transformers fp64 run through transformers' processors, p = 1 bundles as the
greedy and sampling bundles, repeatability, permutation and coalescing, every front-end, launch counts, TFSC_PDL=0 and the
forward hop."""
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
import penalty_ref as pr  # noqa: E402
import test_gpu_generate as gg  # noqa: E402
import test_gpu_gpt2 as g2  # noqa: E402
import test_gpu_sampling as gs  # noqa: E402

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
class Chain:
    """device buffers of one chain of steps over the same rows: done, hist and hist_len0 persist between steps"""

    def __init__(self, x, pos, prompt, mask, vocab, n, word, ptab, off=0, proc=(1.0, 0, 0), eos=-1, seeds=None, cfg=None):
        import torch
        self.torch = torch
        self.rows, self.vp = x.shape
        self.S = prompt.shape[1]
        self.vocab, self.n, self.H, self.off, self.proc, self.eos, self.cfg = vocab, n, word.shape[1], off, proc, eos, cfg
        self.xd, self.pd = _cuda(x), _cuda(pos, np.int32)
        self.idd = _cuda(prompt, np.int32)
        self.md = None if mask is None else _cuda(mask, np.int32)
        self.wd, self.td = _cuda(word, off=off), _cuda(ptab, off=off)
        self.sd = None if seeds is None else _cuda(np.asarray(seeds, np.int32), np.int32)
        self.done = torch.zeros(self.rows, dtype=torch.int32, device="cuda")
        self.hld = self.S + n
        self.hist = torch.full((self.rows, self.hld), -7, dtype=torch.int32, device="cuda")
        self.hl0 = torch.full((self.rows,), -7, dtype=torch.int32, device="cuda")
        self.ids = torch.full((self.rows, n), 12345, dtype=torch.int32, device="cuda")
        self.lp = torch.full((self.rows, n), float("nan"), device="cuda")
        self.ln = torch.full((self.rows,), 777, dtype=torch.int32, device="cuda")
        self.y = torch.full((self.rows * self.H + off,), float("nan"), device="cuda")

    def step(self, t_, x=None):
        if x is not None:
            self.xd = _cuda(x)
        sampling = (_ptr(self.sd), 1, *self.cfg) if self.sd is not None else (None, 0, 1.0, 0, 1.0)
        t._lib.check(lib.tfsc_k_generate_process(
            _ptr(self.xd), self.vp, self.vocab, _ptr(self.pd), t_, int(t_ == self.n - 1), self.eos, _ptr(self.done),
            _ptr(self.ids), self.n, _ptr(self.lp), self.n, _ptr(self.ln), 1, _ptr(self.wd), _ptr(self.td), _ptr(self.y[self.off:]),
            self.rows, self.H, _ptr(self.idd), _ptr(self.md), self.S, _ptr(self.hist), self.hld, _ptr(self.hl0), *self.proc,
            *sampling, None), "generate_process")
        self.torch.cuda.synchronize()
        return (self.ids.cpu().numpy()[:, t_], self.lp.cpu().numpy()[:, t_], self.ln.cpu().numpy(), self.done.cpu().numpy(),
                self.y[self.off:].cpu().numpy().reshape(self.rows, self.H))


def _prompts(rows, S, vocab, seed):
    """ids [rows, S] with out-of-range ids, masks cycling unpadded / right / left / fully padded, and pos"""
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, min(vocab, 12), (rows, S)).astype(np.int32)      # a small alphabet: n-grams repeat
    ids[:, ::7] = rng.integers(-5, vocab + 5, (rows, len(range(0, S, 7))))
    ids[0, 3], ids[0, 4] = -1000, vocab + 1000
    mask = np.ones((rows, S), np.int32)
    pos = np.full(rows, S - 1, np.int32)
    for r in range(rows):
        k = int(rng.integers(2, S))
        if r % 4 == 1:                                                      # right-padded
            mask[r, k:] = 0
            pos[r] = k - 1
        elif r % 4 == 2:                                                    # left-padded
            mask[r, :S - k] = 0
        elif r % 4 == 3 and r % 8 == 7:                                     # fully padded
            mask[r] = 0
            pos[r] = -1
    mask[5, [2, 5, 9]] = 0                                                  # holes in an unpadded row
    return ids, mask, pos


CASES = [(1.3, 3, 2), (0.7, 0, 0), (1.0, 2, 3), (2.9, 1, 0)]


def _case(vocab, vp, misalign, sampled, seed, rows=24):
    """sampling_test's logits rows, _prompts' prompts, tables and (sampled) seeds and a temperature / top-k / top-p config"""
    S, H, P = 128, (768 if not misalign else 30), 160
    x0, _p = gs._rows(rows, vocab, vp, seed)
    rng = np.random.default_rng(seed)
    ids, mask, pos = _prompts(rows, S, vocab, seed)
    if vocab == 100:                                                        # row 4: every id in its prompt, so n = 1 bans all
        ids[4, :100], mask[4], pos[4] = np.arange(100), 1, S - 1
    word = rng.standard_normal((vocab, H)).astype(np.float32)
    ptab = rng.standard_normal((P, H)).astype(np.float32)
    eos = 7
    seeds = rng.integers(-2 ** 31, 2 ** 31, rows).astype(np.int32) if sampled else None
    cfg = (0.9, 40, 0.95) if sampled else None
    return x0, ids, mask, pos, word, ptab, eos, seeds, cfg, S


@pytest.mark.parametrize("vocab,vp", [(50257, 50272), (57344, 57344), (100, 128)])
@pytest.mark.parametrize("misalign", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_process_matches_reference(vocab, vp, misalign, sampled):
    x0, ids, mask, pos, word, ptab, eos, seeds, cfg, S = _case(vocab, vp, misalign, sampled, vocab + misalign)
    rows, steps = len(pos), 4
    for ci, proc in enumerate(CASES):
        m_ = mask if ci != 3 else None                                      # the last case: no mask, every position up to p
        ch = Chain(x0, pos, ids, m_, vocab, steps, word, ptab, off=int(misalign), proc=proc, eos=eos, seeds=seeds, cfg=cfg)
        hist = [pr.history(ids[r], None if m_ is None else m_[r], int(pos[r]), vocab) for r in range(rows)]
        done = np.zeros(rows, bool)
        total = amb = 0
        for t_ in range(steps):
            x = x0.copy()
            x[:, :vocab] = np.roll(x0[:, :vocab], 13 * t_, axis=1) if t_ else x0[:, :vocab]
            if t_ == 2:
                x[6:9, :vocab] = np.roll(x[6:9, :vocab], 1, axis=1)
            g, lp, ln, dn, y = ch.step(t_, x)
            sel = gg._select(x, pos, vocab, t_, t_ == steps - 1, eos, done.astype(np.int32), word, ptab, off=int(misalign))
            L = -sel[1].astype(np.float32)                                  # log(sum) of each row: the argmax has logit m
            m = x[:, :vocab].max(1)
            live = (pos >= 0) & ~done
            assert (g[~live] == -1).all() and (lp[~live] == 0).all() and (ln[live] == t_ + 1).all()
            for r in np.nonzero(live)[0]:
                want, a = pr.pick(x[r, :vocab], hist[r], t_, *proc, eos, None if seeds is None else seeds[r],
                                  *(cfg or (1.0, 0, 1.0)))
                if r != 2:  # the constant row: every draw lies within 1e-5 W of an edge
                    total += 1
                    amb += a
                assert a or g[r] == want, (proc, t_, r, g[r], want)
                exp_lp = np.float32(np.float32(x[r, g[r]]) - m[r]) - L[r]
                assert lp[r].tobytes() == np.float32(exp_lp).tobytes(), (r, lp[r], exp_lp)
                if t_ < steps - 1:
                    assert y[r].tobytes() == (word[g[r]] + ptab[pos[r] + 1 + t_]).astype(np.float32).tobytes(), r
                all_banned = pr.process(x[r, :vocab], hist[r], t_, *proc, eos).max() == -np.inf
                assert all_banned or g[r] not in pr.banned_ngrams(hist[r], proc[1]), (t_, r)
                assert t_ >= proc[2] or g[r] != eos, (t_, r)
            if vocab == 100 and proc[1] == 1 and live[4]:
                assert g[4] == 0                                            # every id banned: the lowest id
            for r in range(rows):
                hist[r].append(int(g[r]) if live[r] else 0)                 # a row that is not live is not checked again
            done = done | ~live | (g == eos)
            assert np.array_equal(dn.astype(bool), done)
        assert amb <= 0.02 * max(total, 1), (amb, total)
        # the row alone gives its bits in the batch
        for r in (0, 2, 5):
            one = Chain(x0[r:r + 1], pos[r:r + 1], ids[r:r + 1], None if m_ is None else m_[r:r + 1], vocab, steps, word, ptab,
                        off=int(misalign), proc=proc, eos=eos, seeds=None if seeds is None else seeds[r:r + 1], cfg=cfg)
            many = Chain(x0, pos, ids, m_, vocab, steps, word, ptab, off=int(misalign), proc=proc, eos=eos, seeds=seeds, cfg=cfg)
            for t_ in range(2):
                for a_, b_ in zip(one.step(t_), many.step(t_)):
                    assert a_.tobytes() == b_[r:r + 1].tobytes(), (r, t_)


@pytest.mark.parametrize("vocab,vp", [(50257, 50272), (100, 128)])
@pytest.mark.parametrize("sampled", [False, True])
def test_penalty_one_is_the_select_and_sample_step(vocab, vp, sampled):
    """p = 1, no n-gram and no minimum: every output bit for bit the select (or sample) step's at each step"""
    x0, ids, mask, pos, word, ptab, eos, seeds, cfg, S = _case(vocab, vp, False, sampled, 3)
    rows = len(pos)
    ch = Chain(x0, pos, ids, mask, vocab, 3, word, ptab, proc=(1.0, 0, 0), eos=eos, seeds=seeds, cfg=cfg)
    done = np.zeros(rows, np.int32)
    for t_ in range(3):
        got = ch.step(t_)
        if sampled:
            want = gs._step("sample", x0, pos, vocab, t_, done, word, ptab, seeds, cfg, last=t_ == 2, eos=eos)
        else:
            want = gg._select(x0, pos, vocab, t_, t_ == 2, eos, done, word, ptab)
        written = (pos >= 0) & (done == 0) if t_ else np.ones(rows, bool)  # a done row's length keeps its step's value
        for i in (0, 1, 3) + ((4,) if t_ < 2 else ()):                      # the last step writes no next input
            assert got[i].tobytes() == want[i].tobytes(), (t_, i)
        assert got[2][written].tobytes() == want[2][written].tobytes(), t_
        done = got[3].astype(np.int32)


def test_process_rejections():
    import torch
    z = torch.zeros(1 << 16, device="cuda")
    i32 = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")  # noqa: E731
    pos, done, prompt, hist, hl0, seed = i32(1), i32(1), i32(4), i32(8), i32(1), i32(1)
    E = t._lib.E_INVALID

    def call(vocab=100, penalty=1.3, n=2, m=0, eos=-1, seeds=False, stride=1, cfg=(1.0, 0, 1.0), hist_=True, hld=8, ids=True):
        return lib.tfsc_k_generate_process(_ptr(z), 128, vocab, _ptr(pos), 0, 1, eos, _ptr(done), None, 0, None, 0, None, 0, None, None,
                                           None, 1, 8, _ptr(prompt) if ids else None, None, 4, _ptr(hist) if hist_ else None, hld,
                                           _ptr(hl0) if hist_ else None, penalty, n, m, _ptr(seed) if seeds else None, stride, *cfg, None)
    assert call() == 0 and call(m=3, eos=99) == 0 and call(seeds=True, cfg=(0.5, 100, 0.5)) == 0 and call(penalty=1.0, n=0) == 0
    for kw in (dict(penalty=0.0), dict(penalty=-1.0), dict(penalty=float("inf")), dict(penalty=float("nan")), dict(penalty=1e-39),
               dict(n=-1), dict(m=-1), dict(m=2), dict(m=2, eos=100), dict(seeds=True, stride=0), dict(seeds=True, cfg=(0.0, 0, 1.0)),
               dict(seeds=True, cfg=(1.0, 101, 1.0)), dict(seeds=True, cfg=(1.0, 0, 0.0)), dict(hist_=False), dict(hld=0), dict(ids=False),
               dict(vocab=57345)):
        assert call(**kw) == E, kw
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ served models ----
def _write(tmp, seq, arch, seed, name="p", outputs=None, model=None, inputs=mf.GPT2_INPUTS):
    return gg._write(tmp, seq, arch, seed, name=name, outputs=_outs(repetition_penalty=1.3, no_repeat_ngram_size=3) if outputs is None
                     else outputs, model=model, inputs=inputs)


def _check_processed(model, x, r, V, proc, eos=-1, sampling=None):
    """teacher-forced against transformers fp64 logits run through transformers' processors on each row's history: every
    token the processed argmax (or draw) unless a near-tie decides it, log-probs within 1e-4 of the raw model's, and exactly
    no banned n-gram and no EOS before step m"""
    penalty, ngram, min_new = proc
    amb = total = 0
    for b in range(len(x["input_ids"])):
        ids, lp, n = r["generated_ids"][b], r["generated_log_probs"][b], r["generated_length"][b]
        assert (ids[:n] >= 0).all() and (ids[:n] < V).all() and (ids[n:] == -1).all()
        mask = x["attention_mask"][b]
        p = int(np.nonzero(mask)[0].max())
        h0 = pr.history(x["input_ids"][b], mask, p, V)
        ref = gg._teacher_forced(model, dict(x, gen=np.where(ids >= 0, ids, 0)[None].repeat(len(x["input_ids"]), 0)), b)[:, :V]
        lse = ref.max(1) + np.log(np.exp(ref - ref.max(1, keepdims=True)).sum(1))
        want_lp = ref[np.arange(n), ids[:n]] - lse[:n]
        assert np.all(np.abs(lp[:n] - want_lp) <= 1e-4 * np.maximum(1.0, np.abs(want_lp))), (b, np.abs(lp[:n] - want_lp).max())
        for s in range(n):
            h = h0 + ids[:s].tolist()
            if ngram:
                assert ids[s] not in pr.banned_ngrams(h, ngram), (b, s)
            if s < min_new:
                assert ids[s] != eos, (b, s)
            zp = pr.transformers_process(ref[s], h, len(h0), penalty, ngram or None, min_new or None, eos, dtype=np.float64)
            total += 1
            if sampling is None:
                srt = np.sort(zp)[::-1]
                clear = srt[0] - srt[1] > 2e-4 * max(1.0, abs(srt[0]))
                amb += not clear
                assert not clear or ids[s] == int(np.argmax(zp)), (b, s)
            else:
                temperature, top_k, top_p = sampling
                want, a = gs.sr.draw(zp, x["seed"][b, 0], s, temperature, top_k, top_p)
                a = a or (ids[s] != want and gs._near(zp, temperature, top_k, top_p, x["seed"][b, 0], s))
                amb += a
                assert a or ids[s] == want, (b, s, ids[s], want)
    assert amb <= 0.5 * total, (amb, total)


SAMPLING = (0.8, 40, 0.95)


@pytest.mark.parametrize("S", [128, 992])
def test_gpt2_small_processing(S, tmp_path):
    import torch
    n, V = 32, 50257
    arch = dict(max_pos=1024)
    m = _write(tmp_path, S, arch, 41, name="g", outputs=gg._outs(n))
    x = ge.gpt2_inputs(8, S, V, seed=S)
    x["input_ids"][0, -12:] = x["input_ids"][0, -24:-12]                   # a repeated tail: the n-gram ban has work at once
    torch.cuda.empty_cache()
    with t.Server(g2._cfg(tmp_path)) as srv:
        greedy = srv.predict("g", "1", x, outputs=NAMES)
        eos = int(greedy["generated_ids"][0, 1])                           # a token greedy emits early
        _write(tmp_path, S, arch, 41, name="p", model=m, outputs=_outs(n, repetition_penalty=1.3, no_repeat_ngram_size=3))
        _write(tmp_path, S, arch, 41, name="pm", model=m, outputs=_outs(n, eos=eos, repetition_penalty=1.3, no_repeat_ngram_size=3,
                                                                         min_new_tokens=6))
        _write(tmp_path, S, arch, 41, name="ps", model=m, inputs=mf.GPT2_SAMPLING_INPUTS,
               outputs=_outs(n, repetition_penalty=1.3, no_repeat_ngram_size=3, temperature=SAMPLING[0], top_k=SAMPLING[1],
                             top_p=SAMPLING[2]))
        _write(tmp_path, S, arch, 41, name="s", model=m, inputs=mf.GPT2_SAMPLING_INPUTS,
               outputs=_outs(n, temperature=SAMPLING[0], top_k=SAMPLING[1], top_p=SAMPLING[2]))
        _write(tmp_path, S, arch, 41, name="one", model=m, outputs=_outs(n, repetition_penalty=1.0))
        _write(tmp_path, S, arch, 41, name="ones", model=m, inputs=mf.GPT2_SAMPLING_INPUTS,
               outputs=_outs(n, repetition_penalty=1.0, temperature=SAMPLING[0], top_k=SAMPLING[1], top_p=SAMPLING[2]))
        r = srv.predict("p", "1", x, outputs=NAMES)
        rm = srv.predict("pm", "1", x, outputs=NAMES)
        xs = gs._inputs(8, S, V, S)
        xs["input_ids"], xs["attention_mask"] = x["input_ids"], x["attention_mask"]
        rs = srv.predict("ps", "1", xs, outputs=NAMES)
        again = srv.predict("ps", "1", xs, outputs=NAMES)
        assert all(again[k].tobytes() == rs[k].tobytes() for k in NAMES)
        one = srv.predict("one", "1", x, outputs=NAMES)
        assert all(one[k].tobytes() == greedy[k].tobytes() for k in NAMES)  # p = 1: the greedy bundle's bits
        ones = srv.predict("ones", "1", xs, outputs=NAMES)
        plain = srv.predict("s", "1", xs, outputs=NAMES)
        assert all(ones[k].tobytes() == plain[k].tobytes() for k in NAMES)  # and the sampling bundle's
    _check_processed(m, x, r, V, (1.3, 3, 0))
    _check_processed(m, x, rm, V, (1.3, 3, 6), eos=eos)
    _check_processed(m, xs, rs, V, (1.3, 3, 0), sampling=SAMPLING)
    assert not np.array_equal(r["generated_ids"], greedy["generated_ids"])


def test_rows_do_not_depend_on_their_batch(tmp_path):
    """a 64-row request and its permutation, and coalesced requests as one request of the same rows: the same bits"""
    S = 40
    _write(tmp_path, S, SMALL, 77, outputs=_outs(eos=3, repetition_penalty=1.2, no_repeat_ngram_size=2, min_new_tokens=2))
    _write(tmp_path, S, SMALL, 77, name="ps", inputs=mf.GPT2_SAMPLING_INPUTS,
           outputs=_outs(repetition_penalty=1.4, no_repeat_ngram_size=1, temperature=1.2, top_k=50, top_p=0.95))
    x = gs._inputs(64, S, SMALL["vocab"], 5)
    x["input_ids"][1], x["attention_mask"][1] = x["input_ids"][0], x["attention_mask"][0]
    xg = {k: v for k, v in x.items() if k != "seed"}
    sizes = [3, 5]
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": 64})) as srv:
        for name, xx in (("p", xg), ("ps", x)):
            whole = srv.predict(name, "1", xx, outputs=NAMES)
            again = srv.predict(name, "1", xx, outputs=NAMES)
            assert all(again[k].tobytes() == whole[k].tobytes() for k in NAMES)
            perm = np.random.default_rng(0).permutation(64)
            shuffled = srv.predict(name, "1", {k: v[perm] for k, v in xx.items()}, outputs=NAMES)
            assert all(shuffled[k].tobytes() == np.ascontiguousarray(whole[k][perm]).tobytes() for k in NAMES)
    with t.Server(g2._cfg(tmp_path, **{"gpu.maxBatch": sum(sizes), "gpu.tickMicros": 3_000_000})) as srv:
        for name, xx in (("p", xg), ("ps", x)):
            joint = srv.predict(name, "1", {k: v[:sum(sizes)] for k, v in xx.items()}, outputs=NAMES)
            st0 = srv.stats()
            parts = ((0, sizes[0]), (sizes[0], sizes[1]))
            tk = [srv.predict_submit(name, "1", {k: v[lo:lo + n] for k, v in xx.items()}, outputs=NAMES) for lo, n in parts]
            outs = [k.wait(30.0) for k in tk]
            [k.release() for k in tk]
            assert srv.stats()["batches"] - st0["batches"] == 1
            for (lo, n), r in zip(parts, outs):
                assert all(r[k].tobytes() == np.ascontiguousarray(joint[k][lo:lo + n]).tobytes() for k in NAMES)


# ----------------------------------------------------------------------------------------- front-ends ----
def test_every_frontend_on_a_processing_bundle(tmp_path):
    import torch
    S, B = 32, 5
    outs = _outs(eos=2, repetition_penalty=1.5, no_repeat_ngram_size=2, min_new_tokens=3)
    _write(tmp_path, S, SMALL, 73, outputs=outs)
    x = ge.gpt2_inputs(B, S, SMALL["vocab"], seed=3)
    with t.Server(g2._cfg(tmp_path)) as srv:
        full = srv.predict("p", "1", x, outputs=NAMES)
        one = srv.predict("p", "1", {k: v[0] for k, v in x.items()}, outputs=NAMES)
        assert one["generated_ids"].shape == (N,) and one["generated_ids"].tobytes() == full["generated_ids"][0].tobytes()
        _spec, g = wire.decode_predict_response(srv.grpc_predict(wire.encode_predict_request("p", 1, x)))
        assert list(g) == NAMES and all(g[k].tobytes() == full[k].tobytes() for k in NAMES)
        st, b = srv.rest_handle("POST", "/v1/models/p/versions/1:predict",
                                json.dumps({"instances": [{k: x[k][i].tolist() for k in x} for i in range(B)]}).encode())
        assert st == 200, b
        for i, p in enumerate(json.loads(b)["predictions"]):
            assert np.array_equal(np.int32(p["generated_ids"]), full["generated_ids"][i])
            assert np.array_equal(np.float32(p["generated_log_probs"]), full["generated_log_probs"][i])
        st, b = srv.rest_handle("POST", "/v1/models/p/versions/1:predict", json.dumps({"inputs": {k: v.tolist() for k, v in x.items()}}).encode())
        cols = json.loads(b)["outputs"]
        assert st == 200 and all(np.array_equal(np.asarray(cols[k], full[k].dtype), full[k]) for k in NAMES)
        srv.ensure(0, "p", 1)
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, SMALL["vocab"]))
        packed = np.concatenate([x[n] for n in mf.packed_input_order(mf.GPT2_INPUTS)], axis=1)
        xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
        yd = torch.full((B, width), float("nan"), device="cuda")
        srv.predict_device(0, "p", 1, _ptr(xd), B, _ptr(yd), 0)
        srv.sync(0)
        dev = mf.split_packed_rows(yd.cpu().numpy(), outs, SMALL["vocab"])
        assert all(dev[k].tobytes() == full[k].tobytes() for k in NAMES)
    for b_ in range(B):
        ids = full["generated_ids"][b_]
        assert 2 not in ids[:3].tolist()


@pytest.mark.parametrize("rows", [1, 8])
def test_launch_counts_equal_the_greedy_bundle(tmp_path, rows):
    S = 64
    m = _write(tmp_path, S, SMALL, 74, outputs=_outs(eos=1, repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=2))
    _write(tmp_path, S, SMALL, 74, name="g", model=m, outputs=gg._outs())
    x = ge.gpt2_inputs(rows, S, SMALL["vocab"], seed=rows)
    counts = []
    with t.Server(g2._cfg(tmp_path)) as srv:
        for name in ("p", "g"):
            srv.predict(name, "1", x, outputs=NAMES)
            s0 = srv.stats()
            srv.predict(name, "1", x, outputs=NAMES)
            counts.append(srv.stats()["kernel_launches"] - s0["kernel_launches"])
    assert counts[0] == counts[1], counts


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_penalty as s
tmp = sys.argv[2]
s._write(tmp, 300, s.SMALL, 75, outputs=s._outs(eos=5, repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=2))
s._write(tmp, 300, s.SMALL, 75, name="ps", inputs=s.mf.GPT2_SAMPLING_INPUTS,
         outputs=s._outs(repetition_penalty=0.8, no_repeat_ngram_size=2, temperature=1.1, top_k=30, top_p=0.9))
out = {}
with t.Server(s.g2._cfg(tmp)) as srv:
    for rows in (1, 8):
        x = s.gs._inputs(rows, 300, s.SMALL["vocab"], rows)
        for name, xx in (("p", {k: v for k, v in x.items() if k != "seed"}), ("ps", x)):
            for k, v in srv.predict(name, "1", xx, outputs=s.NAMES).items():
                out[f"{name}_{k}_r{rows}"] = v
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
    assert sorted(res["default"]) == sorted(res["0"]) and len(res["0"]) == 4 * len(NAMES)
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
                name = f"p{j}"
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


def test_forward_hop_processing():
    world = 2
    base = tempfile.mkdtemp(prefix="tfscpenalty")
    for j in range(N_MODELS):
        _write(base, HOP_S, SMALL, 80 + j, name=f"p{j}",
               outputs=_outs(eos=j, repetition_penalty=1.1 + 0.2 * j, no_repeat_ngram_size=1 + j, min_new_tokens=1 + j))
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
