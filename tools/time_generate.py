"""Time of greedy and sampled generation on GPT-2 small on cuda:0, from CUDA events.

    python -m tools.time_generate [--launches 200] [--repeats 5] [--new 64] [--model-repeats 3] [--profile] [--sampling]
                                  [--processing] [--parent PKGDIR]

1. tfsc_k_decode_attention at rows in {1, 8, 64} and L in {128, 1024} keys, 12 heads of width 64: median of `repeats`
   windows of `launches` back-to-back launches, microseconds per launch, and the GB/s of K and V cache read (2 * rows * L * H
   * 4 bytes) next to the H100 SXM data sheet's 3.35 TB/s.
2. Device-resident GPT-2 small (seeded weights) through tfsc_predict_device, prompt 128 and 960, N = --new tokens, rows in
   {1, 8, 64}: ms per request batch, generated tokens/s, ms per decode step ((batch - prefill) / (N - 1), the prefill timed
   as the N = 1 bundle) and launches per batch. Beside it, the no-cache baseline: N calls of the next-token bundle of
   prompt + N - 1 tokens, right-padded, which is what a client without generation sends for the same tokens.
3. --profile: in a run of its own, torch.profiler's split of the decode steps' kernel time by kernel family at 8 rows and
   prompt 960 (the batch minus a prefill-only batch).
4. --parent PKGDIR: ResNet-50, BERT-base and the tenant MLP (tools/time_convnets.py's comparison), GPT-2 small
   next-token at 8 x 128 (every next-token output, half the rows right-padded) and greedy and sampled (top_k 50, top_p 0.9)
   generation of 32 tokens there,
   against a package built from another commit, alternating the two in child processes: ms per batch over windows of --steps calls, and bit-for-bit outputs.
5. --sampling: tfsc_k_generate_sample against tfsc_k_generate_select at rows in {1, 8, 64}, vocab 50257, for temperature
   only, top_k 50, top_p 0.9 and top_k 200 with top_p 0.95 (microseconds per launch, the two alternating), and a sampling
   bundle (top_k 50, top_p 0.9) against the greedy bundle end to end at prompt {128, 960} x rows {1, 8, 64}, N = --new:
   ms per batch and generated tokens/s, alternating.
6. --processing: tfsc_k_generate_process (repetition_penalty 1.3, no_repeat_ngram_size 0 or 3; greedy, and top_k 50 /
   top_p 0.9 sampled) against tfsc_k_generate_select and tfsc_k_generate_sample at rows in {1, 8, 64}, vocab 50257, histories
   of 128 and 1024 prompt tokens (a t = 1 step: the history built), alternating; and processing bundles (p 1.3, n 3) against
   the greedy and sampling bundles end to end at prompt {128, 960} x rows {1, 8, 64}, N = --new, alternating.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

from tools.time_convnets import _card, _events, _median_us, ab_table
from tools.time_gpt2 import seeded_gpt2_blob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADS, D, H, V = 12, 64, 768, 50257
FAMILIES = ("decode_attention", "generate_select", "gemm_tc", "gemm_f32", "layernorm", "last_token", "dense", "kv_cache")


def decode_table(torch, t, args):
    lib = t._lib.lib
    res = {}
    for rows in (1, 8, 64):
        for L in (128, 1024):
            S, t_ = L - 1, 0                                             # one query at slot S: L keys
            qkv = torch.randn(rows, 3 * H, device="cuda")
            kc, vc = torch.randn(rows, L, H, device="cuda"), torch.randn(rows, L, H, device="cuda")
            pos = torch.full((rows,), S - 1, dtype=torch.int32, device="cuda")
            ctx = torch.empty(rows, H, device="cuda")
            wb = lib.tfsc_k_decode_attention_work_bytes(rows, L, H, HEADS)
            work = torch.zeros(wb // 4, dtype=torch.int32, device="cuda")

            def launch():
                t._lib.check(lib.tfsc_k_decode_attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), pos.data_ptr(), t_, None, S, S,
                                                         L, ctx.data_ptr(), rows, H, HEADS, work.data_ptr(), wb, None), "decode")
            us = _median_us(torch, launch, args.launches, args.repeats)
            gbs = 2 * rows * L * H * 4 / us / 1e3
            res[f"rows{rows}_L{L}"] = {"us": round(us, 2), "cache_GBps": round(gbs, 1), "of_3350_GBps_pct": round(100 * gbs / 3350, 1)}
    return res


def _outs(n):
    return [{"name": k, "kind": k, "max_new_tokens": n} for k in ("generated_ids", "generated_log_probs", "generated_length")]


def model_table(torch, t, args):
    mf = t.modelformat
    tmp = tempfile.mkdtemp(prefix="tfsc_gen_")
    res, N = {}, args.new
    nt = [{"name": "ids", "kind": "next_token_top_k_ids", "k": 1}]
    try:
        bundles = {}
        for S in (128, 960):
            for name, seq, outs in ((f"gen_s{S}", S, _outs(N)), (f"pre_s{S}", S, _outs(1)), (f"nt_s{S}", S + N - 1, nt)):
                man = mf.gpt2_manifest(seq=seq, inputs=mf.GPT2_INPUTS, outputs=outs)
                mf.write_graph_bundle(f"{tmp}/{name}/1", man, seeded_gpt2_blob(man, 0))
                bundles[name] = (seq, sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, V)))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "modelCache.size": 8 << 30, "serving.maxConcurrentModels": 8, "gpu.maxBatch": 64}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for S in (128, 960):
                for rows in (1, 8, 64):
                    ms, launches = {}, {}
                    for name in (f"gen_s{S}", f"pre_s{S}", f"nt_s{S}"):
                        seq, width = bundles[name]
                        srv.ensure(0, name, 1)
                        ids = torch.randint(0, V, (rows, seq), device="cuda", generator=gen, dtype=torch.int32)
                        mask = torch.ones(rows, seq, dtype=torch.int32, device="cuda")
                        if name.startswith("nt"):
                            mask[:, S:] = 0                              # the prompt; each call would attend one more token
                        x = torch.cat([mask, ids], dim=1).contiguous()  # packed row: attention_mask | input_ids
                        y = torch.empty(rows, width, device="cuda")
                        calls = N if name.startswith("nt") else 1

                        def fn():
                            for _ in range(calls):
                                srv.predict_device(0, name, 1, x.data_ptr(), rows, y.data_ptr(), stream.cuda_stream)
                        fn()
                        srv.sync(0)
                        s0 = srv.stats()["kernel_launches"]
                        fn()
                        srv.sync(0)
                        launches[name] = srv.stats()["kernel_launches"] - s0
                        runs = [_events(torch, fn, 1, stream) for _ in range(args.model_repeats)]
                        ms[name] = float(np.median(runs))
                    g, p, b = ms[f"gen_s{S}"], ms[f"pre_s{S}"], ms[f"nt_s{S}"]
                    res[f"prompt{S}_rows{rows}"] = {
                        "new_tokens": N, "ms_per_batch": round(g, 3), "tokens_per_s": round(rows * N / g * 1e3, 1),
                        "ms_per_decode_step": round((g - p) / (N - 1), 4), "prefill_ms": round(p, 3),
                        "launches_per_batch": launches[f"gen_s{S}"], "no_cache_ms": round(b, 3),
                        "no_cache_tokens_per_s": round(rows * N / b * 1e3, 1), "no_cache_launches": launches[f"nt_s{S}"],
                        "speedup_vs_no_cache": round(b / g, 2)}
                    torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


SAMPLING = {"temperature_0.8": (0.8, 0, 1.0), "top_k_50": (1.0, 50, 1.0), "top_p_0.9": (1.0, 0, 0.9),
            "top_k_200_top_p_0.95": (1.0, 200, 0.95)}


def sample_kernel_table(torch, t, args):
    """us per launch of the select step and of the sampling step on the same GPT-2-sized logits, alternating"""
    lib = t._lib.lib
    res = {}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for rows in (1, 8, 64):
        ld = (V + 31) // 32 * 32
        x = torch.randn(rows, ld, device="cuda", generator=gen) * 3
        pos = torch.full((rows,), 10, dtype=torch.int32, device="cuda")
        done = torch.zeros(rows, dtype=torch.int32, device="cuda")
        seeds = torch.arange(rows, dtype=torch.int32, device="cuda")
        ids = torch.empty(rows, 2, dtype=torch.int32, device="cuda")
        lp = torch.empty(rows, 2, device="cuda")
        word, ptab, y = torch.randn(V, H, device="cuda"), torch.randn(64, H, device="cuda"), torch.empty(rows, H, device="cuda")
        common = lambda: (x.data_ptr(), ld, V, pos.data_ptr(), 1, 0, -1, done.data_ptr(), ids.data_ptr(), 2, lp.data_ptr(), 2,  # noqa: E731
                          None, 0, word.data_ptr(), ptab.data_ptr(), y.data_ptr(), rows, H)
        select = lambda: t._lib.check(lib.tfsc_k_generate_select(*common(), None), "select")  # noqa: E731
        row = {}
        for name, (temperature, k, p) in SAMPLING.items():
            def sample():
                t._lib.check(lib.tfsc_k_generate_sample(*common(), seeds.data_ptr(), 1, temperature, k, p, None), "sample")
            us = {"select": [], "sample": []}
            for _ in range(args.repeats):                                 # alternating windows
                us["select"].append(_median_us(torch, select, args.launches, 1))
                us["sample"].append(_median_us(torch, sample, args.launches, 1))
            row[name] = {"select_us": round(float(np.median(us["select"])), 2), "sample_us": round(float(np.median(us["sample"])), 2)}
        res[f"rows{rows}"] = row
    return res


def sampling_model_table(torch, t, args):
    """a sampling bundle against the greedy bundle of the same seeded GPT-2 small, end to end, alternating"""
    mf = t.modelformat
    tmp = tempfile.mkdtemp(prefix="tfsc_samp_")
    res, N = {}, args.new
    try:
        for S in (128, 960):
            for name, outs, inputs in ((f"greedy_s{S}", _outs(N), mf.GPT2_INPUTS),
                                       (f"sample_s{S}", [dict(o, top_k=50, top_p=0.9) for o in _outs(N)], mf.GPT2_SAMPLING_INPUTS)):
                man = mf.gpt2_manifest(seq=S, inputs=inputs, outputs=outs)
                mf.write_graph_bundle(f"{tmp}/{name}/1", man, seeded_gpt2_blob(man, 0))
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(_outs(N), V))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "modelCache.size": 8 << 30, "serving.maxConcurrentModels": 8, "gpu.maxBatch": 64}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for S in (128, 960):
                for rows in (1, 8, 64):
                    ids = torch.randint(0, V, (rows, S), device="cuda", generator=gen, dtype=torch.int32)
                    mask = torch.ones(rows, S, dtype=torch.int32, device="cuda")
                    seed = torch.arange(rows, dtype=torch.int32, device="cuda")[:, None]
                    xs = {"greedy": torch.cat([mask, ids], 1).contiguous(), "sample": torch.cat([mask, ids, seed], 1).contiguous()}
                    y = torch.empty(rows, width, device="cuda")
                    fns = {}
                    for kind in ("greedy", "sample"):
                        name = f"{kind}_s{S}"
                        srv.ensure(0, name, 1)
                        fns[kind] = (lambda name=name, x=xs[kind]: srv.predict_device(0, name, 1, x.data_ptr(), rows, y.data_ptr(),
                                                                                       stream.cuda_stream))
                        fns[kind]()
                    srv.sync(0)
                    ms = {"greedy": [], "sample": []}
                    for _ in range(args.model_repeats):
                        for kind in ("greedy", "sample"):
                            ms[kind].append(_events(torch, fns[kind], 1, stream))
                    g, s_ = float(np.median(ms["greedy"])), float(np.median(ms["sample"]))
                    res[f"prompt{S}_rows{rows}"] = {"new_tokens": N, "greedy_ms": round(g, 3), "sample_ms": round(s_, 3),
                                                    "greedy_tokens_per_s": round(rows * N / g * 1e3, 1),
                                                    "sample_tokens_per_s": round(rows * N / s_ * 1e3, 1)}
                    torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def process_kernel_table(torch, t, args):
    """us per launch of the select and sample steps and of the processing step on the same GPT-2-sized logits, alternating"""
    lib = t._lib.lib
    res = {}
    gen = torch.Generator(device="cuda").manual_seed(0)
    ld = (V + 31) // 32 * 32
    for rows in (1, 8, 64):
        for S in (128, 1024):
            x = torch.randn(rows, ld, device="cuda", generator=gen) * 3
            prompt = torch.randint(0, 64, (rows, S), device="cuda", generator=gen, dtype=torch.int32)  # repeats for the n-gram ban
            mask = torch.ones(rows, S, dtype=torch.int32, device="cuda")
            pos = torch.full((rows,), S - 1, dtype=torch.int32, device="cuda")
            done = torch.zeros(rows, dtype=torch.int32, device="cuda")
            seeds = torch.arange(rows, dtype=torch.int32, device="cuda")
            ids = torch.empty(rows, 2, dtype=torch.int32, device="cuda")
            lp = torch.empty(rows, 2, device="cuda")
            hist = torch.empty(rows, S + 2, dtype=torch.int32, device="cuda")
            hl0 = torch.empty(rows, dtype=torch.int32, device="cuda")
            word, ptab, y = torch.randn(V, H, device="cuda"), torch.randn(S + 2, H, device="cuda"), torch.empty(rows, H, device="cuda")
            common = lambda t_: (x.data_ptr(), ld, V, pos.data_ptr(), t_, 0, -1, done.data_ptr(), ids.data_ptr(), 2, lp.data_ptr(),  # noqa: E731
                                 2, None, 0, word.data_ptr(), ptab.data_ptr(), y.data_ptr(), rows, H)

            def process(n, sampled, t_=1):
                smp = (seeds.data_ptr(), 1, 1.0, 50, 0.9) if sampled else (None, 0, 1.0, 0, 1.0)
                t._lib.check(lib.tfsc_k_generate_process(*common(t_), prompt.data_ptr(), mask.data_ptr(), S, hist.data_ptr(), S + 2,
                                                         hl0.data_ptr(), 1.3, n, 0, *smp, None), "process")
            fns = {"select": lambda: t._lib.check(lib.tfsc_k_generate_select(*common(1), None), "select"),
                   "sample": lambda: t._lib.check(lib.tfsc_k_generate_sample(*common(1), seeds.data_ptr(), 1, 1.0, 50, 0.9, None), "sample")}
            for n in (0, 3):
                fns[f"process_n{n}"] = lambda n=n: process(n, False)
                fns[f"process_sampled_n{n}"] = lambda n=n: process(n, True)
            process(3, False, 0)                                          # t = 0: the history
            torch.cuda.synchronize()
            us = {k: [] for k in fns}
            for _ in range(args.repeats):                                 # alternating windows
                for k, fn in fns.items():
                    us[k].append(_median_us(torch, fn, args.launches, 1))
            res[f"rows{rows}_hist{S}"] = {f"{k}_us": round(float(np.median(v)), 2) for k, v in us.items()}
    return res


def processing_model_table(torch, t, args):
    """processing bundles against the greedy and sampling bundles of the same seeded GPT-2 small, end to end, alternating"""
    mf = t.modelformat
    tmp = tempfile.mkdtemp(prefix="tfsc_proc_")
    res, N = {}, args.new
    proc = dict(repetition_penalty=1.3, no_repeat_ngram_size=3)
    smp = dict(top_k=50, top_p=0.9)
    kinds = {"greedy": ({}, mf.GPT2_INPUTS), "process": (proc, mf.GPT2_INPUTS), "sample": (smp, mf.GPT2_SAMPLING_INPUTS),
             "process_sample": (dict(proc, **smp), mf.GPT2_SAMPLING_INPUTS)}
    try:
        for S in (128, 960):
            for kind, (fields, inputs) in kinds.items():
                man = mf.gpt2_manifest(seq=S, inputs=inputs, outputs=[dict(o, **fields) for o in _outs(N)])
                mf.write_graph_bundle(f"{tmp}/{kind}_s{S}/1", man, seeded_gpt2_blob(man, 0))
        width = sum(w for _n, _o, w, _d in mf.packed_output_layout(_outs(N), V))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "modelCache.size": 8 << 30, "serving.maxConcurrentModels": 8, "gpu.maxBatch": 64}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for S in (128, 960):
                for rows in (1, 8, 64):
                    ids = torch.randint(0, V, (rows, S), device="cuda", generator=gen, dtype=torch.int32)
                    mask = torch.ones(rows, S, dtype=torch.int32, device="cuda")
                    seed = torch.arange(rows, dtype=torch.int32, device="cuda")[:, None]
                    plain, seeded = torch.cat([mask, ids], 1).contiguous(), torch.cat([mask, ids, seed], 1).contiguous()
                    y = torch.empty(rows, width, device="cuda")
                    fns = {}
                    for kind, (_f, inputs) in kinds.items():
                        name = f"{kind}_s{S}"
                        srv.ensure(0, name, 1)
                        x = seeded if inputs is mf.GPT2_SAMPLING_INPUTS else plain
                        fns[kind] = (lambda name=name, x=x: srv.predict_device(0, name, 1, x.data_ptr(), rows, y.data_ptr(), stream.cuda_stream))
                        fns[kind]()
                    srv.sync(0)
                    ms = {k: [] for k in kinds}
                    for _ in range(args.model_repeats):
                        for kind in kinds:
                            ms[kind].append(_events(torch, fns[kind], 1, stream))
                    row = {"new_tokens": N}
                    for kind in kinds:
                        m_ = float(np.median(ms[kind]))
                        row[f"{kind}_ms"] = round(m_, 3)
                        row[f"{kind}_tokens_per_s"] = round(rows * N / m_ * 1e3, 1)
                    res[f"prompt{S}_rows{rows}"] = row
                    torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def profile_table(torch, t, args):
    """kernel time of one batch at 8 rows, prompt 960, minus that of the prefill-only bundle, by family"""
    from torch.profiler import ProfilerActivity, profile
    mf = t.modelformat
    tmp = tempfile.mkdtemp(prefix="tfsc_genp_")
    rows, S, N = 8, 960, args.new
    res = {}
    try:
        for name, outs in (("gen", _outs(N)), ("pre", _outs(1))):
            man = mf.gpt2_manifest(seq=S, inputs=mf.GPT2_INPUTS, outputs=outs)
            mf.write_graph_bundle(f"{tmp}/{name}/1", man, seeded_gpt2_blob(man, 0))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 4, "gpu.maxBatch": rows}
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            part = {}
            for name, outs in (("gen", _outs(N)), ("pre", _outs(1))):
                srv.ensure(0, name, 1)
                x = torch.cat([torch.ones(rows, S, dtype=torch.int32), torch.randint(0, V, (rows, S), dtype=torch.int32)], 1).cuda()
                y = torch.empty(rows, sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, V)), device="cuda")
                for _ in range(2):
                    srv.predict_device(0, name, 1, x.data_ptr(), rows, y.data_ptr(), stream.cuda_stream)
                torch.cuda.synchronize()
                fam = {k: 0.0 for k in FAMILIES + ("other",)}
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    srv.predict_device(0, name, 1, x.data_ptr(), rows, y.data_ptr(), stream.cuda_stream)
                    torch.cuda.synchronize()
                for e in prof.events():
                    if str(e.device_type).endswith("CUDA"):
                        fam[next((k for k in FAMILIES if k in e.name), "other")] += e.time_range.elapsed_us()
                part[name] = fam
            steps = {k: (part["gen"][k] - part["pre"][k]) / (N - 1) for k in part["gen"]}
            tot = sum(steps.values())
            res = {"rows": rows, "prompt": S, "kernel_us_per_decode_step": round(tot, 1),
                   "share_pct": {k: round(100 * v / tot, 1) for k, v in steps.items()} if tot else None}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def gpt2_child(out_path, steps, repeats):
    """this process's library: GPT-2 small next-token at 8 x 128 and greedy generation of 32 tokens at 8 x 128, ms per
    batch, and their outputs on seeded inputs saved to out_path"""
    import torch

    import tfservingcache_b200 as t
    mf = t.modelformat
    outs = [{"name": "next_token_position", "kind": "next_token_position"}] + \
           [{"name": k, "kind": k, "k": 5} for k in mf.NEXT_TOKEN_OUTPUT_KINDS[1:]]
    B, S = 8, 128
    tmp = tempfile.mkdtemp(prefix="tfsc_abg_")
    try:
        man = mf.gpt2_manifest(seq=S, inputs=mf.GPT2_INPUTS, outputs=outs)
        mf.write_graph_bundle(f"{tmp}/gpt2/1", man, seeded_gpt2_blob(man, 0))
        gman = mf.gpt2_manifest(seq=S, inputs=mf.GPT2_INPUTS, outputs=_outs(32))
        mf.write_graph_bundle(f"{tmp}/gen/1", gman, seeded_gpt2_blob(gman, 0))
        sman = mf.gpt2_manifest(seq=S, inputs=mf.GPT2_SAMPLING_INPUTS, outputs=[dict(o, top_k=50, top_p=0.9) for o in _outs(32)])
        mf.write_graph_bundle(f"{tmp}/smp/1", sman, seeded_gpt2_blob(sman, 0))
        rng = np.random.default_rng(0)
        ids = rng.integers(0, V, (B, S)).astype(np.int32)
        mask = np.ones((B, S), np.int32)
        mask[1::2, S // 2:] = 0
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 2, "gpu.maxBatch": B}
        with t.Server(cfg) as srv:
            out = srv.predict("gpt2", "1", {"input_ids": ids, "attention_mask": mask}, outputs=[o["name"] for o in outs])
            gen = srv.predict("gen", "1", {"input_ids": ids, "attention_mask": mask}, outputs=[o["name"] for o in _outs(32)])
            out.update({f"greedy_{k}": v for k, v in gen.items()})
            seed = (np.arange(B, dtype=np.int32) * 7919)[:, None]
            smp = srv.predict("smp", "1", {"input_ids": ids, "attention_mask": mask, "seed": seed}, outputs=[o["name"] for o in _outs(32)])
            out.update({f"sampled_{k}": v for k, v in smp.items()})
            srv.ensure(0, "gpt2", 1)
            srv.ensure(0, "gen", 1)
            stream = torch.cuda.Stream()
            x = torch.from_numpy(np.ascontiguousarray(np.concatenate([mask, ids], axis=1))).cuda()  # attention_mask | input_ids
            y = torch.empty(B, sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, V)), device="cuda")

            def fn():
                srv.predict_device(0, "gpt2", 1, x.data_ptr(), B, y.data_ptr(), stream.cuda_stream)
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            ms = float(np.median([_events(torch, fn, steps, stream) for _ in range(repeats)]))
            yg = torch.empty(B, sum(w for _n, _o, w, _d in mf.packed_output_layout(_outs(32), V)), device="cuda")

            def gfn():
                srv.predict_device(0, "gen", 1, x.data_ptr(), B, yg.data_ptr(), stream.cuda_stream)
            gfn()
            torch.cuda.synchronize()
            gms = float(np.median([_events(torch, gfn, 1, stream) for _ in range(repeats)]))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez(out_path, **out)
    print(json.dumps({"gpt2_next_token_b8_s128": ms, "gpt2_greedy_generate_b8_s128_n32": gms, "lib": t._lib.LIB_PATH}))


def gpt2_ab_table(args):
    tmp = tempfile.mkdtemp(prefix="tfsc_abgr_")
    runs = {"this": [], "parent": []}
    try:
        for rep in range(args.ab_repeats):
            for which in (("this", "parent") if rep % 2 == 0 else ("parent", "this")):
                env = dict(os.environ, PYTHONPATH=ROOT if which == "this" else os.path.abspath(args.parent) + os.pathsep + ROOT)
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--gpt2-child", f"{tmp}/{which}{rep}.npz",
                                    "--steps", str(args.steps), "--model-repeats", str(args.model_repeats)],
                                   capture_output=True, text=True, env=env, cwd=ROOT, timeout=1200)
                assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
                runs[which].append(json.loads(r.stdout.strip().splitlines()[-1]))
        assert runs["this"][0]["lib"] != runs["parent"][0]["lib"], runs["this"][0]["lib"]
        a, b = dict(np.load(f"{tmp}/this0.npz")), dict(np.load(f"{tmp}/parent0.npz"))
        same = {k: bool(a[k].tobytes() == b[k].tobytes()) for k in sorted(a)} if sorted(a) == sorted(b) else {"keys": False}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    res = {"bit_identical_to_parent": same}
    for key in ("gpt2_next_token_b8_s128", "gpt2_greedy_generate_b8_s128_n32"):
        this = [r[key] for r in runs["this"]]
        par = [r[key] for r in runs["parent"]]
        res[key + "_ms"] = {"this": round(float(np.median(this)), 4), "parent": round(float(np.median(par)), 4),
                            "this_runs": [round(v, 4) for v in this], "parent_runs": [round(v, 4) for v in par]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10, help="calls per timed window of the --parent comparison")
    ap.add_argument("--model-repeats", type=int, default=3)
    ap.add_argument("--ab-repeats", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--skip-models", action="store_true")
    ap.add_argument("--sampling", action="store_true")
    ap.add_argument("--processing", action="store_true")
    ap.add_argument("--parent", default=None, help="a tfservingcache_b200 package built from the commit to compare against")
    ap.add_argument("--gpt2-child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.gpt2_child:
        return gpt2_child(args.gpt2_child, args.steps, args.model_repeats)
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_generate needs a CUDA device"
    res = {**_card()}
    res["decode_attention"] = decode_table(torch, t, args)
    if not args.skip_models:
        res["models"] = model_table(torch, t, args)
    if args.sampling:
        res["sample_step"] = sample_kernel_table(torch, t, args)
        res["sampling_models"] = sampling_model_table(torch, t, args)
    if args.processing:
        res["process_step"] = process_kernel_table(torch, t, args)
        res["processing_models"] = processing_model_table(torch, t, args)
    if args.profile:
        res["decode_step_profile"] = profile_table(torch, t, args)
    if args.parent:
        res["vs_parent"] = ab_table(args)
        res["vs_parent"]["gpt2_b8_s128"] = gpt2_ab_table(args)
    res.update({"card_after": _card()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
