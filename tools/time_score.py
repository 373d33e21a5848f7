"""Time of GPT-2 scoring (token_log_probs, token_ranks, token_log_prob_sum, token_count) on cuda:0, from CUDA events.

    python -m tools.time_score [--launches 100] [--repeats 5] [--model-repeats 5] [--parent PKGDIR]

1. tfsc_k_token_score over 1,024 and 8,192 token rows of vocab 50,257 (ld 50,272) in rows of 1,024 unpadded tokens, so every
   token row but each row's last is scored: median of `repeats` windows of `launches` back-to-back launches, microseconds
   per launch, and the GB/s of logits read (scored rows * vocab * 4 bytes) next to the H100 SXM data sheet's 3.35 TB/s.
2. Device-resident GPT-2 small (seeded weights) score bundles through tfsc_predict_device at S in {128, 1024} x rows in
   {1, 8, 64}: ms per batch and scored tokens/s, beside the next-token bundle of the same shape (the trunk's cost: its
   last_token, one-token ln_f, projection and head are small). In a run of its own, torch.profiler's kernel time of one
   batch of each bundle: the score kernel, the score head, and the projection, which is the score bundle's GEMM and dense
   kernel time less the next-token bundle's (the trunk's GEMMs are the same launches in both).
3. --parent PKGDIR: tools/time_generate.py's comparison against a package built from another commit, alternating the two in
   child processes: ResNet-50, BERT-base and the tenant MLP, and GPT-2 small next-token, greedy and sampled generation at
   8 x 128; ms per batch and bit-for-bit outputs.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import shutil
import tempfile

import numpy as np

from tools.time_convnets import _card, _events, _median_us
from tools.time_gpt2 import seeded_gpt2_blob

V, LD = 50257, 50272
PROJECTION = ("gemm", "dense", "cluster")


def kernel_table(torch, t, args):
    lib = t._lib.lib
    res = {}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for n in (1024, 8192):
        S, rows = 1024, n // 1024
        x = torch.randn(n, LD, device="cuda", generator=gen) * 3
        ids = torch.randint(0, V, (rows, S), device="cuda", generator=gen, dtype=torch.int32)
        lp = torch.empty(rows * S, device="cuda")
        rk = torch.empty(rows * S, dtype=torch.int32, device="cuda")

        def launch():
            t._lib.check(lib.tfsc_k_token_score(x.data_ptr(), LD, 0, n, ids.data_ptr(), None, S, rows, S, V, lp.data_ptr(),
                                                rk.data_ptr(), None), "token_score")
        us = _median_us(torch, launch, args.launches, args.repeats)
        gbs = (n - rows) * V * 4 / us / 1e3
        res[f"tokens{n}"] = {"us": round(us, 2), "logits_GBps": round(gbs, 1), "of_3350_GBps_pct": round(100 * gbs / 3350, 1)}
    return res


def _bundles(t, tmp):
    mf = t.modelformat
    score = [{"name": k, "kind": k} for k in mf.SCORE_OUTPUT_KINDS]
    nt = [{"name": "next_token_position", "kind": "next_token_position"}, {"name": "ids", "kind": "next_token_top_k_ids", "k": 5}]
    out = {}
    for S in (128, 1024):
        for kind, outs in (("score", score), ("nt", nt)):
            man = mf.gpt2_manifest(seq=S, inputs=mf.GPT2_INPUTS, outputs=outs)
            mf.write_graph_bundle(f"{tmp}/{kind}_s{S}/1", man, seeded_gpt2_blob(man, 0))
            out[f"{kind}_s{S}"] = sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, S if kind == "score" else V))
    return out


def model_table(torch, t, args):
    from torch.profiler import ProfilerActivity, profile
    tmp = tempfile.mkdtemp(prefix="tfsc_score_")
    res = {}
    try:
        widths = _bundles(t, tmp)
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "modelCache.size": 8 << 30, "serving.maxConcurrentModels": 8, "gpu.maxBatch": 64}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for S in (128, 1024):
                for rows in (1, 8, 64):
                    ids = torch.randint(0, V, (rows, S), device="cuda", generator=gen, dtype=torch.int32)
                    x = torch.cat([torch.ones(rows, S, dtype=torch.int32, device="cuda"), ids], 1).contiguous()  # mask | ids
                    fns = {}
                    for kind in ("score", "nt"):
                        name = f"{kind}_s{S}"
                        y = torch.empty(rows, widths[name], device="cuda")
                        srv.ensure(0, name, 1)
                        fns[kind] = (lambda name=name, y=y: srv.predict_device(0, name, 1, x.data_ptr(), rows, y.data_ptr(),
                                                                                stream.cuda_stream))
                        fns[kind]()
                    srv.sync(0)
                    ms = {"score": [], "nt": []}
                    for _ in range(args.model_repeats):
                        for kind in ("score", "nt"):
                            ms[kind].append(_events(torch, fns[kind], 1, stream))
                    fam = {}
                    for kind in ("score", "nt"):
                        f = {"token_score": 0.0, "score_head": 0.0, "projection_family": 0.0, "other": 0.0}
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            fns[kind]()
                            torch.cuda.synchronize()
                        for e in prof.events():
                            if str(e.device_type).endswith("CUDA"):
                                k = ("token_score" if "token_score" in e.name else "score_head" if "score_head" in e.name
                                     else "projection_family" if any(p in e.name for p in PROJECTION) else "other")
                                f[k] += e.time_range.elapsed_us() / 1e3
                        fam[kind] = f
                    s_ms, nt_ms = float(np.median(ms["score"])), float(np.median(ms["nt"]))
                    proj = fam["score"]["projection_family"] - fam["nt"]["projection_family"]
                    res[f"S{S}_rows{rows}"] = {
                        "score_ms": round(s_ms, 3), "scored_tokens_per_s": round(rows * (S - 1) / s_ms * 1e3, 1),
                        "next_token_ms": round(nt_ms, 3), "score_minus_next_token_ms": round(s_ms - nt_ms, 3),
                        "profiled_ms": {"token_score_kernel": round(fam["score"]["token_score"], 3),
                                        "score_head": round(fam["score"]["score_head"], 3), "projection": round(proj, 3),
                                        "score_bundle_kernels": round(sum(fam["score"].values()), 3),
                                        "next_token_bundle_kernels": round(sum(fam["nt"].values()), 3)},
                        "ms_runs": {k: [round(v, 3) for v in ms[k]] for k in ms}}
                    torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--model-repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10, help="calls per timed window of the --parent comparison")
    ap.add_argument("--ab-repeats", type=int, default=2)
    ap.add_argument("--skip-models", action="store_true")
    ap.add_argument("--parent", default=None, help="a tfservingcache_b200 package built from the commit to compare against")
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_score needs a CUDA device"
    res = {**_card()}
    res["token_score"] = kernel_table(torch, t, args)
    if not args.skip_models:
        res["models"] = model_table(torch, t, args)
    if args.parent:
        from tools.time_generate import ab_table, gpt2_ab_table
        res["vs_parent"] = ab_table(args)
        res["vs_parent"]["gpt2_b8_s128"] = gpt2_ab_table(args)
    res.update({"card_after": _card()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
