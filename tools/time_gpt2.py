"""Time of causal attention and of GPT-2 small on cuda:0, from CUDA events.

    python -m tools.time_gpt2 [--launches 200] [--repeats 5] [--steps 20] [--model-repeats 5] [--parent PKGDIR]

1. tfsc_k_attention_causal against tfsc_k_attention_mask at 8 x 1024 tokens, 12 heads of width 64 (GPT-2 small's shape; the
   key-block kernel): median of `repeats` windows of `launches` back-to-back launches, microseconds per launch.
2. Device-resident GPT-2 small (seeded weights, every output) through tfsc_predict_device at 8 x 128 and 8 x 1024: ms per
   batch, sequences/s and kernel launches per batch; and the split of the batch's kernel time by kernel family, from
   torch.profiler in a separate run.
3. With --parent PKGDIR (a tfservingcache_b200 package built from another commit): ResNet-50 and BERT-base at batch 8 and the
   tenant MLP, this tree's library against that one, alternating in child processes (tools/time_convnets.py's comparison):
   times and bit-for-bit output equality.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import shutil
import tempfile

import numpy as np

from tools.time_convnets import _card, _events, _median_us, ab_table

B, HEADS, D = 8, 12, 64
FAMILIES = ("attention", "gemm_tc", "gemm_f32", "layernorm", "embed_positions", "last_token", "dense", "fill_mask_head")


def attention_table(torch, t, args):
    lib = t._lib.lib
    S, H = 1024, HEADS * D
    gen = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, S, 3 * H, device="cuda", generator=gen)
    ctx = torch.empty(B, S, H, device="cuda")
    mask = torch.ones(B, S, dtype=torch.int32, device="cuda")
    res = {"batch": B, "S": S, "heads": HEADS, "d": D}
    for name, fn in (("causal", lib.tfsc_k_attention_causal), ("non_causal", lib.tfsc_k_attention_mask)):
        def launch():
            t._lib.check(fn(qkv.data_ptr(), mask.data_ptr(), S, ctx.data_ptr(), B, S, H, HEADS, None), name)
        res[f"{name}_us"] = round(_median_us(torch, launch, args.launches, args.repeats), 2)
    res["speedup"] = round(res["non_causal_us"] / res["causal_us"], 3)
    return res


def seeded_gpt2_blob(man, seed):
    """weights of variance 1 / fan_in, biases and LayerNorm beta 0.1 N(0, 1), gamma 1, embeddings 0.1 N(0, 1), the decoder
    the word table transposed and zero-padded"""
    rng = np.random.default_rng(seed)
    blob = np.zeros(man["weights_bytes"] // 4, np.float32)

    def put(off, v):
        blob[off // 4: off // 4 + v.size] = v.astype(np.float32).ravel()

    emb = man["ops"][0]
    word = 0.1 * rng.standard_normal((emb["vocab"], emb["c"]))
    put(emb["word_offset"], word)
    put(emb["pos_offset"], 0.1 * rng.standard_normal(emb["max_pos"] * emb["c"]))
    for o in man["ops"][1:-1]:
        if o["op"] == "conv":
            put(o["w_offset"], rng.standard_normal(o["c"] * o["cout"]) / np.sqrt(o["c"]))
            put(o["b_offset"], 0.1 * rng.standard_normal(o["cout"]))
        elif o["op"] == "layernorm":
            put(o["w_offset"], np.ones(o["c"]))
            put(o["b_offset"], 0.1 * rng.standard_normal(o["c"]))
    dec = man["ops"][-1]
    w = np.zeros((dec["c"], dec["cout"]), np.float32)
    w[:, :emb["vocab"]] = word.T
    put(dec["w_offset"], w)
    return blob


def model_table(torch, t, args):
    mf = t.modelformat
    tmp = tempfile.mkdtemp(prefix="tfsc_gpt2_")
    res = {}
    outs = [{"name": "next_token_position", "kind": "next_token_position"}] + \
           [{"name": k, "kind": k, "k": 5} for k in mf.NEXT_TOKEN_OUTPUT_KINDS[1:]]
    width = sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, 50257))
    try:
        for S in (128, 1024):
            man = mf.gpt2_manifest(seq=S, inputs=mf.GPT2_INPUTS, outputs=outs)
            mf.write_graph_bundle(f"{tmp}/gpt2_s{S}/1", man, seeded_gpt2_blob(man, 0))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 4, "gpu.maxBatch": B}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for S in (128, 1024):
                name = f"gpt2_s{S}"
                srv.ensure(0, name, 1)
                ids = torch.randint(0, 50257, (B, S), device="cuda", generator=gen, dtype=torch.int32)
                mask = torch.ones(B, S, dtype=torch.int32, device="cuda")
                mask[1::2, S // 2:] = 0                                   # half the rows right-padded
                x = torch.cat([mask, ids], dim=1).contiguous()          # packed row: attention_mask | input_ids
                y = torch.empty(B, width, device="cuda")

                def fn():
                    srv.predict_device(0, name, 1, x.data_ptr(), B, y.data_ptr(), stream.cuda_stream)
                for _ in range(5):
                    fn()
                srv.sync(0)
                s0 = srv.stats()["kernel_launches"]
                fn()
                srv.sync(0)
                launches = srv.stats()["kernel_launches"] - s0
                torch.cuda.synchronize()
                assert torch.isfinite(y).all().item()
                runs = [_events(torch, fn, args.steps, stream) for _ in range(args.model_repeats)]
                ms = float(np.median(runs))
                key = f"gpt2_small_b{B}_s{S}"
                res[key] = {"ms_median": round(ms, 4), "ms_runs": [round(v, 4) for v in runs],
                            "seq_per_s": round(B / ms * 1e3, 1), "tokens_per_s": round(B * S / ms * 1e3, 1),
                            "launches_per_batch": launches}
                # kernel split, traced in a run of its own after the timed windows
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        fn()
                    torch.cuda.synchronize()
                tot, part = 0.0, {k: 0.0 for k in FAMILIES + ("other",)}
                for e in prof.events():
                    if str(e.device_type).endswith("CUDA"):
                        d = e.time_range.elapsed_us()
                        tot += d
                        part[next((k for k in FAMILIES if k in e.name), "other")] += d
                res[key]["kernel_share_pct"] = {k: round(100 * v / tot, 1) for k, v in part.items()} if tot else None
                res[key]["kernel_ms_per_batch"] = round(tot / 5 / 1e3, 4)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--model-repeats", type=int, default=5)
    ap.add_argument("--ab-repeats", type=int, default=4)
    ap.add_argument("--parent", default=None, help="a tfservingcache_b200 package built from the commit to compare against")
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_gpt2 needs a CUDA device"
    res = {**_card(), "launches": args.launches, "repeats": args.repeats}
    res["attention"] = attention_table(torch, t, args)
    res["models"] = model_table(torch, t, args)
    if args.parent:
        res["vs_parent"] = ab_table(args)
    res.update({"card_after": _card()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
