"""Time of the Swin Transformer kernels and of swin_t on cuda:0, from CUDA events.

    python -m tools.time_swin [--launches 200] [--repeats 5] [--steps 20] [--model-repeats 5] [--parent PKGDIR]

1. tfsc_k_window_attention alone at Swin-T's four stage shapes (224x224: 56x56 / 3 heads, 28x28 / 6, 14x14 / 12, 7x7 / 24;
   head width 32, window 7, shift 3 but at 7x7), batch 8 and 64: median of `repeats` windows of `launches` back-to-back
   launches, microseconds per launch, and GB/s of algorithmic bytes B*H*W*(3C + C)*4 + heads*N*N*4 (qkv read, ctx written,
   the bias table), beside a device-to-device copy of 256 MB timed the same way and the 3.35 TB/s data-sheet figure.
2. Device-resident swin_t (seeded weights) through tfsc_predict_device at batch 8 and 64: ms per batch, images/s and kernel
   launches per batch; and the split of the batch's kernel time by kernel family, from torch.profiler in a separate run.
3. With --parent PKGDIR (a tfservingcache_b200 package built from another commit): ResNet-50 and BERT-base at batch 8 and the
   tenant MLP, this tree's library against that one, alternating in child processes (tools/time_convnets.py's comparison):
   times and bit-for-bit output equality.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import shutil
import tempfile

import numpy as np

from tools.time_convnets import DATASHEET_GBS, _card, _events, _median_us, ab_table

STAGES = [(56, 3, 3), (28, 6, 3), (14, 12, 3), (7, 24, 0)]   # (H = W, heads, shift) of swin_t at 224 px
D, WS = 32, 7
FAMILIES = ("window_attention", "gemm_tc", "gemm_f32", "layernorm", "patch_merge", "im2col", "dense", "avgpool")


def attention_table(torch, t, args):
    lib = t._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(0)
    src = torch.empty(64 << 20, device="cuda")
    dst = torch.empty_like(src)
    copy_us = _median_us(torch, lambda: dst.copy_(src), args.launches // 4, args.repeats)
    rows, N = [], WS * WS
    for H, heads, shift in STAGES:
        C = heads * D
        bias = torch.randn(heads, N, N, device="cuda", generator=gen)
        for B in (8, 64):
            qkv = torch.randn(B, H, H, 3 * C, device="cuda", generator=gen)
            ctx = torch.empty(B, H, H, C, device="cuda")

            def launch():
                t._lib.check(lib.tfsc_k_window_attention(qkv.data_ptr(), bias.data_ptr(), ctx.data_ptr(), B, H, H, C, heads, WS, shift, None),
                             "window_attention")
            us = _median_us(torch, launch, args.launches, args.repeats)
            nbytes = B * H * H * 4 * C * 4 + heads * N * N * 4
            rows.append({"H": H, "W": H, "C": C, "heads": heads, "shift": shift, "batch": B, "us": round(us, 2),
                         "GBps": round(nbytes / us / 1e3, 1), "pct_datasheet": round(100 * nbytes / us / 1e3 / DATASHEET_GBS, 1)})
    return {"d2d_copy_GBps": round(2 * src.numel() * 4 / copy_us / 1e3, 1), "datasheet_GBps": DATASHEET_GBS, "shapes": rows}


def seeded_swin_blob(man, seed):
    """weights of variance 1 / fan_in, biases and LayerNorm beta 0.1 N(0, 1), gamma 1, relative-position bias N(0, 1)"""
    rng = np.random.default_rng(seed)
    blob = np.zeros(man["weights_bytes"] // 4, np.float32)

    def put(off, v):
        blob[off // 4: off // 4 + v.size] = v.astype(np.float32)

    for o in man["ops"]:
        if o["op"] in ("conv", "dense"):
            fan_in = o.get("kh", 1) * o.get("kw", 1) * o["c"]
            put(o["w_offset"], rng.standard_normal(fan_in * o["cout"]) / np.sqrt(fan_in))
            put(o["b_offset"], 0.1 * rng.standard_normal(o["cout"]))
        elif o["op"] == "layernorm":
            put(o["w_offset"], np.ones(o["c"]))
            put(o["b_offset"], 0.1 * rng.standard_normal(o["c"]))
        elif o["op"] == "window_attention":
            put(o["bias_offset"], rng.standard_normal(o["heads"] * o["window"] ** 4))
    return blob


def model_table(torch, t, args):
    tmp = tempfile.mkdtemp(prefix="tfsc_swin_")
    res = {}
    try:
        man = t.modelformat.swin_manifest()
        t.modelformat.write_graph_bundle(f"{tmp}/swin_t/1", man, seeded_swin_blob(man, 0))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 4, "gpu.maxBatch": 64}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            srv.ensure(0, "swin_t", 1)
            for B in (8, 64):
                x = torch.randn(B, 224, 224, 3, device="cuda", generator=gen)
                y = torch.empty(B, 1000, device="cuda")

                def fn():
                    srv.predict_device(0, "swin_t", 1, x.data_ptr(), B, y.data_ptr(), stream.cuda_stream)
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
                res[f"swin_t_b{B}"] = {"ms_median": round(ms, 4), "ms_runs": [round(v, 4) for v in runs],
                                       "img_per_s": round(B / ms * 1e3, 1), "launches_per_batch": launches}
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
                res[f"swin_t_b{B}"]["kernel_share_pct"] = {k: round(100 * v / tot, 1) for k, v in part.items()} if tot else None
                res[f"swin_t_b{B}"]["kernel_ms_per_batch"] = round(tot / 5 / 1e3, 4)
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
    assert torch.cuda.is_available(), "time_swin needs a CUDA device"
    res = {**_card(), "launches": args.launches, "repeats": args.repeats}
    res["window_attention"] = attention_table(torch, t, args)
    res["models"] = model_table(torch, t, args)
    if args.parent:
        res["vs_parent"] = ab_table(args)
    res.update({"card_after": _card()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
