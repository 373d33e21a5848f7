"""Kernel time of tfsc_k_attention (csrc/nn_kernels.cu) on cuda:0, from CUDA events over back-to-back launches.

    python -m tools.time_attention [--batch 8] [--hidden 768] [--heads 12] [--seqs 128 384 512] [--launches 200] [--repeats 5]

Prints one JSON object: the card name and power limit it ran on, and per sequence length the median / every repeat in
microseconds per launch. Inputs are seeded; ids have no [PAD]. Writes nothing to disk."""
import argparse
import json
import subprocess

import numpy as np


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (s.strip() for s in out.split(",", 1))
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": f"unknown ({e!r})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--hidden", type=int, default=768)
    ap.add_argument("--heads", type=int, default=12)
    ap.add_argument("--seqs", type=int, nargs="+", default=[128, 384, 512])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_attention needs a CUDA device"
    lib = t._lib.lib
    B, H, heads = args.batch, args.hidden, args.heads
    gen = torch.Generator(device="cuda").manual_seed(0)
    res = {**_card(), "batch": B, "hidden": H, "heads": heads, "launches": args.launches, "seqs": {}}
    for S in args.seqs:
        qkv = torch.randn(B, S, 3 * H, device="cuda", generator=gen)
        ids = torch.randint(1, 1000, (B, S), device="cuda", dtype=torch.int32, generator=gen)
        ctx = torch.empty(B, S, H, device="cuda")

        def launch():
            t._lib.check(lib.tfsc_k_attention(qkv.data_ptr(), ids.data_ptr(), ctx.data_ptr(), B, S, H, heads, None), "attention")

        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        runs = []
        for _ in range(args.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                launch()
            e1.record()
            torch.cuda.synchronize()
            runs.append(e0.elapsed_time(e1) * 1e3 / args.launches)
        res["seqs"][str(S)] = {"us_median": round(float(np.median(runs)), 1),
                               "us_runs": [round(r, 1) for r in runs]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
