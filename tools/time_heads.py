"""Time of the classification head of multi-output bundles (csrc/head.cu) on cuda:0, from CUDA events.

    python -m tools.time_heads [--launches 200] [--repeats 5] [--resnet-steps 20] [--resnet-repeats 7]

1. tfsc_k_classify_head alone, writing probabilities, classes and top-5 for rows 8 / 128 and N 1000 / 9216 / 30522: median /
   every repeat in microseconds per launch over back-to-back launches.
2. Device-resident ResNet-50 (224x224, 1000 classes, seeded random weights) at batch 8 through tfsc_predict_device, the
   single-output bundle and the same weights with logits, probabilities, classes and top-5, alternating in one run:
   median / every repeat in milliseconds per batch.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import shutil
import subprocess
import tempfile

import numpy as np

OUTPUTS = [{"name": "logits", "kind": "logits"}, {"name": "probabilities", "kind": "probabilities"},
           {"name": "classes", "kind": "classes"}, {"name": "top_k_classes", "kind": "top_k_classes", "k": 5},
           {"name": "top_k_probabilities", "kind": "top_k_probabilities", "k": 5}]


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (s.strip() for s in out.split(",", 1))
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": f"unknown ({e!r})"}


def _events(torch, fn, n, stream=None):
    """ms per call of fn() over n back-to-back calls, between events on `stream` (the stream fn launches on)"""
    stream = stream or torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _kernel_us(torch, fn, kernel, n=50):
    """mean device duration of `kernel` over n calls of fn(), from torch.profiler's CUDA activity (after the event windows,
    so the tracing does not slow them). Back-to-back launches from Python are bounded by the host's launch rate for small
    heads; this is the kernel alone."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    ds = [e.time_range.elapsed_us() for e in prof.events() if kernel in e.name and str(e.device_type).endswith("CUDA")]
    return round(float(np.mean(ds)), 2) if ds else None


def _resnet_blob(man, seed=0):
    """seeded weights of variance 1 / fan_in, zero biases: finite logits at every depth"""
    rng = np.random.default_rng(seed)
    blob = np.zeros(man["weights_bytes"] // 4, np.float32)
    for o in man["ops"]:
        if o["op"] in ("conv", "dense"):
            fan_in = o.get("kh", 1) * o.get("kw", 1) * o["c"]
            n = fan_in * o["cout"]
            blob[o["w_offset"] // 4: o["w_offset"] // 4 + n] = rng.standard_normal(n).astype(np.float32) / np.sqrt(fan_in)
    return blob


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--resnet-steps", type=int, default=20)
    ap.add_argument("--resnet-repeats", type=int, default=7)
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_heads needs a CUDA device"
    lib = t._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(0)
    res = {**_card(), "k": 5, "launches": args.launches, "head_us": {}}
    for rows in (8, 128):
        for n in (1000, 9216, 30522):
            x = torch.randn(rows, n, device="cuda", generator=gen) * 4
            p = torch.empty(rows, n, device="cuda")
            c = torch.empty(rows, dtype=torch.int64, device="cuda")
            i = torch.empty(rows, 5, dtype=torch.int32, device="cuda")
            tp = torch.empty(rows, 5, device="cuda")

            def launch():
                t._lib.check(lib.tfsc_k_classify_head(x.data_ptr(), rows, n, 5, p.data_ptr(), c.data_ptr(), i.data_ptr(),
                                                      tp.data_ptr(), None), "classify_head")

            for _ in range(20):
                launch()
            torch.cuda.synchronize()
            runs = [_events(torch, launch, args.launches) * 1e3 for _ in range(args.repeats)]
            res["head_us"][f"rows{rows}_n{n}"] = {"us_median": round(float(np.median(runs)), 2), "us_runs": [round(r, 2) for r in runs],
                                                  "kernel_us": _kernel_us(torch, launch, "classify_head_kernel")}

    tmp = tempfile.mkdtemp(prefix="tfsc_heads_")
    try:
        single = t.modelformat.resnet50_manifest()
        multi = t.modelformat.resnet50_manifest(outputs=OUTPUTS)
        blob = _resnet_blob(single)
        t.modelformat.write_graph_bundle(f"{tmp}/single/1", single, blob)
        t.modelformat.write_graph_bundle(f"{tmp}/multi/1", multi, blob)
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 4}
        B = 8
        x = torch.randn(B, 224, 224, 3, device="cuda", generator=gen)
        width = {"single": 1000, "multi": 2 + 1000 + 1000 + 5 + 5}
        ys = {k: torch.empty(B, w, device="cuda") for k, w in width.items()}
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()   # a stream of its own: the events and the launches must share it
            for name in width:
                srv.ensure(0, name, 1)
            fns = {name: (lambda name=name: srv.predict_device(0, name, 1, x.data_ptr(), B, ys[name].data_ptr(), stream.cuda_stream))
                   for name in width}
            for name in width:   # warm every shape the timed windows use
                for _ in range(5):
                    fns[name]()
            torch.cuda.synchronize()
            runs = {name: [] for name in width}
            for rep in range(args.resnet_repeats):
                order = list(width) if rep % 2 == 0 else list(width)[::-1]
                for name in order:
                    runs[name].append(_events(torch, fns[name], args.resnet_steps, stream))
            srv.sync(0)
            # the multi-output bundle's logits are the single-output bundle's bits
            same = bool(torch.equal(ys["single"].view(torch.int32), ys["multi"][:, 2:1002].contiguous().view(torch.int32)))
        med = {name: float(np.median(r)) for name, r in runs.items()}
        res["resnet50_b8_ms"] = {name: {"ms_median": round(med[name], 4), "ms_runs": [round(v, 4) for v in r]} for name, r in runs.items()}
        res["resnet50_b8_head_overhead_pct"] = round(100 * (med["multi"] / med["single"] - 1), 2)
        res["resnet50_logits_bit_identical"] = same
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
