"""Time of the MobileNetV2 / EfficientNet kernels and bundles on cuda:0, from CUDA events.

    python -m tools.time_convnets [--launches 200] [--repeats 5] [--steps 20] [--model-repeats 5] [--parent PKGDIR]

1. tfsc_k_depthwise_conv alone at every distinct depthwise shape of MobileNetV2 and EfficientNet-B0 (224x224), batch 8 and
   64: median of `repeats` windows of `launches` back-to-back launches, microseconds per launch, and GB/s of algorithmic
   bytes B*(H*W*C + OH*OW*C)*4 + (kh*kw + 1)*C*4, beside a device-to-device copy of 256 MB timed the same way and the
   3.35 TB/s data-sheet figure.
2. Device-resident MobileNetV2 and EfficientNet-B0 (seeded weights) through tfsc_predict_device at batch 8 and 64, the two
   bundles alternating: ms per batch, images/s and kernel launches per batch; and the share of the batch time spent in the
   SIMT GEMM (gemm_f32_kernel) and in the depthwise / channel_scale kernels, from torch.profiler in a separate run.
3. With --parent PKGDIR (a tfservingcache_b200 package built from another commit): device-resident ResNet-50 and BERT-base
   at batch 8, this tree's library against that one, alternating in child processes; the logits of ResNet-50, BERT-base and
   the tenant MLP [9216 x 4] of both are compared bit for bit.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATASHEET_GBS = 3350.0
MNV2_DW = [(32, 112, 3, 1, 1), (96, 112, 3, 2, 1), (144, 56, 3, 1, 1), (144, 56, 3, 2, 1), (192, 28, 3, 1, 1), (192, 28, 3, 2, 1),
           (384, 14, 3, 1, 1), (576, 14, 3, 1, 1), (576, 14, 3, 2, 1), (960, 7, 3, 1, 1)]
B0_DW = [(32, 112, 3, 1, 1), (96, 112, 3, 2, 1), (144, 56, 3, 1, 1), (144, 56, 5, 2, 2), (240, 28, 3, 2, 1), (240, 28, 5, 1, 2),
         (480, 14, 3, 1, 1), (480, 14, 5, 1, 2), (672, 14, 5, 1, 2), (672, 14, 5, 2, 2), (1152, 7, 3, 1, 1), (1152, 7, 5, 1, 2)]


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


def _median_us(torch, fn, launches, repeats):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    return float(np.median([_events(torch, fn, launches) * 1e3 for _ in range(repeats)]))


def depthwise_table(torch, t, args):
    lib = t._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(0)
    src = torch.empty(64 << 20, device="cuda")
    dst = torch.empty_like(src)
    copy_us = _median_us(torch, lambda: dst.copy_(src), args.launches // 4, args.repeats)
    rows = []
    for C, H, k, s, p in sorted(set(MNV2_DW + B0_DW), key=lambda v: (-v[1], v[0], v[2], v[3])):
        oh = (H + 2 * p - k) // s + 1
        for B in (8, 64):
            x = torch.randn(B, H, H, C, device="cuda", generator=gen)
            w = torch.randn(k, k, C, device="cuda", generator=gen) / k
            b = torch.randn(C, device="cuda", generator=gen)
            y = torch.empty(B, oh, oh, C, device="cuda")

            def launch():
                t._lib.check(lib.tfsc_k_depthwise_conv(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), B, H, H, C, k, k, s, p, 5,
                                                       None), "depthwise_conv")
            us = _median_us(torch, launch, args.launches, args.repeats)
            nbytes = B * (H * H * C + oh * oh * C) * 4 + (k * k + 1) * C * 4
            rows.append({"C": C, "H": H, "k": k, "stride": s, "pad": p, "batch": B, "us": round(us, 2),
                         "GBps": round(nbytes / us / 1e3, 1), "pct_datasheet": round(100 * nbytes / us / 1e3 / DATASHEET_GBS, 1)})
    return {"d2d_copy_GBps": round(2 * src.numel() * 4 / copy_us / 1e3, 1), "datasheet_GBps": DATASHEET_GBS, "shapes": rows}


def _seeded_blob(man, seed):
    """weights of variance 1 / fan_in and biases 0.1 N(0, 1): finite logits at every depth"""
    rng = np.random.default_rng(seed)
    blob = np.zeros(man["weights_bytes"] // 4, np.float32)
    for o in man["ops"]:
        if o["op"] in ("conv", "dense", "depthwise_conv"):
            fan_in = o.get("kh", 1) * o.get("kw", 1) * (1 if o["op"] == "depthwise_conv" else o["c"])
            n = fan_in * (o["c"] if o["op"] == "depthwise_conv" else o["cout"])
            blob[o["w_offset"] // 4: o["w_offset"] // 4 + n] = rng.standard_normal(n).astype(np.float32) / np.sqrt(fan_in)
            nb = o["c"] if o["op"] == "depthwise_conv" else o["cout"]
            blob[o["b_offset"] // 4: o["b_offset"] // 4 + nb] = 0.1 * rng.standard_normal(nb).astype(np.float32)
    return blob


def model_table(torch, t, args):
    tmp = tempfile.mkdtemp(prefix="tfsc_convnets_")
    res = {}
    try:
        mans = {"mobilenet_v2": t.modelformat.mobilenet_v2_manifest(), "efficientnet_b0": t.modelformat.efficientnet_manifest()}
        for i, (name, man) in enumerate(mans.items()):
            t.modelformat.write_graph_bundle(f"{tmp}/{name}/1", man, _seeded_blob(man, i))
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 4, "gpu.maxBatch": 64}
        gen = torch.Generator(device="cuda").manual_seed(0)
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for name in mans:
                srv.ensure(0, name, 1)
            for B in (8, 64):
                x = torch.randn(B, 224, 224, 3, device="cuda", generator=gen)
                y = torch.empty(B, 1000, device="cuda")
                fns = {n: (lambda n=n: srv.predict_device(0, n, 1, x.data_ptr(), B, y.data_ptr(), stream.cuda_stream)) for n in mans}
                launches = {}
                for n, fn in fns.items():
                    for _ in range(5):
                        fn()
                    srv.sync(0)
                    s0 = srv.stats()["kernel_launches"]
                    fn()
                    srv.sync(0)
                    launches[n] = srv.stats()["kernel_launches"] - s0
                torch.cuda.synchronize()
                runs = {n: [] for n in mans}
                for rep in range(args.model_repeats):
                    for n in (list(mans) if rep % 2 == 0 else list(mans)[::-1]):
                        runs[n].append(_events(torch, fns[n], args.steps, stream))
                for n in mans:
                    ms = float(np.median(runs[n]))
                    res[f"{n}_b{B}"] = {"ms_median": round(ms, 4), "ms_runs": [round(v, 4) for v in runs[n]],
                                        "img_per_s": round(B / ms * 1e3, 1), "launches_per_batch": launches[n]}
                # kernel shares, traced in a run of their own after the timed windows
                from torch.profiler import ProfilerActivity, profile
                for n, fn in fns.items():
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(5):
                            fn()
                        torch.cuda.synchronize()
                    tot, part = 0.0, {"gemm_f32": 0.0, "gemm_tc": 0.0, "depthwise_conv": 0.0, "channel_scale": 0.0}
                    for e in prof.events():
                        if str(e.device_type).endswith("CUDA"):
                            d = e.time_range.elapsed_us()
                            tot += d
                            for key in part:
                                if key in e.name:
                                    part[key] += d
                    res[f"{n}_b{B}"]["kernel_share_pct"] = {k: round(100 * v / tot, 1) for k, v in part.items()} if tot else None
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def ab_child(out_path, steps, repeats):
    """this process's library: ResNet-50 and BERT-base at batch 8 (ms per batch), and the logits of ResNet-50, BERT-base and
    the tenant MLP on seeded inputs, saved to out_path"""
    import torch

    import tfservingcache_b200 as t
    mf = t.modelformat
    tmp = tempfile.mkdtemp(prefix="tfsc_ab_")
    out, res = {}, {}
    try:
        bundles = {"resnet50": (mf.resnet50_manifest(), (8, 224, 224, 3)), "bert_base": (mf.bert_manifest(), (8, 128))}
        for i, (name, (man, _)) in enumerate(bundles.items()):
            mf.write_graph_bundle(f"{tmp}/{name}/1", man, _seeded_blob(man, 10 + i))
        rng = np.random.default_rng(0)
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 4}
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()
            for name, (man, shape) in bundles.items():
                xh = rng.random(shape).astype(np.float32) if name == "resnet50" else rng.integers(1, 30522, shape).astype(np.int32)
                out[name] = srv.predict(name, "1", xh)
                srv.ensure(0, name, 1)
                x = torch.from_numpy(xh).cuda()
                y = torch.empty(8, out[name].shape[1], device="cuda")
                fn = (lambda x=x, y=y, name=name: srv.predict_device(0, name, 1, x.data_ptr(), 8, y.data_ptr(), stream.cuda_stream))
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
                runs = [_events(torch, fn, steps, stream) for _ in range(repeats)]
                res[name] = float(np.median(runs))
        cfg = {"modelProvider.type": "synthetic", "modelProvider.synthetic.dims": [9216] * 4, "modelProvider.synthetic.count": 2,
               "gpu.devices": [0], "gpu.arenaBytes": 2 << 30, "modelCache.size": 4 << 30, "serving.maxConcurrentModels": 2}
        with t.Server(cfg) as srv:
            for rows in (1, 8, 64):
                out[f"mlp_r{rows}"] = srv.predict("m1", "1", rng.standard_normal((rows, 9216)).astype(np.float32))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez(out_path, **out)
    res["lib"] = t._lib.LIB_PATH
    print(json.dumps(res))


def ab_table(args):
    tmp = tempfile.mkdtemp(prefix="tfsc_abr_")
    runs = {"this": [], "parent": []}
    try:
        for rep in range(args.ab_repeats):
            for which in (("this", "parent") if rep % 2 == 0 else ("parent", "this")):
                env = dict(os.environ, PYTHONPATH=ROOT if which == "this" else os.path.abspath(args.parent) + os.pathsep + ROOT)
                # run as a script: its own directory, then PYTHONPATH, lead sys.path, so the package comes from PYTHONPATH
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--ab-child", f"{tmp}/{which}{rep}.npz",
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
    for name in ("resnet50", "bert_base"):
        this = [r[name] for r in runs["this"]]
        par = [r[name] for r in runs["parent"]]
        res[f"{name}_b8_ms"] = {"this": round(float(np.median(this)), 4), "parent": round(float(np.median(par)), 4),
                                "this_runs": [round(v, 4) for v in this], "parent_runs": [round(v, 4) for v in par]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--model-repeats", type=int, default=5)
    ap.add_argument("--ab-repeats", type=int, default=4)
    ap.add_argument("--parent", default=None, help="a tfservingcache_b200 package built from the commit to compare against")
    ap.add_argument("--ab-child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--skip-kernels", action="store_true")
    args = ap.parse_args()
    if args.ab_child:
        return ab_child(args.ab_child, args.steps, args.model_repeats)
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_convnets needs a CUDA device"
    res = {**_card(), "launches": args.launches, "repeats": args.repeats}
    if not args.skip_kernels:
        res["depthwise"] = depthwise_table(torch, t, args)
        res["models"] = model_table(torch, t, args)
    if args.parent:
        res["vs_parent"] = ab_table(args)
    res.update({"card_after": _card()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
