"""Time of the fill-mask kernels of masked-language-model bundles (csrc/mlm.cu) on cuda:0, from CUDA events.

    python -m tools.time_fill_mask [--launches 200] [--repeats 5] [--steps 20]

1. tfsc_k_mask_gather and tfsc_k_fill_mask_head alone at rows x M = 8 x 1, 8 x 20 and 128 x 20 slots (8, 160 and 2560 slot
   rows), S = 128, H = 768, vocab 30522 (Vp = 30528), k = 5: median / every repeat in microseconds per launch over
   `launches` back-to-back launches.
2. The vocabulary projection [rows, 768] x [768, 30528] at 8, 24, 40, 63 and 160 rows on the GEMM path (tfsc_k_gemm: the
   SIMT kernel below 64 rows, the tensor cores from 64) and on the dense path (tfsc_k_dense: the cluster-pair kernel up to
   8 rows, dense_tc above), with each path's largest difference from an fp64 product.
3. Device-resident BERT-base MLM at 8 x 128 through tfsc_predict_device with M = 1 and M = 20 (k = 5), against the encoder
   bundle of the same weights without a pooler (sequence_output), alternating in one run: milliseconds per batch.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np

from tools.time_heads import _card, _events

MASK_ID = 103
H, S, V, K = 768, 128, 30522, 5
VP = (V + 31) // 32 * 32


def _median(torch, fn, launches, repeats, scale=1000.0):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    runs = [_events(torch, fn, launches) * scale for _ in range(repeats)]
    return {"median": round(float(np.median(runs)), 2), "runs": [round(v, 2) for v in runs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_fill_mask needs cuda:0"
    lib, mf = t._lib.lib, t.modelformat
    res = {"card": _card()}
    g = torch.Generator(device="cuda").manual_seed(0)

    # 1. the kernels alone
    kern = {}
    for rows, M in ((8, 1), (8, 20), (128, 20)):
        hidden = torch.randn(rows, S, H, device="cuda", generator=g)
        ids = torch.randint(MASK_ID + 1, V, (rows, S), device="cuda", dtype=torch.int32, generator=g)
        for r in range(rows):
            ids[r, torch.randperm(S, device="cuda", generator=g)[:M]] = MASK_ID
        pos = torch.empty(rows, M, device="cuda", dtype=torch.int32)
        gat = torch.empty(rows, M, H, device="cuda")
        logits = torch.randn(rows * M, VP, device="cuda", generator=g) * 4
        tid = torch.empty(rows, M, K, device="cuda", dtype=torch.int32)
        tp, tl = torch.empty(rows, M, K, device="cuda"), torch.empty(rows, M, K, device="cuda")

        def gather():
            t._lib.check(lib.tfsc_k_mask_gather(hidden.data_ptr(), ids.data_ptr(), None, S, rows, S, H, M, MASK_ID, pos.data_ptr(),
                                                gat.data_ptr(), None), "mask_gather")

        def head():
            t._lib.check(lib.tfsc_k_fill_mask_head(logits.data_ptr(), VP, pos.data_ptr(), rows, M, V, K, tid.data_ptr(),
                                                   tp.data_ptr(), tl.data_ptr(), None), "fill_mask_head")
        gather()
        kern[f"{rows}x{M}"] = {"gather_us": _median(torch, gather, args.launches, args.repeats),
                               "head_us": _median(torch, head, args.launches, args.repeats)}
    res["kernels"] = kern

    # 2. the vocabulary projection: GEMM path against the weight-streaming dense path
    w = torch.randn(H, VP, device="cuda", generator=g) * (1.0 / H) ** 0.5
    b = torch.randn(VP, device="cuda", generator=g) * 0.1
    proj = {}
    for rows in (8, 24, 40, 63, 160):
        x = torch.randn(rows, H, device="cuda", generator=g)
        y0, y1 = torch.empty(rows, VP, device="cuda"), torch.empty(rows, VP, device="cuda")
        wsb = lib.tfsc_k_dense_workspace(rows, H, VP)
        # the split-K counters start at zero, as the executor's cudaMemsetAsync leaves them; the kernels reset them
        ws = torch.zeros(max(wsb, 256), dtype=torch.uint8, device="cuda")

        def gemm():
            t._lib.check(lib.tfsc_k_gemm(x.data_ptr(), w.data_ptr(), b.data_ptr(), None, y0.data_ptr(), rows, VP, H, H, 0, None), "gemm")

        def dense():
            t._lib.check(lib.tfsc_k_dense(x.data_ptr(), w.data_ptr(), b.data_ptr(), y1.data_ptr(), rows, H, VP, 0, ws.data_ptr(), wsb, None),
                         "dense")
        tg = _median(torch, gemm, args.launches // 4, args.repeats)
        td = _median(torch, dense, args.launches // 4, args.repeats)
        torch.cuda.synchronize()
        ref = x.double() @ w.double() + b.double()
        proj[f"rows_{rows}"] = {"gemm_us": tg, "dense_us": td, "gemm_over_dense": round(tg["median"] / td["median"], 2),
                                "gemm_max_abs_err": float((y0.double() - ref).abs().max()),
                                "dense_max_abs_err": float((y1.double() - ref).abs().max()),
                                "weight_mb": round(H * VP * 4 / 1e6, 1)}
    res["vocab_projection"] = proj

    # 3. BERT-base MLM end to end, device-resident
    tmp = tempfile.mkdtemp(prefix="tfscmlm")
    try:
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
        import embed_export as ee
        import mlm_export as me
        m = me.hf_mlm_model(5)
        outs = [{"name": "masked_positions", "kind": "masked_positions"}] + \
               [{"name": k, "kind": k, "k": K} for k in mf.MLM_OUTPUT_KINDS[1:]]
        widths = {}
        for M in (1, 20):
            man = mf.bert_manifest(seq=S, inputs=mf.BERT_INPUTS, outputs=outs, head="mlm", slots=M, mask_token_id=MASK_ID)
            mf.write_graph_bundle(os.path.join(tmp, f"mlm{M}", "1"), man, me.export_mlm_model(m, man))
            widths[f"mlm{M}"] = M + 3 * M * K
        enc = mf.bert_manifest(seq=S, inputs=mf.BERT_INPUTS, outputs=[{"name": "sequence_output", "kind": "sequence_output"}],
                               head="encoder", pooler=False)
        mf.write_graph_bundle(os.path.join(tmp, "enc", "1"), enc, ee.export_bert_model(m.bert, enc))
        widths["enc"] = S * H
        B = 8
        rng = np.random.default_rng(1)
        ids = rng.integers(MASK_ID + 1, V, (B, S)).astype(np.int32)
        ids[:, 1:21] = MASK_ID
        x = np.concatenate([ids, np.ones((B, S), np.int32), np.zeros((B, S), np.int32)], axis=1)  # ids | mask | segments
        xd = torch.from_numpy(x).cuda()
        ys = {n: torch.empty(B, wd, device="cuda") for n, wd in widths.items()}
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "serving.maxConcurrentModels": 8, "modelCache.size": 8 << 30, "gpu.maxBatch": 8}
        stream = torch.cuda.Stream()
        with t.Server(cfg) as srv:
            for n in widths:
                srv.ensure(0, n, 1)
            fns = {n: (lambda n=n: srv.predict_device(0, n, 1, xd.data_ptr(), B, ys[n].data_ptr(), stream.cuda_stream)) for n in widths}
            for n in widths:
                for _ in range(5):
                    fns[n]()
            torch.cuda.synchronize()
            runs = {n: [] for n in widths}
            for rep in range(args.repeats):
                for n in (list(widths) if rep % 2 == 0 else list(widths)[::-1]):
                    runs[n].append(_events(torch, fns[n], args.steps, stream))
            srv.sync(0)
        res["bert_base_b8_s128_ms"] = {n: {"median": round(float(np.median(r)), 4), "runs": [round(v, 4) for v in r]}
                                       for n, r in runs.items()}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
