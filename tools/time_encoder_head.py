"""Time of the encoder head of embedding bundles (csrc/encoder_head.cu) on cuda:0, from CUDA events.

    python -m tools.time_encoder_head [--launches 200] [--repeats 5] [--bert-steps 10] [--bert-repeats 7]

1. tfsc_k_encoder_head alone at (rows, S, H) = (8, 128, 768), (8, 384, 768), (128, 128, 768) and (128, 512, 768), writing
   cls_embedding and mean_embedding (normalised) with and without sequence_output, on rows with a padded tail: median /
   every repeat in microseconds per launch over back-to-back launches, and the achieved GB/s from rows * S * H * 4 bytes
   read (and as many written with sequence_output).
2. Device-resident BERT-base (seeded random weights) at batch 8 x 128 through tfsc_predict_device: the classification
   bundle (pooler + 2-label classifier, one output) and the encoder bundle of the same weights with all four encoder
   outputs, alternating in one run: median / every repeat in milliseconds per batch.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import shutil
import tempfile

import numpy as np

from tools.time_heads import _card, _events, _kernel_us
from tools.time_spans import _bert_blob

SHAPES = ((8, 128, 768), (8, 384, 768), (128, 128, 768), (128, 512, 768))
OUTPUTS = [{"name": "sequence_output", "kind": "sequence_output"}, {"name": "pooled_output", "kind": "pooled_output"},
           {"name": "cls_embedding", "kind": "cls_embedding"}, {"name": "mean_embedding", "kind": "mean_embedding", "normalize": True}]


def _mask(rows, S, seed):
    """mask [rows, S]: half the rows padded from a random position on"""
    rng = np.random.default_rng(seed)
    m = np.ones((rows, S), np.int32)
    for r in range(0, rows, 2):
        m[r, int(rng.integers(1, S + 1)):] = 0
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--bert-steps", type=int, default=10)
    ap.add_argument("--bert-repeats", type=int, default=7)
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_encoder_head needs a CUDA device"
    lib = t._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(0)
    res = {**_card(), "launches": args.launches, "head_us": {}}
    for rows, S, H in SHAPES:
        h = torch.randn(rows, S, H, device="cuda", generator=gen)
        mask = torch.from_numpy(_mask(rows, S, rows + S)).cuda()
        seq = torch.empty(rows, S, H, device="cuda")
        cls, mean = torch.empty(rows, H, device="cuda"), torch.empty(rows, H, device="cuda")
        for with_seq in (False, True):
            def launch():
                t._lib.check(lib.tfsc_k_encoder_head(h.data_ptr(), None, mask.data_ptr(), mask.data_ptr(), S, rows, S, H, 0, 1,
                                                     seq.data_ptr() if with_seq else None, None, cls.data_ptr(), mean.data_ptr(),
                                                     None), "encoder_head")

            for _ in range(20):
                launch()
            torch.cuda.synchronize()
            runs = [_events(torch, launch, args.launches) * 1e3 for _ in range(args.repeats)]
            us = float(np.median(runs))
            nbytes = rows * S * H * 4 * (2 if with_seq else 1)
            res["head_us"][f"rows{rows}_S{S}_H{H}" + ("_seq" if with_seq else "")] = {
                "us_median": round(us, 2), "us_runs": [round(r, 2) for r in runs], "GBps": round(nbytes / us / 1e3, 1),
                "kernel_us": _kernel_us(torch, launch, "encoder_head_kernel")}
        del h, seq

    tmp = tempfile.mkdtemp(prefix="tfsc_encoder_")
    try:
        mf = t.modelformat
        S, B = 128, 8
        single = mf.bert_manifest(seq=S, inputs=mf.BERT_INPUTS)
        multi = mf.bert_manifest(seq=S, inputs=mf.BERT_INPUTS, outputs=OUTPUTS, head="encoder")
        mf.write_graph_bundle(f"{tmp}/classify/1", single, _bert_blob(single))
        mf.write_graph_bundle(f"{tmp}/encoder/1", multi, _bert_blob(multi))   # the same seeded weights up to the pooler
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "modelCache.size": 6 << 30, "serving.maxConcurrentModels": 4}
        m = _mask(B, S, 1)
        ids = np.where(m != 0, np.random.default_rng(1).integers(1000, 30000, (B, S)), 0).astype(np.int32)
        packed = {"input_ids": ids, "input_mask": m, "segment_ids": np.zeros((B, S), np.int32)}
        x = torch.from_numpy(np.ascontiguousarray(np.concatenate([packed[n] for n in mf.packed_input_order(mf.BERT_INPUTS)], 1))).cuda()
        H = 768
        width = {"classify": 2, "encoder": S * H + 3 * H}
        ys = {k: torch.empty(B, w, device="cuda") for k, w in width.items()}
        with t.Server(cfg) as srv:
            stream = torch.cuda.Stream()   # a stream of its own: the events and the launches must share it
            for name in width:
                srv.ensure(0, name, 1)
            fns = {name: (lambda name=name: srv.predict_device(0, name, 1, x.data_ptr(), B, ys[name].data_ptr(), stream.cuda_stream))
                   for name in width}
            for name in width:   # warm every shape the timed windows use
                for _ in range(3):
                    fns[name]()
            torch.cuda.synchronize()
            runs = {name: [] for name in width}
            for rep in range(args.bert_repeats):
                order = list(width) if rep % 2 == 0 else list(width)[::-1]
                for name in order:
                    runs[name].append(_events(torch, fns[name], args.bert_steps, stream))
            srv.sync(0)
        med = {name: float(np.median(r)) for name, r in runs.items()}
        res["bert_base_b8_s128_ms"] = {name: {"ms_median": round(med[name], 4), "ms_runs": [round(v, 4) for v in r]}
                                       for name, r in runs.items()}
        res["bert_base_encoder_vs_classify_pct"] = round(100 * (med["encoder"] / med["classify"] - 1), 2)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
