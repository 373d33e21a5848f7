"""Time of the span head of question-answering bundles (csrc/span.cu) on cuda:0, from CUDA events.

    python -m tools.time_spans [--launches 200] [--repeats 5] [--bert-steps 10] [--bert-repeats 7]

1. tfsc_k_span_head alone at S = 384, max_answer_length 30, k = 20, writing start / end logits and the spans, for rows 8
   and 128 (SQuAD-shaped rows: a question in segment 0, a passage in segment 1, a [PAD] tail): median / every repeat in
   microseconds per launch over back-to-back launches, and the kernel's own device time from torch.profiler.
2. Device-resident BERT-base QA (seeded random weights) at batch 8 x 384 through tfsc_predict_device: the single-output
   bundle ([B, 384, 1, 2] logits) and the same weights with start / end logits and 20 spans, alternating in one run:
   median / every repeat in milliseconds per batch.
Prints one JSON object with the card name and power limit. Bundles go to a temporary directory, removed at the end."""
import argparse
import json
import shutil
import tempfile

import numpy as np

from tools.time_heads import _card, _events, _kernel_us

S, L, K, SEP = 384, 30, 20, 102
OUTPUTS = [{"name": "start_logits", "kind": "start_logits"}, {"name": "end_logits", "kind": "end_logits"}] + [
    {"name": n, "kind": n, "k": K, "max_answer_length": L, "sep_id": SEP} for n in ("span_starts", "span_ends", "span_scores")]


def _qa_rows(rows, seed):
    """ids / mask / segment ids [rows, S]: question up to a third of the row, passage after it, half the rows padded"""
    rng = np.random.default_rng(seed)
    ids = rng.integers(1000, 30000, (rows, S)).astype(np.int32)
    mask = np.ones((rows, S), np.int32)
    seg = np.zeros((rows, S), np.int32)
    for b in range(rows):
        end = S - (b % 2) * int(rng.integers(0, S // 2))
        cut = int(rng.integers(8, S // 3))
        seg[b, cut:end] = 1
        ids[b, cut - 1] = ids[b, end - 1] = SEP
        ids[b, end:], mask[b, end:] = 0, 0
    return ids, mask, seg


def _bert_blob(man, seed=0):
    """seeded weights of variance 1 / fan_in, unit LayerNorm gains, small embeddings: finite logits at every depth"""
    rng = np.random.default_rng(seed)
    blob = np.zeros(man["weights_bytes"] // 4, np.float32)
    for o in man["ops"]:
        if o["op"] in ("conv", "dense"):
            n = o["c"] * o["cout"]
            blob[o["w_offset"] // 4: o["w_offset"] // 4 + n] = rng.standard_normal(n).astype(np.float32) / np.sqrt(o["c"])
        elif o["op"] in ("layernorm", "embed"):
            blob[o["w_offset"] // 4: o["w_offset"] // 4 + o["c"]] = 1.0
            if o["op"] == "embed":
                for key, rows in (("word_offset", o["vocab"]), ("pos_offset", o["max_pos"]), ("type_offset", 2)):
                    n = rows * o["c"]
                    blob[o[key] // 4: o[key] // 4 + n] = rng.standard_normal(n).astype(np.float32) * 0.02
    return blob


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--bert-steps", type=int, default=10)
    ap.add_argument("--bert-repeats", type=int, default=7)
    args = ap.parse_args()
    import torch

    import tfservingcache_b200 as t
    assert torch.cuda.is_available(), "time_spans needs a CUDA device"
    lib = t._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(0)
    res = {**_card(), "S": S, "max_answer_length": L, "k": K, "launches": args.launches, "span_us": {}}
    for rows in (8, 128):
        x = torch.randn(rows, S, 2, device="cuda", generator=gen) * 3
        ids, mask, seg = (torch.from_numpy(a).cuda() for a in _qa_rows(rows, rows))
        st, en = torch.empty(rows, S, device="cuda"), torch.empty(rows, S, device="cuda")
        s, e = torch.empty(rows, K, dtype=torch.int32, device="cuda"), torch.empty(rows, K, dtype=torch.int32, device="cuda")
        v = torch.empty(rows, K, device="cuda")

        def launch():
            t._lib.check(lib.tfsc_k_span_head(x.data_ptr(), ids.data_ptr(), mask.data_ptr(), seg.data_ptr(), S, rows, S, L, K, SEP,
                                              st.data_ptr(), en.data_ptr(), s.data_ptr(), e.data_ptr(), v.data_ptr(), None),
                         "span_head")

        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        runs = [_events(torch, launch, args.launches) * 1e3 for _ in range(args.repeats)]
        res["span_us"][f"rows{rows}"] = {"us_median": round(float(np.median(runs)), 2), "us_runs": [round(r, 2) for r in runs],
                                         "kernel_us": _kernel_us(torch, launch, "span_head_kernel")}

    tmp = tempfile.mkdtemp(prefix="tfsc_spans_")
    try:
        mf = t.modelformat
        single = mf.bert_manifest(seq=S, inputs=mf.BERT_INPUTS, head="span")
        multi = mf.bert_manifest(seq=S, inputs=mf.BERT_INPUTS, outputs=OUTPUTS, head="span")
        blob = _bert_blob(single)
        mf.write_graph_bundle(f"{tmp}/single/1", single, blob)
        mf.write_graph_bundle(f"{tmp}/multi/1", multi, blob)
        cfg = {"modelProvider.type": "diskProvider", "modelProvider.diskProvider.baseDir": tmp, "gpu.devices": [0],
               "gpu.arenaBytes": 4 << 30, "modelCache.size": 6 << 30, "serving.maxConcurrentModels": 4}
        B = 8
        ids, mask, seg = _qa_rows(B, 1)
        packed = {"input_ids": ids, "input_mask": mask, "segment_ids": seg}
        x = torch.from_numpy(np.ascontiguousarray(np.concatenate([packed[n] for n in mf.packed_input_order(mf.BERT_INPUTS)], 1))).cuda()
        width = {"single": 2 * S, "multi": 2 * S + 3 * K}
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
            # the span bundle's start logits are the single-output bundle's even words (packed order: end_logits first)
            lay = {n: (off, w) for n, off, w, _d in mf.packed_output_layout(OUTPUTS, S)}
            off = lay["start_logits"][0]
            same = bool(torch.equal(ys["single"][:, 0::2].contiguous().view(torch.int32),
                                    ys["multi"][:, off:off + S].contiguous().view(torch.int32)))
        med = {name: float(np.median(r)) for name, r in runs.items()}
        res["bert_base_qa_b8_s384_ms"] = {name: {"ms_median": round(med[name], 4), "ms_runs": [round(v, 4) for v in r]}
                                          for name, r in runs.items()}
        res["bert_base_qa_span_overhead_pct"] = round(100 * (med["multi"] / med["single"] - 1), 2)
        res["bert_base_qa_logits_bit_identical"] = same
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
