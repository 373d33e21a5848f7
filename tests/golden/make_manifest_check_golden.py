"""Writes manifest_check_golden.json: tfsc_manifest_check's return code and output (the layout, or the refusal message) for
generate, next-token and BERT bundles that give no repetition-control field, taken from the library built at the commit
before processing bundles existed. tests/test_penalty_cpu.py checks that the library still answers each the same.

    python tests/golden/make_manifest_check_golden.py   (from the repository root, with that commit's library built)"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import tfservingcache_b200 as t  # noqa: E402

mf = t.modelformat
SMALL = dict(hidden=64, layers=2, heads=4, vocab=1000, max_pos=64)


def _outs(n=6, **fields):
    return [dict({"name": k, "kind": k, "max_new_tokens": n}, **fields) for k in mf.GENERATE_OUTPUT_KINDS]


def manifests():
    g = lambda seq=16, inputs=mf.GPT2_INPUTS, outputs=None: mf.gpt2_manifest(seq=seq, **SMALL, inputs=inputs,  # noqa: E731
                                                                               outputs=_outs() if outputs is None else outputs)
    ids_only = [{"name": "input_ids", "role": "ids"}]
    return {
        "greedy": g(),
        "greedy_eos": g(outputs=_outs(eos_token_id=7)),
        "greedy_ids_only": g(inputs=ids_only),
        "greedy_single_input": g(inputs=None),
        "sampling": g(inputs=mf.GPT2_SAMPLING_INPUTS, outputs=_outs(temperature=0.8, top_k=40, top_p=0.9)),
        "next_token": g(outputs=[{"name": "ids", "kind": "next_token_top_k_ids", "k": 3}]),
        "bert": mf.bert_manifest(seq=16, hidden=64, layers=1, heads=4, inter=128, vocab=100, inputs=mf.BERT_INPUTS),
        "refused_eos": g(outputs=_outs(eos_token_id=1000)),
        "refused_max_pos": g(outputs=_outs(50)),
        "refused_top_k": g(inputs=mf.GPT2_SAMPLING_INPUTS, outputs=_outs(top_k=1001)),
        "refused_no_seed": g(outputs=_outs(top_p=0.5)),
        "refused_max_new": g(outputs=_outs(0)),
    }


def check(man):
    buf = C.create_string_buffer(1 << 16)
    rc = t._lib.lib.tfsc_manifest_check(json.dumps(man).encode(), buf, len(buf))
    return rc, buf.value.decode() if rc >= 0 else t._lib.lib.tfsc_last_error().decode()


if __name__ == "__main__":
    out = {k: {"manifest": m, "rc": check(m)[0], "output": check(m)[1]} for k, m in manifests().items()}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "manifest_check_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
