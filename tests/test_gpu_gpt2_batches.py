"""-m gpu: served GPT-2 past 8 rows. In a GPT-2 request the batch size B picks the kernels (Node::run_model,
launch_dense, launch_gemm). On a 132-SM H100, where launch_gt applies its split-K rule:

| op                                | 1-8 rows             | 9-63 rows           | 64-128 rows                  |
|-----------------------------------|----------------------|---------------------|------------------------------|
| prefill decoder GEMMs (M = B * S) | gemm_tc              | gemm_tc             | gemm_tc                      |
| vocabulary projection (a)         | dense_cluster_kernel | dense_tc_kernel (b) | gemm_tc, M = B, BN 128       |
| decode-step projections (c)       | SIMT gemm_f32        | SIMT gemm_f32       | gemm_tc, cluster split-K (d) |

(a) 768 -> 50,272 after last_token, in the prefill and in every decode step.
(b) one pass, 197 strips of 256 columns in two waves, the last strip 96 columns wide.
(c) M = B: c_attn, attn c_proj + residual, c_fc + gelu_tanh, mlp c_proj + residual.
(d) split-K of 2 / 4 / 2 / 8 for the four projections.

Full-size seeded GPT-2 small bundles of one transformers model (next-token, greedy generate, two sampling configs and
top_k = 1 sampling) and GPT-2 medium, served with gpu.maxBatch 128 at row counts on both sides of every column:
next-token against transformers fp64, generation teacher-forced against it, the first generated token bit for bit the
next-token top-1, top_k = 1 bit for bit greedy, coalesced requests across a route boundary bit for bit one request,
tfsc_predict_device at 65 rows and TFSC_PDL=0. The tolerances are test_gpu_gpt2's, test_gpu_generate's and
test_gpu_sampling's, through their own checks."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpt2_export as ge  # noqa: E402
import test_gpu_generate as gg  # noqa: E402
import test_gpu_gpt2 as g2  # noqa: E402
import test_gpu_sampling as gs  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
mf = t.modelformat
V = 50257
S = 128                                    # prompt length of the small bundles
N = 16                                     # greedy and top_k = 1 tokens per row
N_SAMPLED = 4                              # tokens per row of the two sampling configs
S_LONG, N_LONG = 992, 32                   # S + N - 1 = 1023 cache slots: max_pos - 1
SEED = 91
NAMES = gg.NAMES
SAMPLED = {"s_top_p": gs.E2E[1], "s_top_k_p": gs.E2E[2]}
TICK_US = 3_000_000                        # a partial batch waits 3 s for more rows: far longer than submitting tickets


def _cfg(tmp, **kw):
    return g2._cfg(tmp, **dict({"gpu.arenaBytes": 8 << 30, "gpu.maxBatch": 128}, **kw))


def _fields(cfg):
    temperature, top_k, top_p = cfg
    return dict(temperature=temperature, top_p=top_p, **({"top_k": top_k} if top_k else {}))


def _rows(x, lo, hi, seed=True):
    return {k: v[lo:hi] for k, v in x.items() if seed or k != "seed"}


def _fp64(m):
    """the model in fp64 on the GPU, for the references: gpt2_reference copies the model it is given to fp64 on the device
    for each call, and the teacher-forced checks call it once per row, so a device copy of an fp64 model makes each of
    those copies a device-to-device one. The values are those of the fp32 model the bundles were exported from."""
    import copy
    return copy.deepcopy(m).double().cuda()


def _inputs():
    """128 rows of prompt S cycling through unpadded, right- and left-padded, and a seed per row"""
    return gs._inputs(128, S, V, 5)


def _write_small(tmp, m):
    arch = dict(max_pos=1024)
    g2._write_gpt2(tmp, S, arch, SEED, name="nt", model=m)
    gg._write(tmp, S, arch, SEED, name="g", model=m, outputs=gg._outs(N))
    gg._write(tmp, S_LONG, arch, SEED, name="g_long", model=m, outputs=gg._outs(N_LONG))
    for name, cfg in SAMPLED.items():
        gs._write(tmp, S, arch, SEED, name=name, model=m, outputs=gs._outs(N_SAMPLED, **_fields(cfg)))
    gs._write(tmp, S, arch, SEED, name="k1", model=m, outputs=gs._outs(N, temperature=1.3, top_k=1, top_p=0.5))


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    import torch
    tmp = tmp_path_factory.mktemp("gpt2_small")
    m = ge.hf_gpt2_model(SEED, max_pos=1024)
    _write_small(tmp, m)
    m = _fp64(m)
    x = _inputs()
    pos = np.array([max(np.nonzero(mk)[0]) for mk in x["attention_mask"]], np.int32)
    ref = ge.gpt2_reference(m, x["input_ids"], x["attention_mask"], device="cuda", at=pos)
    torch.cuda.empty_cache()
    with t.Server(_cfg(tmp)) as srv:
        yield SimpleNamespace(tmp=tmp, model=m, x=x, pos=pos, ref=ref, srv=srv)


# ------------------------------------------------------------------------------------------- GPT-2 small ----
@pytest.mark.parametrize("B", [8, 9, 16, 17, 33, 49, 63, 64, 65, 128])
def test_next_token_against_fp64(small, B):
    r = small.srv.predict("nt", "1", _rows(small.x, 0, B, seed=False), outputs=g2.NAMES)
    assert r["next_token_top_k_ids"].shape == (B, g2.K)
    g2._check_against_fp64(r, small.ref[:B], small.pos[:B], V)


@pytest.mark.parametrize("B", [8, 9, 33, 63, 64, 65, 128])
def test_greedy_against_fp64(small, B):
    """teacher-forced against transformers fp64, and the first token the next-token bundle's top-1 bit for bit"""
    xb = _rows(small.x, 0, B, seed=False)
    r = small.srv.predict("g", "1", xb, outputs=NAMES)
    assert r["generated_ids"].shape == (B, N) and r["generated_length"].shape == (B,)
    nt = small.srv.predict("nt", "1", xb, outputs=["next_token_top_k_ids"])
    assert r["generated_ids"][:, 0].tobytes() == np.ascontiguousarray(nt["next_token_top_k_ids"][:, 0]).tobytes()
    gg._check_teacher_forced(small.model, xb, r, V)


def test_greedy_fills_the_cache_past_64_rows(small):
    """prompt 992 and N = 32 at 65 rows: the cache's S + N - 1 = 1023 slots (max_pos - 1) fill up, decode attention runs
    up to 16 key blocks per row, and every decode GEMM is on gemm_tc"""
    B = 65
    x = ge.gpt2_inputs(B, S_LONG, V, seed=S_LONG)
    r = small.srv.predict("g_long", "1", x, outputs=NAMES)
    assert r["generated_ids"].shape == (B, N_LONG)
    gg._check_teacher_forced(small.model, x, r, V)


@pytest.mark.parametrize("B", [9, 63, 64, 128])
@pytest.mark.parametrize("name", sorted(SAMPLED))
def test_sampled_against_fp64(small, name, B):
    xb = _rows(small.x, 0, B)
    r = small.srv.predict(name, "1", xb, outputs=NAMES)
    assert r["generated_ids"].shape == (B, N_SAMPLED)
    gs._check_sampled(small.model, xb, r, V, SAMPLED[name])


@pytest.mark.parametrize("B", [9, 65])
def test_top_k_1_is_greedy(small, B):
    k1 = small.srv.predict("k1", "1", _rows(small.x, 0, B), outputs=NAMES)
    greedy = small.srv.predict("g", "1", _rows(small.x, 0, B, seed=False), outputs=NAMES)
    assert all(k1[k].tobytes() == greedy[k].tobytes() for k in NAMES)


@pytest.mark.parametrize("case", ["5+4", "40+24", "60+5", "100+28"])
def test_coalesced_across_a_route_boundary(small, case):
    """gpu.maxBatch is the joint rows, so the batcher holds the first ticket until the others are queued. Each ticket's
    outputs are its slice of one request of the joint rows. 5+4: each part alone would take the cluster kernel, together
    they take dense_tc; 40+24: dense_tc and SIMT decode GEMMs -> gemm_tc; 60+5 and 100+28: past 64 rows."""
    sizes = [int(s) for s in case.split("+")]
    total = sum(sizes)
    starts = np.cumsum([0] + sizes)
    with t.Server(_cfg(small.tmp, **{"gpu.maxBatch": total, "gpu.tickMicros": TICK_US})) as srv:
        for name, names, seed in (("nt", g2.NAMES, False), ("g", NAMES, False), ("s_top_k_p", NAMES, True)):
            joint = srv.predict(name, "1", _rows(small.x, 0, total, seed), outputs=names)     # a full batch does not wait
            st0 = srv.stats()
            tickets = [srv.predict_submit(name, "1", _rows(small.x, starts[i], starts[i + 1], seed), outputs=names)
                       for i in range(len(sizes))]
            outs = [tk.wait(60.0) for tk in tickets]
            [tk.release() for tk in tickets]
            st1 = srv.stats()
            assert (st1["batches"] - st0["batches"], st1["batched_rows"] - st0["batched_rows"]) == (1, total), (name, case)
            for i, r in enumerate(outs):
                lo, hi = starts[i], starts[i + 1]
                assert all(r[k].tobytes() == np.ascontiguousarray(joint[k][lo:hi]).tobytes() for k in names), (name, case, i)


def test_predict_device_at_65_rows(small):
    """tfsc_predict_device's per-stream scratch then holds the KV caches of more than 64 rows"""
    import torch
    B = 65
    xb = _rows(small.x, 0, B, seed=False)
    full = small.srv.predict("g", "1", xb, outputs=NAMES)
    small.srv.ensure(0, "g", 1)
    outs = gg._outs(N)
    width = sum(w for _n, _o, w, _d in mf.packed_output_layout(outs, V))
    packed = np.concatenate([xb[n] for n in mf.packed_input_order(mf.GPT2_INPUTS)], axis=1)
    xd = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
    yd = torch.full((B, width), float("nan"), device="cuda")
    small.srv.predict_device(0, "g", 1, xd.data_ptr(), B, yd.data_ptr(), 0)
    small.srv.sync(0)
    dev = mf.split_packed_rows(yd.cpu().numpy(), outs, V)
    for k in NAMES:
        assert dev[k].shape == full[k].shape and dev[k].tobytes() == full[k].tobytes(), k


def _pdl_outputs(srv):
    """greedy and sampled generation at 9 and 65 rows: the decode loop chains dense_tc or split-K gemm_tc into the select
    / sample step"""
    x, out = _inputs(), {}
    for B in (9, 65):
        for name, seed in (("g", False), ("s_top_k_p", True)):
            for k, v in srv.predict(name, "1", _rows(x, 0, B, seed), outputs=NAMES).items():
                out[f"{name}_{k}_r{B}"] = v
    return out


PDL_SCRIPT = r"""
import sys
import numpy as np
import tfservingcache_b200 as t
sys.path.insert(0, "tests")
import test_gpu_gpt2_batches as b
with t.Server(b._cfg(sys.argv[2])) as srv:
    out = b._pdl_outputs(srv)
np.savez(sys.argv[1], **out)
print("SAVED", len(out))
"""


def test_programmatic_dependent_launch_keeps_the_bits(small, tmp_path):
    """this process launches with programmatic dependent launch (the default); a subprocess with TFSC_PDL=0 without it"""
    if os.environ.get("TFSC_PDL") == "0":
        pytest.skip("this process already runs with TFSC_PDL=0")
    want = _pdl_outputs(small.srv)
    env = dict(os.environ, PYTHONPATH=ROOT, TFSC_PDL="0")
    path = str(tmp_path / "pdl_0.npz")
    run = subprocess.run([sys.executable, "-c", PDL_SCRIPT, path, str(small.tmp)], capture_output=True, text=True, timeout=900,
                         env=env, cwd=ROOT)
    assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]
    got = dict(np.load(path))
    assert sorted(got) == sorted(want) and len(got) == 2 * 2 * len(NAMES)
    for key, y in want.items():
        assert y.tobytes() == got[key].tobytes(), key


# ------------------------------------------------------------------------------------------ GPT-2 medium ----
MEDIUM = dict(hidden=1024, layers=24, heads=16, max_pos=1024)
S_MEDIUM, N_MEDIUM = 64, 4


@pytest.fixture(scope="module")
def medium(tmp_path_factory):
    import torch
    tmp = tmp_path_factory.mktemp("gpt2_medium")
    m = ge.hf_gpt2_model(SEED + 1, **MEDIUM)
    g2._write_gpt2(tmp, S_MEDIUM, MEDIUM, SEED + 1, name="nt", model=m)
    gg._write(tmp, S_MEDIUM, MEDIUM, SEED + 1, name="g", model=m, outputs=gg._outs(N_MEDIUM))
    m = _fp64(m)
    x = ge.gpt2_inputs(65, S_MEDIUM, V, seed=6)
    pos = np.array([max(np.nonzero(mk)[0]) for mk in x["attention_mask"]], np.int32)
    ref = ge.gpt2_reference(m, x["input_ids"], x["attention_mask"], device="cuda", at=pos)
    torch.cuda.empty_cache()
    with t.Server(_cfg(tmp)) as srv:
        yield SimpleNamespace(model=m, x=x, pos=pos, ref=ref, srv=srv)


@pytest.mark.parametrize("B", [8, 9, 64])
def test_medium_next_token_against_fp64(medium, B):
    r = medium.srv.predict("nt", "1", _rows(medium.x, 0, B), outputs=g2.NAMES)
    g2._check_against_fp64(r, medium.ref[:B], medium.pos[:B], V)


@pytest.mark.parametrize("B", [9, 65])
def test_medium_greedy_against_fp64(medium, B):
    xb = _rows(medium.x, 0, B)
    r = medium.srv.predict("g", "1", xb, outputs=NAMES)
    assert r["generated_ids"].shape == (B, N_MEDIUM)
    gg._check_teacher_forced(medium.model, xb, r, V)
