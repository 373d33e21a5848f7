"""-m gpu: the raw kernels at GPT-2's decode shapes past 8 rows, against fp64. A decode step runs its four projections
at M = the batch rows: on the SIMT gemm_f32 below 64 rows, on gemm_tc from 64 rows, where launch_gt splits K over a
cluster on a 132-SM H100 (2 / 4 / 2 / 8 for c_attn, attn c_proj, c_fc, mlp c_proj); the vocabulary projection takes the
cluster kernel up to 8 rows, dense_tc from 9 to 63 and gemm_tc from 64. Decode attention runs one query per row over as
many rows as a served batch. The checks and references are those of test_gpu_graph, test_gpu_tc, test_gpu_parity and
test_gpu_generate: tolerance 1e-4 relative to max(1, |ref|) for the linear kernels, 2e-5 for attention."""
import os
import subprocess
import sys

import numpy as np
import pytest

import tfservingcache_b200 as t

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpt2_ref as gr  # noqa: E402
import test_gpu_generate as gg  # noqa: E402
import test_gpu_graph as ggr  # noqa: E402
import test_gpu_parity as gp  # noqa: E402
import test_gpu_tc as gtc  # noqa: E402

pytestmark = pytest.mark.gpu
lib = t._lib.lib
TOL = 1e-4
ACTS = [0, 1, 2, 3, 7]                     # 7: GPT-2's tanh GELU
# GPT-2 small's c_attn, attn c_proj, c_fc and mlp c_proj as (K, N), then medium's c_attn, c_fc and mlp c_proj
PROJ = [(768, 2304), (768, 768), (768, 3072), (3072, 768), (1024, 3072), (1024, 4096), (4096, 1024)]
# GPT-2 small's and medium's vocabulary projection (50,257 rounded up to a multiple of 32), and the widest vocabulary a
# next-token bundle takes
VOCAB = [(768, 50272), (1024, 50272)]
WIDEST = (768, 57344)


def _linear64(x, w, b):
    """x @ w + b in fp64 (on the GPU: the widest shapes are 11 GFLOP)"""
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(v)).cuda().double() for v in (x, w, b)]
    return (d[0] @ d[1] + d[2]).cpu().numpy()


def _act64(ref, act):
    import torch
    if act == 1:
        return np.maximum(ref, 0)
    if act == 2:
        return torch.nn.functional.gelu(torch.from_numpy(ref)).numpy()
    if act == 3:
        return np.tanh(ref)
    if act == 7:
        return gr.gelu_tanh(ref)
    return ref


# --------------------------------------------------------------------------------------------------- GEMMs ----
def _gemm(fn, m, n, k, act):
    """C = act(A B + bias + R), the residual always given (attn / mlp c_proj add it, c_attn / c_fc have none: the epilogue
    is the same code either way)"""
    import torch
    rng = np.random.default_rng(m * 7 + n + k + act)
    a = rng.standard_normal((m, k), dtype=np.float32)
    b = rng.standard_normal((k, n), dtype=np.float32) / np.float32(np.sqrt(k))
    bias = rng.standard_normal(n, dtype=np.float32)
    r = rng.standard_normal((m, n), dtype=np.float32)
    ad, bd, biasd, rd = (torch.from_numpy(v).cuda() for v in (a, b, bias, r))
    cd = torch.full((m, n), float("nan"), device="cuda")
    t._lib.check(fn(ad.data_ptr(), bd.data_ptr(), biasd.data_ptr(), rd.data_ptr(), cd.data_ptr(), m, n, k, k, act, None), fn.__name__)
    torch.cuda.synchronize()
    ref = _act64(_linear64(a, b, bias) + r, act)
    got = cd.cpu().numpy()
    assert not np.isnan(got).any() and ggr._err(got, ref) <= TOL, ggr._err(got, ref)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("m", [1, 8, 9, 33, 63])
@pytest.mark.parametrize("k,n", PROJ)
def test_k_gemm_at_gpt2_decode_shapes(k, n, m, act):
    """below 64 rows every decode projection runs on the SIMT kernel"""
    _gemm(lib.tfsc_k_gemm, m, n, k, act)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("m", [64, 65, 127, 128])
@pytest.mark.parametrize("k,n", PROJ)
def test_k_gemm_tc_at_gpt2_decode_shapes(k, n, m, act):
    """64-128 rows: one or two 128-row tiles, so launch_gt splits K over a cluster and folds the slices in DSMEM before the
    bias, residual and activation"""
    _gemm(lib.tfsc_k_gemm_tc, m, n, k, act)


@pytest.mark.parametrize("m", [64, 65, 128])
def test_k_gemm_tc_at_gpt2_vocab(m):
    """the vocabulary projection from 64 rows: no activation, no residual in the bundle, both given here"""
    k, n = VOCAB[0]
    _gemm(lib.tfsc_k_gemm_tc, m, n, k, 0)


@pytest.mark.parametrize("splits", ["0", "2", "8"])
def test_gpt2_decode_gemms_with_and_without_the_cluster_fold(splits):
    """the tensor-core cases above with split-K forbidden ("0") and forced to 2 and 8, so each decode shape is compared with
    fp64 both with and without the DSMEM fold (TFSC_GEMM_SPLITK is read once per process, hence the subprocess)"""
    if os.environ.get("TFSC_GEMM_SPLITK"):
        pytest.skip("already inside the forced-split run")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, TFSC_GEMM_SPLITK=splits)
    run = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider",
                          "-k", "gemm_tc_at_gpt2"], capture_output=True, text=True, timeout=900, env=env, cwd=root)
    assert run.returncode == 0, (run.stdout + run.stderr)[-3000:]


# --------------------------------------------------------------------------------------- the dense kernels ----
def _dense_case(rows, k, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, k), dtype=np.float32)
    w = rng.standard_normal((k, n), dtype=np.float32) / np.float32(np.sqrt(k))
    b = rng.standard_normal(n, dtype=np.float32)
    return x, w, b, _linear64(x, w, b)


@pytest.mark.parametrize("rows", [1, 9, 16, 17, 31, 32, 33, 48, 63, 64])
@pytest.mark.parametrize("k,n", VOCAB)
def test_dense_tc_at_gpt2_vocab(k, n, rows):
    """197 strips of 256 columns, the last 96 wide, in two waves over 132 SMs; 9-64 rows cross every RP template"""
    x, w, b, lin = _dense_case(rows, k, n, rows * 1009 + k + n)
    for relu in (False, True):
        got = gtc._run(x, w, b, relu)
        ref = np.maximum(lin, 0) if relu else lin
        assert not np.isnan(got).any() and gtc._err(got, ref) <= TOL, (relu, gtc._err(got, ref))


@pytest.mark.parametrize("rows", [1, 2, 3, 4, 5, 7, 8, 9, 16, 19, 65, 72, 73, 128, 219])
@pytest.mark.parametrize("k,n", VOCAB + [WIDEST])
def test_k_dense_at_gpt2_vocab(k, n, rows):
    """tfsc_k_dense: <= 8 rows on the cluster kernel, 9-63 on dense_tc; 65 / 72 / 73 / 128 / 219 rows as tensor-core
    passes of 64 plus a last pass, SIMT when <= 8 rows, on one split-K workspace whose tensor-core counters outgrow the
    first 256 bytes at n > 16,384"""
    x, w, b, lin = _dense_case(rows, k, n, rows * 7919 + k + n)
    for relu in (False, True):
        got = gp._dense(x, w, b, relu)
        ref = np.maximum(lin, 0) if relu else lin
        assert not np.isnan(got).any() and gp._close(got, ref) <= TOL, (relu, gp._close(got, ref))


# --------------------------------------------------------------------------------------- decode attention ----
@pytest.mark.parametrize("L", [129, 1024])
@pytest.mark.parametrize("rows", [9, 65, 128])
def test_decode_attention_rows_past_8(rows, L):
    """GPT-2's 12 heads x d 64 over as many rows as a served batch: each row with its own padding pattern and prompt
    length, so pos (and with it the query's key block) varies per row. Against fp64, counters left zero (checked by
    gg._decode), and every row's bits those of the row launched alone."""
    heads, d = 12, 64
    H = heads * d
    rng = np.random.default_rng(rows * 10007 + L)
    t_ = L // 8
    S = L - 1 - t_
    qkv = rng.standard_normal((rows, L, 3 * H), dtype=np.float32)
    qkv[..., :2 * H] *= np.float32(3.0 ** 0.5 / d ** 0.25 / 2)
    mask = np.ones((rows, S), np.int32)
    for b in range(rows):
        n = int(rng.integers(1, S + 1))                           # the row's prompt length
        kind = b % 5
        if kind == 1:                                             # right-padded
            mask[b, n:] = 0
        elif kind == 2:                                           # left-padded
            mask[b, :S - n] = 0
        elif kind == 3:                                           # right-padded with masked holes
            mask[b, n:] = 0
            mask[b, rng.integers(0, n, max(1, n // 4))] = 0
        elif kind == 4 and b % 2:                                 # fully padded
            mask[b] = 0
    pos = np.array([max(np.nonzero(m)[0]) if m.any() else -1 for m in mask], np.int32)
    assert len(set(pos.tolist())) >= rows // 3
    ctx, _kc, _vc = gg._decode(qkv, mask, pos, S, t_, heads)
    ref = gg._decode_ref(qkv, mask, pos, t_, heads)
    err = np.abs(ctx - ref).max()
    assert err <= 2e-5 * max(1.0, np.abs(ref).max()), err
    for b in range(rows):
        one, _kc, _vc = gg._decode(qkv[b:b + 1], mask[b:b + 1], pos[b:b + 1], S, t_, heads)
        assert one.tobytes() == ctx[b:b + 1].tobytes(), b
