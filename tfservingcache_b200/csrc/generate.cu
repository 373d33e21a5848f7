// Greedy generation kernels of GPT-2 generate bundles, fp32, sm_90a: the copy of the prompt's keys and values into the KV
// cache, single-query attention over that cache, and the step that picks each row's token and embeds it for the next step.
//
// kv_cache_write_kernel: after each prefill attention op, copies the k | v columns of its packed qkv buffer [rows, S, 3H] to
// slots 0..S-1 of the layer's K and V caches [rows, T, H]. Copies, so the bits are exact; 16-byte vectors, a scalar path
// for layouts that are not 16-byte aligned.
//
// decode_attention_kernel (flash-decoding): one CTA per (row, head, block of kDecodeKeys keys). A CTA stages its block's
// keys in shared memory, a thread scores one key, and the block's max, sum and unnormalised P.V go to the work buffer. The
// last CTA of a (row, head) to finish (an atomic counter, reset by that CTA) combines the blocks in block order, so the
// result does not depend on which CTA finished last. The number of blocks depends on S and the step only, never on the
// batch, and a block beyond a row's query holds no key and is skipped, so a row's bits do not depend on the rest of its
// batch. The step's own key and value are read from the qkv buffer, and the CTA of block 0 appends them to the cache: no
// CTA reads a slot that another writes in the same launch.
//
// generate_select_kernel: one CTA per row, the next-token head's selection (head_select.cuh) with k = 1 and its fp64 sum of
// exponentials for the log-probability, then the next step's input row wte[g] + wpe[slot] (embed_positions_kernel's add).
#include <cuda_runtime.h>

#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdlib>

#include "head_select.cuh"
#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kCacheThreads = 256, kDecodeThreads = 128;

static bool pdl_on() {  // programmatic dependent launch, on unless TFSC_PDL=0, as the heads
  static const bool v = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  return v;
}

template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, int threads, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_on() ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
  g_launches_nn++;
  return e;
}

template <bool kVec>
__global__ void __launch_bounds__(kCacheThreads) kv_cache_write_kernel(const float* __restrict__ qkv, float* __restrict__ kc,
                                                                       float* __restrict__ vc, int64_t tokens, int S, int T, int H) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // launched after the attention op, which reads the same qkv; the op that wrote it finished before that one started
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int Q = kVec ? H >> 2 : H;  // float4s (or floats) per token of one cache
  const int64_t n = tokens * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t tok = i / Q;
    const int q = (int)(i - tok * Q);
    const int64_t r = tok / S, dst = (r * T + (tok - r * S)) * Q + q;
    if (kVec) {
      const float4* src = reinterpret_cast<const float4*>(qkv) + tok * 3 * Q;
      reinterpret_cast<float4*>(kc)[dst] = __ldg(src + Q + q);
      reinterpret_cast<float4*>(vc)[dst] = __ldg(src + 2 * Q + q);
    } else {
      const float* src = qkv + tok * 3 * Q;
      kc[dst] = __ldg(src + Q + q);
      vc[dst] = __ldg(src + 2 * Q + q);
    }
  }
}

cudaError_t launch_kv_cache_write(const float* qkv, float* kc, float* vc, int rows, int S, int T, int H, cudaStream_t s) {
  if (rows < 0 || S < 1 || T < S || H < 1 || !qkv || !kc || !vc) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  const bool vec = H % 4 == 0 && (((uintptr_t)qkv | (uintptr_t)kc | (uintptr_t)vc) & 15) == 0;
  const int64_t tokens = (int64_t)rows * S, n = tokens * (vec ? H / 4 : H);
  int64_t blocks = (n + kCacheThreads - 1) / kCacheThreads;
  if (blocks > (int64_t)device_sm_count() * 8) blocks = (int64_t)device_sm_count() * 8;
  return vec ? launch_pdl(kv_cache_write_kernel<true>, dim3((unsigned)blocks), kCacheThreads, 0, s, qkv, kc, vc, tokens, S, T, H)
             : launch_pdl(kv_cache_write_kernel<false>, dim3((unsigned)blocks), kCacheThreads, 0, s, qkv, kc, vc, tokens, S, T, H);
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// work: int32 counters [rows * heads], then the blocks' max [P], sum [P] and context [P, d], P = rows * heads * blocks
template <bool kVec>
__global__ void __launch_bounds__(kDecodeThreads) decode_attention_kernel(const float* __restrict__ qkv, float* __restrict__ kc,
                                                                          float* __restrict__ vc, const int* __restrict__ pos, int t,
                                                                          const int* __restrict__ mask, int64_t mask_stride, int T,
                                                                          float* __restrict__ ctx, int H, int heads,
                                                                          int* __restrict__ counters, float* __restrict__ part) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float red[kDecodeThreads / 32];
  __shared__ int s_last;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int d = H / heads, ds = d + 4;
  float* Ks = sm;                         // [kDecodeKeys][ds]
  float* qs = Ks + kDecodeKeys * ds;      // [d]
  float* ps = qs + d;                     // [kDecodeKeys] unnormalised weights
  const int bh = blockIdx.x, b = bh / heads, hd = bh - b * heads;
  const int blk = blockIdx.y, blocks = gridDim.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // launched after the op that writes this step's qkv
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int p = __ldg(pos + b);
  const int q = p + 1 + t;                // this token's slot: keys 0..q
  const float* qrow = qkv + (int64_t)b * 3 * H + hd * d;  // q; its k at + H, its v at + 2H
  float* krow = kc + (int64_t)b * T * H + hd * d;         // key j at + j * H
  float* vrow = vc + (int64_t)b * T * H + hd * d;
  const int j0 = blk * kDecodeKeys;
  const int n = min(kDecodeKeys, q + 1 - j0);  // keys of this block (<= 0: none)
  if (blk == 0)
    for (int c = tid; c < d; c += kDecodeThreads) {
      krow[(int64_t)q * H + c] = __ldg(qrow + H + c);
      vrow[(int64_t)q * H + c] = __ldg(qrow + 2 * H + c);
    }
  for (int c = tid; c < d; c += kDecodeThreads) qs[c] = __ldg(qrow + c);
  if (kVec) {
    const int d4 = d >> 2;
    for (int idx = tid; idx < n * d4; idx += kDecodeThreads) {
      const int j = idx / d4, c = (idx - j * d4) << 2;
      const float* src = j0 + j == q ? qrow + H : krow + (int64_t)(j0 + j) * H;
      *reinterpret_cast<float4*>(Ks + j * ds + c) = __ldg(reinterpret_cast<const float4*>(src + c));
    }
  } else {
    for (int idx = tid; idx < n * d; idx += kDecodeThreads) {
      const int j = idx / d, c = idx - j * d;
      const float* src = j0 + j == q ? qrow + H : krow + (int64_t)(j0 + j) * H;
      Ks[j * ds + c] = __ldg(src + c);
    }
  }
  __syncthreads();
  float sc = -FLT_MAX;  // hidden: beyond the query or outside the block
  if (tid < n) {
    const float* kr = Ks + tid * ds;
    float acc = 0.f;
    for (int c = 0; c < d; c += 4) {
      const float4 kv = *reinterpret_cast<const float4*>(kr + c);
      const float4 qv = *reinterpret_cast<const float4*>(qs + c);
      acc = fmaf(qv.x, kv.x, fmaf(qv.y, kv.y, fmaf(qv.z, kv.z, fmaf(qv.w, kv.w, acc))));
    }
    const int j = j0 + tid;
    // a prompt key whose mask is 0 gets the BERT -10000, as in the causal kernel; generated keys (j > p) are never masked
    const float madd = (mask && j <= p && __ldg(mask + (int64_t)b * mask_stride + j) == 0) ? -10000.f : 0.f;
    sc = acc * rsqrtf((float)d) + madd;
  }
  float mx = sc;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < kDecodeThreads / 32; ++w) mx = fmaxf(mx, red[w]);
  const float e = sc == -FLT_MAX ? 0.f : expf(sc - mx);
  if (tid < kDecodeKeys) ps[tid] = e;
  float sum = e;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncthreads();  // every thread has read red
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  float l = red[0];
#pragma unroll
  for (int w = 1; w < kDecodeThreads / 32; ++w) l += red[w];
  const int64_t P = (int64_t)gridDim.x * blocks, slot = (int64_t)bh * blocks + blk;
  float* pm = part;
  float* pl = part + P;
  float* pacc = part + 2 * P;
  // the block's cached keys, then this token's own (the block's last key when it holds the query); a block past the
  // query (n <= 0) has neither
  const int ncached = max(0, min(n, q - j0));
  for (int c = tid; c < d; c += kDecodeThreads) {
    float o = 0.f;
    const float* v = vrow + (int64_t)j0 * H + c;
    for (int j = 0; j < ncached; ++j) o = fmaf(ps[j], __ldg(v + (int64_t)j * H), o);
    if (n > ncached) o = fmaf(ps[n - 1], __ldg(qrow + 2 * H + c), o);
    pacc[slot * d + c] = o;
  }
  if (tid == 0) {
    pm[slot] = mx;  // -FLT_MAX for a block without keys: skipped below
    pl[slot] = l;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(counters + bh, 1) == blocks - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int64_t first = (int64_t)bh * blocks;
  float M = -FLT_MAX;
  for (int c = 0; c < blocks; ++c) M = fmaxf(M, __ldcg(pm + first + c));
  float L = 0.f;
  for (int c = 0; c < blocks; ++c) {
    const float m = __ldcg(pm + first + c);
    if (m != -FLT_MAX) L += __ldcg(pl + first + c) * expf(m - M);
  }
  const float inv = 1.f / L;
  for (int cc = tid; cc < d; cc += kDecodeThreads) {
    float o = 0.f;
    for (int c = 0; c < blocks; ++c) {
      const float m = __ldcg(pm + first + c);
      if (m != -FLT_MAX) o += __ldcg(pacc + (first + c) * d + cc) * expf(m - M);
    }
    ctx[(int64_t)b * H + hd * d + cc] = o * inv;
  }
  if (tid == 0) counters[bh] = 0;
}

cudaError_t launch_decode_attention(const float* qkv, float* kc, float* vc, const int* pos, int t, const int* mask,
                                    int64_t mask_stride, int S, int T, float* ctx, int rows, int H, int heads, void* work,
                                    cudaStream_t s) {
  const int L = S + t + 1;  // the largest key count of any row: pos <= S - 1
  if (rows < 0 || t < 0 || S < 1 || L > T || !decode_attention_supported(L, H, heads) || (mask && mask_stride < S) ||
      (int64_t)rows * heads > 0x7fffffff)
    return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  if (!qkv || !kc || !vc || !pos || !ctx || !work) return cudaErrorInvalidValue;
  const int d = H / heads;
  const bool vec = (((uintptr_t)qkv | (uintptr_t)kc | (uintptr_t)vc) & 15) == 0;
  const dim3 grid((unsigned)(rows * heads), (unsigned)decode_attention_splits(L));
  const size_t smem = ((size_t)kDecodeKeys * (d + 4) + d + kDecodeKeys) * sizeof(float);
  int* counters = static_cast<int*>(work);
  float* part = reinterpret_cast<float*>(static_cast<char*>(work) + align256((size_t)rows * heads * 4));
  return vec ? launch_pdl(decode_attention_kernel<true>, grid, kDecodeThreads, smem, s, qkv, kc, vc, pos, t, mask, mask_stride, T,
                          ctx, H, heads, counters, part)
             : launch_pdl(decode_attention_kernel<false>, grid, kDecodeThreads, smem, s, qkv, kc, vc, pos, t, mask, mask_stride, T,
                          ctx, H, heads, counters, part);
}

template <bool kVec>
__global__ void __launch_bounds__(kHeadThreadsMax) generate_select_kernel(const float* __restrict__ logits, int64_t ld, int vocab,
                                                                          const int* __restrict__ pos, int t, bool last, int eos,
                                                                          int* __restrict__ done, GenerateOutputs o,
                                                                          const float* __restrict__ word,
                                                                          const float* __restrict__ pos_table, float* __restrict__ y,
                                                                          int H) {
  extern __shared__ float xs[];  // the row's vocab logits
  __shared__ float wv[kHeadThreadsMax / 32];
  __shared__ int wi[kHeadThreadsMax / 32];
  __shared__ double wsum[kHeadThreadsMax / 32];
  __shared__ float s_v;
  __shared__ int s_i;
  __shared__ double s_sum;
  __shared__ int sel[1];
  const int64_t row = blockIdx.x;
  // launched after the vocabulary projection; done comes from the previous step's launch
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int p = __ldg(pos + row);
  const bool live = t == 0 ? p >= 0 : done[row] == 0;
  const float m = head_stage_select(logits + row * ld, vocab, 1, xs, wv, wi, &s_v, &s_i, sel);
  const double sum = head_exp_sum(xs, vocab, m, wsum, &s_sum);
  // g < vocab for finite logits; a NaN row can leave the sentinel INT_MAX, which must not index shared memory or a table
  const int g = sel[0], gc = g < 0 ? 0 : (g >= vocab ? vocab - 1 : g);
  if (threadIdx.x == 0) {
    if (o.ids) o.ids[row * o.ids_ld + t] = live ? g : -1;
    if (o.log_probs) o.log_probs[row * o.log_probs_ld + t] = live ? (xs[gc] - m) - (float)log(sum) : 0.f;
    if (o.length && (live || t == 0)) o.length[row * o.length_ld] = live ? t + 1 : 0;
    if (live || t == 0) done[row] = !live || g == eos;
  }
  if (last) return;
  const int64_t slot = p + 1 + t;  // where the token goes: its position embedding
  if (kVec) {
    const float4* w = reinterpret_cast<const float4*>(word + (int64_t)gc * H);
    const float4* pe = reinterpret_cast<const float4*>(pos_table + slot * H);
    float4* dst = reinterpret_cast<float4*>(y + row * H);
    for (int c = threadIdx.x; c < (H >> 2); c += blockDim.x) {
      const float4 a = __ldg(w + c), b = __ldg(pe + c);
      dst[c] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
  } else {
    for (int c = threadIdx.x; c < H; c += blockDim.x) y[row * H + c] = __ldg(word + (int64_t)gc * H + c) + __ldg(pos_table + slot * H + c);
  }
}

cudaError_t launch_generate_select(const float* logits, int64_t ld, int vocab, const int* pos, int t, bool last, int eos,
                                   int* done, const GenerateOutputs& o, const float* word, const float* pos_table, float* y,
                                   int rows, int H, cudaStream_t s) {
  if (rows < 0 || t < 0 || vocab < 1 || vocab > kNextTokenMaxVocab || ld < vocab || H < 1 || !logits || !pos || !done ||
      (!last && (!word || !pos_table || !y)))
    return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    for (cudaError_t e : {cudaFuncSetAttribute(generate_select_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kNextTokenMaxVocab * (int)sizeof(float)),
                          cudaFuncSetAttribute(generate_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kNextTokenMaxVocab * (int)sizeof(float))})
      if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  const bool vec = H % 4 == 0 && (((uintptr_t)word | (uintptr_t)pos_table | (uintptr_t)y) & 15) == 0;
  const size_t smem = (size_t)vocab * sizeof(float);
  // the next-token head's block size for the same vocabulary: its argmax and sum run in the same order
  const int threads = head_threads(vocab);
  return vec ? launch_pdl(generate_select_kernel<true>, dim3((unsigned)rows), threads, smem, s, logits, ld, vocab, pos, t, last, eos,
                          done, o, word, pos_table, y, H)
             : launch_pdl(generate_select_kernel<false>, dim3((unsigned)rows), threads, smem, s, logits, ld, vocab, pos, t, last, eos,
                          done, o, word, pos_table, y, H);
}

}  // namespace tfsc
