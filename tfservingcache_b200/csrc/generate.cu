// Generation kernels of GPT-2 generate bundles, fp32, sm_90a: the copy of the prompt's keys and values into the KV
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
//
// generate_sample_kernel: the select step of sampling bundles. The same staging, maximum and log-probability, then a token
// drawn from the temperature / top-k / top-p distribution with the row's seed (sample_token), written as the select step's.
//
// generate_process_kernel: the step of processing bundles (repetition penalty, no-repeat n-grams, minimum length). The same
// staging, maximum and log-probability, then the row's history of prompt and generated ids (kept in scratch across steps)
// processes the staged row in place, and the token is the processed row's argmax or draw (sample_token).
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

// The select and sample steps' writes for row `row` and its token g (the sentinel INT_MAX of a NaN row clamped to an id): the
// outputs, the done flag and, unless last, the next step's input word[g] + pos_table[p + 1 + t]
template <bool kVec>
__device__ __forceinline__ void generate_write(int64_t row, int t, int p, bool live, int g, const float* xs, int vocab, float m,
                                               double sum, bool last, int eos, int* __restrict__ done, const GenerateOutputs& o,
                                               const float* __restrict__ word, const float* __restrict__ pos_table,
                                               float* __restrict__ y, int H) {
  // g < vocab for finite logits; a NaN row can leave the sentinel INT_MAX, which must not index shared memory or a table
  const int gc = g < 0 ? 0 : (g >= vocab ? vocab - 1 : g);
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
  generate_write<kVec>(row, t, p, live, sel[0], xs, vocab, m, sum, last, eos, done, o, word, pos_table, y, H);
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

// ------------------------------------------------------------------------------------------------- sampling ----
typedef unsigned long long u64;

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011) of counter c under key (k0, k1)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) k0 += 0x9E3779B9u, k1 += 0xBB67AE85u;
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// An order-preserving key of a logit: larger logits have larger keys and -0 ranks as +0, so (key descending, id ascending)
// is the next-token head's rank order for every non-NaN logit
__device__ __forceinline__ uint32_t rank_key(float z) {
  uint32_t u = __float_as_uint(z);
  if (u == 0x80000000u) u = 0;
  return (u & 0x80000000u) ? ~u : u | 0x80000000u;
}

// A token's sampling weight exp((z - m) / temperature) in [0, 1] as a fixed-point integer of 2^-46 units, so that every sum
// of weights is exact and does not depend on its order: 57344 of them stay below 2^62. NaN and inf give 0. inv_t is
// 1 / temperature in fp32, rounded once on the host: a division here would call fp32 division's slow path.
__device__ __forceinline__ u64 weight_q(float z, float m, float inv_t) {
  const float w = expf((z - m) * inv_t);
  return w > 0.f ? __float2ull_rz(fminf(w, 1.f) * 0x1p46f) : 0ull;
}

// hist[b] = the sum of val(key, j) over the staged logits whose key agrees with `prefix` above bit shift + 8, b the key's
// byte at `shift`. Lanes with the same bin add their values first (integers: exact), then one shared atomic per bin.
template <typename Val>
__device__ __forceinline__ void radix_hist(const float* xs, int n, int shift, uint32_t prefix, Val val, u64* hist) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  const uint32_t above = shift == 24 ? 0u : ~0u << (shift + 8);
  const int lane = threadIdx.x & 31;
  for (int j = threadIdx.x; j - lane < n; j += blockDim.x) {  // warp-uniform trip count: every lane reaches the match
    int bin = 256;
    u64 v = 0;
    if (j < n) {
      const uint32_t key = rank_key(xs[j]);
      if (((key ^ prefix) & above) == 0) v = val(key, j);
      if (v) bin = (key >> shift) & 255;
    }
    if (!__any_sync(0xffffffffu, bin < 256)) continue;  // past the first pass most warps hold no element of the prefix
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    // v < 2^47: two 23-bit halves, each summed over at most 32 lanes without overflow
    const unsigned lo = __reduce_add_sync(peers, (unsigned)(v & 0x7fffff)), hi = __reduce_add_sync(peers, (unsigned)(v >> 23));
    if (bin < 256 && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], ((u64)hi << 23) + lo);
  }
  __syncthreads();
}

struct RadixPick {
  int bin;     // -1: the histogram holds less than need
  u64 before;  // the sum of the bins above it
  u64 count;   // its own
  u64 need;
};

// Warp 0 finds the highest bin b whose suffix sum hist[b..255] reaches need; frac > 0 sets need = ceil(frac * total), at
// least 1. Lane l sums bins 255 - 8l down to 248 - 8l, the lanes scan in that order. Every thread gets the result.
__device__ __forceinline__ RadixPick radix_pick(const u64* hist, u64 need, double frac, RadixPick* s_pick) {
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    u64 mine = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) mine += hist[255 - 8 * lane - i];
    u64 incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    const u64 total = __shfl_sync(0xffffffffu, incl, 31);
    if (frac > 0.0) need = total ? min(total, max(1ull, (u64)ceil(frac * (double)total))) : 0;
    if (lane == 0) s_pick->bin = -1, s_pick->need = need;
    __syncwarp();
    if (need >= 1 && incl >= need && incl - mine < need) {
      u64 acc = incl - mine;
      for (int i = 0; i < 8; ++i) {
        const int b = 255 - 8 * lane - i;
        if (acc + hist[b] >= need) {
          s_pick->bin = b, s_pick->before = acc, s_pick->count = hist[b];
          break;
        }
        acc += hist[b];
      }
    }
  }
  __syncthreads();
  const RadixPick r = *s_pick;
  __syncthreads();
  return r;
}

// The first j in [0, n) at which the running sum of v(j) over ascending j exceeds target(total), total the sum over all of
// [0, n); -1 when none does. Each thread sums a contiguous chunk of ids, the chunk sums are scanned in thread order and the
// thread whose chunk holds the crossing walks it. scan: kHeadThreadsMax / 32 words of shared memory.
template <typename V, typename Target>
__device__ __forceinline__ int chunk_find(int n, V v, Target target, u64* scan, int* s_res) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int c = (n + blockDim.x - 1) / blockDim.x, lo = min(n, (int)threadIdx.x * c), hi = min(n, lo + c);
  u64 mine = 0;
  for (int j = lo; j < hi; ++j) mine += v(j);
  u64 incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) scan[warp] = incl;
  if (threadIdx.x == 0) *s_res = -1;
  __syncthreads();
  if (warp == 0) {
    u64 w = lane < nwarps ? scan[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    if (lane < nwarps) scan[lane] = w;
  }
  __syncthreads();
  const u64 total = scan[nwarps - 1], tg = target(total), before = (warp ? scan[warp - 1] : 0) + incl - mine;
  if (tg < total && before <= tg && tg < before + mine) {
    u64 acc = before;
    for (int j = lo; j < hi; ++j)
      if ((acc += v(j)) > tg) {
        *s_res = j;
        break;
      }
  }
  __syncthreads();
  const int r = *s_res;
  __syncthreads();
  return r;
}

// The sampled token of the staged row (DESIGN §3): the rank-order top_k (0: all) and the shortest rank-order prefix of those
// whose weight reaches top_p of theirs (1: all), then the first kept id, ascending, whose running weight exceeds u * W, W
// the kept weight and u the 53-bit uniform of Philox4x32-10 with key (seed, 0) and counter (t, 0, 0, 0). The kept set is
// a rank threshold: key > kt, or key == kt and id <= it. Top-k and top-p boundaries are radix selections over the keys,
// their ties cut in id order; every sum is an integer, so the token is a function of the logits' bits, seed and t.
__device__ __forceinline__ int sample_token(const float* xs, int vocab, float m, float inv_t, int top_k, float top_p,
                                            uint32_t seed, int t, u64* hist, RadixPick* s_pick, int* s_res) {
  uint32_t kt = 0;
  int it = INT_MAX;
  auto kept = [&](uint32_t key, int j) { return key > kt || (key == kt && j <= it); };
  if (top_k > 0 && top_k < vocab) {
    uint32_t prefix = 0;
    RadixPick r = {};
    u64 need = (u64)top_k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      radix_hist(xs, vocab, shift, prefix, [](uint32_t, int) { return 1ull; }, hist);
      r = radix_pick(hist, need, 0.0, s_pick);
      prefix |= (uint32_t)r.bin << shift;
      need -= r.before;
    }
    kt = prefix;
    if (r.count != need) {  // the need-th lowest id among the ties at the boundary
      const uint32_t k = prefix;
      it = chunk_find(vocab, [&](int j) { return (u64)(rank_key(xs[j]) == k); }, [&](u64) { return need - 1; }, hist, s_res);
    }
  }
  if (top_p < 1.f) {
    uint32_t prefix = 0;
    RadixPick r = {};
    u64 need = 0;
    bool none = false;
    for (int shift = 24; shift >= 0 && !none; shift -= 8) {
      radix_hist(xs, vocab, shift, prefix, [&](uint32_t key, int j) { return kept(key, j) ? weight_q(xs[j], m, inv_t) : 0ull; },
                 hist);
      r = radix_pick(hist, need, shift == 24 ? (double)top_p : 0.0, s_pick);
      none = r.bin < 0;  // no kept weight at all (NaN or inf logits): top-p keeps the top-k set
      if (shift == 24) need = r.need;
      prefix |= (uint32_t)(r.bin & 255) << shift;
      need -= none ? 0 : r.before;
    }
    if (!none) {
      const uint32_t k = prefix;
      const int cut = chunk_find(
          vocab, [&](int j) { return rank_key(xs[j]) == k && kept(k, j) ? weight_q(xs[j], m, inv_t) : 0ull; },
          [&](u64) { return need - 1; }, hist, s_res);
      kt = k, it = cut < 0 ? it : cut;
    }
  }
  const uint4 x = philox4x32_10(make_uint4((uint32_t)t, 0, 0, 0), seed, 0);
  const u64 U = ((u64)(x.x >> 5) << 26) | (x.y >> 6);  // u = U * 2^-53
  int g = chunk_find(
      vocab, [&](int j) { return kept(rank_key(xs[j]), j) ? weight_q(xs[j], m, inv_t) : 0ull; },
      [&](u64 W) { return (__umul64hi(U, W) << 11) | ((U * W) >> 53); }, hist, s_res);  // floor(u * W)
  if (g < 0)  // no kept weight: the last kept id
    g = chunk_find(vocab, [&](int j) { return (u64)kept(rank_key(xs[j]), j); }, [](u64 n) { return n - 1; }, hist, s_res);
  return g;
}

template <bool kVec>
__global__ void __launch_bounds__(kHeadThreadsMax) generate_sample_kernel(const float* __restrict__ logits, int64_t ld, int vocab,
                                                                          const int* __restrict__ pos, int t, bool last, int eos,
                                                                          int* __restrict__ done, GenerateOutputs o,
                                                                          const float* __restrict__ word,
                                                                          const float* __restrict__ pos_table, float* __restrict__ y,
                                                                          int H, const int* __restrict__ seeds, int64_t seed_stride,
                                                                          float inv_t, int top_k, float top_p) {
  extern __shared__ float xs[];  // the row's vocab logits
  __shared__ float wv[kHeadThreadsMax / 32];
  __shared__ int wi[kHeadThreadsMax / 32];
  __shared__ double wsum[kHeadThreadsMax / 32];
  __shared__ float s_v;
  __shared__ int s_i;
  __shared__ double s_sum;
  __shared__ int sel[1];
  __shared__ u64 hist[256];  // the radix histograms and the id-order scans, one at a time: 2 KB beside 224 KB of logits
  __shared__ RadixPick s_pick;
  __shared__ int s_res;
  const int64_t row = blockIdx.x;
  // launched after the vocabulary projection; done comes from the previous step's launch
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int p = __ldg(pos + row);
  const bool live = t == 0 ? p >= 0 : done[row] == 0;
  const float m = head_stage_select(logits + row * ld, vocab, 1, xs, wv, wi, &s_v, &s_i, sel);
  const double sum = head_exp_sum(xs, vocab, m, wsum, &s_sum);
  // top_k = 1 is the greedy token; the log-probability is the model's, at temperature 1 and unfiltered, as greedy's
  const int g = top_k == 1 ? sel[0]
                           : sample_token(xs, vocab, m, inv_t, top_k, top_p, (uint32_t)__ldg(seeds + row * seed_stride), t,
                                          hist, &s_pick, &s_res);
  generate_write<kVec>(row, t, p, live, g, xs, vocab, m, sum, last, eos, done, o, word, pos_table, y, H);
}

cudaError_t launch_generate_sample(const float* logits, int64_t ld, int vocab, const int* pos, int t, bool last, int eos,
                                   int* done, const GenerateOutputs& o, const float* word, const float* pos_table, float* y,
                                   int rows, int H, const int* seeds, int64_t seed_stride, float temperature, int top_k,
                                   float top_p, cudaStream_t s) {
  if (rows < 0 || t < 0 || vocab < 1 || vocab > kNextTokenMaxVocab || ld < vocab || H < 1 || !logits || !pos || !done ||
      (!last && (!word || !pos_table || !y)) || !seeds || seed_stride < 1 || !sampling_supported(vocab, temperature, top_k, top_p))
    return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    for (cudaError_t e : {cudaFuncSetAttribute(generate_sample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kNextTokenMaxVocab * (int)sizeof(float)),
                          cudaFuncSetAttribute(generate_sample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kNextTokenMaxVocab * (int)sizeof(float))})
      if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  const bool vec = H % 4 == 0 && (((uintptr_t)word | (uintptr_t)pos_table | (uintptr_t)y) & 15) == 0;
  const size_t smem = (size_t)vocab * sizeof(float);
  // the select step's block size: its maximum and sum of exponentials, so its log-probabilities, are the same bits
  const int threads = head_threads(vocab);
  const float inv_t = 1.f / temperature;
  return vec ? launch_pdl(generate_sample_kernel<true>, dim3((unsigned)rows), threads, smem, s, logits, ld, vocab, pos, t, last, eos,
                          done, o, word, pos_table, y, H, seeds, seed_stride, inv_t, top_k, top_p)
             : launch_pdl(generate_sample_kernel<false>, dim3((unsigned)rows), threads, smem, s, logits, ld, vocab, pos, t, last, eos,
                          done, o, word, pos_table, y, H, seeds, seed_stride, inv_t, top_k, top_p);
}

// --------------------------------------------------------------------------------------- repetition control ----
// The argmax of the staged row in the next-token head's rank order (value descending, ties to the lower id; all -inf: id 0):
// head_stage_select's first round without the staging. Every thread gets the id, and *v its value.
__device__ __forceinline__ int staged_argmax(const float* xs, int n, float* wv, int* wi, float* s_v, int* s_i, float* v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  float bv;
  int bi;
  local_best(xs, n, INFINITY, -1, &bv, &bi);
  warp_best(bv, bi);
  if (lane == 0) {
    wv[warp] = bv;
    wi[warp] = bi;
  }
  __syncthreads();
  if (warp == 0) {
    bv = lane < nwarps ? wv[lane] : -INFINITY;
    bi = lane < nwarps ? wi[lane] : INT_MAX;
    warp_best(bv, bi);
    if (lane == 0) {
      *s_v = bv;
      *s_i = bi;
    }
  }
  __syncthreads();
  *v = *s_v;
  return *s_i;
}

// The step of processing bundles (DESIGN §3): the select step's staging, maximum and sum of the raw logits, then in shared
// memory the repetition penalty over the row's history, the no-repeat n-gram bans and the EOS ban below min_new steps, and
// the argmax (seeds null) or the sampled token (sample_token) of the processed row. At t = 0 the CTA writes the history's
// prompt part, the attended prompt ids in position order, to hist and its length to hist_len0; every step appends its token
// at hist[hist_len0 + t]. hist is ordered across steps as done is: every launch of the chain waits for the one before.
template <bool kVec>
__global__ void __launch_bounds__(kHeadThreadsMax) generate_process_kernel(
    const float* __restrict__ logits, int64_t ld, int vocab, const int* __restrict__ pos, int t, bool last, int eos,
    int* __restrict__ done, GenerateOutputs o, const float* __restrict__ word, const float* __restrict__ pos_table,
    float* __restrict__ y, int H, const int* __restrict__ ids, const int* __restrict__ mask, int64_t stride, int* hist,
    int64_t hist_ld, int* hist_len0, float penalty, int ngram, int min_new, const int* __restrict__ seeds, int64_t seed_stride,
    float inv_t, int top_k, float top_p) {
  extern __shared__ float xs[];  // the row's vocab logits, processed in place
  __shared__ float wv[kHeadThreadsMax / 32];
  __shared__ int wi[kHeadThreadsMax / 32];
  __shared__ double wsum[kHeadThreadsMax / 32];
  __shared__ float s_v;
  __shared__ int s_i;
  __shared__ double s_sum;
  __shared__ int sel[1];
  __shared__ int wcnt[kHeadThreadsMax / 32];
  __shared__ u64 rhist[256];  // sample_token's radix histograms and scans
  __shared__ RadixPick s_pick;
  __shared__ int s_res;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t row = blockIdx.x;
  // launched after the vocabulary projection; done, hist and hist_len0 come from the previous steps' launches
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int p = __ldg(pos + row);
  const bool live = t == 0 ? p >= 0 : done[row] == 0;
  const float* raw = logits + row * ld;
  const float m = head_stage_select(raw, vocab, 1, xs, wv, wi, &s_v, &s_i, sel);
  const double sum = head_exp_sum(xs, vocab, m, wsum, &s_sum);
  int* h = hist + row * hist_ld;
  int L0 = 0;
  if (t == 0) {
    // positions 0..p whose mask is set (all of them without a mask), compacted in order a block of positions at a time:
    // a ballot per warp, the warps' counts in wcnt; ids clamped to [0, vocab) as the embedding clamps them
    const int* irow = ids + row * stride;
    const int* mrow = mask ? mask + row * stride : nullptr;
    for (int base = 0; base <= p; base += blockDim.x) {
      const int j = base + (int)threadIdx.x;
      const bool att = j <= p && (!mrow || __ldg(mrow + j) != 0);
      const unsigned ballot = __ballot_sync(0xffffffffu, att);
      if (lane == 0) wcnt[warp] = __popc(ballot);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < nwarps; ++w) {
        const int c = wcnt[w];
        before += w < warp ? c : 0;
        total += c;
      }
      if (att) {
        const int id = __ldg(irow + j);
        h[L0 + before + __popc(ballot & ((1u << lane) - 1u))] = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
      }
      L0 += total;
      __syncthreads();  // wcnt is rewritten by the next pass; the history is complete after the last
    }
    if (threadIdx.x == 0) hist_len0[row] = L0;
  } else {
    L0 = hist_len0[row];
  }
  const int L = L0 + t;  // the prompt part and g_0 .. g_{t-1}
  // the penalty reads each logit from the unprocessed row in global memory, so an id the history holds twice gets the same
  // value from both writes
  if (penalty != 1.f)
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
      const int id = h[i];
      const float z = __ldg(raw + id);
      xs[id] = z < 0.f ? __fmul_rn(z, penalty) : __fdiv_rn(z, penalty);
    }
  __syncthreads();
  // every h[i + n - 1] whose n - 1 tokens before it are the history's last n - 1 tokens is banned
  for (int i = threadIdx.x; ngram > 0 && i <= L - ngram; i += blockDim.x) {
    bool match = true;
    for (int k = 0; k < ngram - 1 && match; ++k) match = h[i + k] == h[L - ngram + 1 + k];
    if (match) xs[h[i + ngram - 1]] = -INFINITY;
  }
  if (t < min_new && threadIdx.x == 0) xs[eos] = -INFINITY;
  __syncthreads();
  float mp;
  int g = staged_argmax(xs, vocab, wv, wi, &s_v, &s_i, &mp);
  // a sampling bundle draws from the processed row unless top_k = 1 (its argmax) or every logit is banned (id 0, no draw)
  if (seeds && top_k != 1 && mp != -INFINITY)
    g = sample_token(xs, vocab, mp, inv_t, top_k, top_p, (uint32_t)__ldg(seeds + row * seed_stride), t, rhist, &s_pick, &s_res);
  // the log-probability is the raw row's: the select step's bits for the same g
  generate_write<kVec>(row, t, p, live, g, raw, vocab, m, sum, last, eos, done, o, word, pos_table, y, H);
  if (threadIdx.x == 0) h[L] = g < 0 ? 0 : (g >= vocab ? vocab - 1 : g);
}

cudaError_t launch_generate_process(const float* logits, int64_t ld, int vocab, const int* pos, int t, bool last, int eos,
                                    int* done, const GenerateOutputs& o, const float* word, const float* pos_table, float* y,
                                    int rows, int H, const int* ids, const int* mask, int64_t stride, int* hist, int64_t hist_ld,
                                    int* hist_len0, float penalty, int ngram, int min_new, const int* seeds, int64_t seed_stride,
                                    float temperature, int top_k, float top_p, cudaStream_t s) {
  if (rows < 0 || t < 0 || vocab < 1 || vocab > kNextTokenMaxVocab || ld < vocab || H < 1 || !logits || !pos || !done ||
      (!last && (!word || !pos_table || !y)) || !ids || stride < 1 || !hist || hist_ld <= t || !hist_len0 ||
      !processing_supported(penalty, ngram, min_new) || (min_new > 0 && (eos < 0 || eos >= vocab)) ||
      (seeds && (seed_stride < 1 || !sampling_supported(vocab, temperature, top_k, top_p))))
    return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    for (cudaError_t e : {cudaFuncSetAttribute(generate_process_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kNextTokenMaxVocab * (int)sizeof(float)),
                          cudaFuncSetAttribute(generate_process_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kNextTokenMaxVocab * (int)sizeof(float))})
      if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  const bool vec = H % 4 == 0 && (((uintptr_t)word | (uintptr_t)pos_table | (uintptr_t)y) & 15) == 0;
  const size_t smem = (size_t)vocab * sizeof(float);
  // the select step's block size: its maximum and sum of exponentials, so its log-probabilities, are the same bits
  const int threads = head_threads(vocab);
  const float inv_t = seeds ? 1.f / temperature : 1.f;
  return vec ? launch_pdl(generate_process_kernel<true>, dim3((unsigned)rows), threads, smem, s, logits, ld, vocab, pos, t, last,
                          eos, done, o, word, pos_table, y, H, ids, mask, stride, hist, hist_ld, hist_len0, penalty, ngram, min_new,
                          seeds, seed_stride, inv_t, top_k, top_p)
             : launch_pdl(generate_process_kernel<false>, dim3((unsigned)rows), threads, smem, s, logits, ld, vocab, pos, t, last,
                          eos, done, o, word, pos_table, y, H, ids, mask, stride, hist, hist_ld, hist_len0, penalty, ngram, min_new,
                          seeds, seed_stride, inv_t, top_k, top_p);
}

}  // namespace tfsc
