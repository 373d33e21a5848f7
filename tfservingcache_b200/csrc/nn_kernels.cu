// Dense-net building blocks for the graph executor (SURVEY.md 8a rows X4 / X5), fp32, sm_90a:
//   gemm_f32      C[M,N] = act(A[M,K] B[K,N] + bias[N] (+ R[M,N]))   register-tiled FFMA GEMM (exact fp32)
//   im2col_nhwc   NHWC activations -> [B*OH*OW, KH*KW*C (padded to x4)] patch matrix (conv = im2col + GEMM with
//                 the TF HWIO kernel flattened to [KH*KW*Cin, Cout]; 1x1/stride-1 convs skip it)
//   maxpool / global average pool (NHWC), embedding gather + LayerNorm, residual LayerNorm, attention
// launch_gemm dispatches to the wgmma 3xTF32 GEMM of gemm_tc.cu when the shape allows (M >= 64, N % 32 == 0,
// K >= 32); gemm_f32_kernel (CUDA-core FFMA, exact fp32) covers the rest (small M, N = 1000 / 2 heads, conv1's K).
#include <cuda_runtime.h>

#include <atomic>
#include <cfloat>
#include <cstdlib>

#include "act.cuh"
#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;
std::atomic<int64_t> g_launches_nn{0};

// ------------------------------------------------------------------------------------ GEMM ----
constexpr int GBM = 128, GBN = 64, GBK = 16, GTHREADS = 256;

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

template <bool VEC>
__global__ void __launch_bounds__(GTHREADS)
gemm_f32_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ bias,
                const float* __restrict__ R, float* __restrict__ C, int M, int N, int K, int lda, int act) {
  __shared__ __align__(16) float As[2][GBK][GBM + 4];
  __shared__ __align__(16) float Bs[2][GBK][GBN];
  const int tid = threadIdx.x;
  const int ty = tid / 16, tx = tid % 16;  // 16 x 16 threads, 8 x 4 outputs each
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // global -> register staging: A tile 128 x 16 = 512 float4 (2 per thread), B tile 16 x 64 = 256 float4 (1 per thread)
  float4 ra[2], rb;
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = tid / 4 + 64 * i, kq = (tid % 4) * 4;
      const int gm = m0 + row, gk = k0 + kq;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gm < M) {
        const float* p = A + (size_t)gm * lda + gk;
        if (VEC && gk + 3 < K) v = __ldg(reinterpret_cast<const float4*>(p));
        else {
          if (gk < K) v.x = __ldg(p);
          if (gk + 1 < K) v.y = __ldg(p + 1);
          if (gk + 2 < K) v.z = __ldg(p + 2);
          if (gk + 3 < K) v.w = __ldg(p + 3);
        }
      }
      ra[i] = v;
    }
    {
      const int kr = tid / 16, c4 = (tid % 16) * 4;
      const int gk = k0 + kr, gn = n0 + c4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gk < K) {
        const float* p = B + (size_t)gk * N + gn;
        if (VEC && gn + 3 < N) v = __ldg(reinterpret_cast<const float4*>(p));
        else {
          if (gn < N) v.x = __ldg(p);
          if (gn + 1 < N) v.y = __ldg(p + 1);
          if (gn + 2 < N) v.z = __ldg(p + 2);
          if (gn + 3 < N) v.w = __ldg(p + 3);
        }
      }
      rb = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = tid / 4 + 64 * i, kq = (tid % 4) * 4;
      As[buf][kq + 0][row] = ra[i].x;
      As[buf][kq + 1][row] = ra[i].y;
      As[buf][kq + 2][row] = ra[i].z;
      As[buf][kq + 3][row] = ra[i].w;
    }
    const int kr = tid / 16, c4 = (tid % 16) * 4;
    *reinterpret_cast<float4*>(&Bs[buf][kr][c4]) = rb;
  };

  const int nk = (K + GBK - 1) / GBK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * GBK);
#pragma unroll
    for (int k = 0; k < GBK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // epilogue: + bias (folded BN / dense bias), + residual, activation
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + ty * 8 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j] + (bias ? __ldg(bias + gn) : 0.f);
      if (R) v += __ldg(R + (size_t)gm * N + gn);
      if (act == 1) v = fmaxf(v, 0.f);
      else if (act == 2) v = gelu_erf(v);
      else if (act == 3) v = tanhf(v);
      else if (act == 4) v = relu6f(v);
      else if (act == 5) v = siluf(v);
      else if (act == 6) v = sigmoidf(v);
      C[(size_t)gm * N + gn] = v;
    }
  }
}

static bool gemm_tc_enabled() {  // TFSC_GEMM_TC=0 forces the CUDA-core GEMM
  static int v = [] {
    const char* e = getenv("TFSC_GEMM_TC");
    return e ? atoi(e) : 1;
  }();
  return v != 0;
}

cudaError_t launch_gemm(const float* A, const float* B, const float* bias, const float* R, float* C, int M, int N, int K,
                        int lda, int act, cudaStream_t s) {
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (gemm_tc_enabled() && gemm_tc_supported(A, B, bias, R, C, M, N, K, lda))
    return launch_gemm_tc(A, B, bias, R, C, M, N, K, lda, act, s);
  dim3 grid((N + GBN - 1) / GBN, (M + GBM - 1) / GBM);
  const bool vec = (lda % 4 == 0) && (N % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
  if (vec) gemm_f32_kernel<true><<<grid, GTHREADS, 0, s>>>(A, B, bias, R, C, M, N, K, lda, act);
  else gemm_f32_kernel<false><<<grid, GTHREADS, 0, s>>>(A, B, bias, R, C, M, N, K, lda, act);
  g_launches_nn++;
  return cudaGetLastError();
}

// ----------------------------------------------------------------------------------- im2col ----
// col[(b*OH+oh)*OW+ow][(kh*KW+kw)*C + c] = x[b][oh*s-p+kh][ow*s-p+kw][c] (0 outside); row stride ldc >= KH*KW*C
__global__ void __launch_bounds__(256)
im2col_nhwc_kernel(const float* __restrict__ x, float* __restrict__ col, int Bn, int H, int W, int C, int KH, int KW,
                   int stride, int pad, int OH, int OW, int ldc) {
  const int64_t total = (int64_t)Bn * OH * OW * ldc;
  const int Kreal = KH * KW * C;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int kk = (int)(idx % ldc);
    const int64_t row = idx / ldc;
    float v = 0.f;
    if (kk < Kreal) {
      const int c = kk % C, kw = (kk / C) % KW, kh = kk / (C * KW);
      const int ow = (int)(row % OW), oh = (int)((row / OW) % OH), b = (int)(row / ((int64_t)OW * OH));
      const int ih = oh * stride - pad + kh, iw = ow * stride - pad + kw;
      if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(x + (((int64_t)b * H + ih) * W + iw) * C + c);
    }
    col[idx] = v;
  }
}

// Row-parallel version (round 2): a thread keeps its patch column kk = (kh, kw, c) for the whole kernel, so the 64-bit
// div / mod chain of the kernel above runs once per thread instead of once per element; blockDim.y rows per iteration, the
// row index decomposition is uniform per (block, y). Only convs that cannot take the implicit-GEMM path come here (the
// ResNet stem: C = 3 is not a TMA row) -- for it the patch row is 7 runs of 21 contiguous floats, written coalesced.
__global__ void __launch_bounds__(1024)
im2col_rows_kernel(const float* __restrict__ x, float* __restrict__ col, int Bn, int H, int W, int C, int KH, int KW,
                   int stride, int pad, int OH, int OW, int ldc) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // a tensor-core GEMM that follows may start its setup + weight prefetch now (it waits for this grid before touching activations)
  const int Kreal = KH * KW * C;
  const int64_t rows = (int64_t)Bn * OH * OW;
  for (int kk = threadIdx.x; kk < ldc; kk += blockDim.x) {
    const bool real = kk < Kreal;
    const int c = kk % C, kw = (kk / C) % KW, kh = kk / (C * KW);
    for (int64_t row = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; row < rows; row += (int64_t)gridDim.x * blockDim.y) {
      const int ow = (int)(row % OW);
      const int64_t t = row / OW;
      const int oh = (int)(t % OH), b = (int)(t / OH);
      const int ih = oh * stride - pad + kh, iw = ow * stride - pad + kw;
      float v = 0.f;
      if (real && ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(x + (((int64_t)b * H + ih) * W + iw) * C + c);
      col[row * ldc + kk] = v;
    }
  }
}

cudaError_t launch_im2col(const float* x, float* col, int Bn, int H, int W, int C, int KH, int KW, int stride, int pad,
                          int OH, int OW, int ldc, cudaStream_t s) {
  const int64_t rows = (int64_t)Bn * OH * OW;
  if (rows <= 0 || ldc <= 0) return cudaSuccess;
  const int bx = ldc >= 256 ? 256 : (ldc + 31) / 32 * 32;
  const int by = 1024 / bx >= 1 ? (1024 / bx > 8 ? 8 : 1024 / bx) : 1;
  int64_t blocks = (rows + by - 1) / by;
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  im2col_rows_kernel<<<(unsigned)blocks, dim3(bx, by), 0, s>>>(x, col, Bn, H, W, C, KH, KW, stride, pad, OH, OW, ldc);
  g_launches_nn++;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ pools ----
__global__ void __launch_bounds__(256)
maxpool_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int Bn, int H, int W, int C, int KH, int KW, int stride,
                    int pad, int OH, int OW) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // a tensor-core GEMM that follows may start its setup + weight prefetch now (it waits for this grid before touching activations)
  const int64_t total = (int64_t)Bn * OH * OW * C;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const int ow = (int)((idx / C) % OW), oh = (int)((idx / ((int64_t)C * OW)) % OH), b = (int)(idx / ((int64_t)C * OW * OH));
    float m = -FLT_MAX;
    for (int kh = 0; kh < KH; ++kh)
      for (int kw = 0; kw < KW; ++kw) {
        const int ih = oh * stride - pad + kh, iw = ow * stride - pad + kw;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) m = fmaxf(m, __ldg(x + (((int64_t)b * H + ih) * W + iw) * C + c));
      }
    y[idx] = m;
  }
}

cudaError_t launch_maxpool(const float* x, float* y, int Bn, int H, int W, int C, int KH, int KW, int stride, int pad, int OH,
                           int OW, cudaStream_t s) {
  const int64_t total = (int64_t)Bn * OH * OW * C;
  if (total <= 0) return cudaSuccess;
  int64_t blocks = (total + 255) / 256;
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  maxpool_nhwc_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, y, Bn, H, W, C, KH, KW, stride, pad, OH, OW);
  g_launches_nn++;
  return cudaGetLastError();
}

// y[b][c] = mean over H*W of x[b][h][w][c]; sequential fp32 sum per (b,c): deterministic
__global__ void __launch_bounds__(256)
avgpool_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int Bn, int HW, int C) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // a tensor-core GEMM that follows may start its setup + weight prefetch now (it waits for this grid before touching activations)
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Bn * C) return;
  const int c = idx % C, b = idx / C;
  const float* p = x + (size_t)b * HW * C + c;
  float s = 0.f;
  for (int i = 0; i < HW; ++i) s += __ldg(p + (size_t)i * C);
  y[idx] = s / (float)HW;
}

cudaError_t launch_avgpool(const float* x, float* y, int Bn, int HW, int C, cudaStream_t s) {
  if (Bn * C <= 0) return cudaSuccess;
  avgpool_nhwc_kernel<<<(Bn * C + 255) / 256, 256, 0, s>>>(x, y, Bn, HW, C);
  g_launches_nn++;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------- transformer blocks ----
// block-wide sum of (a, b) with 256 threads
__device__ __forceinline__ float2 block_sum2(float a, float b, float2* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sh[w] = make_float2(a, b);
  __syncthreads();
  float2 t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : make_float2(0.f, 0.f);
  if (w == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      t.x += __shfl_xor_sync(0xffffffffu, t.x, o);
      t.y += __shfl_xor_sync(0xffffffffu, t.y, o);
    }
    if (l == 0) sh[0] = t;
  }
  __syncthreads();
  t = sh[0];
  __syncthreads();
  return t;
}

// one CTA per token: y = LayerNorm(v) * gamma + beta, where v = x[token] (+ res[token]) or, for the embedding
// op, word[id] + pos[s] + type[t]. Token b*S + s reads its id at ids[b*stride + s] and its segment t at
// types[b*stride + s] (clamped to 0 / 1, as ids are clamped to the vocabulary); types == nullptr means segment 0.
// Two-pass mean / variance in fp32 (H <= 4096).
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ res, const int* __restrict__ ids,
                 const int* __restrict__ types, int stride, const float* __restrict__ word, const float* __restrict__ pos,
                 const float* __restrict__ type, const float* __restrict__ gamma, const float* __restrict__ beta,
                 float* __restrict__ y, int S, int H, int vocab, float eps) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // a tensor-core GEMM that follows may start its setup + weight prefetch now (it waits for this grid before touching activations)
  __shared__ float2 sh[8];
  extern __shared__ float row[];
  const int token = blockIdx.x;
  const float* xr = nullptr;
  const float* wr = nullptr;
  const float* tr = type;
  if (ids) {
    const size_t at = (size_t)(token / S) * stride + token % S;
    int id = __ldg(ids + at);
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    wr = word + (size_t)id * H;
    if (types && __ldg(types + at) > 0) tr = type + H;
  } else {
    xr = x + (size_t)token * H;
  }
  float s = 0.f;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float v;
    if (ids) v = __ldg(wr + h) + __ldg(pos + (size_t)(token % S) * H + h) + __ldg(tr + h);
    else v = __ldg(xr + h) + (res ? __ldg(res + (size_t)token * H + h) : 0.f);
    row[h] = v;
    s += v;
  }
  const float mean = block_sum2(s, 0.f, sh).x / (float)H;
  float q = 0.f;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    const float d = row[h] - mean;
    q += d * d;
  }
  const float var = block_sum2(q, 0.f, sh).x / (float)H;
  const float inv = rsqrtf(var + eps);
  for (int h = threadIdx.x; h < H; h += blockDim.x)
    y[(size_t)token * H + h] = (row[h] - mean) * inv * __ldg(gamma + h) + __ldg(beta + h);
}

cudaError_t launch_layernorm(const float* x, const float* res, const int* ids, const int* types, int stride, const float* word,
                             const float* pos, const float* type, const float* gamma, const float* beta, float* y, int tokens,
                             int S, int H, int vocab, float eps, cudaStream_t s) {
  if (tokens <= 0) return cudaSuccess;
  if (!layernorm_supported(H)) return cudaErrorInvalidValue;
  layernorm_kernel<<<tokens, 256, (size_t)H * sizeof(float), s>>>(x, res, ids, types, stride, word, pos, type, gamma, beta, y, S,
                                                                   H, vocab, eps);
  g_launches_nn++;
  return cudaGetLastError();
}

// Additive BERT mask of sequence b: key j gets -10000 when mask[b*mask_stride + j] == 0. The mask is the request's
// attention-mask input, or its token ids with mask_stride = S ([PAD] = 0) for bundles that declare no mask. When every
// key of the sequence is masked the same constant is added to every score and softmax is invariant to it, so no key is
// masked: adding -10000 in fp32 would round each score to a multiple of 2^-10 and shift the weights by up to 5e-4. Call
// from every thread of the CTA.
__device__ __forceinline__ bool attention_all_pad(const int* __restrict__ mask, int mask_stride, int b, int S) {
  int real = 0;
  if (mask)
    for (int j = threadIdx.x; j < S && !real; j += blockDim.x) real = __ldg(mask + (size_t)b * mask_stride + j) != 0;
  return mask && !__syncthreads_or(real);
}
__device__ __forceinline__ float attention_mask(const int* __restrict__ mask, int mask_stride, int b, int j, bool all_pad) {
  return (mask && !all_pad && __ldg(mask + (size_t)b * mask_stride + j) == 0) ? -10000.f : 0.f;
}

// Multi-head self-attention on a packed qkv buffer [B, S, 3H] (q | k | v), one CTA per (batch, head): K and V of
// the head are staged in shared memory, each warp owns query rows; softmax with warp shuffles; keys whose token
// id is 0 ([PAD]) get the BERT additive mask -10000. ctx[B, S, H]. Serves head widths the tiled kernels do not take
// (d % 4 != 0, d > 128) while S·(2d+10)+8d floats fit in shared memory.
__global__ void __launch_bounds__(256)
attention_kernel(const float* __restrict__ qkv, const int* __restrict__ mask, int mask_stride, float* __restrict__ ctx, int S, int H,
                 int heads) {
  extern __shared__ float sm[];
  const int d = H / heads;            // 64 for BERT-base
  const int b = blockIdx.x / heads, hd = blockIdx.x % heads;
  float* Ks = sm;                     // [S][d+1]
  float* Vs = Ks + (size_t)S * (d + 1);  // [S][d]
  float* Ps = Vs + (size_t)S * d;     // [8 warps][S]
  float* Qs = Ps + (size_t)8 * S;     // [8 warps][d]
  float* Ms = Qs + 8 * d;             // [S] additive mask
  const float* base = qkv + (size_t)b * S * 3 * H;
  for (int idx = threadIdx.x; idx < S * d; idx += blockDim.x) {
    const int j = idx / d, c = idx - j * d;
    Ks[j * (d + 1) + c] = __ldg(base + (size_t)j * 3 * H + H + hd * d + c);
    Vs[j * d + c] = __ldg(base + (size_t)j * 3 * H + 2 * H + hd * d + c);
  }
  const bool all_pad = attention_all_pad(mask, mask_stride, b, S);
  for (int j = threadIdx.x; j < S; j += blockDim.x) Ms[j] = attention_mask(mask, mask_stride, b, j, all_pad);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float scale = rsqrtf((float)d);
  float* P = Ps + warp * S;
  float* Q = Qs + warp * d;
  for (int i = warp; i < S; i += 8) {
    for (int c = lane; c < d; c += 32) Q[c] = __ldg(base + (size_t)i * 3 * H + hd * d + c);
    __syncwarp();
    float mx = -FLT_MAX;
    for (int j = lane; j < S; j += 32) {
      float sc = 0.f;
      const float* kr = Ks + j * (d + 1);
      for (int c = 0; c < d; ++c) sc = fmaf(Q[c], kr[c], sc);
      sc = sc * scale + Ms[j];
      P[j] = sc;
      mx = fmaxf(mx, sc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < S; j += 32) {
      const float e = expf(P[j] - mx);
      P[j] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    const float inv = 1.f / sum;
    for (int c = lane; c < d; c += 32) {
      float o = 0.f;
      for (int j = 0; j < S; ++j) o = fmaf(P[j], Vs[j * d + c], o);
      ctx[((size_t)b * S + i) * H + hd * d + c] = o * inv;
    }
    __syncwarp();
  }
}

// Register-tiled version (round 2): one CTA per (batch, head, block of 32 query rows), 4 warps x 8 rows. Scores: a lane owns
// keys lane, lane+32, ... (KPL per lane) and accumulates an 8 x KPL tile over d with 128-bit shared loads (K rows padded to
// d+4 floats: conflict-free LDS.128; q rows are broadcasts). Softmax in registers + warp shuffles; the unnormalised
// probabilities go through shared memory once for the P.V product (lane = two output dims). ~10x fewer shared-memory
// instructions per FMA than the row-at-a-time kernel above, and 4x the CTAs (BERT-base, 8 x 128: 384 CTAs, 2 per SM).
template <int KPL>
__global__ void __launch_bounds__(128)
attention_tile_kernel(const float* __restrict__ qkv, const int* __restrict__ mask, int mask_stride, float* __restrict__ ctx, int S,
                      int H, int heads) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // a tensor-core GEMM that follows may start its setup + weight prefetch now (it waits for this grid before touching activations)
  extern __shared__ __align__(16) float sm[];
  constexpr int SP = 32 * KPL;           // padded key count
  const int d = H / heads, ds = d + 4;   // d % 4 == 0
  const int b = blockIdx.y / heads, hd = blockIdx.y % heads, q0 = blockIdx.x * 32;
  float* Ks = sm;                        // [SP][ds]
  float* Vs = Ks + (size_t)SP * ds;      // [SP][d]
  float* Qs = Vs + (size_t)SP * d;       // [32][d]
  float* Ps = Qs + 32 * d;               // [32][SP]
  float* Ms = Ps + 32 * SP;              // [SP] additive mask (-FLT_MAX beyond S)
  const float* base = qkv + (size_t)b * S * 3 * H;
  const int d4 = d >> 2;
  for (int idx = threadIdx.x; idx < SP * d4; idx += 128) {
    const int j = idx / d4, c = (idx - j * d4) << 2;
    float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
    if (j < S) {
      kv = __ldg(reinterpret_cast<const float4*>(base + (size_t)j * 3 * H + H + hd * d + c));
      vv = __ldg(reinterpret_cast<const float4*>(base + (size_t)j * 3 * H + 2 * H + hd * d + c));
    }
    *reinterpret_cast<float4*>(Ks + (size_t)j * ds + c) = kv;
    *reinterpret_cast<float4*>(Vs + (size_t)j * d + c) = vv;
  }
  for (int idx = threadIdx.x; idx < 32 * d4; idx += 128) {
    const int r = idx / d4, c = (idx - r * d4) << 2;
    float4 qv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < S) qv = __ldg(reinterpret_cast<const float4*>(base + (size_t)(q0 + r) * 3 * H + hd * d + c));
    *reinterpret_cast<float4*>(Qs + r * d + c) = qv;
  }
  const bool all_pad = attention_all_pad(mask, mask_stride, b, S);
  for (int j = threadIdx.x; j < SP; j += 128) Ms[j] = j >= S ? -FLT_MAX : attention_mask(mask, mask_stride, b, j, all_pad);
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 8;
  float sc[8][KPL];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int t = 0; t < KPL; ++t) sc[r][t] = 0.f;
  for (int c = 0; c < d; c += 4) {
    float4 kq[KPL];
#pragma unroll
    for (int t = 0; t < KPL; ++t) kq[t] = *reinterpret_cast<const float4*>(Ks + (size_t)(lane + 32 * t) * ds + c);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const float4 qv = *reinterpret_cast<const float4*>(Qs + (r0 + r) * d + c);
#pragma unroll
      for (int t = 0; t < KPL; ++t)
        sc[r][t] = fmaf(qv.x, kq[t].x, fmaf(qv.y, kq[t].y, fmaf(qv.z, kq[t].z, fmaf(qv.w, kq[t].w, sc[r][t]))));
    }
  }
  const float scale = rsqrtf((float)d);
  float inv[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    float mx = -FLT_MAX;
#pragma unroll
    for (int t = 0; t < KPL; ++t) {
      const float m = Ms[lane + 32 * t];
      sc[r][t] = m == -FLT_MAX ? -FLT_MAX : sc[r][t] * scale + m;
      mx = fmaxf(mx, sc[r][t]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < KPL; ++t) {
      const float e = sc[r][t] == -FLT_MAX ? 0.f : expf(sc[r][t] - mx);
      Ps[(r0 + r) * SP + lane + 32 * t] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    inv[r] = 1.f / sum;
  }
  __syncwarp();  // a warp only reads the 8 rows of P it wrote
  const int S4 = (S + 3) & ~3;   // V rows and P columns in [S, S4) are zeros
  for (int dd = lane * 2; dd < d; dd += 64) {
    float2 acc[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r] = make_float2(0.f, 0.f);
    for (int j = 0; j < S4; j += 4) {
      float2 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float2*>(Vs + (size_t)(j + u) * d + dd);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float4 p = *reinterpret_cast<const float4*>(Ps + (r0 + r) * SP + j);
        acc[r].x = fmaf(p.x, v[0].x, fmaf(p.y, v[1].x, fmaf(p.z, v[2].x, fmaf(p.w, v[3].x, acc[r].x))));
        acc[r].y = fmaf(p.x, v[0].y, fmaf(p.y, v[1].y, fmaf(p.z, v[2].y, fmaf(p.w, v[3].y, acc[r].y))));
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (q0 + r0 + r < S)
        *reinterpret_cast<float2*>(ctx + ((size_t)b * S + q0 + r0 + r) * H + hd * d + dd) = make_float2(acc[r].x * inv[r], acc[r].y * inv[r]);
  }
}

// Key-block version for S > 256: the same CTA shape and score / P.V loops as attention_tile_kernel<2>, but K and V pass
// through shared memory 64 keys at a time, so shared memory does not grow with S. Online softmax (Milakov & Gimelshein
// 2018): each row keeps a running max m and its lanes partial sums l; when a block raises m, l and the P.V accumulators
// are rescaled by exp(m_old - m_new). A lane owns output dims lane*2 and 64 + lane*2 (d <= 128, d % 4 == 0).
constexpr int kAttnKeyBlock = 64;
__global__ void __launch_bounds__(128)
attention_keyblock_kernel(const float* __restrict__ qkv, const int* __restrict__ mask, int mask_stride, float* __restrict__ ctx,
                          int S, int H, int heads) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // a tensor-core GEMM that follows may start its setup + weight prefetch now (it waits for this grid before touching activations)
  extern __shared__ __align__(16) float sm[];
  constexpr int KB = kAttnKeyBlock;
  const int d = H / heads, ds = d + 4;
  const int b = blockIdx.y / heads, hd = blockIdx.y % heads, q0 = blockIdx.x * 32;
  float* Ks = sm;                        // [KB][ds]
  float* Vs = Ks + (size_t)KB * ds;      // [KB][d]
  float* Qs = Vs + (size_t)KB * d;       // [32][d]
  float* Ps = Qs + 32 * d;               // [32][KB]
  float* Ms = Ps + 32 * KB;              // [KB] additive mask (-FLT_MAX beyond S)
  const float* base = qkv + (size_t)b * S * 3 * H;
  const int d4 = d >> 2;
  for (int idx = threadIdx.x; idx < 32 * d4; idx += 128) {
    const int r = idx / d4, c = (idx - r * d4) << 2;
    float4 qv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < S) qv = __ldg(reinterpret_cast<const float4*>(base + (size_t)(q0 + r) * 3 * H + hd * d + c));
    *reinterpret_cast<float4*>(Qs + r * d + c) = qv;
  }
  const bool all_pad = attention_all_pad(mask, mask_stride, b, S);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 8;
  const float scale = rsqrtf((float)d);
  float mrow[8], lsum[8];
  float2 acc[2][8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    mrow[r] = -FLT_MAX;
    lsum[r] = 0.f;
    acc[0][r] = acc[1][r] = make_float2(0.f, 0.f);
  }
  for (int j0 = 0; j0 < S; j0 += KB) {
    __syncthreads();  // the previous block's K / V / mask are no longer read
    for (int idx = threadIdx.x; idx < KB * d4; idx += 128) {
      const int j = idx / d4, c = (idx - j * d4) << 2;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (j0 + j < S) {
        kv = __ldg(reinterpret_cast<const float4*>(base + (size_t)(j0 + j) * 3 * H + H + hd * d + c));
        vv = __ldg(reinterpret_cast<const float4*>(base + (size_t)(j0 + j) * 3 * H + 2 * H + hd * d + c));
      }
      *reinterpret_cast<float4*>(Ks + (size_t)j * ds + c) = kv;
      *reinterpret_cast<float4*>(Vs + (size_t)j * d + c) = vv;
    }
    for (int j = threadIdx.x; j < KB; j += 128) Ms[j] = j0 + j >= S ? -FLT_MAX : attention_mask(mask, mask_stride, b, j0 + j, all_pad);
    __syncthreads();

    float sc[8][2];
#pragma unroll
    for (int r = 0; r < 8; ++r) sc[r][0] = sc[r][1] = 0.f;
    for (int c = 0; c < d; c += 4) {
      float4 kq[2];
#pragma unroll
      for (int t = 0; t < 2; ++t) kq[t] = *reinterpret_cast<const float4*>(Ks + (size_t)(lane + 32 * t) * ds + c);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float4 qv = *reinterpret_cast<const float4*>(Qs + (r0 + r) * d + c);
#pragma unroll
        for (int t = 0; t < 2; ++t)
          sc[r][t] = fmaf(qv.x, kq[t].x, fmaf(qv.y, kq[t].y, fmaf(qv.z, kq[t].z, fmaf(qv.w, kq[t].w, sc[r][t]))));
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      float mx = mrow[r];
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const float m = Ms[lane + 32 * t];
        sc[r][t] = m == -FLT_MAX ? -FLT_MAX : sc[r][t] * scale + m;
        mx = fmaxf(mx, sc[r][t]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      // every block holds at least one key < S, so mx is finite from the first block on
      const float alpha = mrow[r] == -FLT_MAX ? 0.f : expf(mrow[r] - mx);
      mrow[r] = mx;
      float part = 0.f;
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const float e = sc[r][t] == -FLT_MAX ? 0.f : expf(sc[r][t] - mx);
        Ps[(r0 + r) * KB + lane + 32 * t] = e;
        part += e;
      }
      lsum[r] = fmaf(lsum[r], alpha, part);
      acc[0][r].x *= alpha;
      acc[0][r].y *= alpha;
      acc[1][r].x *= alpha;
      acc[1][r].y *= alpha;
    }
    __syncwarp();  // a warp only reads the 8 rows of P it wrote
    const int n4 = (min(KB, S - j0) + 3) & ~3;  // V rows and P columns in [S - j0, n4) are zeros
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int dd = lane * 2 + 64 * h;
      if (dd >= d) break;
      for (int j = 0; j < n4; j += 4) {
        float2 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float2*>(Vs + (size_t)(j + u) * d + dd);
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const float4 p = *reinterpret_cast<const float4*>(Ps + (r0 + r) * KB + j);
          acc[h][r].x = fmaf(p.x, v[0].x, fmaf(p.y, v[1].x, fmaf(p.z, v[2].x, fmaf(p.w, v[3].x, acc[h][r].x))));
          acc[h][r].y = fmaf(p.x, v[0].y, fmaf(p.y, v[1].y, fmaf(p.z, v[2].y, fmaf(p.w, v[3].y, acc[h][r].y))));
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    float l = lsum[r];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    const float inv = 1.f / l;
    if (q0 + r0 + r >= S) continue;
    float* out = ctx + ((size_t)b * S + q0 + r0 + r) * H + hd * d;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int dd = lane * 2 + 64 * h;
      if (dd < d) *reinterpret_cast<float2*>(out + dd) = make_float2(acc[h][r].x * inv, acc[h][r].y * inv);
    }
  }
}

static size_t attention_tile_smem(int S, int d, int kpl) {
  const size_t sp = 32 * (size_t)kpl;
  (void)S;
  return (sp * (d + 4) + sp * d + 32 * (size_t)d + 32 * sp + sp) * sizeof(float);
}

static size_t attention_keyblock_smem(int d) {
  const size_t kb = kAttnKeyBlock;
  return (kb * (d + 4) + kb * d + 32 * (size_t)d + 32 * kb + kb) * sizeof(float);
}


template <int KPL>
static cudaError_t launch_attention_tile(const float* qkv, const int* mask, int mask_stride, float* ctx, int Bn, int S, int H, int heads,
                                         cudaStream_t s) {
  const size_t smem = attention_tile_smem(S, H / heads, KPL);
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(attention_tile_kernel<KPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttnSmemCap);
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  attention_tile_kernel<KPL><<<dim3((S + 31) / 32, Bn * heads), 128, smem, s>>>(qkv, mask, mask_stride, ctx, S, H, heads);
  g_launches_nn++;
  return cudaGetLastError();
}

static cudaError_t launch_attention_keyblock(const float* qkv, const int* mask, int mask_stride, float* ctx, int Bn, int S, int H,
                                             int heads, cudaStream_t s) {
  const size_t smem = attention_keyblock_smem(H / heads);
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(attention_keyblock_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)attention_keyblock_smem(128));
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  attention_keyblock_kernel<<<dim3((S + 31) / 32, Bn * heads), 128, smem, s>>>(qkv, mask, mask_stride, ctx, S, H, heads);
  g_launches_nn++;
  return cudaGetLastError();
}

cudaError_t launch_attention(const float* qkv, const int* mask, int mask_stride, float* ctx, int Bn, int S, int H, int heads,
                             cudaStream_t s) {
  if (Bn <= 0) return cudaSuccess;
  const bool al = ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(ctx)) & 15) == 0;
  if (!attention_supported(S, H, heads, al)) return cudaErrorInvalidValue;
  const int d = H / heads;
  if (d % 4 == 0 && H % 4 == 0 && al && d <= 128) {
    const int kpl = (S + 31) / 32;
    if (kpl <= 1 && attention_tile_smem(S, d, 1) <= kAttnSmemCap) return launch_attention_tile<1>(qkv, mask, mask_stride, ctx, Bn, S, H, heads, s);
    if (kpl <= 2 && attention_tile_smem(S, d, 2) <= kAttnSmemCap) return launch_attention_tile<2>(qkv, mask, mask_stride, ctx, Bn, S, H, heads, s);
    if (kpl <= 4 && attention_tile_smem(S, d, 4) <= kAttnSmemCap) return launch_attention_tile<4>(qkv, mask, mask_stride, ctx, Bn, S, H, heads, s);
    if (kpl <= 8 && attention_tile_smem(S, d, 8) <= kAttnSmemCap) return launch_attention_tile<8>(qkv, mask, mask_stride, ctx, Bn, S, H, heads, s);
    return launch_attention_keyblock(qkv, mask, mask_stride, ctx, Bn, S, H, heads, s);
  }
  const size_t smem = attention_smem_bytes(S, H, heads);
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttnSmemCap);
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  attention_kernel<<<Bn * heads, 256, smem, s>>>(qkv, mask, mask_stride, ctx, S, H, heads);
  g_launches_nn++;
  return cudaGetLastError();
}


// ------------------------------------------------------------------------------ X6 / X7 ----
constexpr int kCopySegMax = 64;
struct CopySegTable {
  const char* src[kCopySegMax];
  char* dst[kCopySegMax];
  unsigned long long bytes[kCopySegMax];
};

// grid = (chunks, segments). 16-byte vectors when source, destination and length allow it, 4-byte words otherwise (request
// tensors are fp32 / int32, so lengths are multiples of 4; staging buffers and window slots are 256-byte aligned).
__global__ void __launch_bounds__(256) copy_segments_kernel(const __grid_constant__ CopySegTable tab) {
  const int sg = blockIdx.y;
  const char* __restrict__ src = tab.src[sg];
  char* __restrict__ dst = tab.dst[sg];
  const unsigned long long bytes = tab.bytes[sg];
  const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long nthr = (unsigned long long)gridDim.x * blockDim.x;
  if ((((unsigned long long)src | (unsigned long long)dst | bytes) & 15ull) == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    const unsigned long long n = bytes >> 4;
    for (unsigned long long i = tid; i < n; i += nthr) d4[i] = s4[i];
  } else if ((((unsigned long long)src | (unsigned long long)dst | bytes) & 3ull) == 0) {
    const unsigned int* s1 = reinterpret_cast<const unsigned int*>(src);
    unsigned int* d1 = reinterpret_cast<unsigned int*>(dst);
    const unsigned long long n = bytes >> 2;
    for (unsigned long long i = tid; i < n; i += nthr) d1[i] = s1[i];
  } else {
    for (unsigned long long i = tid; i < bytes; i += nthr) dst[i] = src[i];
  }
}

cudaError_t launch_copy_segments(const CopySeg* segs, int n, cudaStream_t s) {
  for (int base = 0; base < n; base += kCopySegMax) {
    const int m = n - base < kCopySegMax ? n - base : kCopySegMax;
    CopySegTable tab;
    unsigned long long mx = 0;
    for (int i = 0; i < m; ++i) {
      tab.src[i] = static_cast<const char*>(segs[base + i].src);
      tab.dst[i] = static_cast<char*>(segs[base + i].dst);
      tab.bytes[i] = segs[base + i].bytes;
      if (segs[base + i].bytes > mx) mx = segs[base + i].bytes;
    }
    if (mx == 0) continue;
    // 16 KB per block keeps ~64 independent 16-byte requests per thread-block wave in flight (PCIe / NVLink latency);
    // few blocks, no shared memory: the kernel co-resides with the weight-streaming kernels (1 CTA per SM, 544 threads)
    unsigned long long chunks = (mx + 16383) / 16384;
    if (chunks > 32) chunks = 32;
    if (chunks < 1) chunks = 1;
    copy_segments_kernel<<<dim3((unsigned)chunks, (unsigned)m), 256, 0, s>>>(tab);
    g_launches_nn++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace tfsc
