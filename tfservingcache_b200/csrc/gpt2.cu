// GPT-2 kernels of the graph executor, fp32, sm_90a: the embedding without LayerNorm (wte + wpe) and the gather of each
// row's last attended token, the one position a next-token prediction is made from. Causal attention is a flag of the
// tiled and key-block attention kernels (nn_kernels.cu), and the next-token head is the fill-mask head's kernel with one
// slot per row (mlm.cu).
//
// embed_positions_kernel: y[t, :] = word[clamp(id)] + pos[s], one fp32 add per value, 16-byte vectors (a scalar path for
// H % 4 != 0 or misaligned tables). A separate kernel, not a branch of layernorm_kernel, so BERT's embedding is unchanged.
//
// last_token_kernel: one CTA per row. A block-wide max over the mask finds the last attended position p (S - 1 without a
// mask, -1 for a row with none), then the CTA copies the H floats of token p (zeros for p = -1): a copy, so the bits are
// exact. A scalar path covers layouts that are not 16-byte aligned.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdlib>

#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kEmbedThreads = 256, kLastTokenThreads = 256;

static bool pdl_on() {  // programmatic dependent launch, on unless TFSC_PDL=0, as the heads
  static const bool v = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  return v;
}

template <bool kVec>
__global__ void __launch_bounds__(kEmbedThreads) embed_positions_kernel(const int* __restrict__ ids, int64_t stride,
                                                                        const float* __restrict__ word, const float* __restrict__ pos,
                                                                        float* __restrict__ y, int64_t tokens, int S, int H,
                                                                        int vocab) {
  // the ln_1 LayerNorm that follows does not wait on this grid, so it starts after it as usual
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int Q = kVec ? H >> 2 : H;  // float4s (or floats) per token
  const int64_t n = tokens * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / Q;
    const int q = (int)(i - t * Q);
    const int s = (int)(t % S);
    int id = __ldg(ids + (t / S) * stride + s);
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    if (kVec) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(word + (int64_t)id * H) + q);
      const float4 p = __ldg(reinterpret_cast<const float4*>(pos + (int64_t)s * H) + q);
      reinterpret_cast<float4*>(y + t * H)[q] = make_float4(w.x + p.x, w.y + p.y, w.z + p.z, w.w + p.w);
    } else {
      y[t * H + q] = __ldg(word + (int64_t)id * H + q) + __ldg(pos + (int64_t)s * H + q);
    }
  }
}

cudaError_t launch_embed_positions(const int* ids, int64_t stride, const float* word, const float* pos, float* y, int rows, int S,
                                   int H, int vocab, cudaStream_t s) {
  if (rows < 0 || S < 1 || H < 1 || vocab < 1 || stride < S || !ids || !word || !pos || !y) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  const bool vec = H % 4 == 0 && (((uintptr_t)word | (uintptr_t)pos | (uintptr_t)y) & 15) == 0;
  const int64_t tokens = (int64_t)rows * S, n = tokens * (vec ? H / 4 : H);
  int64_t blocks = (n + kEmbedThreads - 1) / kEmbedThreads;
  if (blocks > (int64_t)device_sm_count() * 8) blocks = (int64_t)device_sm_count() * 8;
  if (vec) embed_positions_kernel<true><<<(unsigned)blocks, kEmbedThreads, 0, s>>>(ids, stride, word, pos, y, tokens, S, H, vocab);
  else embed_positions_kernel<false><<<(unsigned)blocks, kEmbedThreads, 0, s>>>(ids, stride, word, pos, y, tokens, S, H, vocab);
  g_launches_nn++;
  return cudaGetLastError();
}

template <bool kVec>
__global__ void __launch_bounds__(kLastTokenThreads) last_token_kernel(const float* __restrict__ hidden, const int* __restrict__ mask,
                                                                       int64_t stride, int S, int H, int* __restrict__ positions,
                                                                       float* __restrict__ gathered) {
  __shared__ int wmax[kLastTokenThreads / 32];
  const int64_t row = blockIdx.x;
  // launched after the op that writes the hidden states, which are that grid's output
  asm volatile("griddepcontrol.wait;" ::: "memory");
  int p = S - 1;
  if (mask) {
    p = -1;
    const int* m = mask + row * stride;
    for (int j = threadIdx.x; j < S; j += blockDim.x)  // ascending j: the last hit is this thread's largest
      if (__ldg(m + j) != 0) p = j;
    p = __reduce_max_sync(0xffffffffu, p);
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = p;
    __syncthreads();
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) p = max(p, wmax[w]);
  }
  if (positions && threadIdx.x == 0) positions[row] = p;
  if (!gathered) return;
  if (kVec) {
    const int Q = H >> 2;
    const float4* src = reinterpret_cast<const float4*>(hidden + (row * S + (p < 0 ? 0 : p)) * H);
    float4* dst = reinterpret_cast<float4*>(gathered + row * H);
    for (int q = threadIdx.x; q < Q; q += blockDim.x) dst[q] = p >= 0 ? __ldg(src + q) : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    const float* src = hidden + (row * S + (p < 0 ? 0 : p)) * H;
    float* dst = gathered + row * H;
    for (int c = threadIdx.x; c < H; c += blockDim.x) dst[c] = p >= 0 ? __ldg(src + c) : 0.f;
  }
}

cudaError_t launch_last_token(const float* hidden, const int* mask, int64_t stride, int rows, int S, int H, int* positions,
                              float* gathered, cudaStream_t s) {
  if (rows < 0 || S < 1 || H < 1 || (mask && stride < S) || (gathered && !hidden)) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  const bool vec = H % 4 == 0 && (((uintptr_t)hidden | (uintptr_t)gathered) & 15) == 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)rows);
  cfg.blockDim = dim3(kLastTokenThreads);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_on() ? 1 : 0;
  cudaError_t e = vec ? cudaLaunchKernelEx(&cfg, last_token_kernel<true>, hidden, mask, stride, S, H, positions, gathered)
                      : cudaLaunchKernelEx(&cfg, last_token_kernel<false>, hidden, mask, stride, S, H, positions, gathered);
  g_launches_nn++;
  return e;
}

}  // namespace tfsc
