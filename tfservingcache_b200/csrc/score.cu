// Scoring kernels of GPT-2 score bundles, fp32, sm_90a: the log-probability and rank of every input token under the logits
// of the attended position before it, and the head that writes a row's outputs.
//
// token_score_kernel: one CTA per token row of a chunk of the vocabulary projection. A row whose position p is masked, or is
// its row's last attended position, predicts nothing and exits. Otherwise the CTA finds s = next(p), stages the row's vocab
// logits and takes its maximum and fp64 exponential sum with the select step's helpers and block size (head_select.cuh), so
// the log-probability has the bits generate_select_kernel writes for the same row; the rank is an integer block count. It
// writes slot s of the [rows, S] log-probabilities and ranks: every scored slot has exactly one writer, and no
// floating-point atomics are used. Once the row is staged the CTA reads no more logits, so it lets the next chunk's
// projection launch (programmatic dependent launch), which overwrites the region only after its griddepcontrol.wait.
//
// score_head_kernel: one CTA per row walks the S positions, copies the scored slots and writes the defaults elsewhere, and
// sums the scored log-probabilities in fp64 in an order fixed by S and the block size.
#include <cuda_runtime.h>

#include <atomic>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>

#include "head_select.cuh"
#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kScoreHeadThreads = 256;

static bool pdl_on() {  // programmatic dependent launch, on unless TFSC_PDL=0, as the generate steps
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

// the smallest position j in [from, S) with mask[j] != 0 (mask nullptr: from), S for none; every thread gets it
__device__ __forceinline__ int first_attended(const int* __restrict__ mask, int from, int S, int* s_min) {
  if (!mask) return from < S ? from : S;
  if (threadIdx.x == 0) *s_min = S;
  __syncthreads();
  for (int j = from + threadIdx.x; j < S; j += blockDim.x)
    if (!mask || __ldg(mask + j) != 0) {
      atomicMin(s_min, j);
      break;
    }
  __syncthreads();
  return *s_min;
}

__global__ void __launch_bounds__(kHeadThreadsMax) token_score_kernel(const float* __restrict__ logits, int64_t ld, int64_t first,
                                                                      const int* __restrict__ ids, const int* __restrict__ mask,
                                                                      int64_t stride, int S, int vocab, float* __restrict__ log_probs,
                                                                      int* __restrict__ ranks) {
  extern __shared__ float xs[];  // the row's vocab logits
  __shared__ float wv[kHeadThreadsMax / 32];
  __shared__ int wi[kHeadThreadsMax / 32];
  __shared__ double wsum[kHeadThreadsMax / 32];
  __shared__ int wcount[kHeadThreadsMax / 32];
  __shared__ float s_v;
  __shared__ int s_i, s_next;
  __shared__ double s_sum;
  __shared__ int sel[1];
  // launched after the projection that wrote this chunk's logits
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int64_t g = first + blockIdx.x, r = g / S;
  const int p = (int)(g - r * S);
  const int* mrow = mask ? mask + r * stride : nullptr;
  if (mrow && __ldg(mrow + p) == 0) return;  // a masked position predicts nothing
  const int s = first_attended(mrow, p + 1, S, &s_next);
  if (s >= S) return;  // the row's last attended position
  const int t = min(max(__ldg(ids + r * stride + s), 0), vocab - 1);
  const float m = head_stage_select(logits + (int64_t)blockIdx.x * ld, vocab, 1, xs, wv, wi, &s_v, &s_i, sel);
  // the row is staged: the next chunk's projection may start and overwrite the logits region
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const double sum = head_exp_sum(xs, vocab, m, wsum, &s_sum);
  const float zt = xs[t];
  int c = 0;
  for (int j = threadIdx.x; j < vocab; j += blockDim.x) {
    const float v = xs[j];
    c += v > zt || (v == zt && j < t);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) wcount[warp] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int rank = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) rank += wcount[w];
    log_probs[r * S + s] = (zt - m) - (float)log(sum);
    ranks[r * S + s] = rank;
  }
}

cudaError_t launch_token_score(const float* logits, int64_t ld, int64_t first, int n, const int* ids, const int* mask,
                               int64_t stride, int S, int vocab, float* log_probs, int* ranks, cudaStream_t s) {
  if (n < 0 || first < 0 || !score_supported(S, vocab) || ld < vocab || stride < S) return cudaErrorInvalidValue;
  if (n == 0) return cudaSuccess;
  if (!logits || !ids || !log_probs || !ranks) return cudaErrorInvalidValue;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(token_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kNextTokenMaxVocab * (int)sizeof(float));
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  // the select step's block size for the same vocabulary: its maximum and sum run in the same order
  return launch_pdl(token_score_kernel, dim3((unsigned)n), head_threads(vocab), (size_t)vocab * sizeof(float), s, logits, ld, first,
                    ids, mask, stride, S, vocab, log_probs, ranks);
}

__global__ void __launch_bounds__(kScoreHeadThreads) score_head_kernel(const float* __restrict__ log_probs,
                                                                       const int* __restrict__ ranks, const int* __restrict__ mask,
                                                                       int64_t stride, int S, ScoreOutputs o) {
  __shared__ double wsum[kScoreHeadThreads / 32];
  __shared__ int wcount[kScoreHeadThreads / 32];
  __shared__ int s_first;
  // launched after the last chunk's score kernel
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int64_t r = blockIdx.x;
  const int* mrow = mask ? mask + r * stride : nullptr;
  const int a0 = first_attended(mrow, 0, S, &s_first);  // the first attended position predicts, it is not scored
  double acc = 0.0;
  int c = 0;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const bool scored = s > a0 && (!mrow || __ldg(mrow + s) != 0);
    const float v = scored ? log_probs[r * S + s] : 0.f;
    if (o.log_probs) o.log_probs[r * o.log_probs_ld + s] = v;
    if (o.ranks) o.ranks[r * o.ranks_ld + s] = scored ? ranks[r * S + s] : -1;
    acc += (double)v;
    c += scored;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, off);
    c += __shfl_xor_sync(0xffffffffu, c, off);
  }
  if (lane == 0) {
    wsum[warp] = acc;
    wcount[warp] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double total = 0.0;
    int count = 0;
    for (int w = 0; w < kScoreHeadThreads / 32; ++w) total += wsum[w], count += wcount[w];
    if (o.sum) o.sum[r * o.sum_ld] = (float)total;
    if (o.count) o.count[r * o.count_ld] = count;
  }
}

cudaError_t launch_score_head(const float* log_probs, const int* ranks, const int* mask, int64_t stride, int rows, int S,
                              const ScoreOutputs& o, cudaStream_t s) {
  if (rows < 0 || S < 1 || S > kScoreMaxS || stride < S) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  if ((o.log_probs && !log_probs) || (o.ranks && !ranks) || (o.sum && !log_probs)) return cudaErrorInvalidValue;
  return launch_pdl(score_head_kernel, dim3((unsigned)rows), kScoreHeadThreads, 0, s, log_probs, ranks, mask, stride, S, o);
}

}  // namespace tfsc
