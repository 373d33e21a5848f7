// Classification head of multi-output bundles (signature.outputs), fp32, sm_90a: one launch turns a batch of logits rows
// into every declared output -- a copy of the logits, softmax probabilities, the argmax class and the top k classes with
// their probabilities -- written at their offsets inside the packed response row.
//
// Layout: one CTA per row. A row of N <= 32768 logits is staged once in shared memory (128 KB at the limit), so the
// softmax passes and the selection never touch HBM again. Selection is k rounds of a block-wide argmax over (value
// descending, index ascending): every thread keeps the best of its own elements (strided j = t, t + T, ...) that ranks
// below the last selected one, a warp-shuffle + shared-memory reduction picks the round's winner, and only the thread
// that owned it rescans its elements. Rounds are exact comparisons on the fp32 logits, so the indices are those of
// tf.math.top_k / a stable argsort, ties to the lower index. Rows are independent, so one CTA each fills the SMs from
// about 132 rows on. Timings are in DESIGN §4.
#include <cuda_runtime.h>

#include <atomic>
#include <climits>
#include <cmath>
#include <cstdlib>

#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kHeadThreadsMax = 512;

__device__ __forceinline__ bool ranks_above(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

__device__ __forceinline__ void warp_best(float& v, int& i) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ranks_above(ov, oi, v, i)) {
      v = ov;
      i = oi;
    }
  }
}

// this thread's best element that ranks below (lv, li); (-inf, INT_MAX) when it has none left
__device__ __forceinline__ void local_best(const float* xs, int n, float lv, int li, float* bv, int* bi) {
  float v0 = -INFINITY;
  int i0 = INT_MAX;
#pragma unroll 4
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float v = xs[j];
    if (ranks_above(lv, li, v, j) && ranks_above(v, j, v0, i0)) {
      v0 = v;
      i0 = j;
    }
  }
  *bv = v0;
  *bi = i0;
}

// one expression for both probability outputs, so top_k_probabilities are the same bits as probabilities[index]
__device__ __forceinline__ float softmax_at(float x, float m, float inv) { return expf(x - m) * inv; }

__global__ void __launch_bounds__(kHeadThreadsMax) classify_head_kernel(const float* __restrict__ logits, int n, int rounds,
                                                                        HeadOutputs o) {
  extern __shared__ float xs[];  // the row's n logits
  __shared__ float wv[kHeadThreadsMax / 32];
  __shared__ int wi[kHeadThreadsMax / 32];
  __shared__ double wsum[kHeadThreadsMax / 32];
  __shared__ float s_v;
  __shared__ int s_i;
  __shared__ double s_sum;
  __shared__ int sel[kHeadMaxK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t row = blockIdx.x;
  // launched after a PDL dense kernel, the logits are that grid's output (a no-op without the launch attribute)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const float* x = logits + row * n;
  // eight independent loads in flight per thread: a 30522-wide row is 60 loads per thread, which one at a time would
  // cost 60 round trips to HBM
  const int T = blockDim.x;
  int j0 = threadIdx.x;
  for (; j0 + 7 * T < n; j0 += 8 * T) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldg(x + j0 + u * T);
#pragma unroll
    for (int u = 0; u < 8; ++u) xs[j0 + u * T] = v[u];
  }
  for (; j0 < n; j0 += T) xs[j0] = __ldg(x + j0);
  __syncthreads();

  float bv;
  int bi;
  local_best(xs, n, INFINITY, -1, &bv, &bi);
  float m = 0.f;
  for (int r = 0; r < rounds; ++r) {
    float v = bv;
    int i = bi;
    warp_best(v, i);
    if (lane == 0) {
      wv[warp] = v;
      wi[warp] = i;
    }
    __syncthreads();
    if (warp == 0) {
      v = lane < nwarps ? wv[lane] : -INFINITY;
      i = lane < nwarps ? wi[lane] : INT_MAX;
      warp_best(v, i);
      if (lane == 0) {
        s_v = v;
        s_i = i;
        sel[r] = i;
      }
    }
    __syncthreads();
    const float gv = s_v;
    const int gi = s_i;
    if (r == 0) m = gv;  // the row maximum
    if (bi == gi) local_best(xs, n, gv, gi, &bv, &bi);
  }

  // softmax: max-subtracted fp32 exponentials, summed in fp64 (a 32768-wide row keeps its sum to ~1 ulp of fp32)
  const bool need_sum = o.probs || o.topk_prob;
  float inv = 0.f;
  if (need_sum) {
    double acc = 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) acc += (double)expf(xs[j] - m);
#pragma unroll
    for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) wsum[warp] = acc;
    __syncthreads();
    if (warp == 0) {
      double a = lane < nwarps ? wsum[lane] : 0.0;
#pragma unroll
      for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
      if (lane == 0) s_sum = a;
    }
    __syncthreads();
    inv = (float)(1.0 / s_sum);
  }
  if (o.logits) {
    float* y = o.logits + row * o.logits_ld;
    for (int j = threadIdx.x; j < n; j += blockDim.x) y[j] = xs[j];
  }
  if (o.probs) {
    float* y = o.probs + row * o.probs_ld;
    for (int j = threadIdx.x; j < n; j += blockDim.x) y[j] = softmax_at(xs[j], m, inv);
  }
  if (o.classes && threadIdx.x < 2) o.classes[row * o.classes_ld + threadIdx.x] = threadIdx.x == 0 ? sel[0] : 0;  // int64 LE
  if ((int)threadIdx.x < rounds) {
    const int j = sel[threadIdx.x];
    if (o.topk_idx) o.topk_idx[row * o.topk_idx_ld + threadIdx.x] = j;
    // j < n for finite logits; a NaN row can leave the sentinel INT_MAX, which must not index shared memory
    if (o.topk_prob) o.topk_prob[row * o.topk_prob_ld + threadIdx.x] = softmax_at(xs[j < n ? j : n - 1], m, inv);
  }
}

cudaError_t launch_classify_head(const float* logits, int rows, int n, int k, const HeadOutputs& o, cudaStream_t s) {
  const bool topk = o.topk_idx || o.topk_prob;
  const int rounds = topk ? k : 1;
  if (!head_supported(n, rounds) || rows < 0 || !logits) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(classify_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHeadMaxN * (int)sizeof(float));
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  // programmatic dependent launch (on unless TFSC_PDL=0): the head is set up while the layer that writes the logits drains,
  // and waits for that grid (griddepcontrol.wait) before its first read
  static const bool pdl = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  // 128 threads cover a ResNet / BERT-classifier head in a few strided loads each; wide vocab heads take 512 so that
  // every thread has at most 64 elements to load and rescan
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)rows);
  cfg.blockDim = dim3(n > 2048 ? kHeadThreadsMax : 128);
  cfg.dynamicSmemBytes = (size_t)n * sizeof(float);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, classify_head_kernel, logits, n, rounds, o);
  g_launches_nn++;
  return e;
}

}  // namespace tfsc
