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

#include "head_select.cuh"
#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

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
  const int64_t row = blockIdx.x;
  // launched after a PDL dense kernel, the logits are that grid's output (a no-op without the launch attribute)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const float m = head_stage_select(logits + row * n, n, rounds, xs, wv, wi, &s_v, &s_i, sel);
  // softmax: max-subtracted fp32 exponentials, summed in fp64
  const bool need_sum = o.probs || o.topk_prob;
  const float inv = need_sum ? head_softmax_inv(xs, n, m, wsum, &s_sum) : 0.f;
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
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)rows);
  cfg.blockDim = dim3(head_threads(n));
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
