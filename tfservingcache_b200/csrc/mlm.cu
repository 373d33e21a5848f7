// Fill-mask (masked-language-model) kernels of BERT MLM bundles, fp32, sm_90a: the mask_gather op that selects the [MASK]
// tokens of each row, and the head that turns each selected slot's vocabulary logits into the top k token ids, their
// probabilities and their logits, written at their offsets inside the packed response row.
//
// mask_gather_kernel: one CTA per row. The candidate scan is an ordered block-wide compaction over the S tokens: each pass
// of blockDim tokens takes a warp ballot of the candidates, a prefix of the per-warp popcounts gives every candidate its
// slot, and the scan stops at the pass that fills the M slots. The H-wide copies of the selected hidden states use 16-byte
// loads and stores (a scalar path for layouts that are not 16-byte aligned); they are copies, so the bits are exact.
//
// fill_mask_head_kernel: one CTA per (row, slot). An empty slot (position -1) writes its fill values and exits. A filled
// slot stages the first `vocab` logits of its Vp-wide row and runs the classification head's selection and softmax
// (head_select.cuh) with the classification head's block size, so its ids and probabilities have the bits
// launch_classify_head gives for those `vocab` logits. Timings are in DESIGN §4.
#include <cuda_runtime.h>

#include <atomic>
#include <cfloat>
#include <cstdint>
#include <cstdlib>

#include "head_select.cuh"
#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kGatherThreads = 256;

static bool pdl_on() {  // programmatic dependent launch, on unless TFSC_PDL=0, as the other heads
  static const bool v = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  return v;
}

template <bool kVec>
__global__ void __launch_bounds__(kGatherThreads) mask_gather_kernel(const float* __restrict__ hidden, const int* __restrict__ ids,
                                                                     const int* __restrict__ mask, int64_t stride, int S, int H,
                                                                     int M, int mask_token_id, int* __restrict__ positions,
                                                                     float* __restrict__ gathered) {
  extern __shared__ int spos[];  // the row's M slot positions
  __shared__ int wcnt[kGatherThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t row = blockIdx.x;
  // launched after the op that writes the hidden states, which are that grid's output
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int* irow = ids + row * stride;
  const int* mrow = mask ? mask + row * stride : nullptr;
  int filled = 0;  // candidates seen so far: the same value in every thread
  for (int base = 0; base < S && filled < M; base += blockDim.x) {
    const int p = base + (int)threadIdx.x;
    const bool cand = p < S && __ldg(irow + p) == mask_token_id && (!mrow || __ldg(mrow + p) != 0);
    const unsigned ballot = __ballot_sync(0xffffffffu, cand);
    if (lane == 0) wcnt[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < nwarps; ++w) {
      const int c = wcnt[w];
      before += w < warp ? c : 0;
      total += c;
    }
    const int slot = filled + before + __popc(ballot & ((1u << lane) - 1u));
    if (cand && slot < M) spos[slot] = p;
    filled += total;
    __syncthreads();  // wcnt is rewritten by the next pass
  }
  filled = min(filled, M);
  for (int s = filled + (int)threadIdx.x; s < M; s += blockDim.x) spos[s] = -1;
  __syncthreads();
  if (positions)
    for (int s = threadIdx.x; s < M; s += blockDim.x) positions[row * M + s] = spos[s];
  if (!gathered) return;
  if (kVec) {
    const int Q = H >> 2;
    const float4* src = reinterpret_cast<const float4*>(hidden) + row * S * Q;
    float4* dst = reinterpret_cast<float4*>(gathered) + row * M * Q;
    for (int i = threadIdx.x; i < M * Q; i += blockDim.x) {
      const int s = i / Q, q = i - s * Q;
      const int p = spos[s];
      dst[i] = p >= 0 ? __ldg(src + (int64_t)p * Q + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else {
    const float* src = hidden + row * S * H;
    float* dst = gathered + row * M * H;
    for (int i = threadIdx.x; i < M * H; i += blockDim.x) {
      const int s = i / H, c = i - s * H;
      const int p = spos[s];
      dst[i] = p >= 0 ? __ldg(src + (int64_t)p * H + c) : 0.f;
    }
  }
}

cudaError_t launch_mask_gather(const float* hidden, const int* ids, const int* mask, int64_t stride, int rows, int S, int H,
                               int M, int mask_token_id, int* positions, float* gathered, cudaStream_t s) {
  if (!mask_gather_supported(S, H, M) || rows < 0 || !ids || stride < S || (gathered && !hidden)) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  const bool vec = H % 4 == 0 && ((uintptr_t)hidden & 15) == 0 && ((uintptr_t)gathered & 15) == 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)rows);
  cfg.blockDim = dim3(kGatherThreads);
  cfg.dynamicSmemBytes = (size_t)M * sizeof(int);  // 32 KB at M = 8192: no opt-in needed
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_on() ? 1 : 0;
  cudaError_t e = vec ? cudaLaunchKernelEx(&cfg, mask_gather_kernel<true>, hidden, ids, mask, stride, S, H, M, mask_token_id,
                                           positions, gathered)
                      : cudaLaunchKernelEx(&cfg, mask_gather_kernel<false>, hidden, ids, mask, stride, S, H, M, mask_token_id,
                                           positions, gathered);
  g_launches_nn++;
  return e;
}

// rounds = 0: masked_positions only (no selection)
__global__ void __launch_bounds__(kHeadThreadsMax) fill_mask_head_kernel(const float* __restrict__ logits, int64_t ld,
                                                                         const int* __restrict__ positions, int M, int vocab,
                                                                         int rounds, FillMaskOutputs o) {
  extern __shared__ float xs[];  // the slot's vocab logits
  __shared__ float wv[kHeadThreadsMax / 32];
  __shared__ int wi[kHeadThreadsMax / 32];
  __shared__ double wsum[kHeadThreadsMax / 32];
  __shared__ float s_v;
  __shared__ int s_i;
  __shared__ double s_sum;
  __shared__ int sel[kHeadMaxK];
  const int64_t slot = blockIdx.x;
  const int64_t row = slot / M;
  const int s = (int)(slot - row * M);
  // launched after the op that writes the vocabulary logits; the positions come from the gather before it
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int pos = __ldg(positions + slot);
  if (o.positions && threadIdx.x == 0) o.positions[row * o.positions_ld + s] = pos;
  if (rounds == 0) return;
  int* ids = o.ids ? o.ids + row * o.ids_ld + (int64_t)s * rounds : nullptr;
  float* probs = o.probs ? o.probs + row * o.probs_ld + (int64_t)s * rounds : nullptr;
  float* lg = o.logits ? o.logits + row * o.logits_ld + (int64_t)s * rounds : nullptr;
  if (pos < 0) {  // an empty slot: the same for the whole CTA
    if ((int)threadIdx.x < rounds) {
      if (ids) ids[threadIdx.x] = -1;
      if (probs) probs[threadIdx.x] = 0.f;
      if (lg) lg[threadIdx.x] = -FLT_MAX;
    }
    return;
  }
  const float m = head_stage_select(logits + slot * ld, vocab, rounds, xs, wv, wi, &s_v, &s_i, sel);
  const float inv = probs ? head_softmax_inv(xs, vocab, m, wsum, &s_sum) : 0.f;
  if ((int)threadIdx.x < rounds) {
    const int j = sel[threadIdx.x];
    // j < vocab for finite logits; a NaN row can leave the sentinel INT_MAX, which must not index shared memory
    const float x = xs[j < vocab ? j : vocab - 1];
    if (ids) ids[threadIdx.x] = j;
    if (probs) probs[threadIdx.x] = softmax_at(x, m, inv);
    if (lg) lg[threadIdx.x] = x;
  }
}

cudaError_t launch_fill_mask_head(const float* logits, int64_t ld, const int* positions, int rows, int M, int vocab, int k,
                                  int max_vocab, const FillMaskOutputs& o, cudaStream_t s) {
  const bool topk = o.ids || o.probs || o.logits;
  // max_vocab: kHeadMaxN for fill-mask bundles (fill_mask_supported), kNextTokenMaxVocab for the next-token head's one slot
  const bool shape_ok = max_vocab == kNextTokenMaxVocab ? M == 1 && next_token_supported(vocab, topk ? k : 1)
                                                         : max_vocab == kHeadMaxN && fill_mask_supported(M, vocab, topk ? k : 1);
  if (!shape_ok || rows < 0 || !positions || (topk && (!logits || ld < vocab))) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    // the largest row either head stages; the opt-in permits more shared memory and changes no launch's code
    cudaError_t e = cudaFuncSetAttribute(fill_mask_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kNextTokenMaxVocab * (int)sizeof(float));
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)((int64_t)rows * M));
  // the classification head's block size for the same row width: its softmax sum runs in the same order
  cfg.blockDim = dim3(topk ? head_threads(vocab) : 32);
  cfg.dynamicSmemBytes = topk ? (size_t)vocab * sizeof(float) : 0;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_on() ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, fill_mask_head_kernel, logits, ld, positions, M, vocab, topk ? k : 0, o);
  g_launches_nn++;
  return e;
}

}  // namespace tfsc
