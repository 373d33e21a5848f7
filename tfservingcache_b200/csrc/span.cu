// Span head of question-answering bundles (signature.outputs start_logits .. span_scores), fp32, sm_90a: one launch turns
// a batch of per-token [S, 2] start / end logits into every declared output -- the start and end logits de-interleaved and
// the k best answer spans with their scores -- written at their offsets inside the packed response row.
//
// Layout: one CTA per row. The row's start[S] and end[S] logits are staged in shared memory with the ineligible tokens
// (mask 0, segment 0, the [SEP] id) replaced by NaN, so a candidate (i, j) -- i <= j < i + L -- scores start[i] + end[j]
// in fp32 and a NaN score ranks nowhere: ineligible and NaN pairs are never selected. Spans are ordered by (score
// descending, i ascending, j ascending). Every thread first finds, for the start positions i = t, t + T, ..., the best
// end j of each (shared best[S], nothing of size S * L is stored). Then warp 0 alone runs k rounds: a warp argmax over the
// per-start bests picks the round's span, and the 32 lanes rescan only the winner's start for its next-best end, so a
// round costs two warp reductions and L / 32 loads per lane, with no block barrier. The comparisons are exact on the fp32
// sums, so the spans are a function of the logits alone. Timings are in DESIGN §4.
#include <cuda_runtime.h>

#include <atomic>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdlib>

#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kSpanThreadsMax = 256;

// (av, ak) ranks above (bv, bk): higher score, then the lower key (key = i * S + j across starts, j within one start)
__device__ __forceinline__ bool span_above(float av, int ak, float bv, int bk) { return av > bv || (av == bv && ak < bk); }

__device__ __forceinline__ void span_warp_best(float& v, int& k) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int ok = __shfl_xor_sync(0xffffffffu, k, o);
    if (span_above(ov, ok, v, k)) {
      v = ov;
      k = ok;
    }
  }
}

// the best of the per-start bests of starts i = lane, lane + 32, ...; (-inf, INT_MAX) when none is left
__device__ __forceinline__ void lane_best(const float* bv, const int* bk, int S, int lane, float* v, int* k) {
  float v0 = -INFINITY;
  int k0 = INT_MAX;
  for (int i = lane; i < S; i += 32)
    if (span_above(bv[i], bk[i], v0, k0)) {
      v0 = bv[i];
      k0 = bk[i];
    }
  *v = v0;
  *k = k0;
}

__global__ void __launch_bounds__(kSpanThreadsMax) span_head_kernel(const float* __restrict__ logits, SpanInputs in, int S, int L,
                                                                    int rounds, SpanOutputs o) {
  extern __shared__ float sm[];  // start[S] | end[S] (ineligible tokens NaN) | best score[S] | best key[S] per start
  float* st = sm;
  float* en = sm + S;
  float* bv = sm + 2 * S;
  int* bk = reinterpret_cast<int*>(sm + 3 * S);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t row = blockIdx.x;
  // launched after the op that writes the per-token logits, which are that grid's output (a no-op without the attribute)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const float* x = logits + row * 2 * S;
  for (int p = threadIdx.x; p < S; p += blockDim.x) {
    const float a = __ldg(x + 2 * p), b = __ldg(x + 2 * p + 1);
    if (o.start_logits) o.start_logits[row * o.start_ld + p] = a;
    if (o.end_logits) o.end_logits[row * o.end_ld + p] = b;
    if (rounds) {
      // the request row as the embedding reads it: ids / mask / segment ids at stride `stride` (no mask: [PAD] = id 0)
      const int64_t q = row * in.stride + p;
      const int id = __ldg(in.ids + q);
      const bool live = in.mask ? __ldg(in.mask + q) != 0 : id != 0;
      const bool ok = live && __ldg(in.types + q) == 1 && (in.sep_id < 0 || id != in.sep_id);
      st[p] = ok ? a : __int_as_float(0x7fc00000);
      en[p] = ok ? b : __int_as_float(0x7fc00000);
    }
  }
  if (rounds == 0) return;
  __syncthreads();
  // the best end of every start (score descending, j ascending)
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const float si = st[i];
    const int jend = min(S, i + L);
    float v0 = -INFINITY;
    int j0 = INT_MAX;
#pragma unroll 4
    for (int j = i; j < jend; ++j) {
      const float v = __fadd_rn(si, en[j]);
      if (span_above(v, j, v0, j0)) {
        v0 = v;
        j0 = j;
      }
    }
    bv[i] = v0;
    bk[i] = j0 == INT_MAX ? INT_MAX : i * S + j0;
  }
  __syncthreads();
  if (warp != 0) return;

  float lv;
  int lk;
  lane_best(bv, bk, S, lane, &lv, &lk);
  int r = 0;
  for (; r < rounds; ++r) {
    float gv = lv;
    int gk = lk;
    span_warp_best(gv, gk);  // every lane holds the winner
    if (gk == INT_MAX) break;  // no candidate left
    const int gi = gk / S, gj = gk - gi * S;
    if (lane == 0) {
      if (o.starts) o.starts[row * o.starts_ld + r] = gi;
      if (o.ends) o.ends[row * o.ends_ld + r] = gj;
      if (o.scores) o.scores[row * o.scores_ld + r] = gv;
    }
    // the winner's start: its best end that ranks below the one just selected
    const float si = st[gi];
    const int jend = min(S, gi + L);
    float cv = -INFINITY;
    int cj = INT_MAX;
    for (int j = gi + lane; j < jend; j += 32) {
      const float v = __fadd_rn(si, en[j]);
      if (span_above(gv, gj, v, j) && span_above(v, j, cv, cj)) {
        cv = v;
        cj = j;
      }
    }
    span_warp_best(cv, cj);
    if (lane == (gi & 31)) {  // the lane that owns the start updates it and its own best
      bv[gi] = cv;
      bk[gi] = cj == INT_MAX ? INT_MAX : gi * S + cj;
      lane_best(bv, bk, S, lane, &lv, &lk);
    }
  }
  // fewer than k candidates: the remaining slots are (-1, -1) with score -FLT_MAX (finite, so JSON bodies stay valid)
  for (int t = r + lane; t < rounds; t += 32) {
    if (o.starts) o.starts[row * o.starts_ld + t] = -1;
    if (o.ends) o.ends[row * o.ends_ld + t] = -1;
    if (o.scores) o.scores[row * o.scores_ld + t] = -FLT_MAX;
  }
}

cudaError_t launch_span_head(const float* logits, const SpanInputs& in, int rows, int S, int L, int k, const SpanOutputs& o,
                             cudaStream_t s) {
  const int rounds = (o.starts || o.ends || o.scores) ? k : 0;
  if (!span_supported(S, rounds ? L : 1, rounds ? k : 1) || rows < 0 || !logits) return cudaErrorInvalidValue;
  if (rounds && (!in.ids || !in.types || in.stride < S)) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {  // 64 KB of dynamic shared memory at S = 4096
    cudaError_t e = cudaFuncSetAttribute(span_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * kSpanMaxS * (int)sizeof(float));
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  // programmatic dependent launch (on unless TFSC_PDL=0), as the classify head: set up while the last op drains
  static const bool pdl = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  // 128 threads give a SQuAD row (S = 384) three start positions each for the first pass; longer rows take 256
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)rows);
  cfg.blockDim = dim3(S > 512 ? kSpanThreadsMax : 128);
  cfg.dynamicSmemBytes = (size_t)S * 4 * sizeof(float);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, span_head_kernel, logits, in, S, rounds ? L : 1, rounds, o);
  g_launches_nn++;
  return e;
}

}  // namespace tfsc
