// Selection and softmax of one logits row, shared by the classification head (head.cu) and the fill-mask head (mlm.cu) so
// that both answer the same bits for the same row: the row is staged in shared memory, the top `rounds` entries are picked
// by block-wide argmax rounds over (value descending, index ascending), and the softmax is a max-subtracted fp32 expf
// summed in fp64 in an order fixed by n and blockDim. Every function is inlined into its kernel; the caller declares the
// shared-memory scratch and must launch the same blockDim for the same n (head_threads) to get the same sums.
#pragma once
#include <cuda_runtime.h>

#include <climits>
#include <cmath>

#include "nn_limits.h"

namespace tfsc {

constexpr int kHeadThreadsMax = 512;

// 128 threads cover a ResNet / BERT-classifier head in a few strided loads each; wide vocab rows take 512 so that every
// thread has at most 64 elements to load and rescan
inline int head_threads(int n) { return n > 2048 ? kHeadThreadsMax : 128; }

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

// one expression for every probability output, so top-k probabilities are the same bits as probabilities[index]
__device__ __forceinline__ float softmax_at(float x, float m, float inv) { return expf(x - m) * inv; }

// Stages x[0, n) in xs and writes the indices of the top `rounds` entries to sel[0, rounds); returns the row maximum.
// wv / wi: kHeadThreadsMax / 32 per-warp slots, s_v / s_i: the round's winner (all shared memory).
__device__ __forceinline__ float head_stage_select(const float* __restrict__ x, int n, int rounds, float* xs, float* wv, int* wi,
                                                   float* s_v, int* s_i, int* sel) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
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
        *s_v = v;
        *s_i = i;
        sel[r] = i;
      }
    }
    __syncthreads();
    const float gv = *s_v;
    const int gi = *s_i;
    if (r == 0) m = gv;  // the row maximum
    if (bi == gi) local_best(xs, n, gv, gi, &bv, &bi);
  }
  return m;
}

// 1 / sum_j expf(xs[j] - m) over the staged row: fp32 exponentials summed in fp64 (a 32768-wide row keeps its sum to ~1 ulp
// of fp32). wsum: kHeadThreadsMax / 32 per-warp slots, s_sum: the total (shared memory).
__device__ __forceinline__ float head_softmax_inv(const float* xs, int n, float m, double* wsum, double* s_sum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
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
    if (lane == 0) *s_sum = a;
  }
  __syncthreads();
  return (float)(1.0 / *s_sum);
}

}  // namespace tfsc
