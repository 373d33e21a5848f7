// Swin Transformer building blocks for the graph executor, fp32 NHWC, sm_90a:
//   window_attention  ctx[b, y, x, h*d:(h+1)*d] = softmax(q k^T * d^-0.5 + bias[h] (+ shift mask)) v within each ws x ws window
//                     of the feature map cyclically shifted by `shift`, reading the packed q | k | v [H, W, 3C]
//   patch_merge       y[b, oy, ox, q*C + c] = x[b, 2oy + (q & 1), 2ox + (q >> 1), c]   (torchvision's x0 | x1 | x2 | x3)
// The qkv and output projections are per-token, so they commute with the roll and the window partition: window_attention
// reads and writes the ordinary NHWC layout and does the shift and the partition in its addressing. Token i of window
// (wy, wx) sits at (y', x') = (wy*ws + i / ws, wx*ws + i % ws) of the shifted frame, which is ((y' + s) mod H, (x' + s) mod W)
// of the feature map. Two tokens whose shifted-frame positions lie in different regions of torchvision's mask ([0, H - ws),
// [H - ws, H - s), [H - s, H) per axis) get -100 added to their score.
// One CTA per (window, head) and a grid-stride over the images: K [N][d+1] (padded against bank conflicts) and V [N][d]
// of the window in shared memory, each of the 4 warps owns query rows; a lane holds the scores of keys lane + 32 t, the
// softmax runs on warp shuffles (max-subtracted expf, fp32 sum) and the P.V product gives one output column per lane.
// Every CTA computes its (image, window, head) with the same instructions in the same order, so a window's bits depend
// neither on the batch nor on the path (16-byte or scalar K / V loads). Both kernels use programmatic dependent launch.
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdlib>

#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kWaThreads = kWindowWarps * 32, kMergeThreads = 256;

static bool pdl_on() {  // programmatic dependent launch, on unless TFSC_PDL=0, as the other graph kernels
  static const bool v = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  return v;
}

// shift-mask region of a shifted-frame coordinate p on an axis of length L
__device__ __forceinline__ int swin_region(int p, int L, int ws, int s) { return p < L - ws ? 0 : p < L - s ? 1 : 2; }

// NT: score slots per lane, N <= 32 * NT. VEC: K / V staged with 16-byte loads (d % 4 == 0, C % 4 == 0, qkv aligned).
// grid: x = windows * heads (head fastest), y = images (grid-stride over the batch)
template <int NT, bool VEC>
__global__ void __launch_bounds__(kWaThreads)
window_attention_kernel(const float* __restrict__ qkv, const float* __restrict__ bias, float* __restrict__ ctx, int Bn, int H, int W,
                        int C, int heads, int ws, int shift, float scale) {
  extern __shared__ float sm[];
  const int d = C / heads, N = ws * ws, C3 = 3 * C;
  const int head = blockIdx.x % heads, win = blockIdx.x / heads;
  const int wy = win / (W / ws), wx = win % (W / ws);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* Ks = sm;                          // [N][d + 1]
  float* Vs = Ks + N * (d + 1);            // [N][d]
  float* Ps = Vs + N * d + warp * N;       // this warp's probabilities [N]
  float* Qs = Vs + N * d + kWindowWarps * N + warp * d;  // this warp's query [d]
  const float* hb = bias + (size_t)head * N * N;
  auto row = [&](int i) {                  // token i of this window -> its pixel in the (unshifted) feature map
    int y = wy * ws + i / ws + shift, x = wx * ws + i % ws + shift;
    y -= y >= H ? H : 0;
    x -= x >= W ? W : 0;
    return y * W + x;
  };
  auto region = [&](int i) { return 3 * swin_region(wy * ws + i / ws, H, ws, shift) + swin_region(wx * ws + i % ws, W, ws, shift); };
  asm volatile("griddepcontrol.wait;" ::: "memory");                // qkv is the previous grid's output
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int img = blockIdx.y; img < Bn; img += gridDim.y) {
    const float* src = qkv + (size_t)img * H * W * C3 + head * d;
    if constexpr (VEC) {
      const int d4 = d / 4;
      for (int idx = threadIdx.x; idx < N * d4; idx += kWaThreads) {
        const int j = idx / d4, c = (idx % d4) * 4;
        const float* p = src + (size_t)row(j) * C3 + c;
        const float4 k = __ldg(reinterpret_cast<const float4*>(p + C));
        const float4 v = __ldg(reinterpret_cast<const float4*>(p + 2 * C));
        float* kr = Ks + j * (d + 1) + c;  // Ks rows are d + 1 wide and Vs starts at N (d + 1): 4-byte stores
        float* vr = Vs + j * d + c;
        kr[0] = k.x, kr[1] = k.y, kr[2] = k.z, kr[3] = k.w;
        vr[0] = v.x, vr[1] = v.y, vr[2] = v.z, vr[3] = v.w;
      }
    } else {
      for (int idx = threadIdx.x; idx < N * d; idx += kWaThreads) {
        const int j = idx / d, c = idx % d;
        const float* p = src + (size_t)row(j) * C3 + c;
        Ks[j * (d + 1) + c] = __ldg(p + C);
        Vs[j * d + c] = __ldg(p + 2 * C);
      }
    }
    __syncthreads();
    float* dst = ctx + (size_t)img * H * W * C + head * d;
    for (int i = warp; i < N; i += kWindowWarps) {
      const int ri = row(i);
      for (int c = lane; c < d; c += 32) Qs[c] = __ldg(src + (size_t)ri * C3 + c);
      __syncwarp();
      float s[NT];
#pragma unroll
      for (int t = 0; t < NT; ++t) s[t] = 0.f;
      for (int c = 0; c < d; ++c) {
        const float q = Qs[c];
#pragma unroll
        for (int t = 0; t < NT; ++t) s[t] = fmaf(q, Ks[min(lane + 32 * t, N - 1) * (d + 1) + c], s[t]);  // j >= N: discarded
      }
      const int gi = shift ? region(i) : 0;
      float m = -INFINITY;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int j = lane + 32 * t;
        if (j < N) {
          s[t] = s[t] * scale + __ldg(hb + i * N + j);
          if (shift && region(j) != gi) s[t] += -100.f;
        } else {
          s[t] = -INFINITY;
        }
        m = fmaxf(m, s[t]);
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      float sum = 0.f;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int j = lane + 32 * t;
        const float e = expf(s[t] - m);  // 0 for j >= N
        sum += e;
        if (j < N) Ps[j] = e;
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      __syncwarp();
      const float inv = 1.f / sum;
      for (int c = lane; c < d; c += 32) {
        float acc = 0.f;
        for (int j = 0; j < N; ++j) acc = fmaf(Ps[j], Vs[j * d + c], acc);
        dst[(size_t)ri * C + c] = acc * inv;
      }
      __syncwarp();
    }
    __syncthreads();  // K / V of the next image overwrite this one's
  }
}

// grid: x = blocks over one image's OH * OW * 4C / VEC outputs, y = images (grid-stride over the batch)
template <int VEC>
__global__ void __launch_bounds__(kMergeThreads)
patch_merge_kernel(const float* __restrict__ x, float* __restrict__ y, int Bn, int H, int W, int C) {
  asm volatile("griddepcontrol.wait;" ::: "memory");                // x is the previous grid's output
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int CV = C / VEC, OW = W / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (H / 2) * OW * 4 * CV) return;
  const int c = (idx % CV) * VEC, q = (idx / CV) % 4, pix = idx / (4 * CV);
  const int iy = 2 * (pix / OW) + (q & 1), ix = 2 * (pix % OW) + (q >> 1);
  const size_t in = (size_t)(iy * W + ix) * C + c, out = (size_t)idx * VEC;
  for (int img = blockIdx.y; img < Bn; img += gridDim.y) {
    const size_t ib = (size_t)img * H * W * C;
    if constexpr (VEC == 4) {
      *reinterpret_cast<float4*>(y + ib + out) = __ldg(reinterpret_cast<const float4*>(x + ib + in));
    } else {
      y[ib + out] = __ldg(x + ib + in);
    }
  }
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
  return e != cudaSuccess ? e : cudaGetLastError();
}

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

cudaError_t launch_window_attention(const float* qkv, const float* bias, float* ctx, int Bn, int H, int W, int C, int heads, int ws,
                                    int shift, cudaStream_t s) {
  if (Bn < 0 || !window_attention_supported(H, W, C, heads, ws, shift) || !qkv || !bias || !ctx) return cudaErrorInvalidValue;
  if (Bn == 0) return cudaSuccess;
  const int d = C / heads, N = ws * ws;
  const float scale = (float)(1.0 / std::sqrt((double)d));
  const bool vec = d % 4 == 0 && C % 4 == 0 && al16(qkv);
  const dim3 grid((H / ws) * (W / ws) * heads, Bn < 65535 ? Bn : 65535);
  const size_t smem = window_attention_smem_bytes(ws, d);
#define TFSC_WA(NT)                                                                                                            \
  (vec ? launch_pdl(window_attention_kernel<NT, true>, grid, kWaThreads, smem, s, qkv, bias, ctx, Bn, H, W, C, heads, ws, shift, \
                    scale)                                                                                                     \
       : launch_pdl(window_attention_kernel<NT, false>, grid, kWaThreads, smem, s, qkv, bias, ctx, Bn, H, W, C, heads, ws, shift, \
                    scale))
  const cudaError_t e = N <= 64 ? TFSC_WA(2) : N <= 160 ? TFSC_WA(5) : TFSC_WA(8);
#undef TFSC_WA
  return e;
}

cudaError_t launch_patch_merge(const float* x, float* y, int Bn, int H, int W, int C, cudaStream_t s) {
  if (Bn < 0 || !patch_merge_supported(H, W, C) || !x || !y) return cudaErrorInvalidValue;
  if (Bn == 0) return cudaSuccess;
  const bool vec = C % 4 == 0 && al16(x) && al16(y);
  const int per_img = (H / 2) * (W / 2) * 4 * (vec ? C / 4 : C);
  const dim3 grid((per_img + kMergeThreads - 1) / kMergeThreads, Bn < 65535 ? Bn : 65535);
  return vec ? launch_pdl(patch_merge_kernel<4>, grid, kMergeThreads, 0, s, x, y, Bn, H, W, C)
             : launch_pdl(patch_merge_kernel<1>, grid, kMergeThreads, 0, s, x, y, Bn, H, W, C);
}

}  // namespace tfsc
