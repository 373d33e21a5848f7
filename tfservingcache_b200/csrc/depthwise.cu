// MobileNet / EfficientNet building blocks for the graph executor, fp32 NHWC, sm_90a:
//   depthwise_conv   y[b, oy, ox, ch] = act(sum_i sum_j x[b, oy*s - p + i, ox*s - p + j, ch] * w[i, j, ch] + bias[ch])
//   channel_scale    y[b, p, ch] = x[b, p, ch] * g[b, ch]   (the squeeze-and-excitation gate)
// Both are bandwidth-bound elementwise-shaped kernels. A thread of depthwise_conv owns one output pixel and 4 channels
// (16-byte loads; 1 channel on the scalar path) and reads its kh x kw input taps straight from global memory: the
// neighbouring pixels of a CTA read the same input rows, so the (k / stride)^2-fold reuse is served by L1, without a
// shared-memory tile or a barrier (DESIGN §4). Taps run i, then j, ascending with fmaf on both paths, and padding taps are
// skipped, so a value's bits depend neither on the batch nor on the path. Both kernels use programmatic dependent
// launch: they wait for the grid before them before their first read and let the next grid launch early.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>

#include "act.cuh"
#include "kernels.h"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

constexpr int kDwThreads = 128, kScaleThreads = 256;

static bool pdl_on() {  // programmatic dependent launch, on unless TFSC_PDL=0, as the other graph kernels
  static const bool v = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  return v;
}

template <int VEC>
struct Vec;
template <>
struct Vec<1> {
  static __device__ __forceinline__ void load(const float* p, float* v) { v[0] = __ldg(p); }
  static __device__ __forceinline__ void store(float* p, const float* v) { *p = v[0]; }
};
template <>
struct Vec<4> {
  static __device__ __forceinline__ void load(const float* p, float* v) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};

// act: 0 none, 1 relu, 4 relu6, 5 silu, 6 sigmoid (the launcher refuses the others)
__device__ __forceinline__ float dw_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 4) return relu6f(v);
  if (act == 5) return siluf(v);
  if (act == 6) return sigmoidf(v);
  return v;
}

// grid: x = blocks over one image's OH * OW * C / VEC outputs, y = images (grid-stride over the batch)
template <int VEC>
__global__ void __launch_bounds__(kDwThreads)
depthwise_conv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                      float* __restrict__ y, int Bn, int H, int W, int C, int KH, int KW, int stride, int pad, int OH, int OW,
                      int act) {
  asm volatile("griddepcontrol.wait;" ::: "memory");                // x is the previous grid's output
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int CV = C / VEC;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= OH * OW * CV) return;
  const int c = (idx % CV) * VEC, pix = idx / CV;
  const int ox = pix % OW, oy = pix / OW;
  const int iy0 = oy * stride - pad, ix0 = ox * stride - pad;
  const int i0 = max(0, -iy0), i1 = min(KH, H - iy0), j0 = max(0, -ix0), j1 = min(KW, W - ix0);
  float b[VEC];
  Vec<VEC>::load(bias + c, b);
  for (int img = blockIdx.y; img < Bn; img += gridDim.y) {
    const float* xb = x + (size_t)img * H * W * C + c;
    float acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
    for (int i = i0; i < i1; ++i) {
      const float* xr = xb + (iy0 + i) * W * C;
      const float* wr = w + i * KW * C + c;
      for (int j = j0; j < j1; ++j) {
        float xv[VEC], wv[VEC];
        Vec<VEC>::load(xr + (ix0 + j) * C, xv);
        Vec<VEC>::load(wr + j * C, wv);
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = fmaf(xv[v], wv[v], acc[v]);
      }
    }
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = dw_act(acc[v] + b[v], act);
    Vec<VEC>::store(y + (size_t)img * OH * OW * C + (size_t)pix * C + c, acc);
  }
}

// grid: x = blocks over one image's HW * C / VEC values, y = images (grid-stride over the batch)
template <int VEC>
__global__ void __launch_bounds__(kScaleThreads)
channel_scale_kernel(const float* __restrict__ x, const float* __restrict__ gate, float* __restrict__ y, int Bn, int HW, int C) {
  asm volatile("griddepcontrol.wait;" ::: "memory");                // the gate is the previous grid's output
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= HW * (C / VEC)) return;
  const int c = (idx % (C / VEC)) * VEC;
  for (int img = blockIdx.y; img < Bn; img += gridDim.y) {
    const size_t off = (size_t)img * HW * C + (size_t)idx * VEC;
    float xv[VEC], g[VEC];
    Vec<VEC>::load(x + off, xv);
    Vec<VEC>::load(gate + (size_t)img * C + c, g);
#pragma unroll
    for (int v = 0; v < VEC; ++v) xv[v] *= g[v];
    Vec<VEC>::store(y + off, xv);
  }
}

template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, int threads, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(threads);
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

cudaError_t launch_depthwise_conv(const float* x, const float* w, const float* bias, float* y, int Bn, int H, int W, int C, int KH,
                                  int KW, int stride, int pad, int act, cudaStream_t s) {
  if (Bn < 0 || !depthwise_supported(H, W, C, KH, KW, stride, pad) || !(act == 0 || act == 1 || (act >= 4 && act <= 6)) || !x ||
      !w || !bias || !y)
    return cudaErrorInvalidValue;
  if (Bn == 0) return cudaSuccess;
  const int OH = (H + 2 * pad - KH) / stride + 1, OW = (W + 2 * pad - KW) / stride + 1;
  const bool vec = C % 4 == 0 && al16(x) && al16(w) && al16(bias) && al16(y);
  const int per_img = OH * OW * (vec ? C / 4 : C);
  const dim3 grid((per_img + kDwThreads - 1) / kDwThreads, Bn < 65535 ? Bn : 65535);
  return vec ? launch_pdl(depthwise_conv_kernel<4>, grid, kDwThreads, s, x, w, bias, y, Bn, H, W, C, KH, KW, stride, pad, OH, OW, act)
             : launch_pdl(depthwise_conv_kernel<1>, grid, kDwThreads, s, x, w, bias, y, Bn, H, W, C, KH, KW, stride, pad, OH, OW, act);
}

cudaError_t launch_channel_scale(const float* x, const float* gate, float* y, int Bn, int HW, int C, cudaStream_t s) {
  if (Bn < 0 || HW < 1 || C < 1 || (long long)HW * C > 0x7fffffffLL || !x || !gate || !y) return cudaErrorInvalidValue;
  if (Bn == 0) return cudaSuccess;
  const bool vec = C % 4 == 0 && al16(x) && al16(gate) && al16(y);
  const int per_img = HW * (vec ? C / 4 : C);
  const dim3 grid((per_img + kScaleThreads - 1) / kScaleThreads, Bn < 65535 ? Bn : 65535);
  return vec ? launch_pdl(channel_scale_kernel<4>, grid, kScaleThreads, s, x, gate, y, Bn, HW, C)
             : launch_pdl(channel_scale_kernel<1>, grid, kScaleThreads, s, x, gate, y, Bn, HW, C);
}

}  // namespace tfsc
