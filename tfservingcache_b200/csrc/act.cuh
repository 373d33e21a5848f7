// The activations MobileNetV2 and EfficientNet add to the GEMM epilogues and the depthwise convolution (act 4, 5, 6 of a
// graph op). One definition, so a value gets the same bits on every path that applies it.
#pragma once
#include <cuda_runtime.h>

namespace tfsc {

__device__ __forceinline__ float relu6f(float x) { return fminf(fmaxf(x, 0.f), 6.f); }
__device__ __forceinline__ float siluf(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

}  // namespace tfsc
