// The activations MobileNetV2 and EfficientNet add to the GEMM epilogues and the depthwise convolution (act 4, 5, 6 of a
// graph op). One definition, so a value gets the same bits on every path that applies it.
#pragma once
#include <cuda_runtime.h>

namespace tfsc {

__device__ __forceinline__ float relu6f(float x) { return fminf(fmaxf(x, 0.f), 6.f); }
__device__ __forceinline__ float siluf(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }
// act 7, GPT-2's GELU (HF gelu_new, TF gelu(approximate=True)): 0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3)))
__device__ __forceinline__ float gelu_tanhf(float x) {
  return 0.5f * x * (1.f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

}  // namespace tfsc
