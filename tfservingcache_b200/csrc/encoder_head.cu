// Encoder head of embedding bundles (signature.outputs sequence_output, pooled_output, cls_embedding, mean_embedding),
// fp32, sm_90a: one launch turns a batch of last hidden states [S, H] (and the pooler's [H]) into every declared output,
// written at its offset inside the packed response row.
//
// Layout: a thread-block cluster per row of ctas = clamp(ceil(S / 16), 1, 8) CTAs; CTA `rank` owns the tokens
// [rank * T, (rank + 1) * T), T = ceil(S / ctas), so even a batch of 8 rows streams through 64 SMs. The hidden states are
// read from HBM once: each thread walks its column quad (one 16-byte load per token, 8 tokens in flight) down its CTA's
// tokens, stores the copy for sequence_output and adds the unmasked tokens into fp32 partial sums, in token order. The
// partials meet in distributed shared memory: rank 0 adds ranks 0, 1, ..., ctas - 1 in that order, divides by the token
// count, optionally normalises, and writes the [H] outputs. Every sum runs in an order fixed by S and H (ctas, T, the
// block size and the norm's reduction tree), never by `rows` or by which SM runs a CTA, so a row's bits do not depend on
// its batch; sequence_output, pooled_output and cls_embedding without normalize are exact copies. Layouts that are not
// 16-byte aligned take a scalar path with the same per-column order, hence the same bits. Timings are in DESIGN §4.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdlib>

#include "kernels.h"

namespace tfsc {

namespace cg = cooperative_groups;

extern std::atomic<int64_t> g_launches_nn;

constexpr int kEncThreadsMax = 256;
constexpr int kEncMaxCtas = 8;           // the portable cluster size
constexpr int kEncTokensPerCta = 16;     // a row gets another CTA for every 16 tokens, up to kEncMaxCtas
constexpr int kEncUnroll = 8;            // tokens in flight per thread
constexpr int kEncMaxSlice = (kEncoderMaxS + kEncMaxCtas - 1) / kEncMaxCtas;

static int encoder_ctas(int S) {
  const int c = (S + kEncTokensPerCta - 1) / kEncTokensPerCta;
  return c < 1 ? 1 : c > kEncMaxCtas ? kEncMaxCtas : c;
}

// one thread per column quad up to 256 threads (H = 1024); a function of H alone, like every reduction order below
static int encoder_threads(int H) {
  const int t = ((H + 3) / 4 + 31) / 32 * 32;
  return t > kEncThreadsMax ? kEncThreadsMax : t;
}

// block-wide sum in a fixed tree (warp butterflies, then warp 0 over the warp sums): the same bits for the same blockDim
__device__ float enc_block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // an earlier call may still be reading red[0]
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.f;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[0] = v;
  }
  __syncthreads();
  return red[0];
}

template <bool kVec>
__global__ void __launch_bounds__(kEncThreadsMax) encoder_head_kernel(const float* __restrict__ hidden, const float* __restrict__ pooled,
                                                                      EncoderInputs in, int S, int H, int ctas, EncoderOutputs o) {
  extern __shared__ float part[];  // [H] fp32 sums of this CTA's unmasked tokens; rank 0 then holds the row's mean there
  __shared__ float red[32];
  __shared__ unsigned char live[kEncMaxSlice];
  const int rank = (int)(blockIdx.x % (unsigned)ctas);  // = the rank in the cluster: clusters are (ctas, 1, 1)
  const int64_t row = blockIdx.x / (unsigned)ctas;
  const int T = (S + ctas - 1) / ctas;
  const int p0 = min(S, rank * T), p1 = min(S, p0 + T);
  const bool mean = o.mean != nullptr;
  // the request row as the embedding reads it (no mask input: [PAD] = id 0)
  const int* mrow = mean ? (in.mask ? in.mask : in.ids) + row * in.stride : nullptr;
  // launched after the op that writes the hidden states or the pooler, which are that grid's output
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const float* h = hidden ? hidden + row * S * H : nullptr;
  float* seq = o.sequence ? o.sequence + row * o.sequence_ld : nullptr;
  if (seq || mean) {
    if (mean) {
      for (int p = p0 + (int)threadIdx.x; p < p1; p += blockDim.x) live[p - p0] = __ldg(mrow + p) != 0;
      __syncthreads();
    }
    if (kVec) {
      const int Q = H >> 2;
      for (int q = threadIdx.x; q < Q; q += blockDim.x) {
        const float4* src = reinterpret_cast<const float4*>(h) + q;  // token p at src[p * Q]
        float4* dst = seq ? reinterpret_cast<float4*>(seq) + q : nullptr;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int p = p0; p < p1; p += kEncUnroll) {
          const int n = min(kEncUnroll, p1 - p);
          float4 v[kEncUnroll];
#pragma unroll
          for (int u = 0; u < kEncUnroll; ++u)
            if (u < n) v[u] = __ldg(src + (p + u) * Q);
#pragma unroll
          for (int u = 0; u < kEncUnroll; ++u) {
            if (u >= n) break;
            if (dst) __stcs(dst + (p + u) * Q, v[u]);
            if (mean && live[p + u - p0]) {
              acc.x += v[u].x;
              acc.y += v[u].y;
              acc.z += v[u].z;
              acc.w += v[u].w;
            }
          }
        }
        if (mean) {
          part[4 * q] = acc.x;
          part[4 * q + 1] = acc.y;
          part[4 * q + 2] = acc.z;
          part[4 * q + 3] = acc.w;
        }
      }
    } else {
      for (int c = threadIdx.x; c < H; c += blockDim.x) {
        float acc = 0.f;
        for (int p = p0; p < p1; p += kEncUnroll) {
          const int n = min(kEncUnroll, p1 - p);
          float v[kEncUnroll];
#pragma unroll
          for (int u = 0; u < kEncUnroll; ++u)
            if (u < n) v[u] = __ldg(h + (p + u) * H + c);
#pragma unroll
          for (int u = 0; u < kEncUnroll; ++u) {
            if (u >= n) break;
            if (seq) __stcs(seq + (p + u) * H + c, v[u]);
            if (mean && live[p + u - p0]) acc += v[u];
          }
        }
        if (mean) part[c] = acc;
      }
    }
  }
  if (mean) {
    if (ctas > 1) {
      cg::cluster_group cl = cg::this_cluster();
      cl.sync();  // every rank's partials are in its shared memory
      if (rank == 0)
        for (int c = threadIdx.x; c < H; c += blockDim.x) {
          float t = part[c];
          for (int r = 1; r < ctas; ++r) t += cl.map_shared_rank(part, r)[c];
          part[c] = t;
        }
      cl.sync();  // the other ranks keep their shared memory until rank 0 has read it
    } else {
      __syncthreads();  // the partials were written column quad by column quad
    }
  }
  if (rank != 0) return;

  if (mean) {
    float cnt = 0.f;
    for (int p = threadIdx.x; p < S; p += blockDim.x) cnt += __ldg(mrow + p) != 0 ? 1.f : 0.f;
    cnt = enc_block_sum(cnt, red);           // exact: an integer <= S
    const float den = cnt > 0.f ? cnt : 1e-9f;  // max(count, 1e-9): a fully masked row's zero sums stay 0
    float ss = 0.f;
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      const float m = part[c] / den;
      part[c] = m;
      ss = fmaf(m, m, ss);
    }
    const float nrm = o.normalize_mean ? fmaxf(sqrtf(enc_block_sum(ss, red)), 1e-12f) : 1.f;
    float* y = o.mean + row * o.mean_ld;
    for (int c = threadIdx.x; c < H; c += blockDim.x) y[c] = o.normalize_mean ? part[c] / nrm : part[c];
  }
  if (o.cls) {  // token 0's hidden state, which rank 0's slice holds
    float ss = 0.f;
    if (o.normalize_cls)
      for (int c = threadIdx.x; c < H; c += blockDim.x) {
        const float v = __ldg(h + c);
        ss = fmaf(v, v, ss);
      }
    const float nrm = o.normalize_cls ? fmaxf(sqrtf(enc_block_sum(ss, red)), 1e-12f) : 1.f;
    float* y = o.cls + row * o.cls_ld;
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      const float v = __ldg(h + c);
      y[c] = o.normalize_cls ? v / nrm : v;
    }
  }
  if (o.pooled) {
    const float* x = pooled + row * H;
    float* y = o.pooled + row * o.pooled_ld;
    for (int c = threadIdx.x; c < H; c += blockDim.x) y[c] = __ldg(x + c);
  }
}

cudaError_t launch_encoder_head(const float* hidden, const float* pooled, const EncoderInputs& in, int rows, int S, int H,
                                const EncoderOutputs& o, cudaStream_t s) {
  if (!encoder_head_supported(S, H) || rows < 0) return cudaErrorInvalidValue;
  if ((!hidden && (o.sequence || o.cls || o.mean)) || (!pooled && o.pooled)) return cudaErrorInvalidValue;
  if (o.mean && (!in.ids || in.stride < S)) return cudaErrorInvalidValue;
  if (rows == 0) return cudaSuccess;
  // only sequence_output and mean_embedding stream all S tokens; cls_embedding and pooled_output need rank 0 alone
  const int ctas = (o.sequence || o.mean) ? encoder_ctas(S) : 1;
  const bool vec = H % 4 == 0 && ((uintptr_t)hidden & 15) == 0 &&
                   (!o.sequence || (((uintptr_t)o.sequence & 15) == 0 && o.sequence_ld % 4 == 0));
  // programmatic dependent launch (on unless TFSC_PDL=0), as the other heads: set up while the last op drains
  static const bool pdl = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)rows * (unsigned)ctas);
  cfg.blockDim = dim3(encoder_threads(H));
  cfg.dynamicSmemBytes = (size_t)H * sizeof(float);  // 32 KB at H = 8192: no opt-in needed
  cfg.stream = s;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (ctas > 1) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = (unsigned)ctas;
    at[na].val.clusterDim.y = 1;
    at[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl) {
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  cudaError_t e = vec ? cudaLaunchKernelEx(&cfg, encoder_head_kernel<true>, hidden, pooled, in, S, H, ctas, o)
                      : cudaLaunchKernelEx(&cfg, encoder_head_kernel<false>, hidden, pooled, in, S, H, ctas, o);
  g_launches_nn++;
  return e;
}

}  // namespace tfsc
