// X2, cluster-pair kernel of the fused dense pass: the DEFAULT for <= 8 rows per pass since round 2 (tfsc_k_dense_variant 0 / 5).
//
//   y[R,N] = act(x[R,K] W[K,N] + b),  R <= 8 rows per pass, fp32.
//
// What it changes against dense_stream_kernel / dense_bulk_kernel (kernels.cu): the split-K tail. Those kernels split K
// eight ways across independent CTAs and fold the partials through an L2 workspace (partials -> fence -> atomic counter
// -> last CTA of the strip re-reads 8 partials), a serial tail of several microseconds that grows with R. Here a
// thread-block CLUSTER of two CTAs (one TPC) owns a 128-column strip, each CTA streams one half of K, and the two halves
// meet in distributed shared memory: no workspace, no atomics, no second pass -- rank 0 reads rank 1's [R,128] result
// with ld.shared::cluster, adds it in fixed order (bit-reproducible), applies bias / ReLU and stores y.
//   * W: one 2-D TMA box {128 n, 64 k} = 32 KB per stage (tensor map over W[K,N], no swizzle; rows beyond K and columns
//     beyond N arrive as zeros), 4-stage mbarrier ring = 128 KB in flight per SM.
//   * x: streamed too (a half of K does not fit beside the ring): chunks of 1024 k, R bulk copies each, double-buffered.
//   * 16 consumer warps: lane = float4 column group of the strip, warp = k-lane (4 consecutive k rows of every stage,
//     so one broadcast LDS.128 yields x[r][k..k+3]); paired-column accumulation; k-lane reduction through shared memory.
//   * programmatic dependent launch (TFSC_PDL=1): W streaming starts before griddepcontrol.wait, x after it.
// Grid: 2 * ceil(N/128) CTAs (144 for N = 9216) in clusters of 2.
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "kernels.h"
#include "tc_ptx.cuh"

namespace tfsc {

std::atomic<int64_t> g_launches_cl{0};

namespace cl {
constexpr int STRIP = 128;             // columns per cluster
constexpr int SK = 64;                 // k rows per W stage
constexpr int STAGES = 4;
constexpr int STAGE_BYTES = STRIP * SK * 4;   // 32 KB
constexpr int XC = 1024;               // k per x chunk
constexpr int CONSUMERS = 512;         // 32 column groups x 16 k-lanes
constexpr int THREADS = CONSUMERS + 32;
constexpr int KLANES = CONSUMERS / 32;
}  // namespace cl

template <int R>
struct ClSmem {
  static constexpr int RING = cl::STAGES * cl::STAGE_BYTES;      // 128 KB
  static constexpr int XS = 2 * R * cl::XC * 4;                  // double-buffered x chunks
  static constexpr int TOTAL = RING + XS + 1024;                 // + alignment slack
};

__device__ __forceinline__ void cl_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void cl_lds_2x64(uint32_t saddr, uint64_t& lo, uint64_t& hi) {
  asm volatile("ld.shared.v2.b64 {%0,%1}, [%2];" : "=l"(lo), "=l"(hi) : "r"(saddr));
}
__device__ __forceinline__ void cl_ffma2(uint64_t& acc, float xs, uint64_t w2) {
  float a0, a1, w0, w1;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(acc));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(w0), "=f"(w1) : "l"(w2));
  asm("mov.b64 %0, {%1, %2};" : "=l"(acc) : "f"(fmaf(xs, w0, a0)), "f"(fmaf(xs, w1, a1)));
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t local_saddr, uint32_t cta_rank) {
  uint32_t raddr;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(local_saddr), "r"(cta_rank));
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(raddr) : "memory");
  return v;
}

template <int R>
__global__ void __launch_bounds__(cl::THREADS, 1)
dense_cluster_kernel(const __grid_constant__ CUtensorMap wmap, const float* __restrict__ x, const float* __restrict__ bias,
                     float* __restrict__ y, int rows, int K, int N, int relu, int k_half) {
  using S = ClSmem<R>;
  extern __shared__ __align__(1024) uint8_t cl_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(cl_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                        // [STAGES][SK][STRIP] fp32
  float* xs = reinterpret_cast<float*>(smem + S::RING);        // [2][R][XC]
  __shared__ __align__(8) uint64_t full[cl::STAGES];
  __shared__ __align__(8) uint64_t empty[cl::STAGES];
  __shared__ __align__(8) uint64_t xfull[2];
  __shared__ __align__(8) uint64_t xempty[2];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t rank = cluster_ctarank();                     // 0 / 1: which half of K
  const int strip = blockIdx.x >> 1;
  const int k_begin = (int)rank * k_half;
  const int k_end = min(K, k_begin + k_half);
  const int kc = max(0, k_end - k_begin);
  const int n_stage = (kc + cl::SK - 1) / cl::SK;
  const int n_chunk = (kc + cl::XC - 1) / cl::XC;
  constexpr int STAGES_PER_CHUNK = cl::XC / cl::SK;            // 16

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < cl::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], cl::KLANES);
    }
    mbar_init(&xfull[0], 1);
    mbar_init(&xfull[1], 1);
    mbar_init(&xempty[0], cl::KLANES);
    mbar_init(&xempty[1], cl::KLANES);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
  }
  // x buffers start as zeros: rows >= `rows` are never copied, and the tail of the last chunk meets W rows that the
  // tensor map zero-fills -- 0 * stale must not be NaN
  for (int i = tid; i < 2 * R * cl::XC; i += cl::THREADS) xs[i] = 0.f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // no-op without the PDL launch attribute

  uint64_t acc[R][2];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r][0] = acc[r][1] = 0ull;

  if (warp == cl::KLANES) {
    // ===================== producer: W stages (TMA 2-D boxes) and x chunks (bulk copies) =====================
    auto issue_x_chunk = [&](int c) {
      const int bsel = c & 1, k0 = c * cl::XC, len = min(cl::XC, kc - k0);
      if (c >= 2) mbar_wait(&xempty[bsel], ((c >> 1) - 1) & 1);   // consumers finished chunk c-2 (same buffer)
      if (lane == 0) mbar_expect_tx(&xfull[bsel], (uint32_t)(rows * len * 4));
      __syncwarp();
      if (lane < rows)
        cl_bulk_g2s(xs + ((size_t)bsel * R + lane) * cl::XC, x + (size_t)lane * K + k_begin + k0, (uint32_t)(len * 4), &xfull[bsel]);
    };
    const int primed = min(cl::STAGES, n_stage) - 1;             // stage index after which the ring is full
    for (int it = 0; it < n_stage; ++it) {
      const int s = it % cl::STAGES;
      if (it >= cl::STAGES) mbar_wait(&empty[s], ((it / cl::STAGES) - 1) & 1);
      if (lane == 0) {
        mbar_expect_tx(&full[s], cl::STAGE_BYTES);
        tma_load_2d(ring + s * cl::STAGE_BYTES, &wmap, &full[s], strip * cl::STRIP, k_begin + it * cl::SK);
      }
      __syncwarp();
      if (it == primed) {
        // W never depends on the previous kernel of the stream, x (its output) does: with programmatic dependent launch
        // the ring fills under the previous kernel's tail and only the first x chunk waits for it
        asm volatile("griddepcontrol.wait;" ::: "memory");
        issue_x_chunk(0);
      }
      // chunk c >= 1 is requested while chunk c-1 is being consumed (at its 5th stage)
      if ((it % STAGES_PER_CHUNK) == cl::STAGES && it / STAGES_PER_CHUNK + 1 < n_chunk) issue_x_chunk(it / STAGES_PER_CHUNK + 1);
    }
    if (n_stage == 0) asm volatile("griddepcontrol.wait;" ::: "memory");
  } else {
    // ===================== consumers: warp = k-lane (rows 4*warp .. 4*warp+3 of every stage), lane = column group =====
    const uint32_t ring_s = smem_u32(ring) + (uint32_t)lane * 16u + (uint32_t)(warp * 4 * cl::STRIP * 4);
    const uint32_t xs_s = smem_u32(xs);
    for (int it = 0; it < n_stage; ++it) {
      const int s = it % cl::STAGES;
      const int c = it / STAGES_PER_CHUNK, b = c & 1;
      if ((it % STAGES_PER_CHUNK) == 0) mbar_wait(&xfull[b], (c >> 1) & 1);
      const int kq = (it % STAGES_PER_CHUNK) * cl::SK + warp * 4;   // this warp's k offset inside the chunk
      if (it == n_stage - 1) {
        // last stage: x positions beyond the valid length meet W rows the tensor map zero-filled; make them zeros too
        // (stale data from an earlier chunk could hold Inf / NaN). Each warp only ever reads its own offsets.
        const int valid = kc - c * cl::XC;
        if (kq + 4 > valid && lane < R) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (kq + j >= valid) xs[((size_t)b * R + lane) * cl::XC + kq + j] = 0.f;
        }
        __syncwarp();
      }
      mbar_wait(&full[s], (it / cl::STAGES) & 1);
      const uint32_t wbase = ring_s + (uint32_t)(s * cl::STAGE_BYTES);
      const uint32_t xk = xs_s + (uint32_t)((b * R * cl::XC + kq) * 4);
      uint64_t w[4][2];
#pragma unroll
      for (int j = 0; j < 4; ++j) cl_lds_2x64(wbase + (uint32_t)(j * cl::STRIP * 4), w[j][0], w[j][1]);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float4 xv = lds_f4(xk + (uint32_t)(r * cl::XC * 4));   // x[r][k..k+3], broadcast
        cl_ffma2(acc[r][0], xv.x, w[0][0]); cl_ffma2(acc[r][1], xv.x, w[0][1]);
        cl_ffma2(acc[r][0], xv.y, w[1][0]); cl_ffma2(acc[r][1], xv.y, w[1][1]);
        cl_ffma2(acc[r][0], xv.z, w[2][0]); cl_ffma2(acc[r][1], xv.z, w[2][1]);
        cl_ffma2(acc[r][0], xv.w, w[3][0]); cl_ffma2(acc[r][1], xv.w, w[3][1]);
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty[s]);
        if ((it % STAGES_PER_CHUNK) == STAGES_PER_CHUNK - 1 || it == n_stage - 1) mbar_arrive(&xempty[b]);
      }
    }
  }

  // ---- k-lane reduction through shared memory (the ring is idle: every full barrier was waited on) ----
  __syncthreads();
  // every thread that is about to write y observes the completion of the prerequisite grid itself (y may be a buffer
  // the previous kernel of the stream still read); long satisfied by now, no-op without the PDL launch attribute
  asm volatile("griddepcontrol.wait;" ::: "memory");
  float* red = reinterpret_cast<float*>(ring);                     // [KLANES][R][STRIP]   (64 KB at R = 8)
  float* res = red + cl::KLANES * R * cl::STRIP;                   // [R][STRIP]           (4 KB at R = 8)
  if (warp < cl::KLANES) {
#pragma unroll
    for (int r = 0; r < R; ++r)
      *reinterpret_cast<ulonglong2*>(red + ((size_t)(warp * R + r) * cl::STRIP) + lane * 4) = make_ulonglong2(acc[r][0], acc[r][1]);
  }
  __syncthreads();
  constexpr int ITEMS = R * (cl::STRIP / 4);                       // float4 items of the [R, 128] result
  for (int idx = tid; idx < ITEMS; idx += cl::THREADS) {
    const int r = idx / (cl::STRIP / 4), c4 = idx - r * (cl::STRIP / 4);
    float4 sacc = *reinterpret_cast<const float4*>(red + (size_t)r * cl::STRIP + c4 * 4);
#pragma unroll
    for (int l = 1; l < cl::KLANES; ++l) {
      const float4 t = *reinterpret_cast<const float4*>(red + ((size_t)(l * R + r) * cl::STRIP) + c4 * 4);
      sacc.x += t.x; sacc.y += t.y; sacc.z += t.z; sacc.w += t.w;
    }
    *reinterpret_cast<float4*>(res + (size_t)r * cl::STRIP + c4 * 4) = sacc;
  }
  // ---- the two halves of K meet in distributed shared memory ----
  cluster_sync_all();                                              // both CTAs published `res`
  if (rank == 0) {
    const uint32_t res_s = smem_u32(res);
    for (int idx = tid; idx < ITEMS; idx += cl::THREADS) {
      const int r = idx / (cl::STRIP / 4), c4 = idx - r * (cl::STRIP / 4);
      const int col = strip * cl::STRIP + c4 * 4;
      if (r >= rows || col >= N) continue;
      float4 a = *reinterpret_cast<const float4*>(res + (size_t)r * cl::STRIP + c4 * 4);
      const float4 o = ld_dsmem_f4(res_s + (uint32_t)((r * cl::STRIP + c4 * 4) * 4), 1u);
      const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
      a.x = a.x + o.x + bv.x; a.y = a.y + o.y + bv.y; a.z = a.z + o.z + bv.z; a.w = a.w + o.w + bv.w;
      if (relu) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f); }
      *reinterpret_cast<float4*>(y + (size_t)r * N + col) = a;
    }
  }
  cluster_sync_all();                                              // rank 1's shared memory stays alive until rank 0 has read it
}

// --------------------------------------------------------------------------------- host side ----
struct ClKey {
  const void* w;
  int k, n;
  bool operator==(const ClKey& o) const { return w == o.w && k == o.k && n == o.n; }
};
struct ClKeyHash {
  size_t operator()(const ClKey& m) const { return std::hash<const void*>()(m.w) ^ ((size_t)m.k * 1315423911u) ^ ((size_t)m.n << 20); }
};

static bool get_cl_map(const float* w, int k, int n, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<ClKey, CUtensorMap, ClKeyHash> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find({w, k, n});
  if (it != cache.end()) {
    *out = it->second;
    return true;
  }
  EncodeTiledFn enc = tc_encode_fn();
  if (!enc) return false;
  CUtensorMap m;
  const cuuint64_t gdim[2] = {(cuuint64_t)n, (cuuint64_t)k};
  const cuuint64_t gstride[1] = {(cuuint64_t)n * 4};
  const cuuint32_t box[2] = {(cuuint32_t)cl::STRIP, (cuuint32_t)cl::SK};
  const cuuint32_t estr[2] = {1, 1};
  if (enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(w), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return false;
  if (cache.size() > 4096) cache.clear();
  cache[{w, k, n}] = m;
  *out = m;
  return true;
}

bool dense_cluster_supported(int rows, int k, int n, const float* w, const float* x, const float* bias, const float* y) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return rows >= 1 && rows <= 8 && n % 4 == 0 && k % 4 == 0 && k >= 2 * cl::SK && al16(w) && al16(x) && al16(bias) && al16(y) &&
         tc_encode_fn() != nullptr;
}

template <int R>
static cudaError_t launch_cl_r(const CUtensorMap& map, const float* x, const float* bias, float* y, int rows, int k, int n, bool relu,
                               cudaStream_t s) {
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(dense_cluster_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, ClSmem<R>::TOTAL);
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  static const bool pdl = [] {  // programmatic dependent launch is on unless TFSC_PDL=0
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  const int strips = (n + cl::STRIP - 1) / cl::STRIP;
  int k_half = ((k + 1) / 2 + cl::SK - 1) / cl::SK * cl::SK;   // rank 0 takes [0, k_half), rank 1 the rest
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * strips);
  cfg.blockDim = dim3(cl::THREADS);
  cfg.dynamicSmemBytes = ClSmem<R>::TOTAL;
  cfg.stream = s;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = 2;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 2 : 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, dense_cluster_kernel<R>, map, x, bias, y, rows, k, n, relu ? 1 : 0, k_half);
  g_launches_cl++;
  return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t launch_dense_cluster(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n, bool relu,
                                 cudaStream_t s) {
  CUtensorMap map;
  if (!get_cl_map(w, k, n, &map)) return cudaErrorNotSupported;
  if (rows == 1) return launch_cl_r<1>(map, x, bias, y, rows, k, n, relu, s);
  if (rows == 2) return launch_cl_r<2>(map, x, bias, y, rows, k, n, relu, s);
  if (rows <= 4) return launch_cl_r<4>(map, x, bias, y, rows, k, n, relu, s);
  return launch_cl_r<8>(map, x, bias, y, rows, k, n, relu, s);
}

}  // namespace tfsc
