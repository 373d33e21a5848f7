// X2, cluster-pair kernel of the fused dense pass: the DEFAULT for <= 8 rows per pass (tfsc_k_dense_variant 0 / 5).
//
//   y[R,N] = act(x[R,K] W[K,N] + b),  R <= 8 rows per pass, fp32.
//
// What it changes against dense_stream_kernel / dense_bulk_kernel (kernels.cu): the split-K tail. Those kernels split K
// eight ways across independent CTAs and fold the partials through an L2 workspace (partials -> fence -> atomic counter
// -> last CTA of the strip re-reads 8 partials), a serial tail of several microseconds that grows with R. Here a
// thread-block CLUSTER of two CTAs (one TPC) owns a column strip, each CTA streams one half of K, and the two halves
// meet in distributed shared memory: no workspace, no atomics, no second pass -- rank 0 reads rank 1's [R,strip] result
// with ld.shared::cluster, adds it in fixed order (bit-reproducible), applies bias / ReLU and stores y.
//   * grid: one wave. The launch never has more clusters than cudaOccupancyMaxActiveClusters reports for it (66 two-CTA
//     clusters on a 132-SM H100, one CTA per SM), and the strip width is sized from N and that count: a multiple of 16
//     columns, at most 144 (N = 9216: 64 strips of 144 columns, 128 CTAs). A 128-column strip would give 72 clusters, and
//     the last 6 would run as a second wave on 12 SMs. When N needs more than 66 strips of 144, a cluster loops over them.
//   * W: one 2-D TMA box {strip, 64 k} (36 KB at 144 columns) per stage (tensor map over W[K,N], no swizzle; rows beyond K
//     and columns beyond N arrive as zeros), 4-stage mbarrier ring = up to 144 KB in flight per SM.
//   * x: streamed too (a half of K does not fit beside the ring): chunks of 1024 k, R bulk copies each, double-buffered.
//   * 576 consumer threads = 16 k-lanes x 36 float4 column groups: k-lane = 4 consecutive k rows of every stage (one
//     broadcast LDS.128 yields x[r][k..k+3]), paired-column accumulation, k-lane reduction through shared memory in k-lane
//     order. The K split and the k-lane rows do not depend on the strip width, so every column sums in the same order.
//   * programmatic dependent launch (TFSC_PDL=1): W streaming starts before griddepcontrol.wait, x after it.
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
constexpr int STRIP_MAX = 144;         // columns per cluster strip (runtime width: a multiple of 16, at most this)
constexpr int GROUPS = STRIP_MAX / 4;  // float4 column groups of the widest strip
constexpr int SK = 64;                 // k rows per W stage
constexpr int STAGES = 4;
constexpr int STAGE_MAX_BYTES = STRIP_MAX * SK * 4;   // 36 KB
constexpr int XC = 1024;               // k per x chunk
constexpr int KLANES = 16;             // 4 consecutive k rows of every stage each
constexpr int CONSUMERS = GROUPS * KLANES;   // 576: thread = (k-lane, column group)
constexpr int CONS_WARPS = CONSUMERS / 32;   // 18
constexpr int THREADS = CONSUMERS + 32;
}  // namespace cl

template <int R>
struct ClSmem {
  static constexpr int RING = cl::STAGES * cl::STAGE_MAX_BYTES;  // 144 KB
  static constexpr int XS = 2 * R * cl::XC * 4;                  // double-buffered x chunks
  static constexpr int TOTAL = RING + XS + 1024;                 // + alignment slack
  static_assert((cl::KLANES + 1) * R * cl::STRIP_MAX * 4 <= RING, "the k-lane reduction overlays the ring");
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

// Grid: one wave of clusters (gridDim.x / 2 <= the co-resident cluster count); cluster c owns strips c, c + clusters, ...
// of `sw` columns each.
template <int R>
__global__ void __launch_bounds__(cl::THREADS, 1)
dense_cluster_kernel(const __grid_constant__ CUtensorMap wmap, const float* __restrict__ x, const float* __restrict__ bias,
                     float* __restrict__ y, int rows, int K, int N, int relu, int k_half, int sw) {
  using S = ClSmem<R>;
  extern __shared__ __align__(1024) uint8_t cl_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(cl_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                        // [STAGES][SK][sw] fp32
  float* xs = reinterpret_cast<float*>(smem + S::RING);        // [2][R][XC]
  __shared__ __align__(8) uint64_t full[cl::STAGES];
  __shared__ __align__(8) uint64_t empty[cl::STAGES];
  __shared__ __align__(8) uint64_t xfull[2];
  __shared__ __align__(8) uint64_t xempty[2];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t rank = cluster_ctarank();                     // 0 / 1: which half of K
  const int clusters = (int)gridDim.x >> 1;
  const int strips = (N + sw - 1) / sw;
  const int stage_bytes = sw * cl::SK * 4;
  const int groups = sw >> 2;                                  // float4 column groups of a strip
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
      mbar_init(&empty[s], cl::CONS_WARPS);
    }
    mbar_init(&xfull[0], 1);
    mbar_init(&xfull[1], 1);
    mbar_init(&xempty[0], cl::CONS_WARPS);
    mbar_init(&xempty[1], cl::CONS_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
  }
  // x buffers start as zeros: rows >= `rows` are never copied
  for (int i = tid; i < 2 * R * cl::XC; i += cl::THREADS) xs[i] = 0.f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // no-op without the PDL launch attribute

  // consumer thread = (k-lane, column group): k-lane kl takes k rows 4*kl .. 4*kl+3 of every stage (as with 16 warps of
  // 32 column groups), so every output column sums in the same order whatever the strip width
  const int kl = tid / cl::GROUPS, grp = tid - kl * cl::GROUPS;
  // ring / x-chunk barrier phases run on across the strips of this cluster
  int it_base = 0, c_base = 0;
  for (int strip = (int)blockIdx.x >> 1; strip < strips; strip += clusters) {
    uint64_t acc[R][2];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r][0] = acc[r][1] = 0ull;

    if (warp == cl::CONS_WARPS) {
      // ===================== producer: W stages (TMA 2-D boxes) and x chunks (bulk copies) =====================
      auto issue_x_chunk = [&](int c) {
        const int gc = c_base + c, bsel = gc & 1, k0 = c * cl::XC, len = min(cl::XC, kc - k0);
        if (gc >= 2) mbar_wait(&xempty[bsel], ((gc >> 1) - 1) & 1);   // consumers finished chunk gc-2 (same buffer)
        if (lane == 0) mbar_expect_tx(&xfull[bsel], (uint32_t)(rows * len * 4));
        __syncwarp();
        if (lane < rows)
          cl_bulk_g2s(xs + ((size_t)bsel * R + lane) * cl::XC, x + (size_t)lane * K + k_begin + k0, (uint32_t)(len * 4), &xfull[bsel]);
      };
      const int primed = min(cl::STAGES, n_stage) - 1;             // stage index after which the ring is full
      for (int it = 0; it < n_stage; ++it) {
        const int gi = it_base + it, s = gi % cl::STAGES;
        if (gi >= cl::STAGES) mbar_wait(&empty[s], ((gi / cl::STAGES) - 1) & 1);
        if (lane == 0) {
          mbar_expect_tx(&full[s], (uint32_t)stage_bytes);
          tma_load_2d(ring + s * stage_bytes, &wmap, &full[s], strip * sw, k_begin + it * cl::SK);
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
      // ===================== consumers =====================
      const bool active = grp < groups;
      const uint32_t ring_s = smem_u32(ring) + (uint32_t)grp * 16u + (uint32_t)(kl * 4 * sw * 4);
      const uint32_t xs_s = smem_u32(xs);
      // one stage: x positions at or beyond `valid` (last stage only) meet W rows the tensor map zero-filled; they count as
      // zeros (stale x from an earlier chunk could hold Inf / NaN)
      auto consume = [&](int it, bool tail) {
        const int gi = it_base + it, s = gi % cl::STAGES;
        const int c = it / STAGES_PER_CHUNK, b = (c_base + c) & 1;
        if ((it % STAGES_PER_CHUNK) == 0) mbar_wait(&xfull[b], ((c_base + c) >> 1) & 1);
        const int kq = (it % STAGES_PER_CHUNK) * cl::SK + kl * 4;   // this k-lane's k offset inside the chunk
        mbar_wait(&full[s], (gi / cl::STAGES) & 1);
        if (active) {
          const uint32_t wbase = ring_s + (uint32_t)(s * stage_bytes);
          const uint32_t xk = xs_s + (uint32_t)((b * R * cl::XC + kq) * 4);
          const int valid = kc - c * cl::XC - kq;
          uint64_t w[4][2];
#pragma unroll
          for (int j = 0; j < 4; ++j) cl_lds_2x64(wbase + (uint32_t)(j * sw * 4), w[j][0], w[j][1]);
#pragma unroll
          for (int r = 0; r < R; ++r) {
            float4 xv = lds_f4(xk + (uint32_t)(r * cl::XC * 4));   // x[r][k..k+3]
            if (tail) {
              if (valid < 4) xv.w = 0.f;
              if (valid < 3) xv.z = 0.f;
              if (valid < 2) xv.y = 0.f;
              if (valid < 1) xv.x = 0.f;
            }
            cl_ffma2(acc[r][0], xv.x, w[0][0]); cl_ffma2(acc[r][1], xv.x, w[0][1]);
            cl_ffma2(acc[r][0], xv.y, w[1][0]); cl_ffma2(acc[r][1], xv.y, w[1][1]);
            cl_ffma2(acc[r][0], xv.z, w[2][0]); cl_ffma2(acc[r][1], xv.z, w[2][1]);
            cl_ffma2(acc[r][0], xv.w, w[3][0]); cl_ffma2(acc[r][1], xv.w, w[3][1]);
          }
        }
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&empty[s]);
          if ((it % STAGES_PER_CHUNK) == STAGES_PER_CHUNK - 1 || it == n_stage - 1) mbar_arrive(&xempty[b]);
        }
      };
      for (int it = 0; it + 1 < n_stage; ++it) consume(it, false);
      if (n_stage > 0) consume(n_stage - 1, true);
    }
    it_base += n_stage;
    c_base += n_chunk;

    // ---- k-lane reduction through shared memory (the ring is idle: every full barrier was waited on) ----
    __syncthreads();
    // every thread that is about to write y observes the completion of the prerequisite grid itself (y may be a buffer
    // the previous kernel of the stream still read); long satisfied by now, no-op without the PDL launch attribute
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float* red = reinterpret_cast<float*>(ring);                     // [KLANES][R][sw]
    float* res = red + cl::KLANES * R * sw;                          // [R][sw]
    if (warp < cl::CONS_WARPS && grp < groups) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        *reinterpret_cast<ulonglong2*>(red + ((size_t)(kl * R + r) * sw) + grp * 4) = make_ulonglong2(acc[r][0], acc[r][1]);
    }
    __syncthreads();
    const int items = R * groups;                                    // float4 items of the [R, sw] result
    for (int idx = tid; idx < items; idx += cl::THREADS) {
      const int r = idx / groups, c4 = idx - r * groups;
      float4 sacc = *reinterpret_cast<const float4*>(red + (size_t)r * sw + c4 * 4);
#pragma unroll
      for (int l = 1; l < cl::KLANES; ++l) {
        const float4 t = *reinterpret_cast<const float4*>(red + ((size_t)(l * R + r) * sw) + c4 * 4);
        sacc.x += t.x; sacc.y += t.y; sacc.z += t.z; sacc.w += t.w;
      }
      *reinterpret_cast<float4*>(res + (size_t)r * sw + c4 * 4) = sacc;
    }
    // ---- the two halves of K meet in distributed shared memory ----
    cluster_sync_all();                                              // both CTAs published `res`
    if (rank == 0) {
      const uint32_t res_s = smem_u32(res);
      for (int idx = tid; idx < items; idx += cl::THREADS) {
        const int r = idx / groups, c4 = idx - r * groups;
        const int col = strip * sw + c4 * 4;
        if (r >= rows || col >= N) continue;
        float4 a = *reinterpret_cast<const float4*>(res + (size_t)r * sw + c4 * 4);
        const float4 o = ld_dsmem_f4(res_s + (uint32_t)((r * sw + c4 * 4) * 4), 1u);
        const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
        a.x = a.x + o.x + bv.x; a.y = a.y + o.y + bv.y; a.z = a.z + o.z + bv.z; a.w = a.w + o.w + bv.w;
        if (relu) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f); }
        *reinterpret_cast<float4*>(y + (size_t)r * N + col) = a;
      }
    }
    // rank 1's shared memory stays alive until rank 0 has read it; the ring is reused by the next strip after this
    cluster_sync_all();
  }
}

// --------------------------------------------------------------------------------- host side ----
struct ClKey {
  const void* w;
  int k, n, sw;
  bool operator==(const ClKey& o) const { return w == o.w && k == o.k && n == o.n && sw == o.sw; }
};
struct ClKeyHash {
  size_t operator()(const ClKey& m) const {
    return std::hash<const void*>()(m.w) ^ ((size_t)m.k * 1315423911u) ^ ((size_t)m.n << 20) ^ ((size_t)m.sw << 44);
  }
};

static bool get_cl_map(const float* w, int k, int n, int sw, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<ClKey, CUtensorMap, ClKeyHash> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find({w, k, n, sw});
  if (it != cache.end()) {
    *out = it->second;
    return true;
  }
  EncodeTiledFn enc = tc_encode_fn();
  if (!enc) return false;
  CUtensorMap m;
  const cuuint64_t gdim[2] = {(cuuint64_t)n, (cuuint64_t)k};
  const cuuint64_t gstride[1] = {(cuuint64_t)n * 4};
  const cuuint32_t box[2] = {(cuuint32_t)sw, (cuuint32_t)cl::SK};
  const cuuint32_t estr[2] = {1, 1};
  if (enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(w), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return false;
  if (cache.size() > 4096) cache.clear();
  cache[{w, k, n, sw}] = m;
  *out = m;
  return true;
}

bool dense_cluster_supported(int rows, int k, int n, const float* w, const float* x, const float* bias, const float* y) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return rows >= 1 && rows <= 8 && n % 4 == 0 && k % 4 == 0 && k >= 2 * cl::SK && al16(w) && al16(x) && al16(bias) && al16(y) &&
         tc_encode_fn() != nullptr;
}

static bool pdl_on() {  // programmatic dependent launch is on unless TFSC_PDL=0
  static const bool pdl = [] {
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  return pdl;
}

static void cl_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute (&at)[2], int R_smem, int clusters, cudaStream_t s) {
  cfg = {};
  cfg.gridDim = dim3(2 * clusters);
  cfg.blockDim = dim3(cl::THREADS);
  cfg.dynamicSmemBytes = R_smem;
  cfg.stream = s;
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = 2;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_on() ? 2 : 1;
}

// Per device and row template: the smem attribute is set and the number of 2-CTA clusters that are co-resident
// (cudaOccupancyMaxActiveClusters for this exact launch configuration; 66 on a 132-SM H100) is cached. The grid never
// exceeds it, so every pass runs in one wave.
template <int R>
static cudaError_t cl_active_clusters(int* out) {
  static int cached[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (cached[dev & 63] > 0) {
    *out = cached[dev & 63];
    return cudaSuccess;
  }
  cudaError_t e = cudaFuncSetAttribute(dense_cluster_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, ClSmem<R>::TOTAL);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at[2];
  cl_config(cfg, at, ClSmem<R>::TOTAL, 1, 0);
  cfg.numAttrs = 1;   // the cluster shape alone decides co-residency
  int n = 0;
  e = cudaOccupancyMaxActiveClusters(&n, dense_cluster_kernel<R>, &cfg);
  if (e != cudaSuccess) return e;
  if (n < 1) return cudaErrorLaunchOutOfResources;
  cached[dev & 63] = n;
  *out = n;
  return cudaSuccess;
}

// Strip width for N columns over `clusters` co-resident clusters: the narrowest multiple of 16 that covers N in one strip
// per cluster, capped at STRIP_MAX (wider N: clusters loop over several strips). N = 9216 on 66 clusters: 144 columns,
// 64 strips.
static int cl_strip_width(int n, int clusters) {
  int sw = ((n + clusters - 1) / clusters + 15) / 16 * 16;
  if (sw > cl::STRIP_MAX) sw = cl::STRIP_MAX;
  if (sw < 16) sw = 16;
  return sw;
}

template <int R>
static cudaError_t launch_cl_r(const float* w, const float* x, const float* bias, float* y, int rows, int k, int n, bool relu,
                               cudaStream_t s) {
  int active = 0;
  cudaError_t e = cl_active_clusters<R>(&active);
  if (e != cudaSuccess) return e;
  const int sw = cl_strip_width(n, active);
  CUtensorMap map;
  if (!get_cl_map(w, k, n, sw, &map)) return cudaErrorNotSupported;
  const int strips = (n + sw - 1) / sw;
  const int clusters = strips < active ? strips : active;
  int k_half = ((k + 1) / 2 + cl::SK - 1) / cl::SK * cl::SK;   // rank 0 takes [0, k_half), rank 1 the rest
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at[2];
  cl_config(cfg, at, ClSmem<R>::TOTAL, clusters, s);
  e = cudaLaunchKernelEx(&cfg, dense_cluster_kernel<R>, map, x, bias, y, rows, k, n, relu ? 1 : 0, k_half, sw);
  g_launches_cl++;
  return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t dense_cluster_grid(int rows, int n, int* active_clusters, int* strip_cols) {
  int active = 0;
  cudaError_t e = rows == 1 ? cl_active_clusters<1>(&active)
                  : rows == 2 ? cl_active_clusters<2>(&active)
                  : rows <= 4 ? cl_active_clusters<4>(&active)
                              : cl_active_clusters<8>(&active);
  if (e != cudaSuccess) return e;
  *active_clusters = active;
  *strip_cols = cl_strip_width(n, active);
  return cudaSuccess;
}

cudaError_t launch_dense_cluster(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n, bool relu,
                                 cudaStream_t s) {
  if (rows == 1) return launch_cl_r<1>(w, x, bias, y, rows, k, n, relu, s);
  if (rows == 2) return launch_cl_r<2>(w, x, bias, y, rows, k, n, relu, s);
  if (rows <= 4) return launch_cl_r<4>(w, x, bias, y, rows, k, n, relu, s);
  return launch_cl_r<8>(w, x, bias, y, rows, k, n, relu, s);
}

}  // namespace tfsc
