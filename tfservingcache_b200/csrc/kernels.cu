// Executor kernels for sm_90a (H100). fp32 SIMT: the per-tenant models of the Zipf mix are run
// at batch <= 8 rows per pass, where y = xW + b is bound by streaming W from HBM once
// (intensity rows/2 FLOP/B, far below the fp32 ridge) -- so the design goal is HBM-rate
// streaming: 128-bit coalesced loads, >= 64 KB in flight per SM, one CTA per SM-sized grid,
// x staged in shared memory and broadcast, deterministic split-K reduction by the last CTA of
// each column strip (no float atomics: bit-reproducible results).
#include "kernels.h"
#include "tc_ptx.cuh"

#include <atomic>
#include <cstdlib>

namespace tfsc {

static std::atomic<int64_t> g_launches{0};
extern std::atomic<int64_t> g_launches_tc;
extern std::atomic<int64_t> g_launches_nn;
extern std::atomic<int64_t> g_launches_cl;
int64_t kernel_launch_count() { return g_launches.load() + g_launches_tc.load() + g_launches_nn.load() + g_launches_cl.load(); }

int device_sm_count() {
  static std::atomic<int> cache[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  int n = cache[dev & 63].load();
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev & 63].store(n);
  }
  return n;
}

// ------------------------------------------------------------------------------------ X1 ----
__global__ void __launch_bounds__(256) affine_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t n,
                                                     const float* __restrict__ pa, const float* __restrict__ pb) {
  const float a = __ldg(pa), b = __ldg(pb);
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n4 = n >> 2;
  const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  if (vec) {
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float4* y4 = reinterpret_cast<float4*>(y);
    for (int64_t j = i; j < n4; j += stride) {
      float4 v = __ldg(x4 + j);
      v.x = fmaf(a, v.x, b); v.y = fmaf(a, v.y, b); v.z = fmaf(a, v.z, b); v.w = fmaf(a, v.w, b);
      y4[j] = v;
    }
    for (int64_t j = (n4 << 2) + i; j < n; j += stride) y[j] = fmaf(a, x[j], b);
  } else {
    for (int64_t j = i; j < n; j += stride) y[j] = fmaf(a, x[j], b);
  }
}

cudaError_t launch_affine(const float* x, float* y, int64_t n, const float* a, const float* b, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  int64_t blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  affine_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, y, n, a, b);
  g_launches++;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ X2 ----
// Tile geometry: a CTA owns a strip of kStripCols columns (2 KB of every W row: long contiguous
// DRAM bursts) and one of `splits` K-chunks. 512 threads = 128 float4 columns x 4 k-lanes; every
// thread keeps kUnroll independent 16-byte loads in flight (64 KB per CTA).
constexpr int kThreads = 512;
constexpr int kColsPerThread = 8;                          // two adjacent 128-bit loads (32 contiguous bytes)
constexpr int kColGroups = 64;                             // 32-byte column groups per strip
constexpr int kStripCols = kColGroups * kColsPerThread;    // 512
constexpr int kKLanes = kThreads / kColGroups;             // 8
constexpr int kUnroll = 4;
constexpr int kMaxChunkK = 4096;                           // x chunk rows staged in smem (8 * 4096 * 4 B = 128 KB)

struct __align__(32) float8 { float v[8]; };

// streaming 32-byte load: no L1 allocation, L2 evict-first (W is read exactly once per pass)
__device__ __forceinline__ float8 ld_stream(const float8* p) {
  float8 r;
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3])
               : "l"(p), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4+16], %5;"
               : "=f"(r.v[4]), "=f"(r.v[5]), "=f"(r.v[6]), "=f"(r.v[7])
               : "l"(p), "l"(pol));
  return r;
}

// Programmatic dependent launch (TFSC_PDL=1; separate instantiations, the default kernels are unchanged): a dense pass may begin while the previous kernel of the stream drains its
// split-K tail. `pdl_trigger` lets the next grid start launching; `pdl_wait` blocks until every prerequisite grid has
// completed and flushed (both are no-ops for a kernel launched without the attribute). Everything that depends on the
// previous kernel (x, the shared split-K workspace, y) is touched only after pdl_wait; W never depends on it.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Workspace layout: [strips] uint32 arrival counters (self-resetting), then partial sums
// float[strips][splits][R][kStripCols].
template <int R, bool PDL = false>
__global__ void __launch_bounds__(kThreads, 1)
dense_stream_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ y, int rows, int K, int N, int relu, int splits, int chunk_k,
                    unsigned int* __restrict__ counters, float* __restrict__ partials) {
  extern __shared__ __align__(32) float smem[];
  float* xs = smem;  // [chunk_k][R]  (k-major so a broadcast LDS.128 yields 4 rows of the batch)

  const int strip = blockIdx.x;
  const int split = blockIdx.y;
  const int tid = threadIdx.x;
  const int cg = tid % kColGroups;
  const int kl = tid / kColGroups;
  const int col0 = strip * kStripCols + cg * kColsPerThread;
  const bool col_ok = col0 < N;  // N % 8 == 0 guaranteed by the host
  const int k_begin = split * chunk_k;
  const int k_end = min(K, k_begin + chunk_k);
  const int kc = max(0, k_end - k_begin);

  if (PDL) {  // TFSC_PDL=1 instantiation only: let the next grid launch early, then wait for the previous one (x, workspace)
    pdl_trigger();
    pdl_wait();
  }
  // stage x[:, k_begin:k_end] transposed into smem: xs[k][r]
  for (int idx = tid; idx < kc * R; idx += kThreads) {
    const int r = idx / kc, k = idx - r * kc;
    xs[k * R + r] = (r < rows) ? __ldg(x + (size_t)r * K + k_begin + k) : 0.f;
  }
  __syncthreads();

  float acc[R][kColsPerThread];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < kColsPerThread; ++c) acc[r][c] = 0.f;

  if (col_ok) {
    const float8* wp = reinterpret_cast<const float8*>(w + (size_t)(k_begin + kl) * N + col0);
    const size_t row_stride8 = (size_t)N / 8 * kKLanes;  // float8 units between this thread's rows
    int k = kl;
    // main loop: kUnroll rows per iteration, all loads issued before the first use
    for (; k + (kUnroll - 1) * kKLanes < kc; k += kUnroll * kKLanes) {
      float8 wv[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) wv[u] = ld_stream(wp + (size_t)u * row_stride8);
      wp += (size_t)kUnroll * row_stride8;
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const float* xr = xs + (k + u * kKLanes) * R;
        float xv[R];
        if (R % 4 == 0) {
#pragma unroll
          for (int q = 0; q < R / 4; ++q) {
            const float4 t = *reinterpret_cast<const float4*>(xr + 4 * q);
            xv[4 * q + 0] = t.x; xv[4 * q + 1] = t.y; xv[4 * q + 2] = t.z; xv[4 * q + 3] = t.w;
          }
        } else if (R == 2) {
          const float2 t = *reinterpret_cast<const float2*>(xr);
          xv[0] = t.x; xv[1] = t.y;
        } else {
#pragma unroll
          for (int r = 0; r < R; ++r) xv[r] = xr[r];
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
          for (int c = 0; c < kColsPerThread; ++c) acc[r][c] = fmaf(xv[r], wv[u].v[c], acc[r][c]);
      }
    }
    for (; k < kc; k += kKLanes) {  // tail rows
      const float8 wv = ld_stream(wp);
      wp += row_stride8;
      const float* xr = xs + k * R;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float xv = xr[r];
#pragma unroll
        for (int c = 0; c < kColsPerThread; ++c) acc[r][c] = fmaf(xv, wv.v[c], acc[r][c]);
      }
    }
  }

  // intra-CTA reduction over the k-lanes (fixed order -> deterministic), through smem
  __syncthreads();  // xs no longer needed
  float* red = smem;  // [kKLanes][R][kStripCols]
#pragma unroll
  for (int r = 0; r < R; ++r) {
    float4* dst = reinterpret_cast<float4*>(red + ((size_t)(kl * R + r) * kStripCols) + cg * kColsPerThread);
    dst[0] = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
    dst[1] = make_float4(acc[r][4], acc[r][5], acc[r][6], acc[r][7]);
  }
  __syncthreads();

  constexpr int kVecPerRow = kStripCols / 4;  // float4 per strip row
  const float4* red4 = reinterpret_cast<const float4*>(red);
  float4* my_partial = reinterpret_cast<float4*>(partials + ((size_t)(strip * splits + split) * R) * kStripCols);
  for (int idx = tid; idx < R * kVecPerRow; idx += kThreads) {
    const int r = idx / kVecPerRow, c = idx - r * kVecPerRow;
    float4 s = red4[(size_t)(0 * R + r) * kVecPerRow + c];
#pragma unroll
    for (int l = 1; l < kKLanes; ++l) {
      const float4 t = red4[(size_t)(l * R + r) * kVecPerRow + c];
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    if (splits == 1) {
      const int col = strip * kStripCols + c * 4;
      if (r < rows && col < N) {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
        s.x += bv.x; s.y += bv.y; s.z += bv.z; s.w += bv.w;
        if (relu) { s.x = fmaxf(s.x, 0.f); s.y = fmaxf(s.y, 0.f); s.z = fmaxf(s.z, 0.f); s.w = fmaxf(s.w, 0.f); }
        *reinterpret_cast<float4*>(y + (size_t)r * N + col) = s;
      }
    } else {
      my_partial[r * kVecPerRow + c] = s;
    }
  }
  if (splits == 1) return;

  // last CTA of this strip folds the `splits` partials in split order, adds bias, activation
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int prev = atomicAdd(&counters[strip], 1u);
    s_last = (prev == (unsigned)splits - 1) ? 1u : 0u;
    if (s_last) counters[strip] = 0u;  // self-reset for the next launch on this stream
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float4* strip_partials = reinterpret_cast<const float4*>(partials + (size_t)strip * splits * R * kStripCols);
  for (int idx = tid; idx < R * kVecPerRow; idx += kThreads) {
    const int r = idx / kVecPerRow, c = idx - r * kVecPerRow;
    const int col = strip * kStripCols + c * 4;
    if (r >= rows || col >= N) continue;
    float4 s = __ldcg(strip_partials + (size_t)(0 * R + r) * kVecPerRow + c);
    for (int sp = 1; sp < splits; ++sp) {
      const float4 t = __ldcg(strip_partials + (size_t)(sp * R + r) * kVecPerRow + c);
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
    s.x += bv.x; s.y += bv.y; s.z += bv.z; s.w += bv.w;
    if (relu) { s.x = fmaxf(s.x, 0.f); s.y = fmaxf(s.y, 0.f); s.z = fmaxf(s.z, 0.f); s.w = fmaxf(s.w, 0.f); }
    *reinterpret_cast<float4*>(y + (size_t)r * N + col) = s;
  }
}

// ------------------------------------------------------------------------- X2, bulk-copy ring ----
// Same strip x K-split decomposition, workspace layout and deterministic fold as dense_stream_kernel, but W reaches
// the SM through the async proxy: a producer warp issues one `cp.async.bulk` (TMA unit, no tensor map) per 2 KB
// row segment into a ring of kBulkStages x 32 KB shared-memory stages guarded by full / empty mbarriers, so the bytes in
// flight per SM (~128 KB) are not bounded by registers. 16 consumer warps = 64 column groups x 8 k-lanes; a thread owns
// the float4 column groups cg and cg + 64 of the strip (both LDS.128 conflict-free) and accumulates with packed
// register pairs (two adjacent columns per 64-bit shared load, x broadcast from a scalar register).
constexpr int kBulkStageRows = 16;
constexpr int kBulkStages = 5;
constexpr int kBulkColGroups = kStripCols / 8;    // 64 threads across a strip, 2 x float4 each
// k-lanes KL (template): 8 -> 512 consumer threads (+ producer warp = 17 warps, 96 registers each), 4 -> 256 (9 warps, 168)
constexpr int kBulkRingFloats = kBulkStages * kBulkStageRows * kStripCols;
constexpr size_t kBulkMaxSmem = 216 * 1024;

__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
// two adjacent fp32 columns as one 64-bit register pair
__device__ __forceinline__ void lds_2x64(uint32_t saddr, uint64_t& lo, uint64_t& hi) {
  asm volatile("ld.shared.v2.b64 {%0,%1}, [%2];" : "=l"(lo), "=l"(hi) : "r"(saddr));
}
__device__ __forceinline__ void ffma2(uint64_t& acc, float xs, uint64_t w2) {
  float a0, a1, w0, w1;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(acc));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(w0), "=f"(w1) : "l"(w2));
  asm("mov.b64 %0, {%1, %2};" : "=l"(acc) : "f"(fmaf(xs, w0, a0)), "f"(fmaf(xs, w1, a1)));
}

template <int R>
__device__ __forceinline__ void bulk_row(uint64_t (&acc)[R][4], uint32_t wrow_saddr, const float* xr) {
  uint64_t w0, w1, w2, w3;
  lds_2x64(wrow_saddr, w0, w1);
  lds_2x64(wrow_saddr + (kStripCols / 2) * 4u, w2, w3);
  float xv[R];
  if (R % 4 == 0) {
#pragma unroll
    for (int q = 0; q < R / 4; ++q) {
      const float4 t = *reinterpret_cast<const float4*>(xr + 4 * q);
      xv[4 * q + 0] = t.x; xv[4 * q + 1] = t.y; xv[4 * q + 2] = t.z; xv[4 * q + 3] = t.w;
    }
  } else if (R == 2) {
    const float2 t = *reinterpret_cast<const float2*>(xr);
    xv[0] = t.x; xv[1] = t.y;
  } else {
#pragma unroll
    for (int r = 0; r < R; ++r) xv[r] = xr[r];
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    ffma2(acc[r][0], xv[r], w0);
    ffma2(acc[r][1], xv[r], w1);
    ffma2(acc[r][2], xv[r], w2);
    ffma2(acc[r][3], xv[r], w3);
  }
}

template <int R, int KL>
__global__ void __launch_bounds__(kBulkColGroups * KL + 32, 1)
dense_bulk_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                  float* __restrict__ y, int rows, int K, int N, int relu, int splits, int chunk_k,
                  unsigned int* __restrict__ counters, float* __restrict__ partials) {
  constexpr int kBulkKLanes = KL, kBulkConsumers = kBulkColGroups * KL, kBulkThreads = kBulkConsumers + 32;
  extern __shared__ __align__(128) float smem_bulk[];
  float* smem = smem_bulk;
  float* ring = smem;                    // [kBulkStages][kBulkStageRows][kStripCols]
  float* xs = smem + kBulkRingFloats;    // [chunk_k][R]
  __shared__ __align__(8) uint64_t full[kBulkStages];
  __shared__ __align__(8) uint64_t empty[kBulkStages];
  __shared__ unsigned int s_last;

  const int strip = blockIdx.x;
  const int split = blockIdx.y;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int k_begin = split * chunk_k;
  const int k_end = min(K, k_begin + chunk_k);
  const int kc = max(0, k_end - k_begin);
  const int strip_cols = min(kStripCols, N - strip * kStripCols);   // multiple of 8 (host guarantees N % 8 == 0)
  const int n_stage = (kc + kBulkStageRows - 1) / kBulkStageRows;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kBulkStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kBulkConsumers / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();  // barriers initialised; the producer starts streaming W while the consumers stage x
  pdl_trigger();

  uint64_t acc[R][4];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0ull;
  const int cg = tid % kBulkColGroups;
  const int kl = (tid / kBulkColGroups) % kBulkKLanes;

  if (warp == kBulkConsumers / 32) {
    // ---- producer: W rows [k_begin, k_end) x this strip's columns, 16 rows per stage
    uint64_t policy;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
    const uint32_t row_bytes = (uint32_t)strip_cols * 4u;
    const float* src0 = w + (size_t)k_begin * N + (size_t)strip * kStripCols;
    for (int it = 0; it < n_stage; ++it) {
      const int s = it % kBulkStages;
      if (it >= kBulkStages) mbar_wait(&empty[s], ((it / kBulkStages) - 1) & 1);
      const int rows_here = min(kBulkStageRows, kc - it * kBulkStageRows);
      if (lane == 0) mbar_expect_tx(&full[s], (uint32_t)rows_here * row_bytes);
      __syncwarp();
      if (lane < rows_here)
        bulk_copy_g2s(ring + ((size_t)s * kBulkStageRows + lane) * kStripCols,
                      src0 + (size_t)(it * kBulkStageRows + lane) * N, row_bytes, &full[s], policy);
    }
    pdl_wait();
  } else {
    // ---- consumers: stage x[:, k_begin:k_end] transposed (xs[k][r]) behind a consumer-only named barrier, then k-lane
    // kl takes rows kl, kl + KL, ... of every stage. Columns >= strip_cols of a partial last strip are never copied:
    // their sums are garbage and are discarded by the column guards of the epilogue.
    pdl_wait();  // x is the previous pass's y
    for (int idx = tid; idx < kc * R; idx += kBulkConsumers) {
      const int r = idx / kc, k = idx - r * kc;
      xs[k * R + r] = (r < rows) ? __ldg(x + (size_t)r * K + k_begin + k) : 0.f;
    }
    asm volatile("bar.sync 1, %0;" ::"r"(kBulkConsumers) : "memory");
    const uint32_t ring_s = smem_u32(ring) + (uint32_t)cg * 16u;
    for (int it = 0; it < n_stage; ++it) {
      const int s = it % kBulkStages;
      mbar_wait(&full[s], (it / kBulkStages) & 1);
      const int kk0 = it * kBulkStageRows + kl;
      const uint32_t base = ring_s + (uint32_t)((s * kBulkStageRows + kl) * kStripCols) * 4u;
      if (it * kBulkStageRows + kBulkStageRows <= kc) {
#pragma unroll
        for (int j = 0; j < kBulkStageRows / KL; ++j)
          bulk_row<R>(acc, base + (uint32_t)(j * KL * kStripCols) * 4u, xs + (size_t)(kk0 + j * KL) * R);
      } else {
#pragma unroll
        for (int j = 0; j < kBulkStageRows / KL; ++j)
          if (kk0 + j * KL < kc) bulk_row<R>(acc, base + (uint32_t)(j * KL * kStripCols) * 4u, xs + (size_t)(kk0 + j * KL) * R);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
  }

  // every full barrier has been waited on by every consumer: no copy is in flight, the ring can be reused
  __syncthreads();
  float* red = smem;  // [kBulkKLanes][R][kStripCols]  (128 KB at R = 8, inside the ring)
  if (warp < kBulkConsumers / 32) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float* dst = red + ((size_t)(kl * R + r) * kStripCols) + cg * 4;
      *reinterpret_cast<ulonglong2*>(dst) = make_ulonglong2(acc[r][0], acc[r][1]);
      *reinterpret_cast<ulonglong2*>(dst + kStripCols / 2) = make_ulonglong2(acc[r][2], acc[r][3]);
    }
  }
  __syncthreads();

  constexpr int kVecPerRow = kStripCols / 4;
  const float4* red4 = reinterpret_cast<const float4*>(red);
  float4* my_partial = reinterpret_cast<float4*>(partials + ((size_t)(strip * splits + split) * R) * kStripCols);
  for (int idx = tid; idx < R * kVecPerRow; idx += kBulkThreads) {
    const int r = idx / kVecPerRow, c = idx - r * kVecPerRow;
    float4 s = red4[(size_t)(0 * R + r) * kVecPerRow + c];
#pragma unroll
    for (int l = 1; l < kBulkKLanes; ++l) {
      const float4 t = red4[(size_t)(l * R + r) * kVecPerRow + c];
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    if (splits == 1) {
      const int col = strip * kStripCols + c * 4;
      if (r < rows && col < N) {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
        s.x += bv.x; s.y += bv.y; s.z += bv.z; s.w += bv.w;
        if (relu) { s.x = fmaxf(s.x, 0.f); s.y = fmaxf(s.y, 0.f); s.z = fmaxf(s.z, 0.f); s.w = fmaxf(s.w, 0.f); }
        *reinterpret_cast<float4*>(y + (size_t)r * N + col) = s;
      }
    } else {
      my_partial[r * kVecPerRow + c] = s;
    }
  }
  if (splits == 1) return;

  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int prev = atomicAdd(&counters[strip], 1u);
    s_last = (prev == (unsigned)splits - 1) ? 1u : 0u;
    if (s_last) counters[strip] = 0u;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float4* strip_partials = reinterpret_cast<const float4*>(partials + (size_t)strip * splits * R * kStripCols);
  for (int idx = tid; idx < R * kVecPerRow; idx += kBulkThreads) {
    const int r = idx / kVecPerRow, c = idx - r * kVecPerRow;
    const int col = strip * kStripCols + c * 4;
    if (r >= rows || col >= N) continue;
    float4 s = __ldcg(strip_partials + (size_t)(0 * R + r) * kVecPerRow + c);
#pragma unroll 8
    for (int sp = 1; sp < splits; ++sp) {
      const float4 t = __ldcg(strip_partials + (size_t)(sp * R + r) * kVecPerRow + c);
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
    s.x += bv.x; s.y += bv.y; s.z += bv.z; s.w += bv.w;
    if (relu) { s.x = fmaxf(s.x, 0.f); s.y = fmaxf(s.y, 0.f); s.z = fmaxf(s.z, 0.f); s.w = fmaxf(s.w, 0.f); }
    *reinterpret_cast<float4*>(y + (size_t)r * N + col) = s;
  }
}

// Generic fallback for shapes the streaming kernel does not cover (N % 8 != 0 or unaligned W):
// one thread per output column, coalesced across columns. Small models only.
__global__ void __launch_bounds__(256)
dense_generic_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ y, int rows, int K, int N, int relu) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (n >= N || r >= rows) return;
  float acc = 0.f;
  const float* xr = x + (size_t)r * K;
  for (int k = 0; k < K; ++k) acc = fmaf(__ldg(xr + k), __ldg(w + (size_t)k * N + n), acc);
  acc += __ldg(bias + n);
  if (relu) acc = fmaxf(acc, 0.f);
  y[(size_t)r * N + n] = acc;
}

struct DensePlan {
  int strips, splits, chunk_k;
};

static DensePlan plan_dense(int k, int n) {
  DensePlan p;
  p.strips = (n + kStripCols - 1) / kStripCols;
  // fill ~one CTA per SM; each chunk must fit the smem x stage
  int splits = device_sm_count() / p.strips;
  if (splits < 1) splits = 1;
  int min_splits = (k + kMaxChunkK - 1) / kMaxChunkK;
  if (splits < min_splits) splits = min_splits;
  if (splits > k / 64 && k >= 64) splits = k / 64;  // keep chunks >= 64 rows
  if (splits < 1) splits = 1;
  int chunk = (k + splits - 1) / splits;
  chunk = (chunk + kKLanes - 1) / kKLanes * kKLanes;
  p.chunk_k = chunk;
  p.splits = (k + chunk - 1) / chunk;
  return p;
}

static size_t stream_workspace_bytes(int k, int n) {
  DensePlan p = plan_dense(k, n);
  size_t counters = ((size_t)p.strips * sizeof(unsigned int) + 255) & ~(size_t)255;
  size_t partials = (size_t)p.strips * p.splits * kMaxRowsPerLaunch * kStripCols * sizeof(float);
  return counters + partials;
}

size_t dense_workspace_bytes(int rows, int k, int n) {
  (void)rows;
  size_t a = stream_workspace_bytes(k, n), b = dense_tc_workspace_bytes(k, n);
  return a > b ? a : b;
}

static int tc_min_rows() {  // rows per group from which the tensor-core path is used (0 = never)
  static int v = [] {
    const char* e = getenv("TFSC_TC_MIN_ROWS");
    return e ? atoi(e) : 9;
  }();
  return v;
}

static bool pdl_enabled() {
  static bool v = [] {
    const char* e = getenv("TFSC_PDL");
    return e && atoi(e) != 0;
  }();
  return v;
}

template <typename... KArgs, typename... Args>
static cudaError_t launch_maybe_pdl(void (*kernel)(KArgs...), dim3 grid, int threads, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <int R>
static cudaError_t launch_dense_r(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n,
                                  bool relu, void* workspace, const DensePlan& p, cudaStream_t s) {
  size_t xs_bytes = (size_t)p.chunk_k * R * sizeof(float);
  size_t red_bytes = (size_t)kKLanes * R * kStripCols * sizeof(float);
  size_t smem = xs_bytes > red_bytes ? xs_bytes : red_bytes;
  static bool attr_set[64] = {};  // function attributes are per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(dense_stream_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return e;
    attr_set[dev & 63] = true;
  }
  unsigned int* counters = static_cast<unsigned int*>(workspace);
  size_t coff = ((size_t)p.strips * sizeof(unsigned int) + 255) & ~(size_t)255;
  float* partials = reinterpret_cast<float*>(static_cast<char*>(workspace) + coff);
  dim3 grid(p.strips, p.splits);
  if (pdl_enabled()) {
    static bool attr_set_pdl[64] = {};
    if (!attr_set_pdl[dev & 63]) {
      cudaError_t e = cudaFuncSetAttribute(dense_stream_kernel<R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (e != cudaSuccess) return e;
      attr_set_pdl[dev & 63] = true;
    }
    cudaError_t le = launch_maybe_pdl(dense_stream_kernel<R, true>, grid, kThreads, smem, s, x, w, bias, y, rows, k, n, relu ? 1 : 0,
                                      p.splits, p.chunk_k, counters, partials);
    g_launches++;
    return le != cudaSuccess ? le : cudaGetLastError();
  }
  dense_stream_kernel<R><<<grid, kThreads, smem, s>>>(x, w, bias, y, rows, k, n, relu ? 1 : 0, p.splits, p.chunk_k,
                                                      counters, partials);
  g_launches++;
  return cudaGetLastError();
}

static bool bulk_fits(int R, const DensePlan& p) {
  return (size_t)kBulkRingFloats * sizeof(float) + (size_t)p.chunk_k * R * sizeof(float) <= kBulkMaxSmem;
}

template <int R, int KL>
static cudaError_t launch_dense_bulk_r(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n,
                                       bool relu, void* workspace, const DensePlan& p, cudaStream_t s) {
  const size_t smem = (size_t)kBulkRingFloats * sizeof(float) + (size_t)p.chunk_k * R * sizeof(float);
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(dense_bulk_kernel<R, KL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBulkMaxSmem);
    if (e != cudaSuccess) return e;
    attr_set[dev & 63] = true;
  }
  unsigned int* counters = static_cast<unsigned int*>(workspace);
  size_t coff = ((size_t)p.strips * sizeof(unsigned int) + 255) & ~(size_t)255;
  float* partials = reinterpret_cast<float*>(static_cast<char*>(workspace) + coff);
  dim3 grid(p.strips, p.splits);
  cudaError_t le = launch_maybe_pdl(dense_bulk_kernel<R, KL>, grid, kBulkColGroups * KL + 32, smem, s, x, w, bias, y, rows, k, n,
                                    relu ? 1 : 0, p.splits, p.chunk_k, counters, partials);
  g_launches++;
  return le != cudaSuccess ? le : cudaGetLastError();
}

static int dense_variant_default() {  // 0 = auto (LDG stream + tensor cores), 1 = LDG stream only, 2 / 4 = bulk ring (8 / 4 k-lanes), 3 = tc
  static int v = [] {
    const char* e = getenv("TFSC_DENSE_VARIANT");
    return e ? atoi(e) : 0;
  }();
  return v;
}

cudaError_t launch_dense(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n,
                         bool relu, void* workspace, size_t workspace_bytes, cudaStream_t s, int variant) {
  if (rows <= 0 || n <= 0) return cudaSuccess;
  if (variant == 0) variant = dense_variant_default();
  const bool stream_ok = (n % 8 == 0) && ((reinterpret_cast<uintptr_t>(w) & 31) == 0) &&
                         ((reinterpret_cast<uintptr_t>(bias) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y) & 15) == 0) &&
                         k >= 1 && workspace && workspace_bytes >= dense_workspace_bytes(rows, k, n);
  if (!stream_ok) {
    for (int r0 = 0; r0 < rows; r0 += 65535) {
      int rr = rows - r0 < 65535 ? rows - r0 : 65535;
      dim3 grid((n + 255) / 256, rr);
      dense_generic_kernel<<<grid, 256, 0, s>>>(x + (size_t)r0 * k, w, bias, y + (size_t)r0 * n, rr, k, n, relu ? 1 : 0);
      g_launches++;
    }
    return cudaGetLastError();
  }
  const DensePlan p = plan_dense(k, n);
  int r_done = 0;
  const int tc_rows = variant == 3 ? 1 : tc_min_rows();
  if (variant != 1 && tc_rows > 0 && rows >= tc_rows && dense_tc_supported(rows > 64 ? 64 : rows, k, n, w, x, bias, y)) {
    // batches of more than 8 rows: one tensor-core pass per 64 rows instead of ceil(rows/8) SIMT passes
    while (rows - r_done >= tc_rows) {
      const int rr = rows - r_done < 64 ? rows - r_done : 64;
      cudaError_t e = launch_dense_tc(x + (size_t)r_done * k, w, bias, y + (size_t)r_done * n, rr, k, n, relu, workspace,
                                      workspace_bytes, s);
      if (e != cudaSuccess) return e;
      r_done += rr;
    }
  }
  for (int r0 = r_done; r0 < rows; r0 += kMaxRowsPerLaunch) {
    const int rr = rows - r0 < kMaxRowsPerLaunch ? rows - r0 : kMaxRowsPerLaunch;
    const float* xp = x + (size_t)r0 * k;
    float* yp = y + (size_t)r0 * n;
    cudaError_t e;
    // default for <= 8 rows: the cluster-pair kernel with programmatic dependent launch (measured round 2: 51.8 us per
    // 9216x9216 layer at 8 rows = the measured HBM copy peak, vs 61.1 us for the LDG stream kernel with its split-K tail)
    if ((variant == 0 || variant == 5) && dense_cluster_supported(rr, k, n, w, xp, bias, yp)) {
      e = launch_dense_cluster(xp, w, bias, yp, rr, k, n, relu, s);
      if (e != cudaSuccess) return e;
      continue;
    }
    if ((variant == 2 || variant == 4) && bulk_fits(rr <= 2 ? rr : (rr <= 4 ? 4 : 8), p)) {
      if (variant == 2) {
        if (rr == 1) e = launch_dense_bulk_r<1, 8>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
        else if (rr == 2) e = launch_dense_bulk_r<2, 8>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
        else if (rr <= 4) e = launch_dense_bulk_r<4, 8>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
        else e = launch_dense_bulk_r<8, 8>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
      } else {
        if (rr == 1) e = launch_dense_bulk_r<1, 4>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
        else if (rr == 2) e = launch_dense_bulk_r<2, 4>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
        else if (rr <= 4) e = launch_dense_bulk_r<4, 4>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
        else e = launch_dense_bulk_r<8, 4>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
      }
      if (e != cudaSuccess) return e;
      continue;
    }
    if (rr == 1) e = launch_dense_r<1>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
    else if (rr == 2) e = launch_dense_r<2>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
    else if (rr <= 4) e = launch_dense_r<4>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
    else e = launch_dense_r<8>(xp, w, bias, yp, rr, k, n, relu, workspace, p, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace tfsc

extern "C" {
int64_t tfsc_kernel_launches(void) { return tfsc::kernel_launch_count(); }
}
