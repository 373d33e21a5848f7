// X3: tensor-core dense layer for batches of 9..64 rows, sm_90a (warpgroup MMA).
//
//   y[rows,N] = act(x[rows,K] W[K,N] + b),  fp32 in / fp32 out, |err| ~1e-6 (3xTF32 split)
//
// The weights are the big streamed operand (1 pass over W per launch, HBM-bound up to ~64 rows), so
// W^T sits on the MMA "M" side: D[n, r] = sum_k W[k][n] x[r][k].
//   * W tiles arrive by TMA (cp.async.bulk.tensor.3d over a 3-D tensor map {32 n, K, N/32}, boxes of 4 rows x
//     8 slabs = 4 x 1 KB contiguous, SWIZZLE_128B) into a 6-stage ring: 192 KB of W in flight per SM.
//   * 4 consumer warpgroups own 64 output columns each. A tf32 operand in shared memory must be K-major and W is
//     N-major, so each warp reads its W fragments from the stage into registers (the wgmma A operand may come from
//     registers in any layout): W_hi = trunc_tf32(W) and W_lo = W - W_hi. All consumers together build
//     B' = [x_hi ; x_lo] (K-major, SWIZZLE_128B) in shared memory from x (double-buffered, one named barrier per k-block).
//   * per 8-wide k step: acc_h += W_hi . x_hi, acc_s += W_hi . x_lo + W_lo . x_hi (N = rows padded to RP);
//     y = acc_h + acc_s: the large term and the small correction terms are kept apart because the tensor core's fp32
//     accumulation truncates.
//   * split-K over CTAs (one CTA per SM), partials folded by the last CTA of a strip in fixed order
//     (same deterministic scheme as dense_stream_kernel), bias + ReLU fused there.
//   * programmatic dependent launch: the W ring fills (TMA) under the previous kernel's tail; x, the
//     split-K workspace and y are touched only after griddepcontrol.wait.
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "kernels.h"
#include "tc_ptx.cuh"

namespace tfsc {

extern std::atomic<int64_t> g_launches_tc;
std::atomic<int64_t> g_launches_tc{0};

namespace tc {
constexpr int BK = 32;                     // k rows per stage = one 128-byte swizzle row of tf32
constexpr int WG_COLS = 64;                // output columns per consumer warpgroup (wgmma M)
constexpr int CONS_WG = 4;
constexpr int STRIP = WG_COLS * CONS_WG;   // 256 output columns per CTA
constexpr int SLABS = STRIP / 32;          // 8 slabs of 32 columns
constexpr int W_BYTES = SLABS * BK * 128;  // 32 KB per stage
constexpr int CONSUMERS = CONS_WG * 128;
constexpr int CONS_WARPS = CONSUMERS / 32;
constexpr int THREADS = CONSUMERS + 32;    // warps 0..15 consumers, warp 16 TMA producer
}  // namespace tc

// smem (dynamic, 1024-aligned): NS stages of W (32 KB each, TMA target, layout [k/4][slab][k%4][32 n] with the
// 128-byte swizzle), 2 buffers of B' = [x_hi ; x_lo] (2*RP rows x 128 B), then the mbarriers.
template <int RP>
struct TcSmem {
  static constexpr int NS = 6;
  static constexpr int B_BYTES = 2 * RP * 128;
  static constexpr int W_TOTAL = NS * tc::W_BYTES;
  static constexpr int TOTAL = W_TOTAL + 2 * B_BYTES + 256 + 1024;
};

template <int RP>
__global__ void __launch_bounds__(tc::THREADS, 1)
dense_tc_kernel(const __grid_constant__ CUtensorMap wmap, const float* __restrict__ x, const float* __restrict__ bias,
                float* __restrict__ y, int rows, int K, int N, int relu, int splits, int chunk_k,
                unsigned int* __restrict__ counters, float* __restrict__ partials) {
  using S = TcSmem<RP>;
  constexpr int NS = S::NS;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bprime = smem + S::W_TOTAL;
  uint64_t* bars = reinterpret_cast<uint64_t*>(bprime + 2 * S::B_BYTES);
  uint64_t* full = bars;             // [NS] TMA landed the W stage
  uint64_t* empty = bars + NS;       // [NS] every consumer warp holds its W fragments of the stage in registers

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // role from a broadcast warpgroup index: ptxas then knows the branch below is warpgroup-uniform and does not serialise
  // the wgmma instructions behind compiler-inserted warpgroup barriers
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int strip = blockIdx.x, split = blockIdx.y;
  const int k_begin = split * chunk_k;
  const int k_end = min(K, k_begin + chunk_k);
  const int n_kblocks = (max(0, k_end - k_begin) + tc::BK - 1) / tc::BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], tc::CONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
  }
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // no-op without the PDL launch attribute

  if (wg == tc::CONS_WG) {
    // ===================== TMA producer: keeps NS x 32 KB of W in flight =====================
    for (int kb = 0; kb < n_kblocks; ++kb) {
      const int s = kb % NS, it = kb / NS;
      if (lane == 0) {
        if (it > 0) mbar_wait(&empty[s], (it - 1) & 1);
        mbar_expect_tx(&full[s], tc::W_BYTES);
        // 8 boxes of {32 n, 4 k, 8 slabs}: every box covers 4 W rows x 1 KB contiguous, so the 128-byte
        // pieces of one DRAM row are requested close together; smem stage = [k/4][slab][k%4][32 n]
#pragma unroll
        for (int g = 0; g < tc::BK / 4; ++g)
          tma_load_3d(smem + s * tc::W_BYTES + g * 4096, &wmap, &full[s], 0, k_begin + kb * tc::BK + g * 4, strip * tc::SLABS);
      }
      __syncwarp();
    }
  } else {
    // ===================== consumers: B' = [x_hi ; x_lo] (smem), W fragments (registers), wgmma =====================
    const int ct = threadIdx.x;       // 0..511
    const int wq = warp & 3, g = lane >> 2, t = lane & 3;
    constexpr int XI = (RP * 8 + tc::CONSUMERS - 1) / tc::CONSUMERS;  // x items (float4) per thread per k-block
    float4 xr[2][XI];                                                // register ring: x is fetched two k-blocks ahead
    auto load_x = [&](int kb, float4* dst) {
      const int k0 = k_begin + kb * tc::BK;
#pragma unroll
      for (int j = 0; j < XI; ++j) {
        const int idx = ct + j * tc::CONSUMERS;
        const int r = idx >> 3, c = idx & 7;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        const int kk = k0 + c * 4;
        if (idx < RP * 8 && r < rows) {
          const float* src = x + (size_t)r * K + kk;
          if (kk + 3 < k_end) v = __ldg(reinterpret_cast<const float4*>(src));
          else {
            if (kk < k_end) v.x = __ldg(src);
            if (kk + 1 < k_end) v.y = __ldg(src + 1);
            if (kk + 2 < k_end) v.z = __ldg(src + 2);
          }
        }
        dst[j] = v;
      }
    };
    asm volatile("griddepcontrol.wait;" ::: "memory");   // x is the previous kernel's output; W (TMA warp) never is
    if (n_kblocks > 0) load_x(0, xr[0]);
    if (n_kblocks > 1) load_x(1, xr[1]);
    // this thread's A fragment columns: n0 = wg*64 + wq*16 + g and n0 + 8 (same 32-column slab), k % 4 == t always.
    // Offset inside a 4-row k group of a stage: row = slab*4 + t (128 B), 16-byte chunk XOR (row % 8).
    const int n0 = wg * tc::WG_COLS + wq * 16 + g, slab = n0 >> 5, row = slab * 4 + t;
    auto w_off = [&](int n) { return (uint32_t)(row * 128 + ((((n & 31) >> 2) ^ (row & 7)) << 4) + (n & 3) * 4); };
    const uint32_t w_base = smem_u32(smem);
    const uint32_t off0 = w_off(n0), off1 = w_off(n0 + 8);
    const uint32_t bp_base = smem_u32(bprime);
    float acc_h[RP / 2], acc_s[RP / 2];
#pragma unroll
    for (int i = 0; i < RP / 2; ++i) acc_h[i] = acc_s[i] = 0.f;
    auto body = [&](int kb, float4* xcur) {
      const int s = kb % NS, it = kb / NS, cb = kb & 1;
      // B'[cb] was last read by the MMAs of k-block kb-2, which every consumer waited for before the barrier of kb-1
      const uint32_t bp = bp_base + cb * S::B_BYTES;
#pragma unroll
      for (int j = 0; j < XI; ++j) {
        const int idx = ct + j * tc::CONSUMERS;
        if (idx < RP * 8) {
          const int r = idx >> 3, c = idx & 7, rl = r + RP;
          const float4 v = xcur[j];
          sts_f4(bp + (uint32_t)(((r >> 3) * 64 + (r & 7) * 8 + (c ^ (r & 7))) * 16), v);
          sts_f4(bp + (uint32_t)(((rl >> 3) * 64 + (rl & 7) * 8 + (c ^ (rl & 7))) * 16),
                 make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w)));
        }
      }
      if (kb + 2 < n_kblocks) load_x(kb + 2, xcur);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // B' writes -> visible to the MMA (async proxy)
      named_bar_sync(1, tc::CONSUMERS);
      mbar_wait(&full[s], it & 1);
      const uint32_t wst = w_base + (uint32_t)(s * tc::W_BYTES);
      uint32_t hi[tc::BK / 8][4], lo[tc::BK / 8][4];
#pragma unroll
      for (int k8 = 0; k8 < tc::BK / 8; ++k8)
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // a[j]: column n0 + 8*(j&1), k = 8*k8 + t + 4*(j>>1)
          const float v = lds_f32(wst + (uint32_t)((k8 * 2 + (j >> 1)) * 4096) + ((j & 1) ? off1 : off0));
          hi[k8][j] = tf32_hi_bits(v);
          lo[k8][j] = __float_as_uint(tf32_lo(v));
        }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);  // this warp is done with the W stage: TMA may refill it
      if constexpr (RP <= 32) {   // fragments final before the warpgroup fence; at 48 / 64 rows it costs spills instead
        fence_regs(hi);
        fence_regs(lo);
      }
      fence_regs(acc_h);
      fence_regs(acc_s);
      wgmma_fence();
#pragma unroll
      for (int k8 = 0; k8 < tc::BK / 8; ++k8) {
        const uint64_t bh = gmma_desc_sw128(bp + k8 * 32), bl = gmma_desc_sw128(bp + RP * 128 + k8 * 32);
        wgmma_tf32_rs<RP>(acc_h, hi[k8], bh);
        wgmma_tf32_rs<RP>(acc_s, hi[k8], bl);
        wgmma_tf32_rs<RP>(acc_s, lo[k8], bh);
      }
      wgmma_commit();
      wgmma_wait_all();
      fence_regs(acc_h);
      fence_regs(acc_s);
    };
    for (int kb = 0; kb < n_kblocks; kb += 2) {
      body(kb, xr[0]);
      if (kb + 1 < n_kblocks) body(kb + 1, xr[1]);
    }
    // ===================== epilogue: accumulators -> split-K partials =====================
    float* my_partial = partials + ((size_t)(strip * splits + split) * RP) * tc::STRIP;
#pragma unroll
    for (int i = 0; i < RP / 2; ++i) {
      const int ncol = n0 + 8 * ((i >> 1) & 1), r = 8 * (i >> 2) + 2 * t + (i & 1);
      my_partial[(size_t)r * tc::STRIP + ncol] = acc_h[i] + acc_s[i];
    }
  }

  // ---- deterministic split-K fold by the last CTA of the strip ----
  __shared__ unsigned int s_last;
  asm volatile("griddepcontrol.wait;" ::: "memory");   // workspace counters / y: every thread observes the prerequisite grid
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(&counters[strip], 1u);
    s_last = (prev == (unsigned)splits - 1) ? 1u : 0u;
    if (s_last) counters[strip] = 0u;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* sp = partials + (size_t)strip * splits * RP * tc::STRIP;
  for (int idx = threadIdx.x; idx < rows * (tc::STRIP / 4); idx += tc::THREADS) {
    const int r = idx / (tc::STRIP / 4), c4 = idx - r * (tc::STRIP / 4);
    const int col = strip * tc::STRIP + c4 * 4;
    if (col >= N) continue;
    float4 acc = __ldcg(reinterpret_cast<const float4*>(sp + (size_t)r * tc::STRIP) + c4);
    for (int s2 = 1; s2 < splits; ++s2) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(sp + ((size_t)s2 * RP + r) * tc::STRIP) + c4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + col));
    acc.x += bv.x; acc.y += bv.y; acc.z += bv.z; acc.w += bv.w;
    if (relu) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
    *reinterpret_cast<float4*>(y + (size_t)r * N + col) = acc;
  }
}

// --------------------------------------------------------------------------------- host side ----
EncodeTiledFn tc_encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

struct MapKey {
  const void* w;
  int k, n;
  bool operator==(const MapKey& o) const { return w == o.w && k == o.k && n == o.n; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& m) const { return std::hash<const void*>()(m.w) ^ ((size_t)m.k * 1315423911u) ^ ((size_t)m.n << 20); }
};

// weights sit at fixed arena addresses while resident: cache the encoded maps
static bool get_wmap(const float* w, int k, int n, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find({w, k, n});
  if (it != cache.end()) {
    *out = it->second;
    return true;
  }
  EncodeTiledFn enc = tc_encode_fn();
  if (!enc) return false;
  CUtensorMap m;
  const cuuint64_t gdim[3] = {32, (cuuint64_t)k, (cuuint64_t)(n / 32)};
  const cuuint64_t gstride[2] = {(cuuint64_t)n * 4, 128};
  const cuuint32_t box[3] = {32, 4, (cuuint32_t)tc::SLABS};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(w), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  if (cache.size() > 4096) cache.clear();
  cache[{w, k, n}] = m;
  *out = m;
  return true;
}

struct TcPlan {
  int strips, splits, chunk_k;
};
static TcPlan plan_tc(int k, int n) {
  TcPlan p;
  p.strips = (n + tc::STRIP - 1) / tc::STRIP;
  int splits = device_sm_count() / p.strips;
  if (splits < 1) splits = 1;
  int max_splits = (k + 4 * tc::BK - 1) / (4 * tc::BK);  // keep >= 4 k-blocks per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int chunk = (k + splits - 1) / splits;
  chunk = (chunk + tc::BK - 1) / tc::BK * tc::BK;
  p.chunk_k = chunk;
  p.splits = (k + chunk - 1) / chunk;
  return p;
}

bool dense_tc_supported(int rows, int k, int n, const float* w, const float* x, const float* bias, const float* y) {
  return rows >= 1 && rows <= 64 && n % 32 == 0 && k % 4 == 0 && k >= 32 &&
         ((reinterpret_cast<uintptr_t>(w) & 15) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
         ((reinterpret_cast<uintptr_t>(bias) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y) & 15) == 0) && tc_encode_fn() != nullptr;
}

size_t dense_tc_workspace_bytes(int k, int n) {
  TcPlan p = plan_tc(k, n);
  size_t counters = ((size_t)p.strips * sizeof(unsigned int) + 255) & ~(size_t)255;
  return counters + (size_t)p.strips * p.splits * 64 * tc::STRIP * sizeof(float);
}

template <int RP>
static cudaError_t launch_tc_rp(const CUtensorMap& map, const float* x, const float* bias, float* y, int rows, int k, int n,
                                bool relu, void* workspace, const TcPlan& p, cudaStream_t s) {
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(dense_tc_kernel<RP>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcSmem<RP>::TOTAL);
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  unsigned int* counters = static_cast<unsigned int*>(workspace);
  size_t coff = ((size_t)p.strips * sizeof(unsigned int) + 255) & ~(size_t)255;
  float* partials = reinterpret_cast<float*>(static_cast<char*>(workspace) + coff);
  static const bool pdl = [] {  // programmatic dependent launch is on unless TFSC_PDL=0
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(p.strips, p.splits);
  cfg.blockDim = dim3(tc::THREADS);
  cfg.dynamicSmemBytes = TcSmem<RP>::TOTAL;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, dense_tc_kernel<RP>, map, x, bias, y, rows, k, n, relu ? 1 : 0, p.splits, p.chunk_k, counters,
                                     partials);
  g_launches_tc++;
  return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t launch_dense_tc(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n, bool relu,
                            void* workspace, size_t workspace_bytes, cudaStream_t s) {
  if (workspace_bytes < dense_tc_workspace_bytes(k, n)) return cudaErrorInvalidValue;
  CUtensorMap map;
  if (!get_wmap(w, k, n, &map)) return cudaErrorNotSupported;
  const TcPlan p = plan_tc(k, n);
  if (rows <= 16) return launch_tc_rp<16>(map, x, bias, y, rows, k, n, relu, workspace, p, s);
  if (rows <= 32) return launch_tc_rp<32>(map, x, bias, y, rows, k, n, relu, workspace, p, s);
  if (rows <= 48) return launch_tc_rp<48>(map, x, bias, y, rows, k, n, relu, workspace, p, s);
  return launch_tc_rp<64>(map, x, bias, y, rows, k, n, relu, workspace, p, s);
}

}  // namespace tfsc
