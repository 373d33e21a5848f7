// Warpgroup-MMA GEMM for the graph executor (conv-as-GEMM, transformer dense layers), sm_90a:
//
//   C[M,N] = act(A[M,K] * B[K,N] + bias[N] (+ R[M,N])),  fp32 in / out, 3xTF32 split (fp32-accurate)
//
//   * A (activations) is K-major: TMA lands the tile [128 m][32 k] (SWIZZLE_128B) either from a row-major matrix (2-D tiled
//     map: dense layers, 1x1 stride-1 convs) or -- IMPLICIT GEMM, no im2col buffer -- straight from the NHWC activation
//     tensor with an im2col tensor map (cuTensorMapEncodeIm2col): the 128 rows are 128 consecutive output pixels, the 32
//     columns are 32 channels of one filter tap (kh, kw); padding arrives as zeros, strided convs through the map's
//     traversal stride. The raw fp32 bits are A_hi (the tensor core ignores the low 13 mantissa bits); the consumers write
//     A_lo = A - trunc_tf32(A) next to it, elementwise at the same (swizzled) offsets.
//   * B (weights [K,N] row-major) is N-major, which a tf32 wgmma operand in shared memory cannot be. So the MMA computes
//     the transposed tile, C^T = B^T A^T: B^T is the register ("A") operand -- each warp reads its fragments from the TMA
//     tile (3-D map {32 n, K, N/32}, SWIZZLE_128B slabs) and splits them into B_hi / B_lo -- and the activation tile is the
//     shared-memory ("B") operand, K-major as it lands.
//   * per 8-wide k step: acc_h += B_hi . A_hi, acc_s += B_hi . A_lo + B_lo . A_hi: the large term and the small corrections
//     have separate accumulators (the tensor core's fp32 accumulate truncates).
//   * two consumer warpgroups: for BN = 128 each owns 64 columns x 128 rows (wgmma N = 128), for BN = 64 each owns the 64
//     columns x 64 rows. The epilogue parks the tile in shared memory and stores it row-contiguous with bias (+ residual)
//     and ReLU / GELU(erf) / tanh / ReLU6 / SiLU / sigmoid.
// One CTA per 128 x BN output tile; small grids (late ResNet stages: M = 392, K = 4608; BERT's K = 3072 projection) split K
// over a thread-block cluster of 2 / 4 / 8 CTAs along grid.z: every CTA parks its partial tile in its own shared memory
// and each CTA folds 128/S rows of the tile over distributed shared memory in fixed rank order (deterministic), then
// applies bias / residual / activation. Warpgroups 0..1 consumers, warpgroup 2 producer (warp 8 issues the TMA); the producer
// warpgroup hands its registers to the consumers with setmaxnreg.
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>
#include <functional>
#include <mutex>
#include <unordered_map>

#include "act.cuh"
#include "kernels.h"
#include "tc_ptx.cuh"

namespace tfsc {

extern std::atomic<int64_t> g_launches_nn;

namespace gt {
constexpr int BM = 128, BK = 32;
constexpr int A_BYTES = BM * BK * 4;  // 16 KB per A tile (hi or lo)
constexpr int CONSUMERS = 256;        // two warpgroups
constexpr int CONS_WARPS = CONSUMERS / 32;
constexpr int THREADS = CONSUMERS + 128;   // + a producer warpgroup (warp 8 issues the TMA)
// register split (setmaxnreg): each 16K register-file quarter holds one producer warp and two consumer warps:
// 40 + 2 * 232 = 504 registers per lane (the BN = 128 accumulators alone take 128)
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
}  // namespace gt

// geometry of an implicit-GEMM conv (A tile = TMA im2col gather from the NHWC activations)
struct ConvGeom {
  int C, KW, OH, OW, stride, pad;
};

template <int BN>
struct GtSmem {
  static constexpr int STAGES = 4;
  static constexpr int SLABS = BN / 32;                 // 32-column slabs of the B tile
  static constexpr int KG_BYTES = SLABS * 512;          // one 4-row k group of B: [slab][k%4][32 n]
  static constexpr int B_BYTES = (gt::BK / 4) * KG_BYTES;
  static constexpr int STAGE_BYTES = 2 * gt::A_BYTES + B_BYTES;   // A_hi | A_lo | B
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 256 + 1024;
  static constexpr int WM = BN == 128 ? 128 : 64;       // tile rows per consumer warpgroup (wgmma N)
  static_assert(gt::BM * (BN + 4) * 4 <= STAGES * STAGE_BYTES, "the parked tile overlays the stages");
};

// TMA im2col gather: coordinates {c, w, h, n} of the base pixel (input space), offsets {kw, kh} of the filter tap
__device__ __forceinline__ void tma_load_im2col_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c, int w, int h, int n,
                                                   uint16_t woff, uint16_t hoff) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(woff), "h"(hoff)
      : "memory");
}

__device__ __forceinline__ float gelu_erf_tc(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
// run-time activation with REAL branches (a noinline body cannot be if-converted into the caller's store loop); every
// activation but ReLU shares one call site, so the store loop of act 0 / 1 carries a single extra compare
__device__ __noinline__ float4 act_call4(float4 v, int act) {
  if (act == 2) return make_float4(gelu_erf_tc(v.x), gelu_erf_tc(v.y), gelu_erf_tc(v.z), gelu_erf_tc(v.w));
  if (act == 3) return make_float4(tanhf(v.x), tanhf(v.y), tanhf(v.z), tanhf(v.w));
  if (act == 4) return make_float4(relu6f(v.x), relu6f(v.y), relu6f(v.z), relu6f(v.w));
  if (act == 5) return make_float4(siluf(v.x), siluf(v.y), siluf(v.z), siluf(v.w));
  if (act == 6) return make_float4(sigmoidf(v.x), sigmoidf(v.y), sigmoidf(v.z), sigmoidf(v.w));
  if (act == 7) return make_float4(gelu_tanhf(v.x), gelu_tanhf(v.y), gelu_tanhf(v.z), gelu_tanhf(v.w));
  return v;
}
__device__ __forceinline__ float4 apply_act_rt(float4 v, int act) {
  if (act == 1) return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
  if (act >= 2) return act_call4(v, act);
  return v;
}
template <int BN, bool IM2COL>
__global__ void __launch_bounds__(gt::THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap bmap,
               const float* __restrict__ bias, const float* __restrict__ R, float* __restrict__ C, int M, int N, int K, int act,
               ConvGeom cg) {
  using S = GtSmem<BN>;
  constexpr int NS = S::STAGES, WM = S::WM;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NS * S::STAGE_BYTES);
  uint64_t* full = bars;            // [NS] TMA landed A_hi and B
  uint64_t* empty = bars + NS;      // [NS] every consumer warp's MMAs on the stage have completed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // role from a broadcast warpgroup index: the consumer branch is then provably warpgroup-uniform for ptxas
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int m0 = blockIdx.y * gt::BM, n0 = blockIdx.x * BN;
  // split-K: grid.z = cluster size S; this CTA (cluster rank = blockIdx.z) takes k blocks [kb0, kb0 + n_kblocks)
  const int splits = (int)gridDim.z, split = (int)blockIdx.z;
  const int total_kblocks = (K + gt::BK - 1) / gt::BK;
  const int per_split = (total_kblocks + splits - 1) / splits;
  const int kb0 = split * per_split;
  const int n_kblocks = max(0, min(total_kblocks, kb0 + per_split) - kb0);
  constexpr int PSTRIDE = BN + 4;   // parked tile [128][BN + 4] fp32 (padded: conflict-free fragment stores)

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], gt::CONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&amap) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&bmap) : "memory");
  }
  __syncthreads();
  // programmatic dependent launch: successors may begin their setup; this kernel waits for its predecessor here -- its
  // own setup above already ran under the predecessor's tail
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  if (wg == gt::CONSUMERS / 128) {
    // ===================== TMA producer =====================
    regs_release<gt::PRODUCER_REGS>();
    int pn = 0, ph = 0, pw = 0;  // im2col: base pixel of the tile's first row, input space
    if (IM2COL) {
      const int per_img = cg.OH * cg.OW;
      pn = m0 / per_img;
      const int rem = m0 - pn * per_img;
      ph = (rem / cg.OW) * cg.stride - cg.pad;
      pw = (rem % cg.OW) * cg.stride - cg.pad;
    }
    if (warp == gt::CONS_WARPS)
    for (int kb = 0; kb < n_kblocks; ++kb) {
      const int s = kb % NS, it = kb / NS;
      if (lane == 0) {
        if (it > 0) mbar_wait(&empty[s], (it - 1) & 1);
        uint8_t* stage = smem + s * S::STAGE_BYTES;
        mbar_expect_tx(&full[s], gt::A_BYTES + BN * gt::BK * 4);
        if (IM2COL) {
          // k block kb = 32 channels [c0, c0+32) of filter tap (kh, kw); K is ordered (kh, kw, c) like the HWIO kernel
          const int k0 = (kb0 + kb) * gt::BK, tap = k0 / cg.C, c0 = k0 - tap * cg.C;
          tma_load_im2col_4d(stage, &amap, &full[s], c0, pw, ph, pn, (uint16_t)(tap % cg.KW), (uint16_t)(tap / cg.KW));
        } else {
          tma_load_2d(stage, &amap, &full[s], (kb0 + kb) * gt::BK, m0);  // A: [128 m][32 k], 128 B rows, SW128
        }
#pragma unroll
        for (int g = 0; g < gt::BK / 4; ++g)                              // B: k group g -> slabs [0, SLABS) of the group
          tma_load_3d(stage + 2 * gt::A_BYTES + g * S::KG_BYTES, &bmap, &full[s], 0, (kb0 + kb) * gt::BK + g * 4, n0 / 32);
      }
      __syncwarp();
    }
  } else {
    // ===================== consumers: A_lo, B fragments, wgmma =====================
    regs_acquire<gt::CONSUMER_REGS>();
    const int ct = threadIdx.x;  // 0..255
    const int wq = warp & 3, g = lane >> 2, t = lane & 3;
    const int n_off = BN == 128 ? wg * 64 : 0, m_off = BN == 128 ? 0 : wg * 64;
    // this thread's B^T fragment columns n and n + 8 (same 32-column slab); k % 4 == t always
    const int nf = n_off + wq * 16 + g, row = (nf >> 5) * 4 + t;
    auto b_off = [&](int n) { return (uint32_t)(row * 128 + ((((n & 31) >> 2) ^ (row & 7)) << 4) + (n & 3) * 4); };
    const uint32_t off0 = b_off(nf), off1 = b_off(nf + 8);
    float acc_h[WM / 2], acc_s[WM / 2];
#pragma unroll
    for (int i = 0; i < WM / 2; ++i) acc_h[i] = acc_s[i] = 0.f;
    for (int kb = 0; kb < n_kblocks; ++kb) {
      const int s = kb % NS, it = kb / NS;
      mbar_wait(&full[s], it & 1);
      const uint32_t ast = smem_u32(smem + s * S::STAGE_BYTES);
#pragma unroll
      for (int i = 0; i < gt::A_BYTES / 16 / gt::CONSUMERS; ++i) {   // A tile: 1024 float4, 4 per thread
        const uint32_t src = ast + (uint32_t)((ct + i * gt::CONSUMERS) * 16);
        const float4 v = lds_f4(src);
        sts_f4(src + gt::A_BYTES, make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w)));
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the MMA (async proxy)
      const uint32_t bsm = ast + 2 * gt::A_BYTES;
      uint32_t hi[gt::BK / 8][4], lo[gt::BK / 8][4];
#pragma unroll
      for (int k8 = 0; k8 < gt::BK / 8; ++k8)
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // a[j]: column nf + 8*(j&1), k = 8*k8 + t + 4*(j>>1)
          const float v = lds_f32(bsm + (uint32_t)((k8 * 2 + (j >> 1)) * S::KG_BYTES) + ((j & 1) ? off1 : off0));
          hi[k8][j] = tf32_hi_bits(v);
          lo[k8][j] = __float_as_uint(tf32_lo(v));
        }
      named_bar_sync(1, gt::CONSUMERS);   // every consumer has written its share of A_lo
      fence_regs(hi);   // fragments and accumulators are final before the warpgroup fence
      fence_regs(lo);
      fence_regs(acc_h);
      fence_regs(acc_s);
      wgmma_fence();
      const uint32_t ahi = ast + (uint32_t)(m_off * 128), alo = ahi + gt::A_BYTES;
#pragma unroll
      for (int k8 = 0; k8 < gt::BK / 8; ++k8) {
        const uint64_t dh = gmma_desc_sw128(ahi + k8 * 32), dl = gmma_desc_sw128(alo + k8 * 32);
        wgmma_tf32_rs<WM>(acc_h, hi[k8], dh);
        wgmma_tf32_rs<WM>(acc_s, hi[k8], dl);
        wgmma_tf32_rs<WM>(acc_s, lo[k8], dh);
      }
      wgmma_commit();
      wgmma_wait_all();
      fence_regs(acc_h);
      fence_regs(acc_s);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // ===================== park the tile: every MMA of this CTA has completed, the stages are idle =====================
    named_bar_sync(1, gt::CONSUMERS);
    float* part = reinterpret_cast<float*>(smem);
#pragma unroll
    for (int i = 0; i < WM / 2; ++i) {
      const int n = nf + 8 * ((i >> 1) & 1), m = m_off + 8 * (i >> 2) + 2 * t + (i & 1);
      part[m * PSTRIDE + n] = acc_h[i] + acc_s[i];
    }
  }

  // ---- the K slices meet in distributed shared memory: rank r folds rows [r*128/S, (r+1)*128/S) of the tile ----
  if (splits > 1) {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");      // every CTA of the cluster parked its partial
  } else {
    __syncthreads();
  }
  const int rows_per = gt::BM / splits;
  const uint32_t part_s = smem_u32(smem);
  constexpr int V4 = BN / 4;
  for (int idx = threadIdx.x; idx < rows_per * V4; idx += gt::THREADS) {
    const int r = split * rows_per + idx / V4, c = (idx % V4) * 4;
    const int gm = m0 + r, gn = n0 + c;
    if (gm >= M || gn >= N) continue;
    const uint32_t off = part_s + (uint32_t)((r * PSTRIDE + c) * 4);
    float4 v;
    if (splits == 1) {
      v = lds_f4(off);
    } else {
      v = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s2 = 0; s2 < splits; ++s2) {                                   // fixed rank order: bit-reproducible
        uint32_t raddr;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(off), "r"((uint32_t)s2));
        float4 t;
        asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(t.x), "=f"(t.y), "=f"(t.z), "=f"(t.w) : "r"(raddr) : "memory");
        v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
      }
    }
    if (bias) {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + gn));
      v.x += bv.x; v.y += bv.y; v.z += bv.z; v.w += bv.w;
    }
    if (R) {
      const float4 rv = __ldg(reinterpret_cast<const float4*>(R + (size_t)gm * N + gn));
      v.x += rv.x; v.y += rv.y; v.z += rv.z; v.w += rv.w;
    }
    v = apply_act_rt(v, act);
    *reinterpret_cast<float4*>(C + (size_t)gm * N + gn) = v;
  }
  if (splits > 1) {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");      // peers may still be reading this CTA's partial
  }
}

// --------------------------------------------------------------------------------- host side ----
struct GKey {
  const void* p;
  int64_t a, b, c;
  bool operator==(const GKey& o) const { return p == o.p && a == o.a && b == o.b && c == o.c; }
};
struct GKeyHash {
  size_t operator()(const GKey& k) const {
    return std::hash<const void*>()(k.p) ^ ((size_t)k.a * 1315423911u) ^ ((size_t)k.b << 21) ^ ((size_t)k.c << 42);
  }
};

static bool cached_map(const GKey& key, const std::function<bool(CUtensorMap*)>& make, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<GKey, CUtensorMap, GKeyHash> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    return true;
  }
  CUtensorMap m;
  if (!make(&m)) return false;
  if (cache.size() > 8192) cache.clear();
  cache[key] = m;
  *out = m;
  return true;
}

bool gemm_tc_supported(const float* A, const float* B, const float* bias, const float* R, const float* C, int M, int N, int K,
                       int lda) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return M >= 64 && N >= 64 && N % 32 == 0 && K >= 32 && lda % 4 == 0 && lda >= K && al16(A) && al16(B) && al16(C) &&
         (!bias || al16(bias)) && (!R || al16(R)) && tc_encode_fn() != nullptr;
}

template <int BN, bool IM2COL>
static cudaError_t launch_gt(const CUtensorMap& am, const CUtensorMap& bm, const float* bias, const float* R, float* C, int M,
                             int N, int K, int act, const ConvGeom& cg, cudaStream_t s) {
  static bool attr[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BN, IM2COL>, cudaFuncAttributeMaxDynamicSharedMemorySize, GtSmem<BN>::TOTAL);
    if (e != cudaSuccess) return e;
    attr[dev & 63] = true;
  }
  const int tiles = ((N + BN - 1) / BN) * ((M + gt::BM - 1) / gt::BM);
  const int kblocks = (K + gt::BK - 1) / gt::BK;
  // split-K over a cluster when the tile grid alone leaves most of the SMs idle and K is long enough to share
  const int sms = device_sm_count();
  int splits = 1;
  while (splits < 8 && tiles * splits * 2 <= sms && kblocks / (splits * 2) >= 6) splits *= 2;
  static const int force = [] {
    const char* e = getenv("TFSC_GEMM_SPLITK");   // 0 = never split (A/B), 2 / 4 / 8 = force where K allows
    return e ? atoi(e) : -1;
  }();
  if (force == 0) splits = 1;
  else if (force > 0) {
    splits = 1;
    while (splits < force && splits < 8 && kblocks / (splits * 2) >= 1) splits *= 2;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((N + BN - 1) / BN, (M + gt::BM - 1) / gt::BM, splits);
  cfg.blockDim = dim3(gt::THREADS);
  cfg.dynamicSmemBytes = GtSmem<BN>::TOTAL;
  cfg.stream = s;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (splits > 1) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = 1;
    at[na].val.clusterDim.y = 1;
    at[na].val.clusterDim.z = splits;
    ++na;
  }
  static const bool pdl = [] {   // programmatic dependent launch is on unless TFSC_PDL=0
    const char* e = getenv("TFSC_PDL");
    return !e || atoi(e) != 0;
  }();
  if (pdl) {
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BN, IM2COL>, am, bm, bias, R, C, M, N, K, act, cg);
  g_launches_nn++;
  return e != cudaSuccess ? e : cudaGetLastError();
}

static int pick_bn(int M, int N) {
  if (N % 128 != 0 && N <= 128) return 64;
  // small problems: 128 x 64 tiles double the CTA count (BERT's N = 768 projections: 48 -> 96 CTAs on 132 SMs)
  const long tiles128 = (long)((N + 127) / 128) * ((M + gt::BM - 1) / gt::BM);
  return tiles128 < 120 && N % 64 == 0 ? 64 : 128;
}

static bool weight_map(const float* B, int K, int N, int BN, CUtensorMap* bm) {
  EncodeTiledFn enc = tc_encode_fn();
  return cached_map({B, K, N, BN}, [&](CUtensorMap* m) {
    const cuuint64_t gdim[3] = {32, (cuuint64_t)K, (cuuint64_t)(N / 32)};
    const cuuint64_t gstride[2] = {(cuuint64_t)N * 4, 128};
    const cuuint32_t box[3] = {32, 4, (cuuint32_t)(BN / 32)};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(B), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }, bm);
}

cudaError_t launch_gemm_tc(const float* A, const float* B, const float* bias, const float* R, float* C, int M, int N, int K,
                           int lda, int act, cudaStream_t s) {
  EncodeTiledFn enc = tc_encode_fn();
  if (!enc) return cudaErrorNotSupported;
  const int BN = pick_bn(M, N);
  // gridDim.y (one CTA row per 128 rows) is capped at 65,535: a taller A runs as consecutive launches over row chunks,
  // each with its own A map (the map cache is keyed by base pointer); one launch below the cap, as before
  constexpr int chunk_rows = kMaxGridY * gt::BM;
  for (int r0 = 0; r0 < M; r0 += chunk_rows) {
    const int rows = M - r0 < chunk_rows ? M - r0 : chunk_rows;
    const float* a = A + (size_t)r0 * lda;
    CUtensorMap am, bm;
    if (!cached_map({a, rows, K, lda}, [&](CUtensorMap* m) {
          const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
          const cuuint64_t gstride[1] = {(cuuint64_t)lda * 4};
          const cuuint32_t box[2] = {(cuuint32_t)gt::BK, (cuuint32_t)gt::BM};
          const cuuint32_t estr[2] = {1, 1};
          return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(a), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
        }, &am))
      return cudaErrorInvalidValue;
    if (!weight_map(B, K, N, BN, &bm)) return cudaErrorInvalidValue;
    const ConvGeom none{};
    const float* r = R ? R + (size_t)r0 * N : nullptr;
    float* c = C + (size_t)r0 * N;
    const cudaError_t e = BN == 128 ? launch_gt<128, false>(am, bm, bias, r, c, rows, N, K, act, none, s)
                                    : launch_gt<64, false>(am, bm, bias, r, c, rows, N, K, act, none, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// ---- implicit-GEMM convolution: NHWC activations x HWIO kernel, A tiles gathered by TMA im2col (no col buffer) ----
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeIm2colFn im2col_encode_fn() {
  static EncodeIm2colFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<EncodeIm2colFn>(p);
  }();
  return fn;
}

bool conv_tc_supported(const float* x, const float* w, const float* bias, const float* R, const float* y, int Bn, int H, int W,
                       int C, int KH, int KW, int stride, int pad, int OH, int OW, int N) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const long M = (long)Bn * OH * OW;
  return C % 32 == 0 && N >= 64 && N % 32 == 0 && M >= 64 && KH >= 1 && KW >= 1 && KH <= 16 && KW <= 16 && stride >= 1 && stride <= 8 &&
         pad >= 0 && pad < KH && pad < KW && H > 0 && W > 0 && al16(x) && al16(w) && al16(y) && (!bias || al16(bias)) &&
         (!R || al16(R)) && tc_encode_fn() != nullptr && im2col_encode_fn() != nullptr;
}

cudaError_t launch_conv_tc(const float* x, const float* w, const float* bias, const float* R, float* y, int Bn, int H, int W, int C,
                           int KH, int KW, int stride, int pad, int OH, int OW, int N, int act, cudaStream_t s) {
  EncodeIm2colFn enc = im2col_encode_fn();
  if (!enc) return cudaErrorNotSupported;
  const int M = Bn * OH * OW, K = KH * KW * C;
  const int BN = pick_bn(M, N);
  // gridDim.y (one CTA row per 128 output pixels) is capped at 65,535: a larger batch runs as consecutive launches over
  // whole images, each with an im2col map over its own images; one launch below the cap, as before
  const int per_img = OH * OW;
  const int chunk = kMaxGridY * gt::BM / per_img > 0 ? kMaxGridY * gt::BM / per_img : 1;
  for (int b0 = 0; b0 < Bn; b0 += chunk) {
    const int nb = Bn - b0 < chunk ? Bn - b0 : chunk;
    const float* xc = x + (size_t)b0 * H * W * C;
    CUtensorMap am, bm;
    if (!cached_map({xc, ((int64_t)nb << 40) | ((int64_t)H << 20) | W, ((int64_t)C << 32) | (KH << 16) | KW, ((int64_t)stride << 8) | pad},
                    [&](CUtensorMap* m) {
          const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)nb};
          const cuuint64_t gstride[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
          // base pixels (top-left corner of the filter window, input space) range over [-pad, dim + pad - K] per axis,
          // visited with the conv stride; tap offsets {kw, kh} are added per load
          const int lower[2] = {-pad, -pad};
          const int upper[2] = {pad - (KW - 1), pad - (KH - 1)};
          const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
          return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(xc), gdim, gstride, lower, upper, (cuuint32_t)gt::BK,
                     (cuuint32_t)gt::BM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
        }, &am))
      return cudaErrorInvalidValue;
    if (!weight_map(w, K, N, BN, &bm)) return cudaErrorInvalidValue;
    const ConvGeom cg{C, KW, OH, OW, stride, pad};
    const size_t out0 = (size_t)b0 * per_img * N;
    const float* r = R ? R + out0 : nullptr;
    const cudaError_t e = BN == 128 ? launch_gt<128, true>(am, bm, bias, r, y + out0, nb * per_img, N, K, act, cg, s)
                                    : launch_gt<64, true>(am, bm, bias, r, y + out0, nb * per_img, N, K, act, cg, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace tfsc
