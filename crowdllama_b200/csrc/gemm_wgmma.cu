// gemm_wgmma.cu — prefill / batched-decode weight projections on the Hopper tensor cores (wgmma).
//
//   Y[t][n] (+)= sum_k X[t][k] * W[n][k]        X bf16 [T][K], W bf16 [N][K] (both K-major), Y fp32
//
// This is the "weight projections as tensor-core tiles for prefill" row of SURVEY.md §8a (kernel table).
//
// Mapping (swap-AB so small token counts waste N, not M):
//   MMA A operand = W tile  [128 rows n ][64 k]  -> accumulator rows    (n)
//   MMA B operand = X tile  [BT  rows t ][64 k]  -> accumulator columns (t)
//   each consumer warpgroup owns 64 of the 128 W rows: wgmma m64 nBT k16, accumulators in registers.
// Warp roles (384 threads, 1 CTA / SM, persistent over tiles):
//   warpgroup 0     TMA producer  : cp.async.bulk.tensor.2d (128B swizzle) into an NST-stage mbarrier ring (one thread)
//   warpgroups 1-2  MMA + epilogue: wgmma.mma_async from the ring, one k-block in flight while the previous one's stage
//                                   is released; then the epilogue straight from the accumulator registers
// Tile order: consecutive tiles share the W tile (t fastest), so W streams from HBM once and X (<= 32 MB) stays
// L2-resident.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace cl {

namespace {

using namespace wg;

struct GemmParams {
  float* Y;
  int T, N, K, ldy;
  int accumulate_into_y;  // 1: Y += result (residual add in place)
  int k_splits;           // > 1: split-K; split s writes its partial to Y + s * T * ldy (the consumer sums in fixed order)
  int pre_stages;         // PDL launches only: W tiles of the first stages requested before griddepcontrol.wait (0 = none)
  __nv_bfloat16* act;     // EPI_SILU: act[t][i] = bf16(silu(gate_i) * up_i), row stride ld_act
  int ld_act;
};
enum { EPI_F32 = 0, EPI_SILU = 1 };

// p is __grid_constant__ so that its fields are read from the parameter bank where they are used: as a plain by-value
// struct the compiler loads them all into registers at kernel entry (+2 to +10 registers per instantiation).
template <int BT, int NST, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, const __grid_constant__ GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr uint32_t A_BYTES = BM * BK * 2;         // 16 KB
  constexpr uint32_t B_BYTES = BT * BK * 2;
  constexpr uint32_t STAGE = A_BYTES + B_BYTES;
  constexpr int NI = BT / 8;                        // accumulator column groups of 8
  // dynamic smem base is only guaranteed 16-byte aligned: round up to 1024 for the 128B swizzle
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)NST * STAGE);
  uint64_t* empty = full + NST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_t = (p.T + BT - 1) / BT, num_n = (p.N + BM - 1) / BM;
  const int ksp = p.k_splits > 1 ? p.k_splits : 1;
  const int num_tiles = num_t * num_n * ksp;          // split index is the slowest dimension
  const int num_kb_all = (p.K + BK - 1) / BK;
  const int kb_per = (num_kb_all + ksp - 1) / ksp;

  if (threadIdx.x == 0) {
    prefetch_tmap(&map_w);
    prefetch_tmap(&map_x);
    for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // one arrival per consumer warpgroup
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // no-ops unless launched with the programmatic-serialization attribute (batched decode step)

  if (warp < 4) {
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      // X is the previous kernel's output; W is constant: the W halves of the first p.pre_stages ring stages are
      // requested before griddepcontrol.wait (while the glue kernel in front still runs), their X halves after it.
      int pre = 0;
      if (p.pre_stages > 0 && (int)blockIdx.x < num_tiles) {
        const int tile = blockIdx.x;
        const int bt_ = tile % (num_t * num_n), ks = tile / (num_t * num_n);
        const int n0 = (bt_ / num_t) * BM;
        const int kb0 = ks * kb_per, kb1 = min(num_kb_all, kb0 + kb_per);
        pre = min(min(p.pre_stages, NST), kb1 - kb0);
        for (int i = 0; i < pre; ++i) {            // fresh barriers: every stage is empty
          mbar_arrive_expect_tx(&full[i], STAGE);
          tma_load_2d(base + (size_t)i * STAGE, &map_w, (kb0 + i) * BK, n0, &full[i]);
        }
      }
      pdl_wait();
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int bt_ = tile % (num_t * num_n), ks = tile / (num_t * num_n);
        const int n0 = (bt_ / num_t) * BM, t0 = (bt_ % num_t) * BT;
        const int kb0 = ks * kb_per, kb1 = min(num_kb_all, kb0 + kb_per);
        for (int kb = kb0; kb < kb1; ++kb) {
          uint8_t* sa = base + (size_t)stage * STAGE;
          if (pre > 0) {                           // W of this stage is already on its way
            --pre;
            tma_load_2d(sa + A_BYTES, &map_x, kb * BK, t0, &full[stage]);
          } else {
            mbar_wait(&empty[stage], phase ^ 1u);
            mbar_arrive_expect_tx(&full[stage], STAGE);
            tma_load_2d(sa, &map_w, kb * BK, n0, &full[stage]);
            tma_load_2d(sa + A_BYTES, &map_x, kb * BK, t0, &full[stage]);
          }
          if (++stage == NST) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ================= consumer warpgroups: rows m0 .. m0 + 63 of every tile =================
    pdl_wait();              // Y / the split-K workspace may still be read by the previous kernel
    const int m0 = (warp >> 2) * 64 - 64;
    const int wq = warp & 3, rq = lane >> 2, cq = lane & 3;
    const bool releaser = wq == 0 && lane == 0;
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int bt_ = tile % (num_t * num_n), ks = tile / (num_t * num_n);
      const int n0 = (bt_ / num_t) * BM, t0 = (bt_ % num_t) * BT;
      const int kb0 = ks * kb_per, num_kb = max(0, min(num_kb_all, kb0 + kb_per) - kb0);
      float acc[BT / 2];
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(base + (size_t)stage * STAGE);
        fence_regs(acc);
        fence();
#pragma unroll
        for (int k = 0; k < BK / UK; ++k)      // advance 32 bytes per MMA K inside the swizzle atom
          mma_ss<BT>(acc, make_desc(sa + (uint32_t)m0 * 128u + (uint32_t)k * 32u), make_desc(sa + A_BYTES + (uint32_t)k * 32u), 1u);
        commit();
        wait<1>();                             // the previous k-block's MMAs are done: release its stage
        fence_regs(acc);
        if (prev >= 0 && releaser) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == NST) { stage = 0; phase ^= 1u; }
      }
      wait<0>();
      fence_regs(acc);
      if (prev >= 0 && releaser) mbar_arrive(&empty[prev]);
      float* Yb = p.Y + (size_t)ks * p.T * p.ldy;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = n0 + m0 + wq * 16 + h * 8 + rq;
        if constexpr (EPI == EPI_F32) {
          if (n < p.N) {
            if (p.accumulate_into_y) {
              // residual add in place: all loads first, then the stores (a load-add-store per token serialises on the
              // load latency: the compiler cannot move the next load above a store it cannot prove disjoint)
              constexpr int NC = NI < 8 ? NI : 8;   // column groups per pass (16 loads in flight)
#pragma unroll
              for (int i0 = 0; i0 < NI; i0 += NC) {
                float y[2 * NC];
#pragma unroll
                for (int i = 0; i < NC; ++i)
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const int t = t0 + (i0 + i) * 8 + 2 * cq + e;
                    y[2 * i + e] = t < p.T ? __ldcg(Yb + (size_t)t * p.ldy + n) : 0.f;
                  }
#pragma unroll
                for (int i = 0; i < NC; ++i)
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const int t = t0 + (i0 + i) * 8 + 2 * cq + e;
                    if (t < p.T) Yb[(size_t)t * p.ldy + n] = y[2 * i + e] + acc[4 * (i0 + i) + 2 * h + e];
                  }
              }
            } else {
#pragma unroll
              for (int i = 0; i < NI; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int t = t0 + i * 8 + 2 * cq + e;
                  if (t < p.T) Yb[(size_t)t * p.ldy + n] = acc[4 * i + 2 * h + e];
                }
            }
          }
        } else {
          // rows are interleaved (2i = gate_i, 2i+1 = up_i): lanes l and l ^ 4 hold rows n and n ^ 1 of the same tokens.
          // Per token pair (c, c + 1) the even-row lane finishes token c (owns g, receives u), the odd-row lane token c + 1
          // (owns u, receives g): one shuffle, one SiLU, one store per lane.
          const int i2 = n >> 1, odd = rq & 1;
#pragma unroll
          for (int i = 0; i < NI; ++i) {
            const float a0 = acc[4 * i + 2 * h], a1 = acc[4 * i + 2 * h + 1];
            const float recv = __shfl_xor_sync(0xffffffffu, odd ? a0 : a1, 4);   // odd sends u[c], even sends g[c + 1]
            const float gt = odd ? recv : a0, up = odd ? a1 : recv;
            const int t = t0 + i * 8 + 2 * cq + odd;
            if (n < p.N && t < p.T)
              p.act[(size_t)t * p.ld_act + i2] = __float2bfloat16_rn(__fdividef(gt, 1.0f + __expf(-gt)) * up);
          }
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 row-major [rows][K] tensor, box = {64 k, box_rows}, 128B swizzle, OOB -> zeros
bool make_map(CUtensorMap* map, const void* ptr, int rows, int K, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

// 2-D bf16 tensor map for KV pools etc.: [rows][cols] row-major, box {box_cols, box_rows}, 128B swizzle
bool make_tmap_2d_bf16(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

namespace {

template <int BT, int NST, int EPI = EPI_F32>
cudaError_t launch_inst(const CUtensorMap& mw, const CUtensorMap& mx, const GemmParams& p, cudaStream_t st, bool pdl) {
  auto kern = gemm_wgmma_kernel<BT, NST, EPI>;
  constexpr size_t smem = (size_t)NST * (BM * BK * 2 + BT * BK * 2) + 1024 + 256;
  static PerDeviceOnce attr;
  if (attr.pending()) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr.mark();
  }
  const int tiles = ((p.T + BT - 1) / BT) * ((p.N + BM - 1) / BM) * (p.k_splits > 1 ? p.k_splits : 1);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  return launch_pdl(kern, dim3(grid), dim3(384), smem, st, pdl, mw, mx, p);
}

}  // namespace

// split s sums k-blocks [s * ceil(nkb / k_splits), ...): every split needs >= 1 k-block (k_splits <= 1: unsplit)
bool gemm_splits_supported(int K, int k_splits) {
  const int nkb = (K + BK - 1) / BK;
  return k_splits <= 1 || (k_splits <= nkb && (nkb + k_splits - 1) / k_splits * (k_splits - 1) < nkb);
}

bool gemm_tc_supported(int T, int N, int K) { return T > 0 && N > 0 && K > 0 && K % 8 == 0 && get_encode() != nullptr; }

// token tile: the smallest of 32 / 64 / 128 that holds T (prefill takes 128-token tiles)
static int token_tile(int T) { return T > 64 ? 128 : T > 32 ? 64 : 32; }

int launch_gemm_bf16(const __nv_bfloat16* X, const __nv_bfloat16* W, float* Y, const float* resid, int T, int N, int K,
                     cudaStream_t st, int k_splits, bool pdl) {
  if (!gemm_tc_supported(T, N, K)) return -1;
  if (resid && resid != Y) return -1;  // residual add is in place
  const int BT = token_tile(T);
  CUtensorMap mw, mx;
  if (!make_map(&mw, W, N, K, BM) || !make_map(&mx, X, T, K, BT)) return -1;
  if (!gemm_splits_supported(K, k_splits) || (k_splits > 1 && resid)) return -1;
  // PDL launches request the W tiles of the whole ring (at most 8 stages) before waiting for the kernel in front
  GemmParams p{Y, T, N, K, N, resid ? 1 : 0, k_splits, pdl ? 8 : 0, nullptr, 0};
  cudaError_t e;
  switch (BT) {
    case 128: e = launch_inst<128, 6>(mw, mx, p, st, pdl); break;
    case 64: e = launch_inst<64, 8>(mw, mx, p, st, pdl); break;
    default: e = launch_inst<32, 8>(mw, mx, p, st, pdl); break;
  }
  return e == cudaSuccess ? 1 : -1;
}

// Prefill gate|up projection with the SiLU epilogue (no fp32 round trip through HBM).  One CTA per 128 x BT tile (no split-K).
int launch_gemm_bf16_silu(const __nv_bfloat16* X, const __nv_bfloat16* W, int T, int N, int K, __nv_bfloat16* act, int ld_act, cudaStream_t st) {
  if (!gemm_tc_supported(T, N, K) || (N & 1)) return -1;
  const int BT = token_tile(T);
  CUtensorMap mw, mx;
  if (!make_map(&mw, W, N, K, BM) || !make_map(&mx, X, T, K, BT)) return -1;
  GemmParams p{nullptr, T, N, K, N, 0, 1, 0, act, ld_act};
  cudaError_t e;
  switch (BT) {
    case 128: e = launch_inst<128, 6, EPI_SILU>(mw, mx, p, st, false); break;
    case 64: e = launch_inst<64, 8, EPI_SILU>(mw, mx, p, st, false); break;
    default: e = launch_inst<32, 8, EPI_SILU>(mw, mx, p, st, false); break;
  }
  return e == cudaSuccess ? 1 : -1;
}

}  // namespace cl
