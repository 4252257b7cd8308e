// decode_kernels.cu — single-token (and small-batch) decode kernels for sm_90a.
//
// These implement the arithmetic that the reference reaches through callOllamaAPI
// (/root/reference/pkg/crowdllama/api.go:108-160 -> ollama v0.9.6 llama.cpp decode loop; SURVEY.md
// §8a row a8): RMSNorm-fused weight GEMVs (HBM-bound), RoPE + paged-KV append + split-KV GQA
// attention, embedding gather, argmax.  All of them are HBM-bound byte streaming: no tensor cores.
//
//   variant 0  gemv_ldg_kernel : coalesced 128-bit LDG (L1 no-allocate, L2 evict-first), warp per row pair
//   variant 1  gemv_ring_kernel: weights streamed by a producer warp with 1-D TMA bulk copies
//                                (cp.async.bulk -> UBLKCP) into an mbarrier ring; 8 consumer warps
//                                keep their x slice in registers.  The producer never waits for
//                                activations, so with PDL the next kernel's ring fills while the
//                                previous kernel drains.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace cl {

static int g_sm_count[64] = {0};   // per device ordinal (one engine per GPU process, but a process may open several)
static bool g_carveout_max = true;
int sm_count() {
  int dev = 0;
  cudaGetDevice(&dev);
  int& n = g_sm_count[dev & 63];
  if (!n) {
    const char* cv = getenv("CL_CARVEOUT_MAX");
    if (cv && *cv == '0') g_carveout_max = false;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Every kernel of the token step asks for the maximum shared-memory carve-out: a different L1/shared
// split per kernel would force the SM to drain before the next kernel's CTAs can become resident,
// which defeats the PDL overlap (and a 101 KB ring kernel would not co-reside with its successor).
template <typename Kern>
static void prefer_max_smem(Kern kern) {
  if (g_carveout_max) cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

template <typename Kern, typename Args>
static cudaError_t launch_ex(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, const Args& args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, args);
}

// ================================================================================================
// shared epilogue
// ================================================================================================
template <int EPI>
__device__ __forceinline__ void gemv_epilogue(const GemvArgs& a, int slot, int row0, float v0, float v1) {
  // (row0, row0+1) is a row pair
  if (EPI == EPI_STORE) {
    float* y = a.y + (size_t)slot * a.y_stride;
    y[row0] = v0;
    y[row0 + 1] = v1;
  } else if (EPI == EPI_RESID) {
    const float* r = a.resid + (size_t)slot * a.y_stride;
    float* y = a.y + (size_t)slot * a.y_stride;
    float r0 = __ldcg(r + row0), r1 = __ldcg(r + row0 + 1);
    y[row0] = r0 + v0;
    y[row0 + 1] = r1 + v1;
  } else if (EPI == EPI_GATEUP) {  // v0 = gate_i, v1 = up_i
    float* y = a.y + (size_t)slot * a.y_stride;
    float si = v0 / (1.0f + __expf(-v0));
    y[row0 >> 1] = bf16_round(si * v1);
  } else {  // EPI_QKV: (v0, v1) = dims (j, j + half) of one head -> RoPE, bf16 round, q out / KV append
    const QkvEpi& e = a.qkv;
    const int HD = e.head_dim, half = HD >> 1;
    const int p = row0 >> 1;
    const int hh = p / half, j = p - hh * half;
    const int pos = e.pos[slot];
    if (hh < e.n_heads + e.n_kv) {
      const float2 cs = e.rope[(size_t)pos * half + j];
      const float r0 = bf16_round(v0 * cs.x - v1 * cs.y), r1 = bf16_round(v1 * cs.x + v0 * cs.y);
      if (hh < e.n_heads) {
        float* y = a.y + (size_t)slot * a.y_stride + (size_t)hh * HD;
        y[j] = r0;
        y[j + half] = r1;
      } else {
        const int g = hh - e.n_heads;
        const int page = e.block_tables[(size_t)slot * e.bt_stride + pos / e.page_size];
        const size_t base = (((size_t)page * e.n_kv + g) * e.page_size + pos % e.page_size) * HD;
        e.kpool[base + j] = __float2bfloat16_rn(r0);
        e.kpool[base + j + half] = __float2bfloat16_rn(r1);
      }
    } else {
      const int g = hh - e.n_heads - e.n_kv;
      const int page = e.block_tables[(size_t)slot * e.bt_stride + pos / e.page_size];
      const size_t base = (((size_t)page * e.n_kv + g) * e.page_size + pos % e.page_size) * HD;
      e.vpool[base + j] = __float2bfloat16_rn(v0);
      e.vpool[base + j + half] = __float2bfloat16_rn(v1);
    }
  }
}

// ================================================================================================
// variant 0: LDG GEMV.  block = 256 threads (8 warps), x (normalised) staged in shared memory.
// ================================================================================================
template <int EPI, bool NORM>
__global__ void __launch_bounds__(256, 2) gemv_ldg_kernel(const GemvArgs a) {
  extern __shared__ __align__(16) float xs[];
  __shared__ float red[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y;
  if (a.pdl_early) pdl_launch_dependents();
  pdl_wait();
  const int slot = a.slots ? a.slots[b] : b;
  const int K = a.K;

  if (NORM) {
    const float* h = a.h + (size_t)slot * a.x_stride;
    float ss = 0.f;
    for (int i = tid * 4; i < K; i += 256 * 4) {
      float4 v = ldcg4(h + i);
      *reinterpret_cast<float4*>(xs + i) = v;
      ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
    }
    ss = warp_sum(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += red[w];
    const float inv = 1.0f / sqrtf(tot / (float)K + a.eps);
    for (int i = tid * 4; i < K; i += 256 * 4) {
      float4 v = *reinterpret_cast<float4*>(xs + i);
      float4 g = *reinterpret_cast<const float4*>(a.gain + i);
      v.x = bf16_round(v.x * inv * g.x); v.y = bf16_round(v.y * inv * g.y);
      v.z = bf16_round(v.z * inv * g.z); v.w = bf16_round(v.w * inv * g.w);
      *reinterpret_cast<float4*>(xs + i) = v;
    }
  } else {
    const float* x = a.x + (size_t)slot * a.x_stride;
    for (int i = tid * 4; i < K; i += 256 * 4)
      *reinterpret_cast<float4*>(xs + i) = ldcg4(x + i);
  }
  __syncthreads();

  const int total_warps = gridDim.x * 8;
  const int gw = blockIdx.x * 8 + warp;
  const int npairs = a.N >> 1;
  const int p0 = (int)(((long long)npairs * gw) / total_warps);
  const int p1 = (int)(((long long)npairs * (gw + 1)) / total_warps);
  const int nchunk = K >> 4;  // 16 bf16 = 32 bytes per lane per load
  const float4* xs4 = reinterpret_cast<const float4*>(xs);

  for (int p = p0; p < p1; ++p) {
    const uint8_t* w0 = reinterpret_cast<const uint8_t*>(a.W + (size_t)(2 * p) * K);
    const uint8_t* w1 = w0 + (size_t)K * 2;
    float acc0 = 0.f, acc1 = 0.f;
    int c = lane;
    for (; c + 32 < nchunk; c += 64) {
      const u32x8 a0 = ldg_stream256(w0 + (size_t)c * 32), a1 = ldg_stream256(w0 + (size_t)(c + 32) * 32);
      const u32x8 b0 = ldg_stream256(w1 + (size_t)c * 32), b1 = ldg_stream256(w1 + (size_t)(c + 32) * 32);
      acc0 = dot16(a0, xs4 + 4 * c, acc0); acc1 = dot16(b0, xs4 + 4 * c, acc1);
      acc0 = dot16(a1, xs4 + 4 * (c + 32), acc0); acc1 = dot16(b1, xs4 + 4 * (c + 32), acc1);
    }
    for (; c < nchunk; c += 32) {
      const u32x8 a0 = ldg_stream256(w0 + (size_t)c * 32);
      const u32x8 b0 = ldg_stream256(w1 + (size_t)c * 32);
      acc0 = dot16(a0, xs4 + 4 * c, acc0);
      acc1 = dot16(b0, xs4 + 4 * c, acc1);
    }
    acc0 = warp_sum(acc0);
    acc1 = warp_sum(acc1);
    if (lane == 0) gemv_epilogue<EPI>(a, slot, 2 * p, acc0, acc1);
    if (!a.pdl_early && p == p1 - 2) pdl_launch_dependents();   // about to start the last row pair
  }
}

// ================================================================================================
// variant 1: TMA-ring streaming GEMV.
//   block = 288 threads: warps 0..7 consume, warp 8 produces.  A stage holds TR full rows
//   (TR*K bf16, contiguous in W -> ONE bulk copy).  Consumer warp w works on row (w / S) of the
//   stage, K-slice (w % S); its CPL*8 x values per lane live in registers for the whole kernel.
//   Per-row partials go to shared memory; one barrier at the end, then a coalesced epilogue.
// ================================================================================================
template <int EPI, bool NORM, int TR, int S, int CPL, int NST>
__global__ void __launch_bounds__(288, 1) gemv_ring_kernel(const GemvArgs a) {
  static_assert(TR * S == 8, "8 consumer warps");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  constexpr int K = S * CPL * 256;
  constexpr uint32_t STAGE_BYTES = (uint32_t)TR * K * 2;
  uint8_t* ring = smem_raw;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)NST * STAGE_BYTES);
  uint64_t* empty = full + NST;
  float* ssw = reinterpret_cast<float*>(empty + NST);  // [8]
  float* part = ssw + 8;                                // [local_rows][S]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y;
  // split in units that keep every row pair (2i, 2i+1) inside one CTA
  constexpr int U = (TR == 1) ? 2 : 1;
  const int NU = a.N / (TR * U);
  const int tile0 = U * (int)(((long long)NU * blockIdx.x) / gridDim.x);
  const int tile1 = U * (int)(((long long)NU * (blockIdx.x + 1)) / gridDim.x);
  const int ntiles = tile1 - tile0;

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  if (a.pdl_early) pdl_launch_dependents();
  const bool stamp = a.tl != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && tid == 0;
  if (stamp) a.tl[0] = gtime_ns();

  if (warp == 8) {
    // ---------------- producer: weights do not depend on the previous kernel -> no pdl_wait here
    if (elect_one()) {
      const uint64_t pol = policy_evict_first();
      const uint8_t* src = reinterpret_cast<const uint8_t*>(a.W) + (size_t)tile0 * STAGE_BYTES;
      for (int it = 0; it < ntiles; ++it) {
        const int st = it % NST;
        const uint32_t par = (uint32_t)(it / NST) & 1u;
        mbar_wait(&empty[st], par ^ 1u);
        mbar_arrive_expect_tx(&full[st], STAGE_BYTES);
        bulk_g2s(ring + (size_t)st * STAGE_BYTES, src + (size_t)it * STAGE_BYTES, STAGE_BYTES, &full[st], pol);
      }
      // every byte this CTA will ever read from HBM is now in flight: let the next kernel's CTAs
      // become resident and start streaming THEIR weights while this one drains
      if (!a.pdl_early) pdl_launch_dependents();
    }
    // the producer warp must stay until the consumers are done with the barriers it arms
  } else {
    // ---------------- consumers
    const int r = warp / S, s = warp % S;
    const int kbase = s * (K / S);
    pdl_wait();
    if (stamp) a.tl[1] = gtime_ns();
    const int slot = a.slots ? a.slots[b] : b;
    float xr[CPL][8];
    if (NORM) {
      const float* h = a.h + (size_t)slot * a.x_stride;
      float ss = 0.f;
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        const int k = kbase + (c * 32 + lane) * 8;
        float4 v0 = ldcg4(h + k);
        float4 v1 = ldcg4(h + k + 4);
        xr[c][0] = v0.x; xr[c][1] = v0.y; xr[c][2] = v0.z; xr[c][3] = v0.w;
        xr[c][4] = v1.x; xr[c][5] = v1.y; xr[c][6] = v1.z; xr[c][7] = v1.w;
#pragma unroll
        for (int j = 0; j < 8; ++j) ss = fmaf(xr[c][j], xr[c][j], ss);
      }
      ss = warp_sum(ss);
      if (lane == 0) ssw[warp] = ss;
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float tot = 0.f;
#pragma unroll
      for (int i = 0; i < S; ++i) tot += ssw[i];  // warps 0..S-1 are row 0, slices 0..S-1: cover K once
      const float inv = 1.0f / sqrtf(tot / (float)K + a.eps);
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        const int k = kbase + (c * 32 + lane) * 8;
        float4 g0 = *reinterpret_cast<const float4*>(a.gain + k);
        float4 g1 = *reinterpret_cast<const float4*>(a.gain + k + 4);
        xr[c][0] = bf16_round(xr[c][0] * inv * g0.x); xr[c][1] = bf16_round(xr[c][1] * inv * g0.y);
        xr[c][2] = bf16_round(xr[c][2] * inv * g0.z); xr[c][3] = bf16_round(xr[c][3] * inv * g0.w);
        xr[c][4] = bf16_round(xr[c][4] * inv * g1.x); xr[c][5] = bf16_round(xr[c][5] * inv * g1.y);
        xr[c][6] = bf16_round(xr[c][6] * inv * g1.z); xr[c][7] = bf16_round(xr[c][7] * inv * g1.w);
      }
    } else {
      const float* x = a.x + (size_t)slot * a.x_stride;
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        const int k = kbase + (c * 32 + lane) * 8;
        float4 v0 = ldcg4(x + k);
        float4 v1 = ldcg4(x + k + 4);
        xr[c][0] = v0.x; xr[c][1] = v0.y; xr[c][2] = v0.z; xr[c][3] = v0.w;
        xr[c][4] = v1.x; xr[c][5] = v1.y; xr[c][6] = v1.z; xr[c][7] = v1.w;
      }
    }

    if (stamp) a.tl[2] = gtime_ns();   // x in registers: start consuming
    const uint32_t row_off = (uint32_t)(r * K + kbase + lane * 8) * 2u;
    for (int it = 0; it < ntiles; ++it) {
      const int st = it % NST;
      const uint32_t par = (uint32_t)(it / NST) & 1u;
      mbar_wait(&full[st], par);
      const uint8_t* base = ring + (size_t)st * STAGE_BYTES + row_off;
      uint4 w[CPL];
#pragma unroll
      for (int c = 0; c < CPL; ++c) w[c] = *reinterpret_cast<const uint4*>(base + c * 512);
      // The stage's next bulk copy writes through the async proxy, which the arrive's release does not order
      // against these generic reads: without the fence the reads may still be in flight when the copy lands.
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        acc = fmaf(bf16_lo(w[c].x), xr[c][0], acc); acc = fmaf(bf16_hi(w[c].x), xr[c][1], acc);
        acc = fmaf(bf16_lo(w[c].y), xr[c][2], acc); acc = fmaf(bf16_hi(w[c].y), xr[c][3], acc);
        acc = fmaf(bf16_lo(w[c].z), xr[c][4], acc); acc = fmaf(bf16_hi(w[c].z), xr[c][5], acc);
        acc = fmaf(bf16_lo(w[c].w), xr[c][6], acc); acc = fmaf(bf16_hi(w[c].w), xr[c][7], acc);
      }
      acc = warp_sum(acc);
      if (lane == 0) part[(it * TR + r) * S + s] = acc;
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    // ---------------- epilogue: one thread per row pair, coalesced
    const int local_pairs = (ntiles * TR) >> 1;
    const int row_base = tile0 * TR;
    for (int p = tid; p < local_pairs; p += 256) {
      float v0 = 0.f, v1 = 0.f;
#pragma unroll
      for (int i = 0; i < S; ++i) { v0 += part[(2 * p) * S + i]; v1 += part[(2 * p + 1) * S + i]; }
      gemv_epilogue<EPI>(a, slot, row_base + 2 * p, v0, v1);
    }
    if (stamp) a.tl[3] = gtime_ns();
  }
}

struct RingCfg { int TR, S, CPL, NST; };
static bool ring_cfg_for(int K, RingCfg* c) {
  switch (K) {
    case 1024: *c = {2, 4, 1, 6}; return true;
    case 2048: *c = {2, 4, 2, 6}; return true;
    case 4096: *c = {2, 4, 4, 6}; return true;
    case 8192: *c = {1, 8, 4, 4}; return true;
    case 14336: *c = {1, 8, 7, 3}; return true;
    default: return false;
  }
}

bool gemv_variant_supported(int variant, int N, int K) {
  if (N <= 0 || K <= 0 || (N & 1) || (K & 15)) return false;
  if (variant == 0) return (size_t)K * 4 <= 200 * 1024;
  RingCfg c;
  if (!ring_cfg_for(K, &c)) return false;
  if (N % (2 * c.TR)) return false;  // each CTA owns whole row pairs
  return true;
}

static int g_last_gemv_ctas = 0;
template <int EPI, bool NORM, int TR, int S, int CPL, int NST>
static cudaError_t launch_ring_inst(const GemvArgs& a, cudaStream_t st, bool pdl) {
  constexpr int K = S * CPL * 256;
  constexpr int U = (TR == 1) ? 2 : 1;
  const int NU = a.N / (TR * U);
  int G = sm_count();
  if (G > NU) G = NU;
  const int max_tiles = U * ((NU + G - 1) / G);
  size_t smem = (size_t)NST * TR * K * 2 + (size_t)2 * NST * 8 + 8 * 4 + (size_t)(max_tiles + 1) * TR * S * 4 + 64;
  auto kern = gemv_ring_kernel<EPI, NORM, TR, S, CPL, NST>;
  static PerDeviceOnce attr_set;
  if (attr_set.pending()) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    prefer_max_smem(kern);
    attr_set.mark();
  }
  if (smem > 160 * 1024) return cudaErrorInvalidValue;
  g_last_gemv_ctas = G * a.batch;
  return launch_ex(kern, dim3(G, a.batch), dim3(288), smem, st, pdl, a);
}

template <int EPI, bool NORM>
static cudaError_t launch_ring(const GemvArgs& a, cudaStream_t st, bool pdl) {
  switch (a.K) {
    case 1024: return launch_ring_inst<EPI, NORM, 2, 4, 1, 6>(a, st, pdl);
    case 2048: return launch_ring_inst<EPI, NORM, 2, 4, 2, 6>(a, st, pdl);
    case 4096:
      // q|k|v and o-proj share the SM with the attention kernel (128 KB KV ring) under PDL: 4 stages (64 KB)
      // (fewer bytes in flight per SM than the bandwidth-latency product needs)
      return launch_ring_inst<EPI, NORM, 2, 4, 4, 6>(a, st, pdl);
    case 8192: return launch_ring_inst<EPI, NORM, 1, 8, 4, 4>(a, st, pdl);
    case 14336: return launch_ring_inst<EPI, NORM, 1, 8, 7, 3>(a, st, pdl);
    default: return cudaErrorInvalidValue;
  }
}

template <int EPI, bool NORM>
static cudaError_t launch_ldg(const GemvArgs& a, cudaStream_t st, bool pdl) {
  auto kern = gemv_ldg_kernel<EPI, NORM>;
  size_t smem = (size_t)a.K * 4;
  static PerDeviceOnce attr_set;
  if (attr_set.pending()) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    prefer_max_smem(kern);
    attr_set.mark();
  }
  int G = sm_count() * 2;
  int npairs = a.N / 2;
  if (G * 8 > npairs) G = (npairs + 7) / 8;
  g_last_gemv_ctas = G * a.batch;
  return launch_ex(kern, dim3(G, a.batch), dim3(256), smem, st, pdl, a);
}

int launch_gemv(int variant, int epi, bool norm, const GemvArgs& a, cudaStream_t st, bool pdl, int* n_ctas) {
  if (variant == 1 && !gemv_variant_supported(1, a.N, a.K)) variant = 0;
  // with TR==1 configs row-pair ownership needs even tile splits; handled in launch_ring_inst
  cudaError_t e = cudaErrorInvalidValue;
#define CL_DISPATCH(FN)                                                                   \
  if (epi == EPI_STORE) e = norm ? FN<EPI_STORE, true>(a, st, pdl) : FN<EPI_STORE, false>(a, st, pdl);   \
  else if (epi == EPI_RESID) e = norm ? FN<EPI_RESID, true>(a, st, pdl) : FN<EPI_RESID, false>(a, st, pdl); \
  else if (epi == EPI_GATEUP) e = norm ? FN<EPI_GATEUP, true>(a, st, pdl) : FN<EPI_GATEUP, false>(a, st, pdl);   \
  else e = norm ? FN<EPI_QKV, true>(a, st, pdl) : FN<EPI_QKV, false>(a, st, pdl);
  if (variant == 1) { CL_DISPATCH(launch_ring) } else { CL_DISPATCH(launch_ldg) }
#undef CL_DISPATCH
  if (n_ctas) *n_ctas = g_last_gemv_ctas;
  return e == cudaSuccess ? 1 : -1;
}

// ================================================================================================
// paged GQA decode attention (split-KV) — v3.
//   grid = (n_kv, nsplit, batch); block = 288: warp 8 streams this split's KV pages with 1-D TMA bulk
//   copies (one (page, kv-head) block of K and of V per stage, 64 KB ring) and warps 0..7 consume them
//   from shared memory.  RoPE and the KV append already happened in the q|k|v GEMV epilogue (EPI_QKV),
//   so the kernel reads roped q and tokens 0..pos from the cache.
//   PDL: everything the producer touches before griddepcontrol.wait (slots, pos, block table, K/V of
//   EARLIER tokens) is immutable during the token step, so the KV stream of this layer overlaps the
//   q|k|v GEMV that precedes it; only the page holding the current token is fetched after the wait.
//   The consumers' short latency-bound phase then overlaps the o-projection's weight prefetch.
// ================================================================================================
static int g_attn_ring_bytes = 64 * 1024;    // + 96 KB GEMV ring of the neighbouring kernel = co-resident under PDL (env CL_ATTN_RING_KB)
constexpr int kAttnRingBytesMax = 128 * 1024;
constexpr int kAttnMaxStages = 8;

template <int REP, int HD>
__global__ void __launch_bounds__(288) attn_decode_kernel(const AttnDecodeArgs a) {
  constexpr int NW = 8;              // consumer warps
  constexpr int LPT = HD / 8;        // lanes per token (16-byte chunk each)
  constexpr int TPW = 32 / LPT;      // tokens per warp pass
  constexpr float LOG2E = 1.4426950408889634f;
  constexpr int MAXS = 64;
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ uint64_t full[kAttnMaxStages], empty[kAttnMaxStages];
  __shared__ float red_m[NW][REP], red_l[NW][REP];
  __shared__ __align__(16) float red_acc[NW][REP][HD];
  __shared__ float cm_s[MAXS][REP], cw_s[MAXS][REP];
  __shared__ float cL_s[REP];
  __shared__ int is_last_s;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = blockIdx.x, split = blockIdx.y, b = blockIdx.z;
  const int P = a.page_size;
  const uint32_t half_bytes = (uint32_t)P * HD * 2;       // K (or V) block of one (page, kv head)
  const uint32_t slot_bytes = 2 * half_bytes;
  int nstg = a.ring_bytes / (int)slot_bytes;
  nstg = nstg > kAttnMaxStages ? kAttnMaxStages : nstg;

  if (tid == 0) {
    for (int i = 0; i < nstg; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NW); }
    fence_barrier_init();
  }
  __syncthreads();
  if (a.pdl_early) pdl_launch_dependents();
  const bool stamp = a.tl != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && tid == 0;
  if (stamp) a.tl[0] = gtime_ns();

  const int slot = a.slots ? a.slots[b] : b;
  const int pos = a.pos[slot];                 // stable for the whole step (written by the previous step's tail)
  const int ctx = pos + 1;
  const int total_pages = (ctx + P - 1) / P;
  const int pages_per_split = (total_pages + a.nsplit - 1) / a.nsplit;
  const int pg0 = split * pages_per_split;
  const int pg1 = min(total_pages, pg0 + pages_per_split);
  const int npg = pg1 > pg0 ? pg1 - pg0 : 0;
  const int* bt = a.block_tables + (size_t)slot * a.bt_stride;

  if (warp == NW) {
    // ---------------- producer
    if (elect_one()) {
      const uint64_t pol = policy_evict_first();
      const int cur_page = pos / P;            // its K/V row is written by the preceding EPI_QKV kernel
      for (int it = 0; it < npg; ++it) {
        const int st = it % nstg;
        const uint32_t par = (uint32_t)(it / nstg) & 1u;
        mbar_wait(&empty[st], par ^ 1u);
        if (pg0 + it == cur_page) pdl_wait();
        const int page = bt[pg0 + it];
        const size_t src = ((size_t)page * a.n_kv + g) * P * HD;
        uint8_t* dst = ring + (size_t)st * slot_bytes;
        mbar_arrive_expect_tx(&full[st], slot_bytes);
        bulk_g2s(dst, a.kpool + src, half_bytes, &full[st], pol);
        bulk_g2s(dst + half_bytes, a.vpool + src, half_bytes, &full[st], pol);
      }
    }
    return;
  }

  // ---------------- consumers (warps 0..7)
  pdl_wait();
  if (stamp) a.tl[1] = gtime_ns();
  const int sub = lane / LPT, j = lane % LPT;
  const float scale2 = rsqrtf((float)HD) * LOG2E;
  float qr[REP][8];
  {
    const float* q = a.q + (size_t)slot * a.q_stride + (size_t)g * REP * HD + j * 8;
#pragma unroll
    for (int hh = 0; hh < REP; ++hh) {
      const float4 q0 = ldcg4(q + hh * HD);
      const float4 q1 = ldcg4(q + hh * HD + 4);
      qr[hh][0] = q0.x; qr[hh][1] = q0.y; qr[hh][2] = q0.z; qr[hh][3] = q0.w;
      qr[hh][4] = q1.x; qr[hh][5] = q1.y; qr[hh][6] = q1.z; qr[hh][7] = q1.w;
    }
  }
  float m[REP], l[REP], acc[REP][8];
#pragma unroll
  for (int hh = 0; hh < REP; ++hh) {
    m[hh] = -INFINITY; l[hh] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[hh][i] = 0.f;
  }

  for (int it = 0; it < npg; ++it) {
    const int st = it % nstg;
    const uint32_t par = (uint32_t)(it / nstg) & 1u;
    mbar_wait(&full[st], par);
    const uint8_t* kbase = ring + (size_t)st * slot_bytes;
    const uint8_t* vbase = kbase + half_bytes;
    const int tok0 = (pg0 + it) * P;
    for (int tl = warp * TPW + sub; tl < P; tl += NW * TPW) {   // warp-uniform trip count (P % (NW*TPW) == 0 or all lanes step together)
      const bool active = tok0 + tl < ctx;
      const uint4 kk = *reinterpret_cast<const uint4*>(kbase + ((size_t)tl * HD + j * 8) * 2);
      const uint4 vv = *reinterpret_cast<const uint4*>(vbase + ((size_t)tl * HD + j * 8) * 2);
      float kf[8], vf[8];
      kf[0] = bf16_lo(kk.x); kf[1] = bf16_hi(kk.x); kf[2] = bf16_lo(kk.y); kf[3] = bf16_hi(kk.y);
      kf[4] = bf16_lo(kk.z); kf[5] = bf16_hi(kk.z); kf[6] = bf16_lo(kk.w); kf[7] = bf16_hi(kk.w);
      vf[0] = bf16_lo(vv.x); vf[1] = bf16_hi(vv.x); vf[2] = bf16_lo(vv.y); vf[3] = bf16_hi(vv.y);
      vf[4] = bf16_lo(vv.z); vf[5] = bf16_hi(vv.z); vf[6] = bf16_lo(vv.w); vf[7] = bf16_hi(vv.w);
      float sc[REP];
#pragma unroll
      for (int hh = 0; hh < REP; ++hh) {
        float p = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) p = fmaf(qr[hh][i], kf[i], p);
        sc[hh] = p;
      }
#pragma unroll
      for (int o = LPT / 2; o > 0; o >>= 1)
#pragma unroll
        for (int hh = 0; hh < REP; ++hh) sc[hh] += __shfl_xor_sync(0xffffffffu, sc[hh], o);
      if (active) {
#pragma unroll
        for (int hh = 0; hh < REP; ++hh) {
          const float s2 = sc[hh] * scale2;
          const float mn = fmaxf(m[hh], s2);
          const float corr = exp2f(m[hh] - mn);   // m = -inf -> 0
          const float p = exp2f(s2 - mn);
          l[hh] = l[hh] * corr + p;
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[hh][i] = fmaf(p, vf[i], acc[hh][i] * corr);
          m[hh] = mn;
        }
      }
    }
    fence_proxy_async();   // order the reads of this stage before the producer's next bulk copy into it
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
  }

  if (stamp) a.tl[2] = gtime_ns();   // all pages consumed
  // ---- merge the TPW token groups of a warp
#pragma unroll
  for (int o = LPT; o < 32; o <<= 1) {
#pragma unroll
    for (int hh = 0; hh < REP; ++hh) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[hh], o);
      const float lo = __shfl_xor_sync(0xffffffffu, l[hh], o);
      const float mn = fmaxf(m[hh], mo);
      const float c0 = (m[hh] == -INFINITY) ? 0.f : exp2f(m[hh] - mn);
      const float c1 = (mo == -INFINITY) ? 0.f : exp2f(mo - mn);
      l[hh] = l[hh] * c0 + lo * c1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float ao = __shfl_xor_sync(0xffffffffu, acc[hh][i], o);
        acc[hh][i] = acc[hh][i] * c0 + ao * c1;
      }
      m[hh] = mn;
    }
  }
  if (sub == 0) {
#pragma unroll
    for (int hh = 0; hh < REP; ++hh) {
      if (j == 0) { red_m[warp][hh] = m[hh]; red_l[warp][hh] = l[hh]; }
#pragma unroll
      for (int i = 0; i < 8; ++i) red_acc[warp][hh][j * 8 + i] = acc[hh][i];
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");

  // ---- CTA partial -> global
  float* part = a.part + ((((size_t)slot * a.n_kv + g) * a.nsplit + split) * REP) * (HD + 2);
  for (int t = tid; t < REP * HD; t += NW * 32) {
    const int hh = t / HD, i = t % HD;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < NW; ++w) M = fmaxf(M, red_m[w][hh]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      const float c = (red_m[w][hh] == -INFINITY) ? 0.f : exp2f(red_m[w][hh] - M);
      L = fmaf(red_l[w][hh], c, L);
      A = fmaf(red_acc[w][hh][i], c, A);
    }
    float* ph = part + (size_t)hh * (HD + 2);
    if (i == 0) { ph[0] = M; ph[1] = L; }
    ph[2 + i] = A;
  }
  if (stamp) a.tl[3] = gtime_ns();   // partial written (CTA 0 is rarely the combining CTA)
  __threadfence();
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (tid == 0) {
    unsigned* cnt = a.counters + (size_t)slot * a.n_kv + g;
    const unsigned old = atomicAdd(cnt, 1u);
    is_last_s = (old == (unsigned)a.nsplit - 1u);
    if (is_last_s) *cnt = 0u;  // re-arm for the next launch (graph replay)
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (!is_last_s) return;
  __threadfence();

  // ---- last split to finish combines all partials of this kv head: one L2 round trip brings every
  // split's (m, l) into shared memory, then the accumulators stream with independent loads.
  const float* pall = a.part + (((size_t)slot * a.n_kv + g) * a.nsplit) * REP * (HD + 2);
  const int ns = a.nsplit;   // host guarantees nsplit <= MAXS
  for (int t = tid; t < ns * REP; t += NW * 32) {
    const int sidx = t / REP, hh = t % REP;
    const float* ph = pall + ((size_t)sidx * REP + hh) * (HD + 2);
    cm_s[sidx][hh] = __ldcg(ph);
    cw_s[sidx][hh] = __ldcg(ph + 1);   // l for now
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (tid < REP) {
    float M = -INFINITY;
    for (int sidx = 0; sidx < ns; ++sidx) M = fmaxf(M, cm_s[sidx][tid]);
    float L = 0.f;
    for (int sidx = 0; sidx < ns; ++sidx) {
      const float ms = cm_s[sidx][tid];
      const float c = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
      L = fmaf(cw_s[sidx][tid], c, L);
      cw_s[sidx][tid] = c;             // weight of this split
    }
    cL_s[tid] = L;
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  // warp w accumulates splits w, w+8, ... for all REP*HD outputs: every load is independent, so the
  // whole partial set arrives in one L2 round trip; then an 8-way shared-memory reduction.
  {
    constexpr int OPL = REP * HD / 32;   // outputs per lane
    float accw[OPL];
#pragma unroll
    for (int k = 0; k < OPL; ++k) accw[k] = 0.f;
    for (int sidx = warp; sidx < ns; sidx += NW) {
      const float* ps = pall + (size_t)sidx * REP * (HD + 2);
#pragma unroll
      for (int k = 0; k < OPL; ++k) {
        const int o = lane + 32 * k, hh = o / HD, i = o % HD;
        accw[k] = fmaf(__ldcg(ps + (size_t)hh * (HD + 2) + 2 + i), cw_s[sidx][hh], accw[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < OPL; ++k) {
      const int o = lane + 32 * k;
      red_acc[warp][o / HD][o % HD] = accw[k];
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float* out = a.out + (size_t)slot * a.out_stride;
  for (int t = tid; t < REP * HD; t += NW * 32) {
    const int hh = t / HD, i = t % HD;
    float A = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) A += red_acc[w][hh][i];
    const float r = bf16_round(A / cL_s[hh]);
    out[(size_t)(g * REP + hh) * HD + i] = r;
    if (a.out_bf16) a.out_bf16[(size_t)b * a.out_stride + (size_t)(g * REP + hh) * HD + i] = __float2bfloat16_rn(r);
  }
}

int launch_attn_decode(const AttnDecodeArgs& a, cudaStream_t st, bool pdl) {
  const int rep = a.n_heads / a.n_kv;
  dim3 grid(a.n_kv, a.nsplit, a.batch), block(288);
  static bool env_read = false;
  if (!env_read) { const char* v = getenv("CL_ATTN_RING_KB"); if (v && atoi(v) >= 16 && atoi(v) <= 128) g_attn_ring_bytes = atoi(v) * 1024; env_read = true; }
  if (a.nsplit > 64 || 2 * a.page_size * a.head_dim * 2 * 2 > g_attn_ring_bytes) return -1;
  const size_t smem = g_attn_ring_bytes;
  AttnDecodeArgs a2 = a;
  a2.ring_bytes = g_attn_ring_bytes;
  cudaError_t e = cudaErrorInvalidValue;
#define CL_ATT(R, D) do { static PerDeviceOnce once; if (once.pending()) { prefer_max_smem(attn_decode_kernel<R, D>);     \
      cudaFuncSetAttribute(attn_decode_kernel<R, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnRingBytesMax); once.mark(); } \
    e = launch_ex(attn_decode_kernel<R, D>, grid, block, smem, st, pdl, a2); } while (0)
  if (a.head_dim == 128) {
    if (rep == 1) CL_ATT(1, 128); else if (rep == 2) CL_ATT(2, 128); else if (rep == 4) CL_ATT(4, 128);
    else if (rep == 8) CL_ATT(8, 128);
  } else if (a.head_dim == 64) {
    if (rep == 1) CL_ATT(1, 64); else if (rep == 2) CL_ATT(2, 64); else if (rep == 4) CL_ATT(4, 64);
    else if (rep == 8) CL_ATT(8, 64);
  }
#undef CL_ATT
  return e == cudaSuccess ? 1 : -1;
}

// ================================================================================================
// embedding gather, argmax + sequence advance, synthetic weights
// ================================================================================================
__global__ void embed_kernel(const __nv_bfloat16* __restrict__ table, int d, const int* __restrict__ tok, float* h,
                             int h_stride, const int* __restrict__ slots) {
  pdl_launch_dependents();
  pdl_wait();
  const int slot = slots ? slots[blockIdx.y] : blockIdx.y;
  const int id = tok[slot];
  const uint4* row = reinterpret_cast<const uint4*>(table + (size_t)id * d);
  float* out = h + (size_t)slot * h_stride;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < d / 8; c += gridDim.x * blockDim.x) {
    const uint4 w = row[c];
    float4 a = make_float4(bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y));
    float4 b2 = make_float4(bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w));
    *reinterpret_cast<float4*>(out + c * 8) = a;
    *reinterpret_cast<float4*>(out + c * 8 + 4) = b2;
  }
}

int launch_embed(const __nv_bfloat16* table, int d, const int* tok, float* h, int h_stride, const int* slots, int batch,
                 cudaStream_t st) {
  int threads = 128;
  int blocks = (d / 8 + threads - 1) / threads;
  static PerDeviceOnce once;
  if (once.pending()) { prefer_max_smem(embed_kernel); once.mark(); }
  embed_kernel<<<dim3(blocks, batch), threads, 0, st>>>(table, d, tok, h, h_stride, slots);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ---- device sampler of the step tail: the host sampler (host_util.cpp sample_token) step for step ------------------
// A candidate is the 64-bit key (orderable(v) << 32) | (0xFFFFFFFF - id): keys are distinct, and "largest k keys" is
// exactly the host's top-k order (value descending, id ascending).  -0 is keyed as +0 because the host compares them equal.
__device__ __forceinline__ unsigned long long sample_key(float v, int id) {
  uint32_t u = __float_as_uint(v);
  if ((u << 1) == 0u) u = 0u;
  u ^= (u >> 31) ? 0xFFFFFFFFu : 0x80000000u;
  return ((unsigned long long)u << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)id);
}
__device__ __forceinline__ float sample_key_value(unsigned long long k) {
  const uint32_t o = (uint32_t)(k >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o ^ 0x80000000u) : ~o);
}
__device__ __forceinline__ int sample_key_id(unsigned long long k) { return (int)(0xFFFFFFFFu - (uint32_t)k); }

// Smallest T such that exactly k of the nonzero keys get(0..n-1) are >= T (8-bit radix select, most significant digit
// first; stops at the first digit whose whole bucket is taken).  Needs at least k nonzero keys.  All 256 threads call it.
template <class Get>
__device__ unsigned long long block_topk_threshold(const Get& get, int n, int k) {
  __shared__ unsigned hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_need, s_done;
  const int tid = threadIdx.x, lane = tid & 31;
  unsigned long long prefix = 0ull, mask = 0ull;
  int need = k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    hist[tid] = 0u;
    __syncthreads();
    for (int i = tid; i < n; i += 256) {
      const unsigned long long key = get(i);
      if (key != 0ull && (key & mask) == prefix) atomicAdd(&hist[(unsigned)(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid < 32) {   // lane l owns buckets 255 - 8l down to 248 - 8l
      unsigned c[8], s = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[255 - 8 * lane - j]; s += c[j]; }
      unsigned incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const unsigned hit = __ballot_sync(0xffffffffu, incl >= (unsigned)need);
      if (lane == __ffs(hit) - 1) {
        unsigned acc = incl - s, cnt = 0u;
        int d = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (cnt == 0u && acc + c[j] >= (unsigned)need) { d = 255 - 8 * lane - j; cnt = c[j]; }
          else if (cnt == 0u) acc += c[j];
        s_prefix = prefix | ((unsigned long long)d << shift);
        s_need = need - (int)acc;
        s_done = cnt == (unsigned)(need - (int)acc);
      }
    }
    __syncthreads();
    prefix = s_prefix; need = s_need;
    const int done = s_done;
    mask |= 0xFFull << shift;
    __syncthreads();
    if (done) break;
  }
  return prefix;
}

__device__ __forceinline__ double sample_uniform01(unsigned long long seed, unsigned long long step) {   // host_util.cpp uniform01
  const unsigned long long x = mix64(seed * 0x9E3779B97F4A7C15ull + step + 0x632BE59BD9B4E019ull);
  return __dmul_rn((double)(x >> 11), 1.0 / 9007199254740992.0);
}

// History of a draw: the slot's ring (ids 0 .. ring_len - 1, id i at ring[i % kSampleHistMax]) followed by n_extra ids
// that are not in the ring yet (a decode step's input; the inputs of a verify pass up to its row).
struct TailHist {
  const int* ring;
  int ring_len;
  const int* extra;
  int n_extra;
};

// The draw of one logits row, called by all kTailBlocks blocks of the row: each block keys its vocabulary slice (repeat
// penalty applied) and leaves its top-k keys in cand[blockIdx.x]; the last block to finish merges them and draws at RNG
// step *step + step_add.  Returns the id on thread 0 of the last block, -1 on every other thread.
__device__ __forceinline__ int tail_draw(const float* lg_row, int V, const SampleParams& sp, const TailHist& h,
                                         unsigned long long* cand_row, unsigned* counter, const unsigned long long* step,
                                         int step_add) {
  __shared__ unsigned long long keys[kSampleSliceMax];
  __shared__ unsigned pen[kSampleSliceMax / 32];
  __shared__ unsigned long long top[kSampleTopKMax], sorted[kSampleTopKMax];
  __shared__ double p[kSampleTopKMax];
  __shared__ int n_out, is_last_s;
  __shared__ double s_den;
  const int tid = threadIdx.x;
  const int K = sp.top_k;
  const int slice = (V + (int)gridDim.x - 1) / (int)gridDim.x;
  const int lo = blockIdx.x * slice, n = max(0, min(slice, V - lo));
  const float* lg = lg_row + lo;

  for (int i = tid; i < kSampleSliceMax / 32; i += 256) pen[i] = 0u;
  if (tid == 0) n_out = 0;
  __syncthreads();
  if (sp.repeat_penalty != 1.0f && sp.repeat_last_n != 0) {   // the distinct in-range ids of the last repeat_last_n
    const int total = h.ring_len + h.n_extra;
    const int w = sp.repeat_last_n > 0 && total > sp.repeat_last_n ? sp.repeat_last_n : total;
    for (int j = tid; j < w; j += 256) {
      const int idx = total - w + j;
      const int id = idx < h.ring_len ? h.ring[idx % kSampleHistMax] : h.extra[idx - h.ring_len];
      if (id >= lo && id < lo + n) atomicOr(&pen[(id - lo) >> 5], 1u << ((id - lo) & 31));
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += 256) {
    float v = lg[i];
    if (pen[i >> 5] & (1u << (i & 31))) v = v > 0.f ? __fdiv_rn(v, sp.repeat_penalty) : __fmul_rn(v, sp.repeat_penalty);
    keys[i] = sample_key(v, lo + i);
  }
  __syncthreads();
  const unsigned long long t1 = n > K ? block_topk_threshold([&](int i) { return keys[i]; }, n, K) : 1ull;
  unsigned long long* cand = cand_row + (size_t)blockIdx.x * kSampleTopKMax;
  for (int i = tid; i < n; i += 256)
    if (keys[i] >= t1) cand[atomicAdd(&n_out, 1)] = keys[i];
  __syncthreads();
  for (int j = n_out + tid; j < K; j += 256) cand[j] = 0ull;   // short slice: empty entries
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned old = atomicAdd(counter, 1u);
    is_last_s = (old == gridDim.x - 1);
    if (is_last_s) *counter = 0u;
    n_out = 0;
  }
  __syncthreads();
  if (!is_last_s) return -1;
  __threadfence();

  // merge: the k largest of the kTailBlocks * k candidates, sorted descending
  const unsigned long long* cs = cand_row;
  auto cget = [&](int i) { return __ldcg(cs + (size_t)(i / K) * kSampleTopKMax + (i % K)); };
  const int nc = (int)gridDim.x * K;
  const unsigned long long t2 = block_topk_threshold(cget, nc, K);
  for (int i = tid; i < nc; i += 256) {
    const unsigned long long key = cget(i);
    if (key != 0ull && key >= t2) top[atomicAdd(&n_out, 1)] = key;
  }
  __syncthreads();
  if (tid < K) {
    const unsigned long long mine = top[tid];
    int rank = 0;
    for (int j = 0; j < K; ++j) rank += top[j] > mine;
    sorted[rank] = mine;
  }
  __syncthreads();
  // p_i = exp((double)(v_i - max) / T); the sums run sequentially in rank order, as on the host
  const float mx = sample_key_value(sorted[0]);
  if (tid < K) p[tid] = exp(__ddiv_rn((double)__fsub_rn(sample_key_value(sorted[tid]), mx), (double)sp.temperature));
  __syncthreads();
  if (tid == 0) {
    double den = 0.0;
    for (int i = 0; i < K; ++i) den = __dadd_rn(den, p[i]);
    s_den = den;
  }
  __syncthreads();
  __shared__ double q[kSampleTopKMax];
  if (tid < K) q[tid] = __ddiv_rn(p[tid], s_den);
  __syncthreads();
  if (tid != 0) return -1;
  int keep = K;
  if (sp.top_p > 0.f && sp.top_p < 1.f) {
    double cum = 0.0;
    for (int i = 0; i < K; ++i) { cum = __dadd_rn(cum, q[i]); if (cum >= (double)sp.top_p) { keep = i + 1; break; } }
  }
  double tot = 0.0;
  for (int i = 0; i < keep; ++i) tot = __dadd_rn(tot, p[i]);
  const double u = __dmul_rn(sample_uniform01(sp.seed, *step + (unsigned long long)step_add), tot);
  double cum = 0.0;
  int pick = sample_key_id(sorted[keep - 1]);
  for (int i = 0; i < keep; ++i) { cum = __dadd_rn(cum, p[i]); if (u < cum) { pick = sample_key_id(sorted[i]); break; } }
  return pick;
}

// Greedy choice of one logits row (largest value, lowest index on ties), called by all kTailBlocks blocks of the row:
// per-block partials in part_val / part_idx, merged by the last block to finish.  Returns the id on lane 0 of warp 0 of
// the last block, -1 on every other thread.
__device__ __forceinline__ int tail_argmax(const float* lg, int V, float* part_val, int* part_idx, unsigned* counter) {
  __shared__ float sv[8];
  __shared__ int si[8];
  __shared__ int is_last_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = blockIdx.x * 256 + tid; i < V; i += gridDim.x * 256) {
    const float v = lg[i];
    if (v > best || (v == best && i < bi)) { best = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
    part_val[blockIdx.x] = best;
    part_idx[blockIdx.x] = bi;
    __threadfence();
    const unsigned old = atomicAdd(counter, 1u);
    is_last_s = (old == gridDim.x - 1);
    if (is_last_s) *counter = 0u;
  }
  __syncthreads();
  if (!is_last_s || warp != 0) return -1;
  __threadfence();
  best = -INFINITY; bi = 0x7fffffff;
  for (int i = lane; i < (int)gridDim.x; i += 32) {
    const float v = __ldcg(part_val + i);
    const int id = __ldcg(part_idx + i);
    if (v > best || (v == best && id < bi)) { best = v; bi = id; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane != 0) return -1;
  return bi == 0x7fffffff ? 0 : bi;   // all-NaN logits: stay in range
}

// Log-probabilities of one logits row (kernels.h LogprobRecord), called by all kTailBlocks blocks of the row before the
// choice: each block leaves its slice's (max, sum of expf(v - max)) in part_row and its top-n keys in cand_row; the last
// block to finish merges them and writes lse, n_top and the top-n into rec (and rec2 when not nullptr).  The id and its
// logprob are written by the choosing block afterwards (tail_logprob_pick): every record write of this function is fenced
// before this block takes part in the choice, whose last block therefore sees lse.
//
// The top-n are n rounds of "largest key below the previous one" (keys as sample_key: value descending, id ascending): per
// block over its slice, then one warp merges the kTailBlocks sorted lists.  A radix select (block_topk_threshold) needs
// its own histogram per instantiation, and the tail kernels' shared memory would then no longer fit 8 blocks per SM.
__device__ __forceinline__ void tail_logprobs(const float* lg_row, int V, int N, float2* part_row, unsigned long long* cand_row,
                                           unsigned* counter, LogprobRecord* rec, LogprobRecord* rec2) {
  __shared__ float red[8];
  __shared__ unsigned long long kred[2][8];
  __shared__ int is_last_s;
  __shared__ double s_lse;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int slice = (V + (int)gridDim.x - 1) / (int)gridDim.x;
  const int lo = blockIdx.x * slice, n = max(0, min(slice, V - lo));
  const float* x = lg_row + lo;
  if (N > V) N = V;

  float m = -INFINITY;
  for (int i = tid; i < n; i += 256) m = fmaxf(m, x[i]);
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float s = 0.f;
  if (m > -INFINITY)
    for (int i = tid; i < n; i += 256) s += expf(x[i] - m);
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (tid == 0) {
    float tot = 0.f;
    for (int w = 0; w < 8; ++w) tot += red[w];
    part_row[blockIdx.x] = make_float2(m, tot);
  }
  unsigned long long* cand = cand_row + (size_t)blockIdx.x * kLogprobTopMax;
  unsigned long long below = ~0ull;
  for (int j = 0; j < N; ++j) {   // a short slice leaves empty (0) entries
    unsigned long long best = 0ull;
    for (int i = tid; i < n; i += 256) {
      const unsigned long long k = sample_key(x[i], lo + i);
      if (k < below && k > best) best = k;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) kred[j & 1][warp] = best;
    __syncthreads();
    best = kred[j & 1][0];
#pragma unroll
    for (int w = 1; w < 8; ++w) best = max(best, kred[j & 1][w]);
    if (tid == 0) cand[j] = best;
    below = best;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned old = atomicAdd(counter, 1u);
    is_last_s = (old == gridDim.x - 1);
    if (is_last_s) *counter = 0u;
  }
  __syncthreads();
  if (!is_last_s) return;
  __threadfence();

  // lse = M + log(sum_b s_b exp(m_b - M)), in double and in block order
  if (tid == 0) {
    float M = -INFINITY;
    for (int b = 0; b < (int)gridDim.x; ++b) M = fmaxf(M, __ldcg(&part_row[b].x));
    double S = 0.0;
    for (int b = 0; b < (int)gridDim.x; ++b) {
      const float2 p = __ldcg(part_row + b);
      if (p.y > 0.f) S += (double)p.y * exp((double)p.x - (double)M);
    }
    s_lse = (double)M + log(S);
    rec->lse = s_lse;
    rec->n_top = N;
    if (rec2) { rec2->lse = s_lse; rec2->n_top = N; }
  }
  __syncthreads();
  if (N > 0 && warp == 0) {
    // k-way merge of the blocks' descending lists: lane l holds the heads of lists l and l + 32 (kTailBlocks = 64)
    static_assert(kTailBlocks == 64, "two lists per lane");
    const double lse = s_lse;
    int h0 = 0, h1 = 0;
    const unsigned long long* c0 = cand_row + (size_t)lane * kLogprobTopMax;
    const unsigned long long* c1 = cand_row + (size_t)(lane + 32) * kLogprobTopMax;
    unsigned long long k0 = __ldcg(c0), k1 = __ldcg(c1);
    for (int j = 0; j < N; ++j) {
      unsigned long long best = max(k0, k1);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
      // keys are distinct, so exactly one head equals best
      if (k0 == best) k0 = ++h0 < N ? __ldcg(c0 + h0) : 0ull;
      else if (k1 == best) k1 = ++h1 < N ? __ldcg(c1 + h1) : 0ull;
      if (lane == 0) {
        const int id = sample_key_id(best);
        const float lp = __double2float_rn(__dsub_rn((double)sample_key_value(best), lse));
        rec->top_ids[j] = id; rec->top_logprobs[j] = lp;
        if (rec2) { rec2->top_ids[j] = id; rec2->top_logprobs[j] = lp; }
      }
    }
  }
  __threadfence();
  __syncthreads();
}

// The choosing thread of an armed row: the chosen id and logit[id] - lse into the record(s) tail_logprobs filled.
__device__ __forceinline__ void tail_logprob_pick(const float* lg_row, int pick, LogprobRecord* rec, LogprobRecord* rec2) {
  const float lp = __double2float_rn(__dsub_rn((double)lg_row[pick], __ldcg(&rec->lse)));
  rec->id = pick; rec->logprob = lp;
  if (rec2) { rec2->id = pick; rec2->logprob = lp; }
}

__global__ void __launch_bounds__(256, 8) step_tail_kernel(const StepTailArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const int slot = a.slots ? a.slots[b] : b;
  const float* lg = a.logits + (size_t)slot * a.vocab;
  const SampleState& S = a.sample;
  const bool sampled = S.mode && S.mode[slot];
  const LogprobState& P = a.lp;
  const int lp_n = P.top_n ? P.top_n[slot] : -1;
  LogprobRecord* lp_ring = nullptr;
  if (lp_n >= 0) {
    if (P.ring) lp_ring = P.ring + (size_t)(*a.step_counter % a.ring_steps) * a.ring_stride + b;
    tail_logprobs(lg, a.vocab, lp_n, P.part + (size_t)slot * gridDim.x, P.cand + (size_t)slot * gridDim.x * kLogprobTopMax,
                  P.counters + slot, P.last + slot, lp_ring);
  }
  int pick;
  if (sampled) {
    const TailHist h{S.hist + (size_t)slot * kSampleHistMax, S.hist_len[slot], a.tok + slot, S.push_input};
    pick = tail_draw(lg, a.vocab, S.par[slot], h, S.cand + (size_t)slot * gridDim.x * kSampleTopKMax, a.counters + slot,
                     S.step + slot, 0);
  } else {
    pick = tail_argmax(lg, a.vocab, a.part_val + (size_t)slot * gridDim.x, a.part_idx + (size_t)slot * gridDim.x, a.counters + slot);
  }
  if (pick < 0) return;
  if (lp_n >= 0) tail_logprob_pick(lg, pick, P.last + slot, lp_ring);
  if (sampled) {
    if (S.push_input) {
      const int hlen = S.hist_len[slot];
      S.hist[(size_t)slot * kSampleHistMax + hlen % kSampleHistMax] = a.tok[slot];
      S.hist_len[slot] = hlen + 1;
    }
    S.step[slot] += 1;
  }
  a.tok[slot] = pick;
  a.pos[slot] += 1;
  const int step = *a.step_counter;  // same value for every batch entry of this step
  a.ids_ring[(size_t)(step % a.ring_steps) * a.ring_stride + b] = pick;
  // the step counter itself is bumped by step_bump_kernel after every batch entry has read it
}

// Verify pass (Engine::verify_batch): row r of the logits [T][vocab] makes the choice the step tail would make after the
// inputs x0, d1 .. dr: greedy, or on an armed slot the draw with history = ring + inputs[0..r] and RNG step step + r.
// Each row has its own partial, candidate and counter buffers.  Nothing of the slot is written here.
__global__ void __launch_bounds__(256, 8) spec_tail_kernel(const SpecTailArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.y, slot = a.slot;
  const float* lg = a.logits + (size_t)r * a.vocab;
  const SampleState& S = a.sample;
  const LogprobState& P = a.lp;
  const int lp_n = P.top_n ? P.top_n[slot] : -1;
  if (lp_n >= 0)
    tail_logprobs(lg, a.vocab, lp_n, P.part + (size_t)r * gridDim.x, P.cand + (size_t)r * gridDim.x * kLogprobTopMax, P.counters + r,
                  P.last + r, nullptr);
  int pick;
  if (S.mode[slot]) {
    const TailHist h{S.hist + (size_t)slot * kSampleHistMax, S.hist_len[slot], a.inputs, r + 1};
    pick = tail_draw(lg, a.vocab, S.par[slot], h, a.cand + (size_t)r * gridDim.x * kSampleTopKMax, a.counters + r, S.step + slot, r);
  } else {
    pick = tail_argmax(lg, a.vocab, a.part_val + (size_t)r * gridDim.x, a.part_idx + (size_t)r * gridDim.x, a.counters + r);
  }
  if (pick >= 0) {
    a.choice[r] = pick;
    if (lp_n >= 0) tail_logprob_pick(lg, pick, P.last + r, nullptr);
  }
}

// One block after spec_tail_kernel: a = the drafts d_1 .. d_a that equal the choices y_1 .. y_a; the pass emits
// y_1 .. y_{a+1} and leaves the slot as a + 1 decode steps would: next input y_{a+1} at position len + a + 1, and on an
// armed slot x0, d1 .. da pushed into the history ring and the RNG step advanced by a + 1.
__global__ void spec_accept_kernel(const SpecTailArgs a) {
  __shared__ int s_acc;
  pdl_wait();
  const int tid = threadIdx.x, k = a.T - 1, slot = a.slot;
  if (tid == 0) {
    int acc = 0;
    while (acc < k && a.choice[acc] == a.inputs[acc + 1]) ++acc;
    s_acc = acc;
    a.out[0] = acc + 1;
    a.tok[slot] = a.choice[acc];
    a.pos[slot] = a.len + acc + 1;
  }
  __syncthreads();
  const int acc = s_acc;
  if (tid <= acc) a.out[1 + tid] = a.choice[tid];
  const SampleState& S = a.sample;
  if (!S.mode[slot]) return;
  const int hlen = S.hist_len[slot];
  if (tid <= acc) S.hist[(size_t)slot * kSampleHistMax + (hlen + tid) % kSampleHistMax] = a.inputs[tid];
  __syncthreads();   // every thread has read hist_len
  if (tid == 0) {
    S.hist_len[slot] = hlen + acc + 1;
    S.step[slot] += (unsigned long long)(acc + 1);
  }
}

// step counter bump: tiny kernel keeps the protocol obviously correct (1 thread).
__global__ void step_bump_kernel(int* step_counter, unsigned* sync_counters, int n_sync) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) *step_counter += 1;
  for (int i = threadIdx.x; i < n_sync; i += blockDim.x) sync_counters[i] = 0u;   // re-arm the persistent kernel's counters
}

int launch_step_tail(const StepTailArgs& a, cudaStream_t st) {
  static PerDeviceOnce once;
  if (once.pending()) { prefer_max_smem(step_tail_kernel); prefer_max_smem(step_bump_kernel); once.mark(); }
  step_tail_kernel<<<dim3(kTailBlocks, a.batch), 256, 0, st>>>(a);
  if (cudaGetLastError() != cudaSuccess) return -1;
  step_bump_kernel<<<1, 256, 0, st>>>(a.step_counter, a.sync_counters, a.n_sync_counters);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_spec_tail(const SpecTailArgs& a, cudaStream_t st, bool pdl) {
  static PerDeviceOnce once;
  if (once.pending()) { prefer_max_smem(spec_tail_kernel); prefer_max_smem(spec_accept_kernel); once.mark(); }
  if (launch_ex(spec_tail_kernel, dim3(kTailBlocks, a.T), dim3(256), 0, st, pdl, a) != cudaSuccess) return -1;
  return launch_ex(spec_accept_kernel, dim3(1), dim3(32), 0, st, true, a) == cudaSuccess ? 2 : -1;
}

__global__ void synth_bf16_kernel(__nv_bfloat16* out, int64_t n, int k_cols, int row_mult, int row_off, uint64_t seed,
                                  int key, float scale, int rope_hd) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / k_cols;
    const int64_t c = i - r * k_cols;
    const float v = (float)synth_int(seed, key, (uint64_t)i) * scale;
    if (rope_hd > 0) {  // logical row (head, w) -> stored row head*hd + (w < hd/2 ? 2w : 2(w - hd/2) + 1)
      const int64_t head = r / rope_hd;
      const int w = (int)(r - head * rope_hd), half = rope_hd >> 1;
      r = head * rope_hd + (w < half ? 2 * w : 2 * (w - half) + 1);
    }
    out[(r * row_mult + row_off) * k_cols + c] = __float2bfloat16_rn(v);
  }
}
int launch_synth_bf16(__nv_bfloat16* out, int64_t n_logical, int k_cols, int row_mult, int row_off, uint64_t seed,
                      int key, float scale, cudaStream_t st, int rope_hd) {
  int blocks = (int)((n_logical + 255) / 256);
  if (blocks > sm_count() * 16) blocks = sm_count() * 16;
  if (blocks < 1) blocks = 1;
  synth_bf16_kernel<<<blocks, 256, 0, st>>>(out, n_logical, k_cols, row_mult, row_off, seed, key, scale, rope_hd);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}
__global__ void synth_gain_kernel(float* out, int n, uint64_t seed, int key, float scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = 1.0f + (float)synth_int(seed, key, (uint64_t)i) * scale;
}
int launch_synth_gain(float* out, int n, uint64_t seed, int key, float scale, cudaStream_t st) {
  synth_gain_kernel<<<(n + 255) / 256, 256, 0, st>>>(out, n, seed, key, scale);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}
__global__ void bf16_to_f32_kernel(const __nv_bfloat16* in, float* out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __bfloat162float(in[i]);
}
int launch_bf16_to_f32(const __nv_bfloat16* in, float* out, int64_t n, cudaStream_t st) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  if (blocks < 1) blocks = 1;
  bf16_to_f32_kernel<<<blocks, 256, 0, st>>>(in, out, n);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ---- parity aid: fill a sequence's paged K/V with the oracle's cheap pattern (oracle/llama_oracle.c oc_seq_fake_fill:
// every value is n/128 with n in [-128, 127], exact in bf16), the same in every layer.  i = token * kv_dim + head * hd + dim.
__global__ void fake_fill_kv_kernel(__nv_bfloat16* kpool, __nv_bfloat16* vpool, size_t layer_elems, int n_layers, const int* bt,
                                    int page, int n_kv, int hd, long long n_elems) {
  const int kvd = n_kv * hd;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_elems; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long u = (unsigned long long)i;
    const float kv = (float)((int)(((u * 2654435761ull) >> 24) & 0xffull) - 128) * (1.0f / 128.0f);
    const float vv = (float)((int)(((u * 40503ull) >> 8) & 0xffull) - 128) * (1.0f / 128.0f);
    const int t = (int)(i / kvd), r = (int)(i - (long long)t * kvd), g = r / hd, j = r - g * hd;
    const size_t dst = (((size_t)bt[t / page] * n_kv + g) * page + (t % page)) * hd + j;
    const __nv_bfloat16 kb = __float2bfloat16_rn(kv), vb = __float2bfloat16_rn(vv);
    for (int l = 0; l < n_layers; ++l) { kpool[(size_t)l * layer_elems + dst] = kb; vpool[(size_t)l * layer_elems + dst] = vb; }
  }
}
int launch_fake_fill_kv(__nv_bfloat16* kpool, __nv_bfloat16* vpool, size_t layer_elems, int n_layers, const int* block_table,
                        int page_size, int n_kv, int head_dim, int n_tokens, cudaStream_t st) {
  const long long n = (long long)n_tokens * n_kv * head_dim;
  if (n <= 0) return 0;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  fake_fill_kv_kernel<<<blocks, 256, 0, st>>>(kpool, vpool, layer_elems, n_layers, block_table, page_size, n_kv, head_dim, n);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// parity aid: gather one layer's cached K or V rows of a sequence from the paged pool -> dense fp32 [n][n_kv*hd]
__global__ void gather_kv_kernel(const __nv_bfloat16* pool, const int* bt, int page, int n_kv, int hd, int t0, long long n_elems, float* out) {
  const int kvd = n_kv * hd;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_elems; i += (long long)gridDim.x * blockDim.x) {
    const int t = t0 + (int)(i / kvd), r = (int)(i % kvd), g = r / hd, j = r - g * hd;
    out[i] = __bfloat162float(pool[(((size_t)bt[t / page] * n_kv + g) * page + (t % page)) * hd + j]);
  }
}
int launch_gather_kv(const __nv_bfloat16* pool_layer, const int* block_table, int page_size, int n_kv, int head_dim, int t0, int n,
                     float* out, cudaStream_t st) {
  const long long ne = (long long)n * n_kv * head_dim;
  if (ne <= 0) return 0;
  int blocks = (int)((ne + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  gather_kv_kernel<<<blocks, 256, 0, st>>>(pool_layer, block_table, page_size, n_kv, head_dim, t0, ne, out);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace cl
