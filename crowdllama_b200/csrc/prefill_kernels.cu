// prefill_kernels.cu — the non-GEMM kernels of the prompt (prefill) path: embedding rows,
// RMSNorm -> bf16, RoPE + paged-KV scatter, causal GQA attention over the paged cache, SiLU*mul.
// (Upstream counterparts, SURVEY.md §2.2: ggml-cuda rms_norm / rope / cpy / flash_attn_ext / silu.)
//
// The attention kernel is a FlashAttention-2 style mma.sync (m16n8k16 bf16) kernel: it is the
// round-1 baseline for prompts; attn_prefill_tc.cu replaces it for head_dim 128.
#include "common.cuh"
#include "kernels.h"

namespace cl {

// ------------------------------------------------------------------------------------------------
__global__ void embed_rows_kernel(const __nv_bfloat16* __restrict__ table, int d, const int* __restrict__ ids, float* h) {
  const int t = blockIdx.x;
  const uint4* row = reinterpret_cast<const uint4*>(table + (size_t)ids[t] * d);
  float* out = h + (size_t)t * d;
  for (int c = threadIdx.x; c < d / 8; c += blockDim.x) {
    const uint4 w = row[c];
    *reinterpret_cast<float4*>(out + c * 8) = make_float4(bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y));
    *reinterpret_cast<float4*>(out + c * 8 + 4) = make_float4(bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w));
  }
}
int launch_embed_rows(const __nv_bfloat16* table, int d, const int* ids_dev, float* h, int T, cudaStream_t st) {
  embed_rows_kernel<<<T, 128, 0, st>>>(table, d, ids_dev, h);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rmsnorm_bf16_kernel(const float* __restrict__ h, const float* __restrict__ gain, float eps,
                                                           __nv_bfloat16* __restrict__ out, int d) {
  __shared__ float red[8];
  const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* x = h + (size_t)t * d;
  float ss = 0.f;
  for (int i = tid * 4; i < d; i += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(x + i);
    ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
  }
  ss = warp_sum(ss);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float inv = 1.0f / sqrtf(tot / (float)d + eps);
  __nv_bfloat16* o = out + (size_t)t * d;
  for (int i = tid * 4; i < d; i += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(x + i);
    const float4 g = *reinterpret_cast<const float4*>(gain + i);
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x * inv * g.x, v.y * inv * g.y);
    __nv_bfloat162 b = __floats2bfloat162_rn(v.z * inv * g.z, v.w * inv * g.w);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(o + i) = pk;
  }
}
int launch_rmsnorm_bf16(const float* h, const float* gain, float eps, __nv_bfloat16* out, int T, int d, cudaStream_t st) {
  rmsnorm_bf16_kernel<<<T, 256, 0, st>>>(h, gain, eps, out, d);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rope_scatter_kernel(const RopeScatterArgs a) {
  const int t = blockIdx.x;
  const int pos = a.row_seq ? a.row_pos[t] : a.pos0 + t;
  const int* bt = a.row_seq ? a.block_table + (size_t)a.row_seq[t] * a.bt_stride : a.block_table;
  const int HD = a.head_dim, half = HD / 2;
  const float* row = a.qkv + (size_t)t * a.qkv_stride;
  const float2* rope = a.rope + (size_t)pos * half;
  const int qd = a.n_heads * HD, kvd = a.n_kv * HD;
  // split-K GEMM output (short prompts): the value is the fixed-order sum of n_split partials, split_stride floats apart
  auto val = [&](int col) {
    float v = row[col];
    for (int s = 1; s < a.n_split; ++s) v += row[(size_t)s * a.split_stride + col];
    return v;
  };
  // q heads
  for (int i = threadIdx.x; i < a.n_heads * half; i += blockDim.x) {
    const int hh = i / half, j = i % half;
    const float2 cs = rope[j];
    const float x0 = val(hh * HD + 2 * j), x1 = val(hh * HD + 2 * j + 1);   // rope-pair-interleaved GEMM output
    a.q_out[(size_t)t * qd + hh * HD + j] = __float2bfloat16_rn(x0 * cs.x - x1 * cs.y);
    a.q_out[(size_t)t * qd + hh * HD + j + half] = __float2bfloat16_rn(x1 * cs.x + x0 * cs.y);
  }
  const int page = bt[pos / a.page_size], off = pos % a.page_size;
  for (int i = threadIdx.x; i < a.n_kv * half; i += blockDim.x) {
    const int g = i / half, j = i % half;
    const float2 cs = rope[j];
    const float x0 = val(qd + g * HD + 2 * j), x1 = val(qd + g * HD + 2 * j + 1);
    const size_t base = (((size_t)page * a.n_kv + g) * a.page_size + off) * HD;
    a.kpool[base + j] = __float2bfloat16_rn(x0 * cs.x - x1 * cs.y);
    a.kpool[base + j + half] = __float2bfloat16_rn(x1 * cs.x + x0 * cs.y);
  }
  for (int i = threadIdx.x; i < kvd; i += blockDim.x) {
    const int g = i / HD, w = i % HD;                      // stored column w -> dim (w even ? w/2 : w/2 + half)
    const int j = (w & 1) ? (w >> 1) + half : (w >> 1);
    const size_t base = (((size_t)page * a.n_kv + g) * a.page_size + off) * HD;
    a.vpool[base + j] = __float2bfloat16_rn(val(qd + kvd + i));
  }
}
int launch_rope_scatter(const RopeScatterArgs& a, cudaStream_t st) {
  rope_scatter_kernel<<<a.T, 256, 0, st>>>(a);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// causal GQA attention for T new tokens against the paged cache (which already holds them)
// grid = (ceil(T/64), n_heads), block = 128 (4 warps x 16 query rows), KV blocks of 64 keys,
// double-buffered cp.async, XOR-swizzled shared tiles, mma.sync.m16n8k16 bf16 -> fp32.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
template <int D>
__global__ void __launch_bounds__(128) attn_prefill_kernel(const AttnPrefillArgs a) {
  constexpr int CH = D / 8;            // 16-byte chunks per row
  constexpr int TILE = 64 * D * 2;     // bytes of a 64-row tile
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: Q tile | K stage0 | V stage0 | K stage1 | V stage1 ; chunk c of row r lives at (c ^ (r & 7))
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sKV = sQ + TILE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * 64, head = blockIdx.y;
  const int rep = a.n_heads / a.n_kv, g = head / rep;
  const int qd = a.n_heads * D;
  const int P = a.page_size;
  const int n_keys = min(a.pos0 + a.T, a.pos0 + q0 + 64);   // keys any query of this CTA may see
  const int n_blocks = (n_keys + 63) / 64;

  auto swz = [](int r, int c) { return (uint32_t)((r * CH + (c ^ (r & 7))) * 16); };

  // ---- Q tile -> smem
  for (int i = tid; i < 64 * CH; i += 128) {
    const int r = i / CH, c = i % CH;
    const int t = min(q0 + r, a.T - 1);
    cp_async16(sQ + swz(r, c), a.q + (size_t)t * qd + (size_t)head * D + c * 8);
  }
  auto load_kv = [&](int kb, int stage) {
    const uint32_t sK = sKV + stage * 2 * TILE, sV = sK + TILE;
    for (int i = tid; i < 64 * CH; i += 128) {
      const int r = i / CH, c = i % CH;
      const int t = min(kb * 64 + r, n_keys - 1);
      const size_t base = (((size_t)a.block_table[t / P] * a.n_kv + g) * P + t % P) * D + c * 8;
      cp_async16(sK + swz(r, c), a.kpool + base);
      cp_async16(sV + swz(r, c), a.vpool + base);
    }
  };
  load_kv(0, 0);
  asm volatile("cp.async.commit_group;" ::: "memory");

  uint32_t qf[D / 16][4];
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows (lane/4) and (lane/4 + 8)
  const float scale2 = rsqrtf((float)D) * 1.4426950408889634f;
  const int qrow0 = a.pos0 + q0 + warp * 16 + (lane >> 2);     // absolute position of row lane/4
  const int qrow1 = qrow0 + 8;
  const int warp_qmax = a.pos0 + q0 + warp * 16 + 15;

  for (int kb = 0; kb < n_blocks; ++kb) {
    const int stage = kb & 1;
    if (kb + 1 < n_blocks) load_kv(kb + 1, stage ^ 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    if (kb == 0) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const int id = lane >> 3;
        ldsm_x4(qf[kk], sQ + swz(warp * 16 + (id & 1) * 8 + (lane & 7), 2 * kk + (id >> 1)));
      }
    }
    if (kb * 64 <= warp_qmax) {
      const uint32_t sK = sKV + stage * 2 * TILE, sV = sK + TILE;
      // ---- S = Q K^T  (16 x 64 per warp)
      float s[8][4];
#pragma unroll
      for (int nj = 0; nj < 8; ++nj) { s[nj][0] = s[nj][1] = s[nj][2] = s[nj][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {   // pairs of 8-key groups
          uint32_t kf[4];
          const int id = lane >> 3;
          ldsm_x4(kf, sK + swz((2 * np + (id >> 1)) * 8 + (lane & 7), 2 * kk + (id & 1)));
          mma_bf16(s[2 * np], qf[kk], kf[0], kf[1]);
          mma_bf16(s[2 * np + 1], qf[kk], kf[2], kf[3]);
        }
      }
      // ---- scale, causal mask, online softmax
      const bool need_mask = kb * 64 + 63 > a.pos0 + q0 + warp * 16;
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nj = 0; nj < 8; ++nj) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = s[nj][e] * scale2;
          if (need_mask) {
            const int key = kb * 64 + nj * 8 + 2 * (lane & 3) + (e & 1);
            const int qp = (e < 2) ? qrow0 : qrow1;
            if (key > qp) v = -INFINITY;
          }
          s[nj][e] = v;
        }
        mx0 = fmaxf(mx0, fmaxf(s[nj][0], s[nj][1]));
        mx1 = fmaxf(mx1, fmaxf(s[nj][2], s[nj][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      // key 0 is visible to every query, so after the first block mn is finite
      const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
      m0 = mn0; m1 = mn1;
      float rs0 = 0.f, rs1 = 0.f;
      uint32_t pf[4][4];   // P as A fragments for 4 k-slices of 16 keys
#pragma unroll
      for (int nj = 0; nj < 8; ++nj) {
        const float p0 = exp2f(s[nj][0] - mn0), p1 = exp2f(s[nj][1] - mn0);
        const float p2 = exp2f(s[nj][2] - mn1), p3 = exp2f(s[nj][3] - mn1);
        rs0 += p0 + p1; rs1 += p2 + p3;
        pf[nj >> 1][(nj & 1) * 2 + 0] = pack_bf16(p0, p1);
        pf[nj >> 1][(nj & 1) * 2 + 1] = pack_bf16(p2, p3);
      }
      l0 = l0 * c0 + rs0; l1 = l1 * c1 + rs1;
#pragma unroll
      for (int nd = 0; nd < D / 8; ++nd) { o[nd][0] *= c0; o[nd][1] *= c0; o[nd][2] *= c1; o[nd][3] *= c1; }
      // ---- O += P V
#pragma unroll
      for (int j = 0; j < 4; ++j) {          // 16-key slices
#pragma unroll
        for (int nd = 0; nd < D / 8; nd += 2) {
          uint32_t vf[4];
          const int id = lane >> 3;
          ldsm_x4_t(vf, sV + swz(j * 16 + (id & 1) * 8 + (lane & 7), nd + (id >> 1)));
          mma_bf16(o[nd], pf[j], vf[0], vf[1]);
          mma_bf16(o[nd + 1], pf[j], vf[2], vf[3]);
        }
      }
    }
    __syncthreads();   // everyone done with this stage before it is refilled
  }
  // ---- finalise: the 4 lanes of a row hold partial sums of l
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  const int t0 = q0 + warp * 16 + (lane >> 2), t1 = t0 + 8;
#pragma unroll
  for (int nd = 0; nd < D / 8; ++nd) {
    const int col = head * D + nd * 8 + 2 * (lane & 3);
    if (t0 < a.T) *reinterpret_cast<uint32_t*>(a.out + (size_t)t0 * qd + col) = pack_bf16(o[nd][0] * i0, o[nd][1] * i0);
    if (t1 < a.T) *reinterpret_cast<uint32_t*>(a.out + (size_t)t1 * qd + col) = pack_bf16(o[nd][2] * i1, o[nd][3] * i1);
  }
}

int launch_attn_prefill(const AttnPrefillArgs& a, cudaStream_t st) {
  dim3 grid((a.T + 63) / 64, a.n_heads), block(128);
  cudaError_t e = cudaErrorInvalidValue;
  if (a.head_dim == 128) {
    constexpr int smem = 5 * 64 * 128 * 2;
    static PerDeviceOnce attr;
    if (attr.pending()) { cudaFuncSetAttribute(attn_prefill_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr.mark(); }
    attn_prefill_kernel<128><<<grid, block, smem, st>>>(a);
    e = cudaGetLastError();
  } else if (a.head_dim == 64) {
    constexpr int smem = 5 * 64 * 64 * 2;
    attn_prefill_kernel<64><<<grid, block, smem, st>>>(a);
    e = cudaGetLastError();
  }
  return e == cudaSuccess ? 1 : -1;
}

}  // namespace cl
