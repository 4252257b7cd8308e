// batch_kernels.cu — glue kernels of the BATCHED decode step (continuous batching, B >= 2 sequences).
// The weight projections of a batched step run on the tensor cores (gemm_wgmma.cu, token tile 32,
// split-K so that every SM streams weights); everything here is per-sequence element-wise work
// between those GEMMs.  Sequences live in "slots"; slots[b] maps batch index -> slot.
#include "common.cuh"
#include "kernels.h"

namespace cl {

// h[slot] += sum_s ypart[s][b]  (fixed order);  xn[b] = bf16(rmsnorm(h[slot]) * gain)
// one CTA of 1024 threads per sequence: every thread owns <= 2 float4 of the row, all loads of a pass are independent
__global__ void __launch_bounds__(1024) batch_resid_norm_kernel(float* __restrict__ h, int d, const float* __restrict__ ypart, int n_split,
                                                                int B, const float* __restrict__ gain, float eps,
                                                                __nv_bfloat16* __restrict__ xn, const int* __restrict__ slots) {
  __shared__ float red[32];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* hr = h + (size_t)slots[b] * d;
  float4 v[2], g[2];
  float ss = 0.f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = (tid + r * 1024) * 4;
    v[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    g[r] = v[r];
    if (i < d) {
      v[r] = *reinterpret_cast<const float4*>(hr + i);
      g[r] = *reinterpret_cast<const float4*>(gain + i);
      float4 y[8];
      for (int s0 = 0; s0 < n_split; s0 += 8) {
#pragma unroll
        for (int s = 0; s < 8; ++s)
          y[s] = s0 + s < n_split ? __ldcg(reinterpret_cast<const float4*>(ypart + ((size_t)(s0 + s) * B + b) * d + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int s = 0; s < 8; ++s) { v[r].x += y[s].x; v[r].y += y[s].y; v[r].z += y[s].z; v[r].w += y[s].w; }
      }
      if (n_split > 0) *reinterpret_cast<float4*>(hr + i) = v[r];
    }
    ss = fmaf(v[r].x, v[r].x, ss); ss = fmaf(v[r].y, v[r].y, ss); ss = fmaf(v[r].z, v[r].z, ss); ss = fmaf(v[r].w, v[r].w, ss);
  }
  ss = warp_sum(ss);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 32; ++w) tot += red[w];
  const float inv = 1.0f / sqrtf(tot / (float)d + eps);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = (tid + r * 1024) * 4;
    if (i < d) {
      uint2 pk;
      pk.x = pack_bf16(v[r].x * inv * g[r].x, v[r].y * inv * g[r].y);
      pk.y = pack_bf16(v[r].z * inv * g[r].z, v[r].w * inv * g[r].w);
      *reinterpret_cast<uint2*>(xn + (size_t)b * d + i) = pk;
    }
  }
}
int launch_batch_resid_norm(float* h, int d, const float* ypart, int n_split, int B, const float* gain, float eps, __nv_bfloat16* xn,
                            const int* slots, cudaStream_t st, bool pdl) {
  if (d > 8192 || d % 4) return -1;
  return launch_pdl(batch_resid_norm_kernel, dim3(B), dim3(1024), 0, st, pdl, h, d, ypart, n_split, B, gain, eps, xn, slots) == cudaSuccess ? 1 : -1;
}

// q|k|v partials (rope-pair-interleaved columns) -> RoPE at pos[slot] -> q (fp32, bf16-rounded) and the paged cache
__global__ void __launch_bounds__(256) batch_rope_append_kernel(const float* __restrict__ ypart, int n_split, int B, QkvEpi e,
                                                                float* __restrict__ q_out, int q_stride, const int* __restrict__ slots) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y, slot = slots[b];
  const int HD = e.head_dim, half = HD >> 1;
  const int qkv_dim = (e.n_heads + 2 * e.n_kv) * HD;
  const int pos = e.pos[slot];
  const int page = e.block_tables[(size_t)slot * e.bt_stride + pos / e.page_size], off = pos % e.page_size;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < qkv_dim / 2; p += gridDim.x * blockDim.x) {
    float v0 = 0.f, v1 = 0.f;
    for (int s = 0; s < n_split; ++s) {
      const float2 y = *reinterpret_cast<const float2*>(ypart + ((size_t)s * B + b) * qkv_dim + 2 * p);
      v0 += y.x; v1 += y.y;
    }
    const int hh = p / half, j = p - hh * half;
    if (hh < e.n_heads + e.n_kv) {
      const float2 cs = e.rope[(size_t)pos * half + j];
      const float r0 = bf16_round(v0 * cs.x - v1 * cs.y), r1 = bf16_round(v1 * cs.x + v0 * cs.y);
      if (hh < e.n_heads) {
        float* q = q_out + (size_t)slot * q_stride + (size_t)hh * HD;
        q[j] = r0; q[j + half] = r1;
      } else {
        const size_t base = (((size_t)page * e.n_kv + (hh - e.n_heads)) * e.page_size + off) * HD;
        e.kpool[base + j] = __float2bfloat16_rn(r0);
        e.kpool[base + j + half] = __float2bfloat16_rn(r1);
      }
    } else {
      const size_t base = (((size_t)page * e.n_kv + (hh - e.n_heads - e.n_kv)) * e.page_size + off) * HD;
      e.vpool[base + j] = __float2bfloat16_rn(v0);
      e.vpool[base + j + half] = __float2bfloat16_rn(v1);
    }
  }
}
int launch_batch_rope_append(const float* ypart, int n_split, int B, const QkvEpi& e, float* q_out, int q_stride, const int* slots,
                             cudaStream_t st, bool pdl) {
  const int pairs = (e.n_heads + 2 * e.n_kv) * e.head_dim / 2;
  return launch_pdl(batch_rope_append_kernel, dim3((pairs + 255) / 256, B), dim3(256), 0, st, pdl, ypart, n_split, B, e, q_out, q_stride, slots) ==
                 cudaSuccess ? 1 : -1;
}

// gate|up partials (interleaved pairs) -> act[b][i] = bf16(silu(g) * u)
__global__ void batch_silu_kernel(const float* __restrict__ ypart, int n_split, int B, int d_ff, __nv_bfloat16* __restrict__ act) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d_ff; i += gridDim.x * blockDim.x) {
    float g = 0.f, u = 0.f;
    for (int s = 0; s < n_split; ++s) {
      const float2 y = *reinterpret_cast<const float2*>(ypart + ((size_t)s * B + b) * 2 * d_ff + 2 * i);
      g += y.x; u += y.y;
    }
    act[(size_t)b * d_ff + i] = __float2bfloat16_rn(g / (1.0f + __expf(-g)) * u);
  }
}
int launch_batch_silu(const float* ypart, int n_split, int B, int d_ff, __nv_bfloat16* act, cudaStream_t st, bool pdl) {
  return launch_pdl(batch_silu_kernel, dim3((d_ff + 255) / 256, B), dim3(256), 0, st, pdl, ypart, n_split, B, d_ff, act) == cudaSuccess ? 1 : -1;
}

// logits partial/tmp [b][vocab] -> logits[slot][vocab]
__global__ void batch_scatter_rows_kernel(const float* __restrict__ y, int n, float* __restrict__ out, int out_stride,
                                          const int* __restrict__ slots) {
  const int b = blockIdx.y;
  float* dst = out + (size_t)slots[b] * out_stride;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += gridDim.x * blockDim.x * 4)
    *reinterpret_cast<float4*>(dst + i) = *reinterpret_cast<const float4*>(y + (size_t)b * n + i);
}
int launch_batch_scatter_rows(const float* y, int n, float* out, int out_stride, const int* slots, int B, cudaStream_t st) {
  batch_scatter_rows_kernel<<<dim3(std::min((n / 4 + 255) / 256, 128), B), 256, 0, st>>>(y, n, out, out_stride, slots);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ids[b] = tok[slots[b]]: a step's input ids in row order, for a pass that embeds rows (deterministic mode's step)
__global__ void gather_tok_kernel(const int* __restrict__ tok, const int* __restrict__ slots, int B, int* __restrict__ ids) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) ids[b] = tok[slots[b]];
}
int launch_gather_tok(const int* tok, const int* slots, int B, int* ids, cudaStream_t st) {
  gather_tok_kernel<<<(B + 127) / 128, 128, 0, st>>>(tok, slots, B, ids);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace cl
