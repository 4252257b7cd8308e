// kv_shift.cu — context shift of a paged sequence: the kept K rows are rotated by -delta in place (or into a private copy
// of a shared page), and the rows of the partial page after num_keep move into the page that keeps num_keep.
//
// RoPE is a rotation per dimension pair, R(p - delta) = R(-delta) R(p), so the K a prefill wrote at position p becomes the
// K of position p - delta with one more rotation, and V does not depend on the position at all.
//
// One CTA handles one (item, layer, kv head): rows [off0, off1) of a page, head_dim bf16 each.  A unit is one thread's
// share of one row: the 16-byte vectors of dims [8u, 8u + 8) and [8u + D/2, 8u + D/2 + 8), i.e. eight whole rotation pairs,
// so an in-place rotation reads exactly what the same thread later writes.  Every thread loads all of its units (K, and V
// when it moves) before it stores any, which keeps up to kUnits x 2 (K) + kUnits x 2 (V) 16-byte loads in flight.
//
// No griddepcontrol.launch_dependents: a kernel launched after this one with programmatic dependent launch loads KV pages
// before its griddepcontrol.wait and must not see rows this kernel has not written yet.
#include "common.cuh"
#include "kernels.h"

namespace cl {

namespace {

constexpr int kShiftThreads = 128;
constexpr int kUnits = 4;   // units per thread: 64 rows x 8 units (head_dim 128, page 64) fit one pass of 128 threads

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
  const __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&b);
}

__global__ void __launch_bounds__(kShiftThreads) kv_shift_kernel(KvShiftArgs a) {
  const int per_item = a.n_layers * a.n_kv;
  const int item = blockIdx.x / per_item, r = blockIdx.x % per_item;
  const int layer = r / a.n_kv, g = r % a.n_kv;
  const KvShiftItem it = a.items[item];
  const int D = a.head_dim, half = D / 2, upr = D / 16;   // units per row
  const size_t blk = (size_t)a.n_kv * a.page_size * D;
  const size_t src0 = (size_t)layer * a.layer_elems + (size_t)it.src * blk + (size_t)g * a.page_size * D;
  const size_t dst0 = (size_t)layer * a.layer_elems + (size_t)it.dst * blk + (size_t)g * a.page_size * D;
  const int n_units = (it.off1 - it.off0) * upr;
  const bool move_v = it.src != it.dst;
  uint4 k0[kUnits], k1[kUnits], v0[kUnits], v1[kUnits];
  for (int base = 0; base < n_units; base += kShiftThreads * kUnits) {
#pragma unroll
    for (int u = 0; u < kUnits; ++u) {
      const int unit = base + threadIdx.x + u * kShiftThreads;
      if (unit >= n_units) continue;
      const size_t e = (size_t)(it.off0 + unit / upr) * D + (unit % upr) * 8;
      k0[u] = *reinterpret_cast<const uint4*>(a.kpool + src0 + e);
      k1[u] = *reinterpret_cast<const uint4*>(a.kpool + src0 + e + half);
      if (move_v) {
        v0[u] = *reinterpret_cast<const uint4*>(a.vpool + src0 + e);
        v1[u] = *reinterpret_cast<const uint4*>(a.vpool + src0 + e + half);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnits; ++u) {
      const int unit = base + threadIdx.x + u * kShiftThreads;
      if (unit >= n_units) continue;
      const int j0 = (unit % upr) * 8;
      const size_t e = (size_t)(it.off0 + unit / upr) * D + j0;
      if (it.rot) {
        uint32_t* x = reinterpret_cast<uint32_t*>(&k0[u]);
        uint32_t* y = reinterpret_cast<uint32_t*>(&k1[u]);
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          const float2 c0 = a.rope_row[j0 + 2 * w], c1 = a.rope_row[j0 + 2 * w + 1];
          const float a0 = bf_lo(x[w]), a1 = bf_hi(x[w]), b0 = bf_lo(y[w]), b1 = bf_hi(y[w]);
          // R(-delta): explicit roundings, no contraction into an FMA, so the host restatement is bit-identical
          x[w] = pack_bf2(__fadd_rn(__fmul_rn(a0, c0.x), __fmul_rn(b0, c0.y)), __fadd_rn(__fmul_rn(a1, c1.x), __fmul_rn(b1, c1.y)));
          y[w] = pack_bf2(__fsub_rn(__fmul_rn(b0, c0.x), __fmul_rn(a0, c0.y)), __fsub_rn(__fmul_rn(b1, c1.x), __fmul_rn(a1, c1.y)));
        }
      }
      *reinterpret_cast<uint4*>(a.kpool + dst0 + e) = k0[u];
      *reinterpret_cast<uint4*>(a.kpool + dst0 + e + half) = k1[u];
      if (move_v) {
        *reinterpret_cast<uint4*>(a.vpool + dst0 + e) = v0[u];
        *reinterpret_cast<uint4*>(a.vpool + dst0 + e + half) = v1[u];
      }
    }
  }
}

}  // namespace

int launch_kv_shift(const KvShiftArgs& a, cudaStream_t st) {
  if (a.n_items <= 0) return 0;
  const long long blocks = (long long)a.n_items * a.n_layers * a.n_kv;
  if (blocks >= (1LL << 31)) return -1;
  kv_shift_kernel<<<(unsigned)blocks, kShiftThreads, 0, st>>>(a);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace cl
