// kv_host.cu — the host tier of the prefix cache: copies of whole KV pages between the paged pool in HBM and pinned,
// mapped host pages, made by the kernels themselves over the host link (no staging buffer, no cudaMemcpy per block).
//
// A work item is one (move, K|V, layer) block: page `page` of one layer of the pool, [n_kv][page_size][head_dim] bf16,
// which is contiguous there and in the host page ([K|V][layer][n_kv][page_size][head_dim]).  One CTA copies one block
// with 16-byte accesses, kUnroll of them in flight per thread, so that a fill keeps enough reads of host memory
// outstanding to cover the link's latency.
//
// Neither kernel triggers its dependents early (no griddepcontrol.launch_dependents): the decode and attention kernels
// issue their KV page loads before griddepcontrol.wait, so a kernel launched after a fill with programmatic dependent
// launch must not start before the fill has finished writing.
#include "common.cuh"
#include "kernels.h"

namespace cl {

namespace {

constexpr int kMoveThreads = 256;
constexpr int kUnroll = 8;

template <bool kToHost>
__device__ __forceinline__ void kv_move_block(const KvMoveArgs& a) {
  const int items = 2 * a.n_layers;
  const int m = blockIdx.x / items, r = blockIdx.x % items;   // r = (K|V) * n_layers + layer
  const int2 mv = a.moves[m];                                 // (device page, host page)
  const int layer = r % a.n_layers;
  __nv_bfloat16* pool = (r < a.n_layers ? a.kpool : a.vpool) + (size_t)layer * a.layer_elems;
  uint4* dev = reinterpret_cast<uint4*>(pool) + (size_t)mv.x * a.blk_vec;
  uint4* host = a.host + ((size_t)mv.y * items + r) * a.blk_vec;
  const uint4* src = kToHost ? dev : host;
  uint4* dst = kToHost ? host : dev;
  for (int i0 = threadIdx.x; i0 < a.blk_vec; i0 += kMoveThreads * kUnroll) {
    uint4 v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int i = i0 + u * kMoveThreads;
      if (i < a.blk_vec) v[u] = src[i];
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int i = i0 + u * kMoveThreads;
      if (i < a.blk_vec) dst[i] = v[u];
    }
  }
}

__global__ void __launch_bounds__(kMoveThreads) kv_spill_kernel(KvMoveArgs a) { kv_move_block<true>(a); }
__global__ void __launch_bounds__(kMoveThreads) kv_fill_kernel(KvMoveArgs a) { kv_move_block<false>(a); }

}  // namespace

int launch_kv_move(bool to_host, const KvMoveArgs& a, cudaStream_t st) {
  if (a.n_moves <= 0) return 0;
  const dim3 grid((unsigned)(a.n_moves * 2 * a.n_layers));
  if (to_host) kv_spill_kernel<<<grid, kMoveThreads, 0, st>>>(a);
  else kv_fill_kernel<<<grid, kMoveThreads, 0, st>>>(a);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace cl
