// attn_decode_tc.cu — paged GQA decode attention on the tensor cores, stand-alone kernel for the BATCHED step.
//
// The CUDA-core kernel of decode_kernels.cu is issue-bound once many sequences share a step (many warp instructions per
// byte of KV).  This is phase P1 of the
// persistent kernel (decode_mega.cu) as a kernel of its own:
//   grid = (n_kv, nsplit, batch), 288 threads: warp 8 streams this split's KV pages as 128B-swizzled 2-D TMA tiles
//   (two 32-token pages = K lo|hi, V lo|hi per 32 KB ring slot), warps 0-7 take one page each:
//   S[16 x 32] = Q K^T with the 4 query heads of the kv group in rows 0-3 of an m16n8k16 A tile (ldmatrix on the
//   swizzled tiles), online softmax on the fragments, O += P V with P split into hi + lo bf16 terms (fp32-accurate
//   probabilities, DESIGN.md §2), then the warp merge, the split partial, and the last split to arrive combines
//   (same tail as attn_decode_kernel: fp32 output for the GEMV path, bf16 copy = X operand of the o-projection).
// Shapes: head_dim 128, 4 query heads per kv head, page 32 (Llama-3-8B / Mistral-7B); others use the CUDA-core kernel.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace cl {

namespace {

constexpr int HD = 128, REP = 4, P = 32;
// Two shapes of the same kernel (template parameters NW = consumer warps, NS = ring slots of 32 KB, MINB = CTAs per SM):
//   <8, 4, 1>  one CTA per SM, 8 warps, 128 KB of KV in flight — few (kv head, split, sequence) items, long chains;
//   <4, 2, 2>  two CTAs per SM, 4 warps each, 2 x 64 KB in flight — more items than SMs (B >= 19):
//              the prologue (block table, q) and the epilogue (warp merge, split combine) of one CTA overlap the page
//              loop of its neighbour, and the waves of short items halve.
constexpr uint32_t SLOT = 32 * 1024;
constexpr int MAXS = 64;
constexpr float LOG2E = 1.4426950408889634f;

struct TcArgs {
  AttnDecodeArgs a;
  long long layer_row0;                    // first row of this layer in the pool-wide tensor maps
};

template <int NW, int NS, int MINB>
__global__ void __launch_bounds__((NW + 1) * 32, MINB)
attn_decode_tc_kernel(const __grid_constant__ CUtensorMap kmap, const __grid_constant__ CUtensorMap vmap, const TcArgs t) {
  const AttnDecodeArgs& a = t.a;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)NS * SLOT);
  uint64_t* empty = full + NS;
  float* red_m = reinterpret_cast<float*>(empty + NS);       // [NW][REP]
  float* red_l = red_m + NW * REP;                           // [NW][REP]
  float* red_acc = red_l + NW * REP;                         // [NW][REP][HD]
  float* cm_s = red_acc + NW * REP * HD;                     // [MAXS][REP]
  float* cw_s = cm_s + MAXS * REP;                           // [MAXS][REP]
  float* cL_s = cw_s + MAXS * REP;                           // [REP]
  int* is_last_s = reinterpret_cast<int*>(cL_s + REP);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    for (int i = 0; i < NS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NW); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  const bool is_producer = warp == NW;
  if (is_producer) {
    if (!elect_one()) return;
    prefetch_tmap(&kmap);
    prefetch_tmap(&vmap);
  }
  // Items = (kv head, split, sequence), kv head fastest.  One item per CTA when the grid covers them; with fewer CTAs
  // (persistent launch, nsplit == 1) every CTA walks its items and the ring keeps running across them: the producer is
  // already loading the next item's pages while the consumer warps merge and store the current one.
  const int n_items = a.n_kv * a.nsplit * a.batch;
  int tile_base = 0;                           // ring tiles of the items this CTA has finished (same in every warp)
  bool waited = false;                         // producer: griddepcontrol.wait executed
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
  const int g = item % a.n_kv, sp = (item / a.n_kv) % a.nsplit, b = item / (a.n_kv * a.nsplit);
  const int slot = a.slots ? a.slots[b] : b;
  const int pos = a.pos[slot];                 // stable for the whole step
  const int ctx = pos + 1;
  const int total_pages = (ctx + P - 1) / P;
  const int pps = (total_pages + a.nsplit - 1) / a.nsplit;
  const int pg0 = sp * pps;
  const int pg1 = min(total_pages, pg0 + pps);
  const int npg = pg1 > pg0 ? pg1 - pg0 : 0;
  const int n_tiles = (npg + 1) / 2;
  const int* bt = a.block_tables + (size_t)slot * a.bt_stride;

  if (is_producer) {
    // ---------------- producer: everything it touches before griddepcontrol.wait (pos, block table, K/V of EARLIER
    // tokens) is immutable during the step; only the page that receives the current token waits
    const int cur_page = pos / P;
    for (int it = 0; it < n_tiles; ++it) {
      const int T = tile_base + it, st = T % NS;
      mbar_wait(&empty[st], ((uint32_t)(T / NS) & 1u) ^ 1u);
      const int pa = pg0 + 2 * it, pb = pa + 1;
      const bool two = pb < pg1;
      if (!waited && (pa == cur_page || (two && pb == cur_page))) { pdl_wait(); waited = true; }
      uint8_t* dst = ring + (size_t)st * SLOT;
      mbar_arrive_expect_tx(&full[st], two ? 32768u : 16384u);
      for (int pgi = 0; pgi < (two ? 2 : 1); ++pgi) {
        const long long row = t.layer_row0 + ((long long)bt[pa + pgi] * a.n_kv + g) * P;
        uint8_t* d = dst + pgi * 16384;
        tma_load_2d(d, &kmap, 0, (int)row, &full[st]);
        tma_load_2d(d + 4096, &kmap, 64, (int)row, &full[st]);
        tma_load_2d(d + 8192, &vmap, 0, (int)row, &full[st]);
        tma_load_2d(d + 12288, &vmap, 64, (int)row, &full[st]);
      }
    }
    tile_base += n_tiles;
    continue;
  }

  // ---------------- consumers (warps 0..7)
  pdl_wait();                                  // q is the previous kernel's output
  const int rq = lane >> 2, cq = lane & 3;     // fragment row (head) / column pair
  const float scale2 = rsqrtf((float)HD) * LOG2E;
  uint32_t qf[HD / 16][4];
  {
    const float* q = a.q + (size_t)slot * a.q_stride + (size_t)g * REP * HD;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      qf[kk][1] = 0u; qf[kk][3] = 0u;          // rows 8..15: padding
      if (rq < REP) {
        const float2 lo = __ldcg(reinterpret_cast<const float2*>(q + rq * HD + kk * 16 + 2 * cq));
        const float2 hi = __ldcg(reinterpret_cast<const float2*>(q + rq * HD + kk * 16 + 8 + 2 * cq));
        qf[kk][0] = pack_bf16(lo.x, lo.y);
        qf[kk][2] = pack_bf16(hi.x, hi.y);
      } else {
        qf[kk][0] = 0u; qf[kk][2] = 0u;
      }
    }
  }
  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float mrow = -INFINITY, lrow = 0.f;          // row rq (valid for rq < REP)
  for (int it = 0; it < n_tiles; ++it) {
    const int T = tile_base + it, st = T % NS;
    mbar_wait(&full[st], (uint32_t)(T / NS) & 1u);
    const int npage = (pg0 + 2 * it + 1 < pg1) ? 2 : 1;
    for (int pgi = 0; pgi < npage; ++pgi) {
      if (((2 * it + pgi) & (NW - 1)) != warp) continue;   // page -> warp (round robin)
      const uint32_t kb = smem_u32(ring + (size_t)st * SLOT + pgi * 16384), vb = kb + 8192;
      const int tok0 = (pg0 + 2 * it + pgi) * P;
      float sacc[4][4];
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) { sacc[nj][0] = sacc[nj][1] = sacc[nj][2] = sacc[nj][3] = 0.f; }
      const int id = lane >> 3;
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        const uint32_t kh = kb + (kk >> 2) * 4096;          // dims 0-63 | 64-127
#pragma unroll
        for (int np = 0; np < 2; ++np) {
          uint32_t kf[4];
          const int row = (2 * np + (id >> 1)) * 8 + (lane & 7), ch = (kk & 3) * 2 + (id & 1);
          ldsm_x4(kf, kh + row * 128 + ((ch ^ (row & 7)) << 4));
          mma_bf16(sacc[2 * np], qf[kk], kf[0], kf[1]);
          mma_bf16(sacc[2 * np + 1], qf[kk], kf[2], kf[3]);
        }
      }
      float mx = -INFINITY;
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int tok = tok0 + nj * 8 + 2 * cq + e;
          const float v = tok < ctx ? sacc[nj][e] * scale2 : -INFINITY;
          sacc[nj][e] = v;
          mx = fmaxf(mx, v);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(mrow, mx);                     // finite: every page of a split holds >= 1 valid token
      const float corr = exp2f(mrow - mn);
      mrow = mn;
      float rs = 0.f;
      uint32_t pf[2][4], pl[2][4];                          // P = hi + lo bf16 terms
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
        const float p0 = exp2f(sacc[nj][0] - mn), p1 = exp2f(sacc[nj][1] - mn);
        rs += p0 + p1;
        const float h0 = bf16_round(p0), h1 = bf16_round(p1);
        pf[nj >> 1][(nj & 1) * 2] = pack_bf16(h0, h1);
        pf[nj >> 1][(nj & 1) * 2 + 1] = 0u;                 // rows 8..15
        pl[nj >> 1][(nj & 1) * 2] = pack_bf16(p0 - h0, p1 - h1);
        pl[nj >> 1][(nj & 1) * 2 + 1] = 0u;
      }
      lrow = lrow * corr + rs;
#pragma unroll
      for (int nd = 0; nd < HD / 8; ++nd) { o[nd][0] *= corr; o[nd][1] *= corr; }
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {                      // 16-token k-steps
#pragma unroll
        for (int nd = 0; nd < HD / 8; nd += 2) {
          uint32_t vf[4];
          const int row = jj * 16 + (id & 1) * 8 + (lane & 7), chunk = nd + (id >> 1);
          ldsm_x4_t(vf, vb + (chunk >> 3) * 4096 + row * 128 + (((chunk & 7) ^ (row & 7)) << 4));
          mma_bf16(o[nd], pf[jj], vf[0], vf[1]);
          mma_bf16(o[nd + 1], pf[jj], vf[2], vf[3]);
          mma_bf16(o[nd], pl[jj], vf[0], vf[1]);
          mma_bf16(o[nd + 1], pl[jj], vf[2], vf[3]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
  }
  lrow += __shfl_xor_sync(0xffffffffu, lrow, 1);
  lrow += __shfl_xor_sync(0xffffffffu, lrow, 2);
  if (rq < REP) {
    if (cq == 0) { red_m[warp * REP + rq] = mrow; red_l[warp * REP + rq] = lrow; }
#pragma unroll
    for (int nd = 0; nd < HD / 8; ++nd) {
      red_acc[(warp * REP + rq) * HD + nd * 8 + 2 * cq] = o[nd][0];
      red_acc[(warp * REP + rq) * HD + nd * 8 + 2 * cq + 1] = o[nd][1];
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");

  // ---- CTA partial (merge of the 8 warps) -> global, or straight to the output when there is one split
  float* part = a.part + ((((size_t)slot * a.n_kv + g) * a.nsplit + sp) * REP) * (HD + 2);
  float* out = a.out + (size_t)slot * a.out_stride;
  for (int e = tid; e < REP * HD; e += NW * 32) {
    const int hh = e / HD, i = e % HD;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < NW; ++w) M = fmaxf(M, red_m[w * REP + hh]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      const float mw = red_m[w * REP + hh];
      const float c = (mw == -INFINITY) ? 0.f : exp2f(mw - M);
      L = fmaf(red_l[w * REP + hh], c, L);
      A = fmaf(red_acc[(w * REP + hh) * HD + i], c, A);
    }
    if (a.nsplit == 1) {
      const float r = bf16_round(A / L);
      out[(size_t)(g * REP + hh) * HD + i] = r;
      if (a.out_bf16) a.out_bf16[(size_t)b * a.out_stride + (size_t)(g * REP + hh) * HD + i] = __float2bfloat16_rn(r);
    } else {
      float* ph = part + (size_t)hh * (HD + 2);
      if (i == 0) { ph[0] = M; ph[1] = L; }
      ph[2 + i] = A;
    }
  }
  bool combine = false;                        // uniform over the consumer warps
  if (a.nsplit > 1) {
    __threadfence();
    asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
    if (tid == 0) {
      unsigned* cnt = a.counters + (size_t)slot * a.n_kv + g;
      const unsigned old = atomicAdd(cnt, 1u);
      *is_last_s = (old == (unsigned)a.nsplit - 1u);
      if (*is_last_s) *cnt = 0u;  // re-arm for the next launch (graph replay)
    }
    asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
    combine = *is_last_s != 0;
  }
  if (combine) {
  __threadfence();

  // ---- the last split to finish combines all partials of this kv head (fixed split order)
  const float* pall = a.part + (((size_t)slot * a.n_kv + g) * a.nsplit) * REP * (HD + 2);
  const int ns = a.nsplit;
  for (int e = tid; e < ns * REP; e += NW * 32) {
    const int sidx = e / REP, hh = e % REP;
    const float* ph = pall + ((size_t)sidx * REP + hh) * (HD + 2);
    cm_s[sidx * REP + hh] = __ldcg(ph);
    cw_s[sidx * REP + hh] = __ldcg(ph + 1);   // l for now
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  if (tid < REP) {
    float M = -INFINITY;
    for (int sidx = 0; sidx < ns; ++sidx) M = fmaxf(M, cm_s[sidx * REP + tid]);
    float L = 0.f;
    for (int sidx = 0; sidx < ns; ++sidx) {
      const float ms = cm_s[sidx * REP + tid];
      const float c = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
      L = fmaf(cw_s[sidx * REP + tid], c, L);
      cw_s[sidx * REP + tid] = c;             // weight of this split
    }
    cL_s[tid] = L;
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  for (int e = tid; e < REP * HD; e += NW * 32) {
    const int hh = e / HD, i = e % HD;
    float A = 0.f;
    for (int sidx = 0; sidx < ns; ++sidx)
      A = fmaf(__ldcg(pall + ((size_t)sidx * REP + hh) * (HD + 2) + 2 + i), cw_s[sidx * REP + hh], A);
    const float r = bf16_round(A / cL_s[hh]);
    out[(size_t)(g * REP + hh) * HD + i] = r;
    if (a.out_bf16) a.out_bf16[(size_t)b * a.out_stride + (size_t)(g * REP + hh) * HD + i] = __float2bfloat16_rn(r);
  }
  }  // combine
  tile_base += n_tiles;
  // the merge buffers (and is_last_s / the combine scratch) are reused by this CTA's next item
  if (item + (int)gridDim.x < n_items) asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  }  // items
}

}  // namespace

bool attn_decode_tc_supported(int n_heads, int n_kv, int head_dim, int page_size, int nsplit) {
  return head_dim == HD && n_kv > 0 && n_heads == REP * n_kv && page_size == P && nsplit >= 1 && nsplit <= MAXS;
}

namespace {
template <int NW, int NS, int MINB>
int launch_variant(const AttnDecodeArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st, bool pdl) {
  constexpr size_t smem = (size_t)NS * SLOT + 2 * NS * 8 + (2 * NW * REP + NW * REP * HD + 2 * MAXS * REP + REP + 4) * 4 + 1024 + 64;
  auto kern = attn_decode_tc_kernel<NW, NS, MINB>;
  static PerDeviceOnce attr;
  if (attr.pending()) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
    attr.mark();
  }
  TcArgs t{a, layer_row0};
  // persistent launch (single split, more items than resident CTAs): MINB CTAs per SM walk the items instead of one CTA
  // per item.
  const int n_items = a.n_kv * a.nsplit * a.batch, resident = MINB * sm_count();
  const int grid = (a.nsplit == 1 && n_items > resident) ? resident : n_items;
  return launch_pdl(kern, dim3(grid), dim3((NW + 1) * 32), smem, st, pdl, kmap, vmap, t) == cudaSuccess ? 1 : -1;
}
}  // namespace

// KV splits per sequence and kernel shape for a batched step of `batch` sequences: one wave of 8-warp CTAs while the
// items fit the machine, otherwise the 4-warp shape with two CTAs per SM.
void attn_decode_tc_plan(int n_kv, int batch, int nsplit_max, int cta_budget, int* nsplit, int* small) {
  const int items = n_kv * batch;
  *small = items > cta_budget;   // small shape once the items exceed one wave
  const int budget = *small ? 2 * cta_budget : cta_budget;
  *nsplit = std::max(1, std::min(std::min(nsplit_max, MAXS), budget / std::max(items, 1)));
}

int launch_attn_decode_tc(const AttnDecodeArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st,
                          bool pdl) {
  if (!attn_decode_tc_supported(a.n_heads, a.n_kv, a.head_dim, a.page_size, a.nsplit)) return -1;
  return a.tc_small ? launch_variant<4, 2, 2>(a, kmap, vmap, layer_row0, st, pdl) : launch_variant<8, 4, 1>(a, kmap, vmap, layer_row0, st, pdl);
}

}  // namespace cl
