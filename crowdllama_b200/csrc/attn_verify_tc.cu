// attn_verify_tc.cu — paged GQA attention of a few consecutive query rows per sequence over a long cache, on the tensor
// cores: the attention of a verify pass over several sequences (Engine::verify_batch).
//
// attn_decode_tc_kernel with R <= 16 query positions per sequence instead of one:
//   grid = (kv head, split, segment), 160 threads: warp 4 streams the split's KV pages as 128B-swizzled 2-D TMA tiles (two
//   32-token pages = K lo|hi, V lo|hi per 32 KB ring slot).  The A-tile rows are the pairs (row r, query head h of the kv
//   group), A row 4 r + h: up to 64 rows, four m16 tiles.  Consumer warp w takes m16 tile w over every page of the
//   split (4 warps, not 8: with 8 the 12-warp register allocation would cap a thread at 168 registers and spill): S = Q K^T (ldmatrix on the swizzled tiles, mma.sync.m16n8k16), the causal mask (row r sees keys
//   < len + r + 1), online softmax on the fragments, O += P V with P split into hi + lo bf16 terms (fp32-accurate
//   probabilities, DESIGN.md §2); with several splits the last split to arrive combines the partials in split order, so the result is bit-reproducible.
// Output: bf16 attention rows [row][q_dim], the X operand of the o-projection.  The split plan of a segment depends on
// that segment alone (AttnVerifyArgs), so its rows come out the same whatever else shares the launch.
// Shapes: head_dim 128, 4 query heads per kv head, page 32 (attn_decode_tc_supported's); others run the prefill kernels.
#include <algorithm>
#include <cstdio>

#include "common.cuh"
#include "kernels.h"

namespace cl {

namespace {

constexpr int HD = 128, REP = 4, P = 32;
constexpr int NS = 3;                         // ring slots
constexpr int MAXS = 64;
constexpr uint32_t PAGE_BYTES = 16 * 1024;    // one 32-token page: K lo|hi, V lo|hi
constexpr float LOG2E = 1.4426950408889634f;
// Two instantiations.  <4, 2>: 4 consumer warps (one per m16 tile, up to kVerifyMaxRows rows per segment) and two pages
// per ring slot, one CTA per SM.  <1, 1>: one consumer warp (segments of one row, whose 4 A rows sit in m16 tile 0) and
// one page per slot, about 64 KB of shared memory: three CTAs per SM (launches of kVerifyOneWarpMinSegs or more
// segments of one row).  A row's instruction sequence is the same in both:
// the same fragments, pages in the same order each with its own online-softmax update, hi + lo P, split-order combine.
template <int NW, int PPS>
struct VerifyShape {
  static constexpr int ROWS = NW * 16;        // A rows: 4 per segment row
  static constexpr uint32_t SLOT = PPS * PAGE_BYTES;
  static constexpr size_t SMEM = (size_t)NS * SLOT + 2 * NS * 8 + (2 * NW * 16 + NW * 16 * HD + 2 * MAXS * ROWS + ROWS + 4) * 4 + 1024 + 64;
};
static_assert(VerifyShape<4, 2>::ROWS == kVerifyMaxRows * REP, "the 4-warp kernel covers the largest segment");

struct VerifyTcArgs {
  AttnVerifyArgs a;
  long long layer_row0;                       // first row of this layer in the pool-wide tensor maps
};

template <int NW, int PPS>
__global__ void __launch_bounds__((NW + 1) * 32, NW == 1 ? 3 : 1)
attn_verify_tc_kernel(const __grid_constant__ CUtensorMap kmap, const __grid_constant__ CUtensorMap vmap, const VerifyTcArgs t) {
  constexpr int ROWS = VerifyShape<NW, PPS>::ROWS;
  constexpr uint32_t SLOT = VerifyShape<NW, PPS>::SLOT;
  const AttnVerifyArgs& a = t.a;
  const int g = blockIdx.x, sp = blockIdx.y, sg = blockIdx.z;
  const int4 s0 = reinterpret_cast<const int4*>(a.segs)[2 * sg], s1 = reinterpret_cast<const int4*>(a.segs)[2 * sg + 1];
  const int seq = s0.x, row0 = s0.y, R = s0.z, len = s0.w, part_off = s1.x, ns = s1.y;
  if (sp >= ns) return;                       // this segment takes fewer splits than the grid has
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)NS * SLOT);
  uint64_t* empty = full + NS;
  float* red_m = reinterpret_cast<float*>(empty + NS);       // [NW][16]
  float* red_l = red_m + NW * 16;                            // [NW][16]
  float* red_acc = red_l + NW * 16;                          // [NW][16][HD]
  float* cm_s = red_acc + NW * 16 * HD;                      // [MAXS][ROWS]
  float* cw_s = cm_s + MAXS * ROWS;                          // [MAXS][ROWS]
  float* cL_s = cw_s + MAXS * ROWS;                          // [ROWS]
  int* is_last_s = reinterpret_cast<int*>(cL_s + ROWS);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    for (int i = 0; i < NS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NW); }
    fence_barrier_init();
  }
  __syncthreads();
  const int ctx = len + R;                    // keys of the last row
  const int total_pages = (ctx + P - 1) / P;
  const int pps = a.split_pages > 0 ? a.split_pages : (total_pages + ns - 1) / ns;
  const int pg0 = sp * pps;
  const int pg1 = min(total_pages, pg0 + pps);
  const int npg = pg1 > pg0 ? pg1 - pg0 : 0;
  const int n_tiles = (npg + PPS - 1) / PPS;
  const int* bt = a.block_tables + (size_t)seq * a.bt_stride;

  if (warp == NW) {
    // ---------------- producer: the new rows' K/V were written by the launch before this one (stream order)
    if (!elect_one()) return;
    prefetch_tmap(&kmap);
    prefetch_tmap(&vmap);
    for (int it = 0; it < n_tiles; ++it) {
      const int st = it % NS;
      mbar_wait(&empty[st], ((uint32_t)(it / NS) & 1u) ^ 1u);
      const int pa = pg0 + PPS * it;
      const int npage = min(PPS, pg1 - pa);
      uint8_t* dst = ring + (size_t)st * SLOT;
      mbar_arrive_expect_tx(&full[st], (uint32_t)npage * PAGE_BYTES);
      for (int pgi = 0; pgi < npage; ++pgi) {
        const long long row = t.layer_row0 + ((long long)bt[pa + pgi] * a.n_kv + g) * P;
        uint8_t* d = dst + pgi * PAGE_BYTES;
        tma_load_2d(d, &kmap, 0, (int)row, &full[st]);
        tma_load_2d(d + 4096, &kmap, 64, (int)row, &full[st]);
        tma_load_2d(d + 8192, &vmap, 0, (int)row, &full[st]);
        tma_load_2d(d + 12288, &vmap, 64, (int)row, &full[st]);
      }
    }
    return;
  }

  // ---------------- consumers: warp = m16 tile
  const int mt = warp;
  const bool active = mt * 4 < R;
  const int rq = lane >> 2, cq = lane & 3;     // fragment rows rq and rq + 8, column pair cq
  const int r0 = mt * 4 + (rq >> 2), r1 = r0 + 2, h = rq & 3;   // A row x -> (row mt * 4 + x / 4, head x % 4)
  // causal limit of each fragment row; rows past R (padding) take the last row's, their output is never written
  const int lim0 = len + min(r0, R - 1) + 1, lim1 = len + min(r1, R - 1) + 1;
  const float scale2 = rsqrtf((float)HD) * LOG2E;
  uint32_t qf[HD / 16][4];
  {
    const __nv_bfloat16* q0 = a.q + (size_t)(row0 + r0) * a.q_stride + (size_t)(g * REP + h) * HD;
    const __nv_bfloat16* q1 = a.q + (size_t)(row0 + r1) * a.q_stride + (size_t)(g * REP + h) * HD;
    const bool v0 = r0 < R, v1 = r1 < R;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      qf[kk][0] = v0 ? *reinterpret_cast<const uint32_t*>(q0 + kk * 16 + 2 * cq) : 0u;
      qf[kk][2] = v0 ? *reinterpret_cast<const uint32_t*>(q0 + kk * 16 + 8 + 2 * cq) : 0u;
      qf[kk][1] = v1 ? *reinterpret_cast<const uint32_t*>(q1 + kk * 16 + 2 * cq) : 0u;
      qf[kk][3] = v1 ? *reinterpret_cast<const uint32_t*>(q1 + kk * 16 + 8 + 2 * cq) : 0u;
    }
  }
  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int it = 0; it < n_tiles; ++it) {
    const int st = it % NS;
    mbar_wait(&full[st], (uint32_t)(it / NS) & 1u);
    const int npage = min(PPS, pg1 - (pg0 + PPS * it));
    for (int pgi = 0; pgi < npage && active; ++pgi) {
      const uint32_t kb = smem_u32(ring + (size_t)st * SLOT + pgi * PAGE_BYTES), vb = kb + 8192;
      const int tok0 = (pg0 + PPS * it + pgi) * P;
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
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int tok = tok0 + nj * 8 + 2 * cq + e;
          sacc[nj][e] = tok < lim0 ? sacc[nj][e] * scale2 : -INFINITY;
          sacc[nj][2 + e] = tok < lim1 ? sacc[nj][2 + e] * scale2 : -INFINITY;
          mx0 = fmaxf(mx0, sacc[nj][e]);
          mx1 = fmaxf(mx1, sacc[nj][2 + e]);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      // a row may have no key yet: the page can lie past its causal limit.  Its maximum then stays -inf and a finite
      // reference (0) keeps corr and p at 0 instead of NaN.
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      const float ref0 = mn0 == -INFINITY ? 0.f : mn0, ref1 = mn1 == -INFINITY ? 0.f : mn1;
      const float corr0 = exp2f(m0 - ref0), corr1 = exp2f(m1 - ref1);
      m0 = mn0; m1 = mn1;
      float rs0 = 0.f, rs1 = 0.f;
      uint32_t pf[2][4], pl[2][4];                          // P = hi + lo bf16 terms
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
        const float p0 = exp2f(sacc[nj][0] - ref0), p1 = exp2f(sacc[nj][1] - ref0);
        const float p2 = exp2f(sacc[nj][2] - ref1), p3 = exp2f(sacc[nj][3] - ref1);
        rs0 += p0 + p1;
        rs1 += p2 + p3;
        const float h0 = bf16_round(p0), h1 = bf16_round(p1), h2 = bf16_round(p2), h3 = bf16_round(p3);
        pf[nj >> 1][(nj & 1) * 2] = pack_bf16(h0, h1);
        pf[nj >> 1][(nj & 1) * 2 + 1] = pack_bf16(h2, h3);
        pl[nj >> 1][(nj & 1) * 2] = pack_bf16(p0 - h0, p1 - h1);
        pl[nj >> 1][(nj & 1) * 2 + 1] = pack_bf16(p2 - h2, p3 - h3);
      }
      l0 = l0 * corr0 + rs0;
      l1 = l1 * corr1 + rs1;
#pragma unroll
      for (int nd = 0; nd < HD / 8; ++nd) { o[nd][0] *= corr0; o[nd][1] *= corr0; o[nd][2] *= corr1; o[nd][3] *= corr1; }
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
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  if (cq == 0) {
    red_m[warp * 16 + rq] = m0; red_l[warp * 16 + rq] = l0;
    red_m[warp * 16 + rq + 8] = m1; red_l[warp * 16 + rq + 8] = l1;
  }
#pragma unroll
  for (int nd = 0; nd < HD / 8; ++nd) {
    float* r0p = red_acc + (size_t)(warp * 16 + rq) * HD + nd * 8 + 2 * cq;
    float* r1p = red_acc + (size_t)(warp * 16 + rq + 8) * HD + nd * 8 + 2 * cq;
    r0p[0] = o[nd][0]; r0p[1] = o[nd][1];
    r1p[0] = o[nd][2]; r1p[1] = o[nd][3];
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");

  // ---- the m16 tile's rows -> the output (one split) or this split's partial
  const int nrows = REP * R;                   // A row a = 4 r + h = mt * 16 + x
  float* part = a.part + part_off + ((size_t)g * ns + sp) * nrows * (HD + 2);
  for (int e = tid; e < nrows * HD; e += NW * 32) {
    const int ar = e / HD, i = e % HD;            // warp ar / 16, fragment row ar % 16
    const float M = red_m[ar], L = red_l[ar], A = red_acc[(size_t)ar * HD + i];
    if (ns == 1) {
      a.out[(size_t)(row0 + (ar >> 2)) * a.out_stride + (size_t)(g * REP + (ar & 3)) * HD + i] = __float2bfloat16_rn(A / L);
    } else {
      float* ph = part + (size_t)ar * (HD + 2);
      if (i == 0) { ph[0] = M; ph[1] = L; }
      ph[2 + i] = A;
    }
  }
  if (ns == 1) return;
  __threadfence();
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  if (tid == 0) {
    unsigned* cnt = a.counters + (size_t)sg * a.n_kv + g;
    const unsigned old = atomicAdd(cnt, 1u);
    *is_last_s = (old == (unsigned)ns - 1u);
    if (*is_last_s) *cnt = 0u;                 // re-arm for the next launch
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  if (!*is_last_s) return;
  __threadfence();

  // ---- the last split to finish combines the partials of this (segment, kv head) in split order
  const float* pall = a.part + part_off + (size_t)g * ns * nrows * (HD + 2);
  for (int e = tid; e < ns * nrows; e += NW * 32) {
    const int sidx = e / nrows, ar = e % nrows;
    const float* ph = pall + ((size_t)sidx * nrows + ar) * (HD + 2);
    cm_s[sidx * ROWS + ar] = __ldcg(ph);
    cw_s[sidx * ROWS + ar] = __ldcg(ph + 1);  // l for now
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  if (tid < nrows) {
    float M = -INFINITY;
    for (int sidx = 0; sidx < ns; ++sidx) M = fmaxf(M, cm_s[sidx * ROWS + tid]);
    float L = 0.f;
    for (int sidx = 0; sidx < ns; ++sidx) {
      const float ms = cm_s[sidx * ROWS + tid];
      const float c = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
      L = fmaf(cw_s[sidx * ROWS + tid], c, L);
      cw_s[sidx * ROWS + tid] = c;            // weight of this split
    }
    cL_s[tid] = L;
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
  for (int e = tid; e < nrows * HD; e += NW * 32) {
    const int ar = e / HD, i = e % HD;
    float A = 0.f;
    for (int sidx = 0; sidx < ns; ++sidx)
      A = fmaf(__ldcg(pall + ((size_t)sidx * nrows + ar) * (HD + 2) + 2 + i), cw_s[sidx * ROWS + ar], A);
    a.out[(size_t)(row0 + (ar >> 2)) * a.out_stride + (size_t)(g * REP + (ar & 3)) * HD + i] = __float2bfloat16_rn(A / cL_s[ar]);
  }
}

}  // namespace

bool attn_verify_tc_supported(int n_heads, int n_kv, int head_dim, int page_size) {
  return attn_decode_tc_supported(n_heads, n_kv, head_dim, page_size, 1);
}

int attn_verify_max_splits() { return MAXS; }

namespace {
template <int NW, int PPS>
int launch_inst(const AttnVerifyArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st) {
  constexpr size_t SMEM = VerifyShape<NW, PPS>::SMEM;
  static PerDeviceOnce attr;
  if (attr.pending()) {
    if (cudaFuncSetAttribute(attn_verify_tc_kernel<NW, PPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess) {
      fprintf(stderr, "[clengine] attn_verify_tc: %zu B of shared memory refused\n", SMEM);
      return -1;
    }
    attr.mark();
  }
  VerifyTcArgs t{a, layer_row0};
  attn_verify_tc_kernel<NW, PPS><<<dim3(a.n_kv, a.nsplit, a.n_segs), (NW + 1) * 32, SMEM, st>>>(kmap, vmap, t);
  return cudaPeekAtLastError() == cudaSuccess ? 1 : -1;   // a failed launch stays visible to the caller's report
}
}  // namespace

int launch_attn_verify_tc(const AttnVerifyArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st) {
  if (!attn_verify_tc_supported(a.n_heads, a.n_kv, a.head_dim, a.page_size) || a.nsplit < 1 || a.nsplit > MAXS || a.n_segs < 1 ||
      a.max_rows < 1 || a.max_rows > kVerifyMaxRows)
    return -1;
  // the one-warp kernel where every segment has one row and there are enough of them to fill the SMs with its three CTAs
  // per SM: a deterministic step of B = 8 / 64 behind 4096 tokens spends 0.96 / 0.73 of its time with it, one of B = 1
  // 1.08 (H100 80GB HBM3, profiles/h100_deterministic.json)
  const bool one_warp = a.max_rows == 1 && a.n_segs >= kVerifyOneWarpMinSegs;
  return one_warp ? launch_inst<1, 1>(a, kmap, vmap, layer_row0, st) : launch_inst<4, 2>(a, kmap, vmap, layer_row0, st);
}

}  // namespace cl
