// attn_prefill_tc.cu — causal GQA prefill attention over the paged KV cache on the Hopper tensor cores (wgmma).
//
// "prefill causal attention | T x T per head, d = 128 | tensor pipe" row of SURVEY.md §8a.
// Replaces the mma.sync kernel of prefill_kernels.cu for head_dim 128 / page 32 (that one stays for head_dim 64).
//
// One work item = one query head x 128 consecutive query rows.  Persistent CTAs (one per SM) take items round-robin from a
// heaviest-first order.  Each of the two consumer warpgroups owns 64 of the 128 rows; per 64-token KV block j:
//     S = Q K_j^T            wgmma m64 n64 k16 x 8 (head dim), Q and K K-major 128B-swizzled tiles, fp32 in registers
//     P = exp2(S - m)        online softmax on the accumulator fragments (row maximum over the 4 lanes of a row),
//                            P rounded to bf16 straight into the A-operand fragments of the next MMA
//     O += P V_j             wgmma m64 n64 k16 x 4 (tokens) x 2 (head-dim halves), A = P from registers, V straight from
//                            the paged cache as an MN-major (token rows, dims contiguous) 128B-swizzled operand
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread: the Q tile, K / V pages through a 4 x 32 KB ring,
// 2-D tensor maps over the whole pool), warpgroups 1-2 = MMA + softmax.  While one warpgroup runs its exponentials the
// tensor core works for the other.
// Numerics (cl-llama v1, DESIGN.md §3): q, K, V bf16; scores, softmax, accumulation fp32; P rounded to bf16 before P.V
// (the documented deviation of the prefill path); output rounded to bf16 = the o-projection's GEMM operand.
//
// Two instantiations of the one body:
//   LONG = false (variant 1): the block table staged in shared memory (MAX_BT pages, 10240 tokens), one item sweeps every
//     KV block of its (head, tile).
//   LONG = true (variant 2, any length): the producer reads block-table entries from global memory (a 128K-token row is
//     16 KB and stays in L2), and an item is (head, tile, KV split): the tile's blocks 0 .. nblk-1 spread evenly over
//     nsplit contiguous ranges.  With one split the item writes its bf16 rows as variant 1 does, bit for bit.  Otherwise
//     each split leaves fp32 (m, l, O) for its 128 rows in a workspace, and the split that arrives last for a (tile, head)
//     folds them in split order (so the result does not depend on arrival order) and re-arms its counter.
#include <cuda.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace cl {

namespace {

using namespace wg;

constexpr int HD = 128;                 // head dim
constexpr int TQ = 128;                 // query rows per item (two warpgroups of 64)
constexpr int TKV = 64;                 // tokens per KV block
constexpr int PAGE = 32;
constexpr uint32_t Q_BYTES = TQ * HD * 2;     // two [128 rows][128 B] swizzled slabs (dims 0-63 | 64-127)
constexpr uint32_t Q_SLAB = TQ * 128;
constexpr uint32_t KV_SLAB = TKV * 128;       // [64 tokens][128 B]
constexpr uint32_t KV_TILE = 2 * KV_SLAB;     // K or V of one block: 16 KB
constexpr uint32_t SLOT = 2 * KV_TILE;        // K | V
constexpr int NRING = 4;
constexpr int MAX_BT = 320;             // block-table entries staged in shared memory (10240 tokens)
constexpr int PART_ROW = HD + 2;        // a partial row: m, l, O[HD] (fp32)

struct AttnTcParams {
  const int* block_table;               // this sequence
  int n_bt;                             // entries of block_table that are valid (pages covering pos0 + T tokens)
  int pos0, T, n_heads, n_kv;
  long long layer_row0;                 // first row of this layer in the pool-wide K / V tensor maps
  __nv_bfloat16* out;                   // [T][n_heads * HD]
  float scale2;                         // 1/sqrt(HD) * log2(e)
  int nsplit;                           // variant 2: KV splits per (tile, head), 1 .. the lightest tile's block count
  float* part;                          // variant 2, nsplit > 1: [tile * n_heads + head][nsplit][TQ][PART_ROW]
  unsigned* counters;                   // variant 2, nsplit > 1: [tile * n_heads + head], zero between launches
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// work item -> (first query row, head, KV blocks kb0 .. kb1-1 of the tile's nblk); heaviest (latest rows) first, heads
// fastest, so the query heads of one kv group stream the same K / V pages through L2 at the same time
struct Item { int q0, head, split, kb0, kb1; };
template <bool LONG>
__device__ __forceinline__ bool get_item(const AttnTcParams& p, int idx, int n_tiles, Item* it) {
  const int ns = LONG ? p.nsplit : 1;
  if (idx >= n_tiles * p.n_heads * ns) return false;
  it->head = idx % p.n_heads;
  const int r = idx / p.n_heads;
  it->split = r % ns;
  it->q0 = (n_tiles - 1 - r / ns) * TQ;
  const int last = min(it->q0 + TQ, p.T) - 1;                      // last real query row of the item
  const int nblk = (p.pos0 + last) / TKV + 1;                      // KV blocks 0 .. nblk-1 hold keys <= its position
  it->kb0 = it->split * nblk / ns;                                 // nsplit <= nblk of every tile: no split is empty
  it->kb1 = (it->split + 1) * nblk / ns;
  return true;
}

// Variant 2 with nsplit > 1, run by the 256 consumer threads: this split's unnormalised rows (m, l, O) go to the workspace,
// and the split that arrives last for the (tile, head) folds every split's rows in split order into the bf16 output and
// re-arms the counter.  r = the thread's first row in the tile (its second is r + 8), as in the bf16 epilogue.
__device__ __forceinline__ void split_epilogue(const AttnTcParams& p, const Item& it, int r, int cq, const float (&o)[2][32],
                                               const float (&m_run)[2], const float (&l_run)[2], int* last_s) {
  const size_t th = (size_t)(it.q0 / TQ) * p.n_heads + it.head;
  const size_t split_floats = (size_t)TQ * PART_ROW;
  float* part = p.part + (th * p.nsplit + it.split) * split_floats;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* row = part + (size_t)(r + h * 8) * PART_ROW;
    if (cq == 0) { row[0] = m_run[h]; row[1] = l_run[h]; }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<float2*>(row + 2 + hh * 64 + i * 8 + 2 * cq) = make_float2(o[hh][4 * i + 2 * h], o[hh][4 * i + 2 * h + 1]);
  }
  __threadfence();
  asm volatile("bar.sync 3, 256;" ::: "memory");
  const int t = threadIdx.x - 128;
  if (t == 0) {
    unsigned* cnt = p.counters + th;
    const unsigned old = atomicAdd(cnt, 1u);
    *last_s = old == (unsigned)p.nsplit - 1u;
    if (*last_s) *cnt = 0u;                                          // re-arm for the next launch
  }
  asm volatile("bar.sync 3, 256;" ::: "memory");
  if (!*last_s) return;
  __threadfence();
  // two threads per row, 64 dims each
  const int row = t >> 1, c0 = (t & 1) * 64, qrow = it.q0 + row;
  if (qrow < p.T) {
    const float* base = p.part + th * p.nsplit * split_floats + (size_t)row * PART_ROW;
    float M = -INFINITY;
    for (int sp = 0; sp < p.nsplit; ++sp) M = fmaxf(M, __ldcg(base + sp * split_floats));
    float acc[64], L = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int sp = 0; sp < p.nsplit; ++sp) {
      const float* ph = base + sp * split_floats;
      const float ms = __ldcg(ph);
      const float c = ms == -INFINITY ? 0.f : exp2f(ms - M);
      L = fmaf(__ldcg(ph + 1), c, L);
#pragma unroll
      for (int i = 0; i < 64; i += 2) {
        const float2 v = __ldcg(reinterpret_cast<const float2*>(ph + 2 + c0 + i));
        acc[i] = fmaf(v.x, c, acc[i]);
        acc[i + 1] = fmaf(v.y, c, acc[i + 1]);
      }
    }
    __nv_bfloat16* orow = p.out + (size_t)qrow * ((size_t)p.n_heads * HD) + (size_t)it.head * HD + c0;
#pragma unroll
    for (int i = 0; i < 64; i += 2) *reinterpret_cast<uint32_t*>(orow + i) = pack_bf16(acc[i] / L, acc[i + 1] / L);
  }
}

template <bool LONG>
__global__ void __launch_bounds__(384, 1)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                       const __grid_constant__ CUtensorMap map_v, const AttnTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_s = base;                                  // [2 slabs][128 rows][128 B]
  uint8_t* ring = base + Q_BYTES;                       // [NRING][K lo | K hi | V lo | V hi]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)NRING * SLOT);
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 1;
  uint64_t* kv_full = bars + 2;                         // [NRING]
  uint64_t* kv_empty = kv_full + NRING;                 // [NRING]
  int* bt_s = reinterpret_cast<int*>(kv_empty + NRING); // [MAX_BT]; variant 2: bt_s[0] = "this split arrived last"

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (p.T + TQ - 1) / TQ;
  const int g_rep = p.n_heads / p.n_kv;

  if (threadIdx.x == 0) {
    prefetch_tmap(&map_q); prefetch_tmap(&map_k); prefetch_tmap(&map_v);
    mbar_init(q_full, 1); mbar_init(q_empty, 2);        // one arrival per consumer warpgroup
    for (int i = 0; i < NRING; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 2); }
    fence_barrier_init();
  }
  if (!LONG)
    for (int i = threadIdx.x; i < p.n_bt && i < MAX_BT; i += blockDim.x) bt_s[i] = p.block_table[i];
  __syncthreads();

  if (warp < 4) {
    // ======================================= TMA producer =======================================
    if (warp == 0 && lane == 0) {
      uint32_t ring_it = 0, nq = 0;
      Item it;
      for (int idx = blockIdx.x; get_item<LONG>(p, idx, n_tiles, &it); idx += gridDim.x, ++nq) {
        const int g = it.head / g_rep;
        mbar_wait(q_empty, (nq & 1u) ^ 1u);                        // both warpgroups are past the previous item's last S
        mbar_arrive_expect_tx(q_full, Q_BYTES);
        tma_load_2d(q_s, &map_q, it.head * HD, it.q0, q_full);
        tma_load_2d(q_s + Q_SLAB, &map_q, it.head * HD + 64, it.q0, q_full);
        for (int j = it.kb0; j < it.kb1; ++j, ++ring_it) {
          const int slot = (int)(ring_it % NRING);
          mbar_wait(&kv_empty[slot], ((ring_it / NRING) & 1u) ^ 1u);
          mbar_arrive_expect_tx(&kv_full[slot], SLOT);
          uint8_t* dst = ring + (size_t)slot * SLOT;
#pragma unroll
          for (int i = 0; i < TKV / PAGE; ++i) {
            int pi = j * (TKV / PAGE) + i;
            if (pi >= p.n_bt) pi = 0;                               // past the sequence: any valid page (its keys are masked)
            const long long row = p.layer_row0 + ((long long)(LONG ? __ldg(p.block_table + pi) : bt_s[pi]) * p.n_kv + g) * PAGE;
            uint8_t* d = dst + i * (PAGE * 128);
            tma_load_2d(d, &map_k, 0, (int)row, &kv_full[slot]);
            tma_load_2d(d + KV_SLAB, &map_k, 64, (int)row, &kv_full[slot]);
            tma_load_2d(d + KV_TILE, &map_v, 0, (int)row, &kv_full[slot]);
            tma_load_2d(d + KV_TILE + KV_SLAB, &map_v, 64, (int)row, &kv_full[slot]);
          }
        }
      }
    }
  } else {
    // ======================================= consumer warpgroups =======================================
    const int m0 = (warp >> 2) * 64 - 64;                          // rows m0 .. m0 + 63 of the item
    const int wq = warp & 3, rq = lane >> 2, cq = lane & 3;
    const bool leader = wq == 0 && lane == 0;
    const uint32_t qaddr = smem_u32(q_s) + (uint32_t)m0 * 128u;
    uint32_t ring_it = 0, nq = 0;
    Item it;
    for (int idx = blockIdx.x; get_item<LONG>(p, idx, n_tiles, &it); idx += gridDim.x, ++nq) {
      int qabs[2];                                                  // positions of this thread's two rows
#pragma unroll
      for (int h = 0; h < 2; ++h) qabs[h] = p.pos0 + it.q0 + m0 + wq * 16 + h * 8 + rq;
      float o[2][32];                                               // head-dim halves 0-63 | 64-127
#pragma unroll
      for (int i = 0; i < 32; ++i) { o[0][i] = 0.f; o[1][i] = 0.f; }
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      mbar_wait(q_full, nq & 1u);
      for (int j = it.kb0; j < it.kb1; ++j, ++ring_it) {
        const int slot = (int)(ring_it % NRING);
        mbar_wait(&kv_full[slot], (ring_it / NRING) & 1u);
        const uint32_t kaddr = smem_u32(ring + (size_t)slot * SLOT), vaddr = kaddr + KV_TILE;
        float s[32];
        fence_regs(s);
        fence();
#pragma unroll
        for (int k = 0; k < HD / UK; ++k) {
          const uint32_t off = (uint32_t)(k & 3) * 32u;           // 32 bytes per MMA K inside the 64-dim slab k / 4
          mma_ss<TKV>(s, make_desc(qaddr + (uint32_t)(k >> 2) * Q_SLAB + off), make_desc(kaddr + (uint32_t)(k >> 2) * KV_SLAB + off),
                      k ? 1u : 0u);
        }
        commit();
        wait<0>();
        fence_regs(s);
        if (j == it.kb1 - 1) {                                      // last S of the item: the Q tile may be replaced
          asm volatile("bar.sync %0, 128;" ::"r"(warp >> 2) : "memory");
          if (leader) mbar_arrive(q_empty);
        }
        // scaled, masked scores; block maximum per row (4 lanes share a row)
        const int k0 = j * TKV;
        float mb[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < TKV / 8; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int h = e >> 1, key = k0 + i * 8 + 2 * cq + (e & 1);
            const float v = key <= qabs[h] ? s[4 * i + e] * p.scale2 : -INFINITY;
            s[4 * i + e] = v;
            mb[h] = fmaxf(mb[h], v);
          }
        float corr[2], ref[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          mb[h] = fmaxf(mb[h], __shfl_xor_sync(0xffffffffu, mb[h], 1));
          mb[h] = fmaxf(mb[h], __shfl_xor_sync(0xffffffffu, mb[h], 2));
          const float mn = fmaxf(m_run[h], mb[h]);                  // variant 1: finite, block 0 holds key 0 <= every position
          // a later split's first blocks can lie past a row's position: its maximum stays -inf, and a finite reference
          // (0) keeps corr and p at 0 instead of NaN
          ref[h] = LONG && mn == -INFINITY ? 0.f : mn;
          corr[h] = ex2_approx(m_run[h] - ref[h]);
          m_run[h] = mn;
          l_run[h] *= corr[h];
        }
        // P = 2^(s - m) -> bf16 A fragments (16-token k-step kk = accumulator column groups 2 kk, 2 kk + 1)
        uint32_t pa[TKV / 16][4];
#pragma unroll
        for (int i = 0; i < TKV / 8; ++i) {
          const float p0 = ex2_approx(s[4 * i] - ref[0]), p1 = ex2_approx(s[4 * i + 1] - ref[0]);
          const float p2 = ex2_approx(s[4 * i + 2] - ref[1]), p3 = ex2_approx(s[4 * i + 3] - ref[1]);
          l_run[0] += p0 + p1;
          l_run[1] += p2 + p3;
          pa[i >> 1][(i & 1) * 2] = pack_bf16(p0, p1);
          pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16(p2, p3);
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float c = corr[(i >> 1) & 1];
          o[0][i] *= c;
          o[1][i] *= c;
        }
        fence_regs(o[0]);
        fence_regs(o[1]);
        fence();
#pragma unroll
        for (int kk = 0; kk < TKV / UK; ++kk)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            mma_rs_tb<64>(o[hh], pa[kk], make_desc(vaddr + (uint32_t)hh * KV_SLAB + (uint32_t)kk * (UK * 128u), KV_SLAB), 1u);
        commit();
        wait<0>();
        fence_regs(o[0]);
        fence_regs(o[1]);
        asm volatile("bar.sync %0, 128;" ::"r"(warp >> 2) : "memory");
        if (leader) mbar_arrive(&kv_empty[slot]);
      }
      // epilogue: O / l -> bf16 -> out[qrow][head * HD ..]
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
      }
      if (LONG && p.nsplit > 1) {
        split_epilogue(p, it, m0 + wq * 16 + rq, cq, o, m_run, l_run, bt_s);
        continue;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float inv = 1.0f / l_run[h];
        const int qrow = it.q0 + m0 + wq * 16 + h * 8 + rq;
        if (qrow < p.T) {
          __nv_bfloat16* orow = p.out + (size_t)qrow * ((size_t)p.n_heads * HD) + (size_t)it.head * HD;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int i = 0; i < 8; ++i)
              *reinterpret_cast<uint32_t*>(orow + hh * 64 + i * 8 + 2 * cq) =
                  pack_bf16(o[hh][4 * i + 2 * h] * inv, o[hh][4 * i + 2 * h + 1] * inv);
        }
      }
    }
  }
}

constexpr size_t kSmem = (size_t)Q_BYTES + (size_t)NRING * SLOT + (2 + 2 * NRING) * 8 + MAX_BT * 4 + 1024;

}  // namespace

bool attn_prefill_tc_supported(int n_heads, int n_kv, int head_dim, int page_size, int pos0, int T) {
  return attn_prefill_long_supported(n_heads, n_kv, head_dim, page_size) && T > 0 && (pos0 + T + PAGE - 1) / PAGE <= MAX_BT;
}

bool attn_prefill_long_supported(int n_heads, int n_kv, int head_dim, int page_size) {
  return head_dim == HD && page_size == PAGE && n_kv > 0 && n_heads % n_kv == 0;
}

// Split plan of variant 2, from the shape alone.  Splits are taken only while the unsplit items, n_tiles x n_heads, leave
// SMs idle; then the count that minimises the waves of equal-sized items per split (ceil(items x s / sms) / s, the smaller
// s on a tie) among those that keep
//   - every split at >= kAttnLongMinSplitBlocks KV blocks of the lightest tile: a split's partial (128 rows x 130 fp32,
//     66.5 KB written once and read once by the combine) stays under 7 % of the 1 MB of K/V it streams, and
//   - items x s <= 2 x sms: the workspace bound attn_prefill_long_part_floats.
// force > 0 asks for that count instead, clamped to 1 .. the lightest tile's block count (every split non-empty).
int attn_prefill_long_splits(int pos0, int T, int n_heads, int sms, int force) {
  if (T <= 0 || pos0 < 0 || n_heads <= 0 || sms <= 0) return 1;
  const int items = ((T + TQ - 1) / TQ) * n_heads;
  const int nblk_min = (pos0 + std::min(TQ, T) - 1) / TKV + 1;
  if (force > 0) return std::min(force, nblk_min);
  if (items >= sms) return 1;
  const int cap = std::max(1, std::min(2 * sms / items, nblk_min / kAttnLongMinSplitBlocks));
  int best = 1;
  long long best_waves = ((long long)items + sms - 1) / sms;
  for (int s = 2; s <= cap; ++s) {
    const long long waves = ((long long)items * s + sms - 1) / sms;
    if (waves * best < best_waves * s) { best = s; best_waves = waves; }
  }
  return best;
}

size_t attn_prefill_long_part_floats(int sms) { return (size_t)2 * sms * TQ * PART_ROW; }
size_t attn_prefill_long_counters(int sms) { return (size_t)sms; }

namespace {

template <bool LONG>
int launch_tc(const AttnPrefillArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, int nsplit, float* part,
              unsigned* counters, cudaStream_t st) {
  CUtensorMap qmap;
  if (!make_tmap_2d_bf16(&qmap, a.q, (uint64_t)a.T, (uint64_t)a.n_heads * HD, 64, TQ)) return -1;
  static PerDeviceOnce attr;
  if (attr.pending()) {
    if (cudaFuncSetAttribute(attn_prefill_tc_kernel<LONG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem) != cudaSuccess) return -1;
    attr.mark();
  }
  AttnTcParams p;
  p.block_table = a.block_table; p.n_bt = (a.pos0 + a.T + PAGE - 1) / PAGE; p.pos0 = a.pos0; p.T = a.T; p.n_heads = a.n_heads; p.n_kv = a.n_kv;
  p.layer_row0 = layer_row0; p.out = a.out; p.scale2 = 1.4426950408889634f / sqrtf((float)HD);
  p.nsplit = nsplit; p.part = part; p.counters = counters;
  const int items = ((a.T + TQ - 1) / TQ) * a.n_heads * nsplit;
  const int grid = items < sm_count() ? items : sm_count();
  attn_prefill_tc_kernel<LONG><<<grid, 384, kSmem, st>>>(qmap, kmap, vmap, p);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace

// q: [T][n_heads*128] bf16 (roped); K / V through the pool-wide tensor maps (box {64, 32}, 128B swizzle);
// layer_row0 = first row of this layer in those maps
int launch_attn_prefill_tc(const AttnPrefillArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st) {
  if (!attn_prefill_tc_supported(a.n_heads, a.n_kv, a.head_dim, a.page_size, a.pos0, a.T)) return -1;
  return launch_tc<false>(a, kmap, vmap, layer_row0, 1, nullptr, nullptr, st);
}

int launch_attn_prefill_long(const AttnPrefillArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, int nsplit,
                             float* part, unsigned* counters, cudaStream_t st) {
  if (!attn_prefill_long_supported(a.n_heads, a.n_kv, a.head_dim, a.page_size) || a.T <= 0 || a.pos0 < 0 || nsplit < 1 ||
      nsplit > (a.pos0 + std::min(TQ, a.T) - 1) / TKV + 1 || (nsplit > 1 && (!part || !counters)))
    return -1;
  return launch_tc<true>(a, kmap, vmap, layer_row0, nsplit, part, counters, st);
}

}  // namespace cl
