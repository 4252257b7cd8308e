// decode_mega_batch.cu — one BATCHED decode step (B = 2..32 sequences) of the whole transformer stack as a single
// persistent kernel: the continuous-batching inner loop of the worker (scheduler.cpp) without ~10 kernel launches per
// layer.  Same idea as decode_mega.cu (B = 1), with the projections on the tensor cores (wgmma):
//
//   grid = one CTA per SM, 352 threads: warp 0 = TMA producer of W / KV tiles, warp 10 = TMA producer of the token operand,
//   warps 2-9 = consumers (paged tensor-core attention; per-token reductions); consumer warps 4-7 form warpgroup 1, which
//   also runs the projections' MMAs and writes their fp32 split-K partials (warp 1 is idle).
//   Projections are Y[n][b] = sum_k W[n][k] X[b][k] with W tile [128 rows x 64 k] = MMA A (16 KB, 2-D TMA, 128B
//   swizzle, two m64 halves), the B <= 32 token columns [32 x 64 k] = MMA B (4 KB), accumulators in registers.
//   Every projection is cut into (row tile, k split) units — split counts from the engine's pick_splits — so that all
//   SMs stream weights; fp32 partials go to a workspace and are folded in FIXED order by the next phase
//   (deterministic run to run).
//   The producer streams W k-blocks, this CTA's KV pages and again W k-blocks through ONE ring of 16 KB slots in
//   program order and never waits for activations with W: at a phase boundary it first primes the ring with the next
//   projection's weights and only then waits for the grid barrier that publishes the token operand (X tiles travel in
//   a small ring of their own).  HBM therefore keeps streaming while the consumers sit in barriers and reductions.
//
// Phases per layer (grid barriers between them; counters zeroed by the step tail):
//   R0  h_b += sum_s down-partials(prev layer); xn_b = bf16(rmsnorm(h_b) g)            token b on CTA b
//   G0  q|k|v partials                                                               all CTAs, split-K
//   AT  attention unit (b, kv head, split): q / k / v from the partials (+RoPE, K/V append into the paged cache),
//       mma.sync m16n8k16 over TMA-swizzled pages (P = hi + lo bf16), the last split to finish combines -> bf16 attn_b
//   G1  o partials   R1  h_b += ..., xn_b = norm   G2  gate|up partials   R2  act = bf16(SiLU(g) u)   G3  down partials
// then the final norm; the LM head follows as a separate GEMM launch (gemm_wgmma.cu).
// Built for the Llama-3-8B / Mistral-7B layer shape (d 4096, d_ff 14336, head_dim 128, 4 q heads per kv head, page 32).
#include <cuda.h>

#include <cstdlib>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace cl {

namespace {

using namespace wg;

constexpr int D = 4096, F = 14336, HD = 128, REP = 4, P = 32, HALF = HD / 2;
constexpr int BT = 32;                       // token columns (MMA N)
constexpr int NSW = 6;                       // W / KV ring slots of 16 KB (at most max_flight of them in flight)
constexpr uint32_t WSLOT = 16384;
constexpr int NSX = 25;                      // resident X tiles of 4 KB: the k range of one split (<= 25 k-blocks)
constexpr uint32_t XSLOT = 4096;
constexpr int NC = 8;                        // consumer warps
constexpr int MAXS = 32;                     // max KV splits per (sequence, kv head)
constexpr float LOG2E = 1.4426950408889634f;

struct Proj {                                // one projection of one layer
  const CUtensorMap* wmap;                   // device-resident tensor map of W [N][K], box {64, 128}
  int N, K, S;                               // rows, depth, k splits
};

__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// grid-wide barrier among the consumer warps of all CTAs (producer / MMA warps do not take part)
// pause: while this CTA's consumers sit in the barrier its producer issues no new bulk copy — the barrier's red / poll round
// trips queue behind bulk traffic in front of the L2 slices (tools/bench_barrier.cu)
// pause[1] counts the barriers this CTA has left: its producer waits for "barrier n passed" on that shared-memory word
// instead of adding one more poller per SM to the global counter.
__device__ __forceinline__ void grid_barrier(unsigned* cnt, int ctid, volatile int* pause) {
  bar_consumers();
  if (ctid == 0) {
    pause[0] = 1;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(cnt) : "memory");
    const long long t0 = clock64();
    while (ld_acquire_u32(cnt) < gridDim.x) {
      if (clock64() - t0 > (1ll << 31)) __trap();
    }
    pause[0] = 0;
    __threadfence_block();
    pause[1] = pause[1] + 1;
  }
  bar_consumers();
}
// producer thread: has this CTA's consumer side left its n-th grid barrier (counted in shared memory)?  Then one acquire
// load of the global counter (already complete) orders the other CTAs' writes before this thread's TMA loads.
__device__ __forceinline__ void wait_counter(const unsigned* cnt, volatile int* done, int n) {
  const long long t0 = clock64();
  while (*done < n) {
    if (clock64() - t0 > (1ll << 31)) __trap();
  }
  while (ld_acquire_u32(cnt) < gridDim.x) {
    if (clock64() - t0 > (1ll << 31)) __trap();
  }
}

// attention work of this step: unit u = ((b * n_kv) + g) * nsplit + sp, u = blockIdx.x, blockIdx.x + gridDim.x, ...
struct AttUnit { int b, g, sp, slot, pos, pg0, pg1, owner; };
__device__ __forceinline__ bool att_unit(const BatchMegaArgs& a, int u, AttUnit* o) {
  if (u >= a.B * a.n_kv * a.nsplit) return false;
  o->sp = u % a.nsplit;
  const int bg = u / a.nsplit;
  o->g = bg % a.n_kv;
  o->b = bg / a.n_kv;
  o->slot = a.slots[o->b];
  o->pos = a.pos[o->slot];
  const int total = o->pos / P + 1;                          // pages holding tokens 0..pos
  const int pps = (total + a.nsplit - 1) / a.nsplit;
  o->pg0 = o->sp * pps;
  o->pg1 = min(total, o->pg0 + pps);
  if (o->pg1 < o->pg0) o->pg1 = o->pg0;
  o->owner = (o->pos / P) / pps;                             // the split whose range holds the current token's page
  return true;
}

// GEMM work of one projection: (row tile, k split) units.  A CTA keeps ONE split for the whole phase (ks = blockIdx.x mod S),
// so the token operand of that split (<= 25 tiles of [32 x 64 k]) is loaded once and stays resident in shared memory for
// all of the CTA's row tiles; row tiles go round-robin over the CTAs that share the split.
struct GemmPlan { int RT, nkb, kbp, ks, kb0, nk, m, M; };
__device__ __forceinline__ GemmPlan gemm_plan(const Proj& pr) {
  GemmPlan g;
  g.RT = (pr.N + BM - 1) / BM;
  g.nkb = pr.K / BK;
  g.kbp = (g.nkb + pr.S - 1) / pr.S;
  g.ks = (int)blockIdx.x % pr.S;
  g.m = (int)blockIdx.x / pr.S;
  g.M = ((int)gridDim.x - g.ks + pr.S - 1) / pr.S;                 // CTAs that work on split ks
  g.kb0 = g.ks * g.kbp;
  g.nk = max(0, min(g.nkb, g.kb0 + g.kbp) - g.kb0);
  return g;
}

__global__ void __launch_bounds__(352, 1) decode_mega_batch_kernel(const __grid_constant__ BatchMegaArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* wring = base;                                            // [NSW][16 KB]
  uint8_t* xres = base + (size_t)NSW * WSLOT;                       // [NSX][4 KB] resident token operand of this CTA's split
  uint64_t* bars = reinterpret_cast<uint64_t*>(xres + (size_t)NSX * XSLOT);
  uint64_t* w_full = bars;                   // [NSW]
  uint64_t* w_empty = w_full + NSW;          // [NSW]
  uint64_t* x_full = w_empty + NSW;          // [NSX]  tile i of this GEMM phase's token operand has landed
  uint64_t* kv_ready = x_full + NSX;         // [1]  consumers -> producer: the current token's K/V rows are in the cache
  float* red_m = reinterpret_cast<float*>(kv_ready + 1);     // [NC][REP]
  float* red_l = red_m + NC * REP;                           // [NC][REP]
  float* red_acc = red_l + NC * REP;                         // [NC][REP][HD]
  float* qs = red_acc + NC * REP * HD;                       // [REP][HD]   roped, bf16-rounded query of the unit
  float* cm_s = qs + REP * HD;                               // [MAXS][REP]
  float* cw_s = cm_s + MAXS * REP;                           // [MAXS][REP]
  float* cL_s = cw_s + MAXS * REP;                           // [REP]
  float* ssw = cL_s + REP;                                   // [NC]
  int* flag_s = reinterpret_cast<int*>(ssw + NC);
  volatile int* pause_s = flag_s + 1;                        // consumers are inside a grid barrier

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = (int)gridDim.x;
  if (threadIdx.x == 0) {
    for (int i = 0; i < NSW; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 1); }
    for (int i = 0; i < NSX; ++i) mbar_init(&x_full[i], 1);
    mbar_init(kv_ready, 1);
    pause_s[0] = 0; pause_s[1] = 0;
    fence_barrier_init();
  }
  __syncthreads();

  // the four projections of layer l, then the LM head (l == n_layers, j == 0)
  auto proj = [&](int l, int j) -> Proj {
    if (l == a.n_layers) return Proj{a.wmaps + (size_t)a.n_layers * 4, a.vocab, D, 1};
    const CUtensorMap* m = a.wmaps + (size_t)l * 4 + j;
    switch (j) {
      case 0: return Proj{m, a.qkv_dim, D, a.s_qkv};
      case 1: return Proj{m, D, a.q_dim, a.s_o};
      case 2: return Proj{m, 2 * F, D, a.s_gu};
      default: return Proj{m, D, F, a.s_dn};
    }
  };
  // grid barrier that publishes the token operand of projection j of layer l (see the phase list in the header)
  auto xready = [&](int l, int j) -> const unsigned* {
    if (l == a.n_layers) return a.bars + (size_t)a.n_layers * 8;
    return a.bars + (size_t)l * 8 + 2 * j;           // j = 0: after R0, 1: after AT, 2: after R1, 3: after R2
  };
  auto xmap = [&](int l, int j) -> const CUtensorMap* { return (l == a.n_layers || j == 0 || j == 2) ? &a.map_xn : j == 1 ? &a.map_attn : &a.map_act; };
  // pages this CTA's attention units stream in one layer (identical in every layer)
  int att_pages = 0;
  {
    AttUnit u;
    for (int i = blockIdx.x; att_unit(a, i, &u); i += G) att_pages += u.pg1 - u.pg0;
  }

  if (warp == 0) {
    // =============================================== producer ===============================================
    if (lane == 0) {
    prefetch_tmap(&a.map_xn); prefetch_tmap(&a.map_attn); prefetch_tmap(&a.map_act); prefetch_tmap(&a.kmap); prefetch_tmap(&a.vmap);
    uint32_t wit = 0, att_n = 0;                    // ring items issued; attention units issued (kv_ready phases)
    uint32_t wtail = 0;                             // oldest ring item not yet known to have landed
    long long c_empty = 0, c_flight = 0, c_kv = 0;   // diagnostics: cycles blocked (CL_TIMELINE)
    const long long c_start = clock64();
    const int max_flight = a.max_flight > 0 ? a.max_flight : NSW;
    // a free slot, at most max_flight 16 KB copies in flight (the ring still fills all NSW slots over time), and no new
    // copy while the consumers are inside a grid barrier
    auto w_acquire = [&]() -> int {
      const int s = (int)(wit % NSW);
      long long t0 = clock64();
      mbar_wait(&w_empty[s], ((wit / NSW) & 1u) ^ 1u);
      long long t1 = clock64();
      c_empty += t1 - t0;
      for (uint32_t spins = 0; (int)(wit - wtail) >= max_flight; ++spins) {
        if (mbar_try_wait(&w_full[wtail % NSW], (wtail / NSW) & 1u)) ++wtail;
        if (spins > (1u << 24)) __trap();
      }
      if (a.pause_in_barrier)
        for (uint32_t spins = 0; *pause_s; ++spins) if (spins > (1u << 26)) __trap();
      c_flight += clock64() - t1;
      return s;
    };
    // W k-blocks of this CTA's units of projection j of layer l, in unit order.  No dependency on activations: the
    // weight stream runs ahead of the phases by the depth of the ring (the token operand has its own producer, warp 10).
    auto gemm_items = [&](int l, int j) {
      const Proj pr = proj(l, j);
      const GemmPlan g = gemm_plan(pr);
      for (int rt = g.m; rt < g.RT && g.nk > 0; rt += g.M)
        for (int kb = g.kb0; kb < g.kb0 + g.nk; ++kb) {
          const int s = w_acquire();
          mbar_arrive_expect_tx(&w_full[s], WSLOT);
          tma_load_2d(wring + (size_t)s * WSLOT, pr.wmap, kb * BK, rt * BM, &w_full[s]);
          ++wit;
        }
    };
    for (int l = 0; l < a.n_layers; ++l) {
      gemm_items(l, 0);
      // ---- attention pages of this CTA's units: one page (K lo|hi, V lo|hi = 16 KB) per ring slot
      AttUnit u;
      for (int i = blockIdx.x; att_unit(a, i, &u); i += G, ++att_n) {
        const int* bt = a.block_tables + (size_t)u.slot * a.bt_stride;
        const int cur = u.pos / P;
        for (int pg = u.pg0; pg < u.pg1; ++pg) {
          const int s = w_acquire();
          if (pg == cur) {                          // this page receives the current token's K/V from THIS unit's prologue
            const long long t0 = clock64();
            mbar_wait(kv_ready, att_n & 1u);
            c_kv += clock64() - t0;
            fence_proxy_async_all();
          }
          const long long row = (long long)l * a.kv_layer_rows + ((long long)bt[pg] * a.n_kv + u.g) * P;
          uint8_t* d = wring + (size_t)s * WSLOT;
          mbar_arrive_expect_tx(&w_full[s], WSLOT);
          tma_load_2d(d, &a.kmap, 0, (int)row, &w_full[s]);
          tma_load_2d(d + 4096, &a.kmap, 64, (int)row, &w_full[s]);
          tma_load_2d(d + 8192, &a.vmap, 0, (int)row, &w_full[s]);
          tma_load_2d(d + 12288, &a.vmap, 64, (int)row, &w_full[s]);
          ++wit;
        }
        if (u.sp != u.owner) {                      // units that do not own the current page never wait: keep the phases aligned
          mbar_wait(kv_ready, att_n & 1u);
        }
      }
      gemm_items(l, 1);
      gemm_items(l, 2);
      gemm_items(l, 3);
    }
    if (a.tl != nullptr && blockIdx.x == 0) {
      long long* dbg = a.tl + (size_t)a.n_layers * 16;
      dbg[0] = clock64() - c_start; dbg[1] = c_empty; dbg[2] = c_flight; dbg[5] = c_kv;
    }
    }
  } else if (warp == 10) {
    // =============================================== X producer ===============================================
    // token-operand tiles [32 x 64 k] (4 KB, L2-resident) of every GEMM k-block, gated only by the grid barrier that
    // publishes the operand
    if (lane == 0) {
      uint32_t gp = 0;                             // GEMM phases so far: every x_full barrier completes once per phase
      long long c_xempty = 0, c_phase = 0;
      auto x_items = [&](int l, int j) {
        const Proj pr = proj(l, j);
        const GemmPlan g = gemm_plan(pr);
        const CUtensorMap* xm = xmap(l, j);
        { const long long t0 = clock64(); wait_counter(xready(l, j), pause_s + 1, l * 8 + 2 * j + 1); c_phase += clock64() - t0; }
        fence_proxy_async_all();                     // X was written with generic-proxy stores by other CTAs
        // The previous phase's MMAs are long complete: this operand only exists after grid barriers that follow them.
        const bool work = g.m < g.RT && g.nk > 0;
        for (int i = 0; i < NSX; ++i) {
          if (work && i < g.nk) {
            mbar_arrive_expect_tx(&x_full[i], XSLOT);
            tma_load_2d(xres + (size_t)i * XSLOT, xm, (g.kb0 + i) * BK, 0, &x_full[i]);
          } else {
            mbar_arrive(&x_full[i]);                 // unused tile: complete the phase so that parities stay aligned
          }
        }
        ++gp;
      };
      for (int l = 0; l < a.n_layers; ++l)
        for (int j = 0; j < 4; ++j) x_items(l, j);
      if (a.tl != nullptr && blockIdx.x == 0) {
        long long* dbg = a.tl + (size_t)a.n_layers * 16;
        dbg[3] = c_xempty; dbg[4] = c_phase;
      }
    }
  } else if (warp >= 2 && warp < 2 + NC) {
    // =============================================== consumers ===============================================
    const int cw = warp - 2, ctid = cw * 32 + lane;          // consumer warp 0..7, consumer thread 0..255
    uint32_t wit = 0, att_n = 0, gp = 0;                     // ring items consumed; attention units; GEMM phases
    // ---- projections: warpgroup 1 (warps 4-7) runs the MMAs of this CTA's units and writes the split-K partials
    // partial[ks][b][n] fp32 (LM head: the logits); the other consumer warps only keep the ring count
    auto gemm_units = [&](int l, int j) {
      const Proj pr = proj(l, j);
      const GemmPlan g = gemm_plan(pr);
      const bool mma = warp >= 4 && warp < 8;
      const int wq = warp & 3, rq = lane >> 2, cq = lane & 3;
      bool first = true;                            // the X tiles are waited for once, by the phase's first unit
      for (int rt = g.m; rt < g.RT && g.nk > 0; rt += g.M) {
        if (!mma) { wit += (uint32_t)g.nk; continue; }
        float acc[2][BT / 2];                       // W rows 0-63 | 64-127 of the tile
#pragma unroll
        for (int i = 0; i < BT / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
        int prev = -1;
        for (int kb = 0; kb < g.nk; ++kb, ++wit) {
          const int s = (int)(wit % NSW);
          mbar_wait(&w_full[s], (wit / NSW) & 1u);
          if (first) mbar_wait(&x_full[kb], gp & 1u);
          const uint32_t wa = smem_u32(wring + (size_t)s * WSLOT), xa = smem_u32(xres + (size_t)kb * XSLOT);
          fence_regs(acc[0]); fence_regs(acc[1]);
          fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
              mma_ss<BT>(acc[hf], make_desc(wa + (uint32_t)hf * 8192u + (uint32_t)k * 32u), make_desc(xa + (uint32_t)k * 32u), 1u);
          commit();
          wait<1>();                                // the previous k-block's MMAs are done: release its slot
          fence_regs(acc[0]); fence_regs(acc[1]);
          if (prev >= 0 && ctid == 64) mbar_arrive(&w_empty[prev]);
          prev = s;
        }
        wait<0>();
        fence_regs(acc[0]); fence_regs(acc[1]);
        if (prev >= 0 && ctid == 64) mbar_arrive(&w_empty[prev]);
        first = false;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int n = rt * BM + hf * 64 + wq * 16 + h * 8 + rq;
            if (n >= pr.N) continue;
#pragma unroll
            for (int i = 0; i < BT / 8; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int b = i * 8 + 2 * cq + e;
                if (b >= a.B) continue;
                const float v = acc[hf][4 * i + 2 * h + e];
                if (l == a.n_layers) a.logits[(size_t)a.slots[b] * a.vocab + n] = v;     // LM head: logits[slot][n]
                else a.part[((size_t)g.ks * BT + b) * pr.N + n] = v;
              }
          }
      }
      // observe EVERY x_full barrier in EVERY phase (tiles beyond this split's range, or all of them when this CTA has no
      // unit in the phase): a warp that skipped a phase of a barrier would pass its next wait on stale parity
      if (mma)
        for (int i = first ? 0 : g.nk; i < NSX; ++i) mbar_wait(&x_full[i], gp & 1u);
      ++gp;
    };
    // ---- h_b += sum_s partial[s][b][:] (fixed order; n_split == 0: nothing to add); xn_b = bf16(rmsnorm(h_b) * gain)
    auto resid_norm = [&](const float* gain, int n_split) {
      for (int b = blockIdx.x; b < a.B; b += G) {
        float* hr = a.h + (size_t)a.slots[b] * D;
        float4 v[4];
        float ss = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) v[r] = *reinterpret_cast<const float4*>(hr + (ctid + r * 256) * 4);
        // partials in groups of 4 splits: 16 independent loads in flight per thread, added in fixed order
        for (int s0 = 0; s0 < n_split; s0 += 4) {
          float4 y[4][4];
#pragma unroll
          for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int r = 0; r < 4; ++r)
              y[s][r] = s0 + s < n_split ? __ldcg(reinterpret_cast<const float4*>(a.part + ((size_t)(s0 + s) * BT + b) * D + (ctid + r * 256) * 4))
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int r = 0; r < 4; ++r) { v[r].x += y[s][r].x; v[r].y += y[s][r].y; v[r].z += y[s][r].z; v[r].w += y[s][r].w; }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          if (n_split > 0) *reinterpret_cast<float4*>(hr + (ctid + r * 256) * 4) = v[r];
          ss = fmaf(v[r].x, v[r].x, ss); ss = fmaf(v[r].y, v[r].y, ss); ss = fmaf(v[r].z, v[r].z, ss); ss = fmaf(v[r].w, v[r].w, ss);
        }
        ss = warp_sum(ss);
        if (lane == 0) ssw[cw] = ss;
        bar_consumers();
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < NC; ++w) tot += ssw[w];
        const float inv = 1.0f / sqrtf(tot / (float)D + a.eps);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = (ctid + r * 256) * 4;
          const float4 g = *reinterpret_cast<const float4*>(gain + i);
          uint2 pk;
          pk.x = pack_bf16(v[r].x * inv * g.x, v[r].y * inv * g.y);
          pk.y = pack_bf16(v[r].z * inv * g.z, v[r].w * inv * g.w);
          *reinterpret_cast<uint2*>(a.xn + (size_t)b * D + i) = pk;
        }
        bar_consumers();                             // ssw is reused by the next token of this CTA
      }
    };

    const bool stamp = a.tl != nullptr && blockIdx.x == 0 && ctid == 0;
#define CL_STAMP(k) do { if (stamp) a.tl[(size_t)l * 16 + (k)] = gtime_ns(); } while (0)
    for (int l = 0; l < a.n_layers; ++l) {
      const BatchMegaLayer& L = a.layers[l];
      unsigned* bars_l = a.bars + (size_t)l * 8;
      // ------------------------------------------------------------------ R0
      if (l > 0) grid_barrier(a.bars + (size_t)(l - 1) * 8 + 7, ctid, pause_s);      // previous layer's down partials complete
      CL_STAMP(15);
      resid_norm(L.attn_norm, l > 0 ? a.s_dn : 0);
      CL_STAMP(0);
      grid_barrier(bars_l + 0, ctid, pause_s);
      CL_STAMP(1);
      // ------------------------------------------------------------------ G0: q|k|v partials
      gemm_units(l, 0);
      CL_STAMP(2);
      grid_barrier(bars_l + 1, ctid, pause_s);
      CL_STAMP(3);
      // ------------------------------------------------------------------ AT
      {
        AttUnit u;
        for (int ui = blockIdx.x; att_unit(a, ui, &u); ui += G, ++att_n) {
          const int ctx = u.pos + 1;
          const int* bt = a.block_tables + (size_t)u.slot * a.bt_stride;
          // prologue: q of the 4 heads (and, in the owner split, k / v of the current token) from the q|k|v partials
          {
            const int hh = ctid >> 6, j = ctid & 63;                        // 256 threads = 4 heads x 64 rotation pairs
            const float2 cs = __ldg(a.rope + (size_t)u.pos * HALF + j);
            const int col = (u.g * REP + hh) * HD + 2 * j;
            float v0 = 0.f, v1 = 0.f;
            for (int s = 0; s < a.s_qkv; ++s) {
              const float2 y = __ldcg(reinterpret_cast<const float2*>(a.part + ((size_t)s * BT + u.b) * a.qkv_dim + col));
              v0 += y.x; v1 += y.y;
            }
            qs[hh * HD + j] = bf16_round(v0 * cs.x - v1 * cs.y);
            qs[hh * HD + j + HALF] = bf16_round(v1 * cs.x + v0 * cs.y);
            if (u.sp == u.owner && ctid < 128) {
              const bool isk = ctid < 64;
              const int jj = ctid & 63;
              const int c2 = a.q_dim + (isk ? 0 : a.n_kv * HD) + u.g * HD + 2 * jj;
              float w0 = 0.f, w1 = 0.f;
              for (int s = 0; s < a.s_qkv; ++s) {
                const float2 y = __ldcg(reinterpret_cast<const float2*>(a.part + ((size_t)s * BT + u.b) * a.qkv_dim + c2));
                w0 += y.x; w1 += y.y;
              }
              const float2 c = __ldg(a.rope + (size_t)u.pos * HALF + jj);
              const size_t dst = (((size_t)bt[u.pos / P] * a.n_kv + u.g) * P + (u.pos % P)) * HD;
              __nv_bfloat16* pool = isk ? L.kpool : L.vpool;
              pool[dst + jj] = __float2bfloat16_rn(isk ? w0 * c.x - w1 * c.y : w0);
              pool[dst + jj + HALF] = __float2bfloat16_rn(isk ? w1 * c.x + w0 * c.y : w1);
            }
          }
          __threadfence();
          bar_consumers();
          if (ctid == 0) { fence_proxy_async_all(); mbar_arrive(kv_ready); }   // the producer may load the current page now
          // Q fragments: heads in rows 0..3 of the m16n8k16 A tile
          const int rq = lane >> 2, cq = lane & 3;
          uint32_t qf[HD / 16][4];
#pragma unroll
          for (int kk = 0; kk < HD / 16; ++kk) {
            qf[kk][1] = 0u; qf[kk][3] = 0u;
            if (rq < REP) {
              qf[kk][0] = pack_bf16(qs[rq * HD + kk * 16 + 2 * cq], qs[rq * HD + kk * 16 + 2 * cq + 1]);
              qf[kk][2] = pack_bf16(qs[rq * HD + kk * 16 + 8 + 2 * cq], qs[rq * HD + kk * 16 + 8 + 2 * cq + 1]);
            } else {
              qf[kk][0] = 0u; qf[kk][2] = 0u;
            }
          }
          const float scale2 = rsqrtf((float)HD) * LOG2E;
          float o[HD / 8][4];
#pragma unroll
          for (int i = 0; i < HD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
          float mrow = -INFINITY, lrow = 0.f;
          const int npg = u.pg1 - u.pg0;
          for (int it = 0; it < npg; ++it, ++wit) {
            // EVERY warp observes every page's barrier in ring order (a waiter that skipped a phase of the same slot
            // would see "parity differs" for a page that has not landed: mbarrier waits are only safe one phase at a
            // time); only the owner warp (round robin) touches the data and frees the slot
            const int s = (int)(wit % NSW);
            mbar_wait(&w_full[s], (wit / NSW) & 1u);
            if ((it & (NC - 1)) != cw) continue;
            {
              const uint32_t kb = smem_u32(wring + (size_t)s * WSLOT), vb = kb + 8192;
              const int tok0 = (u.pg0 + it) * P;
              float sacc[4][4];
#pragma unroll
              for (int nj = 0; nj < 4; ++nj) { sacc[nj][0] = sacc[nj][1] = sacc[nj][2] = sacc[nj][3] = 0.f; }
              const int id = lane >> 3;
#pragma unroll
              for (int kk = 0; kk < HD / 16; ++kk) {
                const uint32_t kh = kb + (kk >> 2) * 4096;
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
                  const float vv = tok < ctx ? sacc[nj][e] * scale2 : -INFINITY;
                  sacc[nj][e] = vv;
                  mx = fmaxf(mx, vv);
                }
              }
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
              const float mn = fmaxf(mrow, mx);       // finite: every page of a split holds >= 1 valid token
              const float corr = exp2f(mrow - mn);
              mrow = mn;
              float rs = 0.f;
              uint32_t pf[2][4], pl[2][4];            // P = hi + lo bf16 terms (DESIGN.md §2)
#pragma unroll
              for (int nj = 0; nj < 4; ++nj) {
                const float p0 = exp2f(sacc[nj][0] - mn), p1 = exp2f(sacc[nj][1] - mn);
                rs += p0 + p1;
                const float h0 = bf16_round(p0), h1 = bf16_round(p1);
                pf[nj >> 1][(nj & 1) * 2] = pack_bf16(h0, h1);
                pf[nj >> 1][(nj & 1) * 2 + 1] = 0u;
                pl[nj >> 1][(nj & 1) * 2] = pack_bf16(p0 - h0, p1 - h1);
                pl[nj >> 1][(nj & 1) * 2 + 1] = 0u;
              }
              lrow = lrow * corr + rs;
#pragma unroll
              for (int nd = 0; nd < HD / 8; ++nd) { o[nd][0] *= corr; o[nd][1] *= corr; }
#pragma unroll
              for (int jj = 0; jj < 2; ++jj) {
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
            if (lane == 0) mbar_arrive(&w_empty[s]);
          }
          lrow += __shfl_xor_sync(0xffffffffu, lrow, 1);
          lrow += __shfl_xor_sync(0xffffffffu, lrow, 2);
          if (rq < REP) {
            if (cq == 0) { red_m[cw * REP + rq] = mrow; red_l[cw * REP + rq] = lrow; }
#pragma unroll
            for (int nd = 0; nd < HD / 8; ++nd) {
              red_acc[(cw * REP + rq) * HD + nd * 8 + 2 * cq] = o[nd][0];
              red_acc[(cw * REP + rq) * HD + nd * 8 + 2 * cq + 1] = o[nd][1];
            }
          }
          bar_consumers();
          // merge of the 8 warps -> bf16 output (one split) or the split partial
          float* part = a.att_part + ((((size_t)u.slot * a.n_kv + u.g) * a.nsplit + u.sp) * REP) * (HD + 2);
          __nv_bfloat16* outb = a.attn + (size_t)u.b * a.q_dim + (size_t)u.g * REP * HD;
          for (int e = ctid; e < REP * HD; e += 256) {
            const int hh = e / HD, i = e % HD;
            float M = -INFINITY;
#pragma unroll
            for (int w = 0; w < NC; ++w) M = fmaxf(M, red_m[w * REP + hh]);
            float Ls = 0.f, A = 0.f;
#pragma unroll
            for (int w = 0; w < NC; ++w) {
              const float mw = red_m[w * REP + hh];
              const float c = (mw == -INFINITY) ? 0.f : exp2f(mw - M);
              Ls = fmaf(red_l[w * REP + hh], c, Ls);
              A = fmaf(red_acc[(w * REP + hh) * HD + i], c, A);
            }
            if (a.nsplit == 1) {
              outb[hh * HD + i] = __float2bfloat16_rn(A / Ls);
            } else {
              float* ph = part + (size_t)hh * (HD + 2);
              if (i == 0) { ph[0] = M; ph[1] = Ls; }
              ph[2 + i] = A;
            }
          }
          if (a.nsplit > 1) {
            __threadfence();
            bar_consumers();
            if (ctid == 0) {
              unsigned* cnt = a.att_cnt + (size_t)u.slot * a.n_kv + u.g;
              const unsigned old = atomicAdd(cnt, 1u);
              *flag_s = (old == (unsigned)a.nsplit - 1u);
              if (*flag_s) *cnt = 0u;                 // re-armed for the next layer / step
            }
            bar_consumers();
            if (*flag_s) {                            // the last split to finish combines (fixed split order)
              __threadfence();
              const float* pall = a.att_part + (((size_t)u.slot * a.n_kv + u.g) * a.nsplit) * REP * (HD + 2);
              const int ns = a.nsplit;
              for (int e = ctid; e < ns * REP; e += 256) {
                const int sidx = e / REP, hh = e % REP;
                const float* ph = pall + ((size_t)sidx * REP + hh) * (HD + 2);
                cm_s[sidx * REP + hh] = __ldcg(ph);
                cw_s[sidx * REP + hh] = __ldcg(ph + 1);
              }
              bar_consumers();
              if (ctid < REP) {
                float M = -INFINITY;
                for (int sidx = 0; sidx < ns; ++sidx) M = fmaxf(M, cm_s[sidx * REP + ctid]);
                float Ls = 0.f;
                for (int sidx = 0; sidx < ns; ++sidx) {
                  const float ms = cm_s[sidx * REP + ctid];
                  const float c = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
                  Ls = fmaf(cw_s[sidx * REP + ctid], c, Ls);
                  cw_s[sidx * REP + ctid] = c;
                }
                cL_s[ctid] = Ls;
              }
              bar_consumers();
              for (int e = ctid; e < REP * HD; e += 256) {
                const int hh = e / HD, i = e % HD;
                float A = 0.f;
                for (int sidx = 0; sidx < ns; ++sidx)
                  A = fmaf(__ldcg(pall + ((size_t)sidx * REP + hh) * (HD + 2) + 2 + i), cw_s[sidx * REP + hh], A);
                outb[hh * HD + i] = __float2bfloat16_rn(A / cL_s[hh]);
              }
            }
          }
          bar_consumers();                            // qs / red_* / flag_s are reused by the next unit
        }
      }
      CL_STAMP(4);
      grid_barrier(bars_l + 2, ctid, pause_s);
      CL_STAMP(5);
      // ------------------------------------------------------------------ G1: o partials
      gemm_units(l, 1);
      CL_STAMP(6);
      grid_barrier(bars_l + 3, ctid, pause_s);
      CL_STAMP(7);
      // ------------------------------------------------------------------ R1
      resid_norm(L.ffn_norm, a.s_o);
      CL_STAMP(8);
      grid_barrier(bars_l + 4, ctid, pause_s);
      CL_STAMP(9);
      // ------------------------------------------------------------------ G2: gate|up partials
      gemm_units(l, 2);
      CL_STAMP(10);
      grid_barrier(bars_l + 5, ctid, pause_s);
      CL_STAMP(11);
      // ------------------------------------------------------------------ R2: act = bf16(SiLU(g) * u)
      {
        const int total = a.B * F;
        for (int e = blockIdx.x * 256 + ctid; e < total; e += G * 256) {
          const int b = e / F, i = e - b * F;
          float gt = 0.f, up = 0.f;
          for (int s = 0; s < a.s_gu; ++s) {
            const float2 y = __ldcg(reinterpret_cast<const float2*>(a.part + ((size_t)s * BT + b) * (2 * F) + 2 * i));
            gt += y.x; up += y.y;
          }
          a.act[(size_t)b * F + i] = __float2bfloat16_rn(gt / (1.0f + __expf(-gt)) * up);
        }
      }
      CL_STAMP(12);
      grid_barrier(bars_l + 6, ctid, pause_s);
      CL_STAMP(13);
      // ------------------------------------------------------------------ G3: down partials
      gemm_units(l, 3);
      CL_STAMP(14);
      // its barrier (bars_l + 7) is taken at the top of the next layer / before the final norm
    }
    grid_barrier(a.bars + (size_t)(a.n_layers - 1) * 8 + 7, ctid, pause_s);
    resid_norm(a.final_norm, a.s_dn);                 // xn = final norm: the LM head (K = 64 k-blocks, more than the resident
                                                      // operand holds) runs as a plain GEMM launch after this kernel
#undef CL_STAMP
  }
}

constexpr size_t kSmem = (size_t)NSW * WSLOT + (size_t)NSX * XSLOT + (2 * NSW + NSX + 1) * 8 +
                         (2 * NC * REP + NC * REP * HD + REP * HD + 2 * MAXS * REP + REP + NC + 8) * 4 + 1024 + 64;

bool g_ready[64] = {false}, g_ok[64] = {false};

}  // namespace

bool batch_mega_supported(int d, int d_ff, int head_dim, int n_heads, int n_kv, int page_size, int vocab) {
  return d == D && d_ff == F && head_dim == HD && n_kv > 0 && n_heads == REP * n_kv && page_size == P && vocab > 0;
}

bool batch_mega_prepare_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 63;
  if (!g_ready[dev]) {
    g_ready[dev] = true;
    int nb = 0;
    g_ok[dev] = cudaFuncSetAttribute(decode_mega_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem) == cudaSuccess &&
                cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, decode_mega_batch_kernel, 352, kSmem) == cudaSuccess && nb >= 1;
    if (!g_ok[dev]) cudaGetLastError();
  }
  return g_ok[dev];
}

// tensor map of one weight matrix [N][K] bf16, box {64 k, 128 rows}, 128B swizzle (host side; copied into a device array)
bool make_wmap(CUtensorMap* map, const void* W, int N, int K) { return make_tmap_2d_bf16(map, W, (uint64_t)N, (uint64_t)K, 64, 128); }

int launch_decode_mega_batch(const BatchMegaArgs& a, cudaStream_t st) {
  if (!batch_mega_prepare_device() || a.B < 1 || a.B > BT || a.nsplit < 1 || a.nsplit > MAXS) return -1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(sm_count()); cfg.blockDim = dim3(352); cfg.dynamicSmemBytes = kSmem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;        // all CTAs co-resident (grid barriers), or the launch fails
  at[0].val.cooperative = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, decode_mega_batch_kernel, a) == cudaSuccess ? 1 : -1;
}

}  // namespace cl
