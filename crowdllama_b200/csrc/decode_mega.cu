// decode_mega.cu — the whole transformer stack of ONE decode token as a single persistent kernel.
//
// Why: with one kernel per op (decode_kernels.cu) the weight stream stops at every kernel boundary:
// a CL_TIMELINE trace shows a large share of each layer spent in dependency release at 5 boundaries,
// x/RMSNorm prologues and the attention latency chain,
// during which at most 96 KB/SM of prefetched weights keep HBM busy.  Here:
//   * grid = one CTA per SM, 288 threads: warp 8 is the producer, warps 0..7 consume;
//   * the producer streams EVERY byte the CTA will need — q|k|v rows, this CTA's KV pages, o rows,
//     gate|up rows, down rows, layer after layer — through ONE 6 x 32 KB shared-memory ring with
//     1-D TMA bulk copies; it never waits for activations (only for free slots, and once per layer for
//     the page that holds the current token), so HBM stays busy across every phase boundary;
//   * phases are separated by grid-wide counter barriers (release-add / acquire-poll on a per-phase
//     counter, zeroed at the end of every step), ~1 us instead of a kernel boundary;
//   * the arithmetic of each phase is the code of decode_kernels.cu (same numerics contract).
// Phases per layer: P0 RMSNorm + q|k|v GEMV + RoPE + KV append | P1 split-KV attention partials |
// P2 cross-split combine + o-proj (+residual) | P3 RMSNorm + gate|up GEMV + SiLU*mul | P4 down (+residual).
// The LM head and the argmax tail stay separate kernels (decode_kernels.cu).
// Built for the Llama-3-8B / Mistral-7B layer shape (d 4096, d_ff 14336, head_dim 128, 4 q heads per kv
// head, page 32); other shapes use the per-op path.
#include "common.cuh"
#include "kernels.h"

namespace cl {

namespace {

constexpr int NS = 6;                       // ring slots
constexpr uint32_t SLOT = 32 * 1024;        // bytes per slot
constexpr int NW = 8;                       // consumer warps
constexpr int D = 4096, F = 14336, HD = 128, REP = 4, P = 32, HALF = HD / 2;
constexpr int MAXS = 32;                    // max KV splits (lane-parallel combine)
constexpr int CAP4 = 96;                    // max 4-row tiles one CTA may claim per phase (avg 48.4 for gate|up)
constexpr int CAP1 = 96;                    // max 1-row tiles (down-proj; avg 27.7)
constexpr float LOG2E = 1.4426950408889634f;

struct Ring {
  uint8_t* base;
  uint64_t* full;
  uint64_t* empty;
  int* tile_id;                             // [NS] global tile index carried by each slot (-1 = end of phase)
  uint32_t git;                             // tiles issued / consumed so far by this thread's role
  uint32_t tail;                            // producer only: oldest tile not yet known to have landed
  __device__ __forceinline__ int slot() const { return (int)(git % NS); }
  __device__ __forceinline__ uint32_t parity() const { return (git / NS) & 1u; }
};

__device__ __forceinline__ void tile_range(int ntiles, int unit, int& t0, int& t1) {
  // contiguous, balanced, in multiples of `unit` tiles (keeps row pairs inside one CTA)
  const int nu = ntiles / unit;
  t0 = unit * (int)(((long long)nu * blockIdx.x) / gridDim.x);
  t1 = unit * (int)(((long long)nu * (blockIdx.x + 1)) / gridDim.x);
}

// ---- grid-wide barrier among the consumer halves of all CTAs (producer warps do not take part) ----
__device__ __forceinline__ void grid_barrier(unsigned* cnt, int tid, volatile int* pause = nullptr) {
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (tid == 0) {
    if (pause) *pause = 1;
    // release-increment without waiting for the atomic's return value, then poll
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(cnt) : "memory");
    const long long t0 = clock64();
    while (ld_acquire_u32(cnt) < gridDim.x) {
      if (clock64() - t0 > (1ll << 31)) __trap();
    }
    if (pause) *pause = 0;
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

// ---- producer: DYNAMIC tile scheduling.  SMs do not get equal bandwidth (GPCs hold 16-20 SMs behind the
// same crossbar port; the timeline shows ~20 % spread), so a static split makes every phase as slow as the
// slowest SM.  Tiles are claimed in chunks of CH from a per-(layer, phase) counter; the claim for the next
// chunk is issued before the current chunk's copies so its latency is hidden.  A slot with tile_id = -1 ends
// the phase for this CTA.
constexpr int CH = 1;

// ---- L2 lookahead.  Whenever a producer finds its ring full (the consumers sit in an epilogue, a grid barrier,
// a norm prologue or attention, with HBM idle) it pulls weight tiles that lie AHEAD of every
// CTA's ring into the L2 (50 MB on H100) with cp.async.bulk.prefetch.L2.  All weight tiles of the step form one sequence
// in consumption order (per layer: q|k|v, o, gate|up, down); `ctr` is the global prefetch frontier in that
// numbering.  The frontier is kept between (own demand position + kPfMin) and (+ kPfBudget) tiles, so the
// lookahead never outgrows L2.  When the consumers resume, the ring refills from L2 faster than HBM could feed
// it, the producers block again and the frontier moves on: HBM keeps streaming through the barriers.
constexpr int PFCH = 2;
constexpr int kPfMin = 900, kPfBudget = 4096;   // tiles
struct Lookahead {
  unsigned* ctr;         // nullptr: no lookahead
  unsigned known;        // lower bound of the frontier as last seen by this CTA
  unsigned total;        // n_layers * tiles per layer
  int t_qkv, tl;         // tiles in the q|k|v segment / per layer
  unsigned n_pf, n_lim, n_jump, n_calls;   // diagnostics (CL_TIMELINE)
};
__device__ __forceinline__ void lookahead_step(Lookahead& la, const MegaArgs& a, unsigned mypos) {
  if (!la.ctr) return;
  ++la.n_calls;
  const unsigned lim = mypos + (unsigned)kPfBudget;
  if (la.known >= lim || la.known >= la.total) { ++la.n_lim; return; }
  const unsigned p = atomicAdd(la.ctr, (unsigned)PFCH);
  la.known = p + PFCH;
  if (p < mypos + (unsigned)kPfMin) {      // frontier fell behind the demand stream: jump ahead
    atomicMax(la.ctr, mypos + (unsigned)kPfMin);
    la.known = mypos + (unsigned)kPfMin;
    ++la.n_jump;
    return;
  }
  if (p >= lim) return;
  la.n_pf += PFCH;
#pragma unroll
  for (int i = 0; i < PFCH; ++i) {
    const unsigned gidx = p + i;
    if (gidx >= la.total) break;
    const int l = (int)(gidx / (unsigned)la.tl);
    int idx = (int)(gidx - (unsigned)l * (unsigned)la.tl);
    const MegaLayer& L = a.layers[l];
    const uint8_t* src;
    uint32_t bytes = SLOT;
    if (idx < la.t_qkv) src = reinterpret_cast<const uint8_t*>(L.wqkv) + (size_t)idx * SLOT;
    else if ((idx -= la.t_qkv) < D / 4) src = reinterpret_cast<const uint8_t*>(L.wo) + (size_t)idx * SLOT;
    else if ((idx -= D / 4) < 2 * F / 4) src = reinterpret_cast<const uint8_t*>(L.wgu) + (size_t)idx * SLOT;
    else { idx -= 2 * F / 4; bytes = (uint32_t)F * 2u; src = reinterpret_cast<const uint8_t*>(L.wdown) + (size_t)idx * bytes; }
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
  }
}
// wait for a free ring slot; while blocked, run the L2 lookahead.  Then cap the number of copies IN FLIGHT:
// a few 32 KB copies per SM already saturate HBM (tools/bench_barrier.cu measures it), while every further tile in
// flight only deepens the queues in front of the L2 slices — and the grid barriers' red/poll round trips wait in
// those queues.  The ring still fills all NS slots.
constexpr int kMaxFlight = 2;
__device__ __forceinline__ void wait_slot(Ring& r, int st, Lookahead& la, const MegaArgs& a, unsigned mypos) {
  // (try_wait, not test_wait: a tightly polling producer warp measurably slows the two consumer warps that share
  // its scheduler)
  for (uint32_t spins = 0; !mbar_try_wait(&r.empty[st], r.parity() ^ 1u); ++spins) {
    lookahead_step(la, a, mypos);
    if (spins > (1u << 22)) __trap();
  }
  if (a.pause_in_barrier) {
    volatile int* pause = r.tile_id + 7;
    for (uint32_t spins = 0; *pause; ++spins) if (spins > (1u << 26)) __trap();
  }
  for (uint32_t spins = 0; (int)(r.git - r.tail) >= kMaxFlight; ++spins) {
    const uint32_t n = r.tail;
    if (mbar_try_wait(&r.full[n % NS], (n / NS) & 1u)) ++r.tail;
    else lookahead_step(la, a, mypos);
    if (spins > (1u << 22)) __trap();
  }
}

__device__ __forceinline__ void produce_dynamic(Ring& r, const uint8_t* w, int total, uint32_t bytes, unsigned* ctr, int cap,
                                                uint64_t pol, Lookahead& la, const MegaArgs& a, unsigned gbase) {
  int issued = 0;
  int cur = (int)atomicAdd(ctr, (unsigned)CH);
  while (cur < total) {
    const int nxt = (issued + 2 * CH <= cap) ? (int)atomicAdd(ctr, (unsigned)CH) : total;
    const int end = min(cur + CH, total);
    for (int t = cur; t < end; ++t) {
      const int st = r.slot();
      wait_slot(r, st, la, a, gbase + (unsigned)t);
      r.tile_id[st] = t;
      mbar_arrive_expect_tx(&r.full[st], bytes);
      bulk_g2s(r.base + (size_t)st * SLOT, w + (size_t)t * bytes, bytes, &r.full[st], pol);
      ++r.git;
      ++issued;
    }
    cur = nxt;
  }
  const int st = r.slot();
  wait_slot(r, st, la, a, gbase + (unsigned)total);
  r.tile_id[st] = -1;
  mbar_arrive(&r.full[st]);
  ++r.git;
}

// ---- consumer GEMV over this CTA's tiles.  x lives in registers (xr[CPL][8], already bf16-rounded).
// Partial row sums go to part[(local_row) * S + s]; the caller runs the epilogue after a CTA barrier.
template <int TR, int S, int CPL>
__device__ __forceinline__ int consume_dynamic(Ring& r, const float (&xr)[CPL][8], float* part, int* ids, int warp, int lane) {
  // 8 warps cover TR rows x S k-slices; a warp owns slice (warp % S) of RPW rows: warp / S + j * (8 / S).
  // (registers are allocated for 12 warps when 9 are launched, so <= 168 per thread: small x slices matter)
  // Returns the number of tiles this CTA processed; ids[i] = global tile index of local tile i.
  constexpr int K = S * CPL * 256;
  constexpr int RPW = TR * S / 8, RSTEP = 8 / S;
  static_assert(RPW >= 1 && RPW * 8 == TR * S, "8 consumer warps");
  const int s = warp % S, row0 = warp / S;
  const uint32_t off = (uint32_t)(row0 * K + s * (K / S) + lane * 8) * 2u;
  int n = 0;
  while (true) {
    const int st = r.slot();
    mbar_wait(&r.full[st], r.parity());
    const int tile = r.tile_id[st];
    if (tile < 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&r.empty[st]);
      ++r.git;
      break;
    }
    const uint8_t* b = r.base + (size_t)st * SLOT + off;
    uint4 w[RPW][CPL];
#pragma unroll
    for (int j = 0; j < RPW; ++j)
#pragma unroll
      for (int c = 0; c < CPL; ++c) w[j][c] = *reinterpret_cast<const uint4*>(b + (size_t)j * RSTEP * K * 2 + c * 512);
    __syncwarp();
    if (lane == 0) mbar_arrive(&r.empty[st]);
    ++r.git;
#pragma unroll
    for (int j = 0; j < RPW; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        acc = fmaf(bf16_lo(w[j][c].x), xr[c][0], acc); acc = fmaf(bf16_hi(w[j][c].x), xr[c][1], acc);
        acc = fmaf(bf16_lo(w[j][c].y), xr[c][2], acc); acc = fmaf(bf16_hi(w[j][c].y), xr[c][3], acc);
        acc = fmaf(bf16_lo(w[j][c].z), xr[c][4], acc); acc = fmaf(bf16_hi(w[j][c].z), xr[c][5], acc);
        acc = fmaf(bf16_lo(w[j][c].w), xr[c][6], acc); acc = fmaf(bf16_hi(w[j][c].w), xr[c][7], acc);
      }
      acc = warp_sum(acc);
      if (lane == 0) part[(n * TR + row0 + j * RSTEP) * S + s] = acc;
    }
    if (warp == 0 && lane == 0) ids[n] = tile;
    ++n;
  }
  return n;
}

// x slice of this warp -> registers.  NORM: RMSNorm(h) * gain, bf16-rounded (gains are prefetched by the caller)
template <int S, int CPL>
__device__ __forceinline__ void load_x(const float* x, float (&xr)[CPL][8], int warp, int lane) {
  constexpr int K = S * CPL * 256;
  const int kbase = (warp % S) * (K / S);
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int k = kbase + (c * 32 + lane) * 8;
    const float4 v0 = ldcg4(x + k), v1 = ldcg4(x + k + 4);
    xr[c][0] = v0.x; xr[c][1] = v0.y; xr[c][2] = v0.z; xr[c][3] = v0.w;
    xr[c][4] = v1.x; xr[c][5] = v1.y; xr[c][6] = v1.z; xr[c][7] = v1.w;
  }
}

template <int S, int CPL>
__device__ __forceinline__ void load_x_norm(const float* h, const float (&gr)[CPL][8], float eps, float* ssw, float (&xr)[CPL][8],
                                            int warp, int lane) {
  constexpr int K = S * CPL * 256;
  load_x<S, CPL>(h, xr, warp, lane);
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(xr[c][j], xr[c][j], ss);
  ss = warp_sum(ss);
  if (lane == 0) ssw[warp] = ss;
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < S; ++i) tot += ssw[i];   // warps 0..S-1 = row 0, slices 0..S-1: cover K once
  const float inv = 1.0f / sqrtf(tot / (float)K + eps);
#pragma unroll
  for (int c = 0; c < CPL; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) xr[c][j] = bf16_round(xr[c][j] * inv * gr[c][j]);
  asm volatile("bar.sync 1, 256;" ::: "memory");   // ssw may be reused by the next phase
}

template <int S, int CPL>
__device__ __forceinline__ void load_gain(const float* gain, float (&gr)[CPL][8], int warp, int lane) {
  constexpr int K = S * CPL * 256;
  const int kbase = (warp % S) * (K / S);
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int k = kbase + (c * 32 + lane) * 8;
    const float4 g0 = *reinterpret_cast<const float4*>(gain + k), g1 = *reinterpret_cast<const float4*>(gain + k + 4);
    gr[c][0] = g0.x; gr[c][1] = g0.y; gr[c][2] = g0.z; gr[c][3] = g0.w;
    gr[c][4] = g1.x; gr[c][5] = g1.y; gr[c][6] = g1.z; gr[c][7] = g1.w;
  }
}

__global__ void __launch_bounds__(288, 1) decode_mega_kernel(const __grid_constant__ MegaArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // the KV tiles are 128B-swizzled TMA boxes: ring slots must be 1024-byte aligned
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring_base = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)NS * SLOT);
  uint64_t* empty = full + NS;
  int* tile_id = reinterpret_cast<int*>(empty + NS);         // [NS] (+2 pad)
  int* ids = tile_id + 8;                                    // [CAP4] local tile list of the current phase
  float* ssw = reinterpret_cast<float*>(ids + CAP4);         // [8]
  float* part = ssw + 8;                                     // [CAP4 tiles * 4 rows * 4 slices]
  float* red_m = part + CAP4 * 16;                           // [NW][REP]
  float* red_l = red_m + NW * REP;                           // [NW][REP]
  float* red_acc = red_l + NW * REP;                         // [NW][REP][HD]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    tile_id[7] = 0;
    for (int i = 0; i < NS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NW); }
    fence_barrier_init();
  }
  __syncthreads();

  const int slot = a.slots ? a.slots[0] : 0;
  const int pos = a.pos[slot];
  const int ctx = pos + 1;
  const int* bt = a.block_tables + (size_t)slot * a.bt_stride;
  // attention work of this CTA: (kv head g, split sp) over pages [pg0, pg1)
  const int n_att = a.n_kv * a.nsplit;
  const bool has_att = (int)blockIdx.x < n_att;
  const int g = has_att ? blockIdx.x / a.nsplit : 0, sp = has_att ? blockIdx.x % a.nsplit : 0;
  const int total_pages = (ctx + P - 1) / P;
  const int pps = (total_pages + a.nsplit - 1) / a.nsplit;
  const int pg0 = has_att ? sp * pps : 0;
  const int pg1 = has_att ? min(total_pages, pg0 + pps) : 0;
  const int npg = pg1 > pg0 ? pg1 - pg0 : 0;
  const int n_att_tiles = (npg + 1) / 2;

  const int T_QKV = a.qkv_dim / 4, T_O = D / 4, T_GU = 2 * F / 4, T_DN = D;   // tiles per phase
  Ring r{ring_base, full, empty, tile_id, 0u, 0u};

  if (warp == NW) {
    // =============================== producer ===============================
    if (!elect_one()) return;
    prefetch_tmap(&a.kmap);
    prefetch_tmap(&a.vmap);
    const uint64_t pol = policy_evict_first();
    const int cur_page = pos / P;
    const int TL = T_QKV + T_O + T_GU + T_DN;
    Lookahead la{a.pf_ctr, 0u, (unsigned)(a.n_layers * TL), T_QKV, TL, 0u, 0u, 0u, 0u};
    for (int l = 0; l < a.n_layers; ++l) {
      const MegaLayer& L = a.layers[l];
      unsigned* ctr = a.tile_ctr + (size_t)l * 4;
      const unsigned g0 = (unsigned)(l * TL), g1 = g0 + T_QKV, g2 = g1 + T_O, g3 = g2 + T_GU;
      produce_dynamic(r, reinterpret_cast<const uint8_t*>(L.wqkv), T_QKV, SLOT, ctr + 0, CAP4, pol, la, a, g0);
      for (int t = 0; t < n_att_tiles; ++t) {
        const int st = r.slot();
        wait_slot(r, st, la, a, g1);
        const int pa = pg0 + 2 * t, pb = pa + 1;
        const bool two = pb < pg1;
        if (pa == cur_page || (two && pb == cur_page)) {
          // this page receives the current token's K/V in phase P0 of THIS layer: wait for barrier B0
          const unsigned* b0 = a.bars + (size_t)l * 6 + 0;
          const long long t0 = clock64();
          while (ld_acquire_u32(b0) < gridDim.x) { if (clock64() - t0 > (1ll << 31)) __trap(); }
          fence_proxy_async_all();
        }
        uint8_t* dst = r.base + (size_t)st * SLOT;
        mbar_arrive_expect_tx(&r.full[st], two ? 32768u : 16384u);
        // per page: K dims 0-63 | K dims 64-127 | V dims 0-63 | V dims 64-127, each a [32 tokens][128 B] swizzled box
        for (int pgi = 0; pgi < (two ? 2 : 1); ++pgi) {
          const long long row = (long long)l * a.kv_layer_rows + ((long long)bt[pa + pgi] * a.n_kv + g) * P;
          uint8_t* d = dst + pgi * 16384;
          tma_load_2d(d, &a.kmap, 0, (int)row, &r.full[st]);
          tma_load_2d(d + 4096, &a.kmap, 64, (int)row, &r.full[st]);
          tma_load_2d(d + 8192, &a.vmap, 0, (int)row, &r.full[st]);
          tma_load_2d(d + 12288, &a.vmap, 64, (int)row, &r.full[st]);
        }
        ++r.git;
      }
      produce_dynamic(r, reinterpret_cast<const uint8_t*>(L.wo), T_O, SLOT, ctr + 1, CAP4, pol, la, a, g1);
      produce_dynamic(r, reinterpret_cast<const uint8_t*>(L.wgu), T_GU, SLOT, ctr + 2, CAP4, pol, la, a, g2);
      produce_dynamic(r, reinterpret_cast<const uint8_t*>(L.wdown), T_DN, (uint32_t)F * 2u, ctr + 3, CAP1, pol, la, a, g3);
    }
    if (a.tl != nullptr && blockIdx.x == (unsigned)a.tl_cta) {
      long long* dbg = a.tl + (size_t)a.n_layers * 16;
      dbg[0] = la.n_pf; dbg[1] = la.n_lim; dbg[2] = la.n_jump; dbg[3] = la.n_calls; dbg[4] = r.git;
    }
    return;
  }

  // =============================== consumers ===============================
  float* h = a.h + (size_t)slot * D;
  float* qbuf = a.q + (size_t)slot * a.q_dim;
  float* xatt = a.attn_x + (size_t)slot * a.q_dim;
  float* act = a.act + (size_t)slot * F;
  // RoPE row of the current position: one row serves all 32 layers, so it is staged in shared memory once — the P0
  // epilogue sits between the q|k|v GEMV and barrier B0, where a global load costs a loaded L2 round trip per layer
  float2* rope = reinterpret_cast<float2*>(red_acc + NW * REP * HD);   // [HALF]
  for (int i = tid; i < HALF; i += 256) rope[i] = __ldg(a.rope + (size_t)pos * HALF + i);
  asm volatile("bar.sync 1, 256;" ::: "memory");
  const int cur_pg = bt[pos / P], cur_off = pos % P;
  const float scale2 = rsqrtf((float)HD) * LOG2E;

  volatile int* pz = a.pause_in_barrier ? tile_id + 7 : nullptr;
  const bool stamp = a.tl != nullptr && blockIdx.x == (unsigned)a.tl_cta && tid == 0;
#define CL_STAMP(k) do { if (stamp) a.tl[(size_t)l * 16 + (k)] = gtime_ns(); } while (0)
  for (int l = 0; l < a.n_layers; ++l) {
    const MegaLayer& L = a.layers[l];
    unsigned* bars = a.bars + (size_t)l * 6;
    // ------------------------------------------------------------------ P0: norm + q|k|v + RoPE + append
    {
      float gr[4][8], xr[4][8];
      load_gain<4, 4>(L.attn_norm, gr, warp, lane);
      if (l > 0) grid_barrier(a.bars + (size_t)(l - 1) * 6 + 5, tid, pz);   // previous layer's down-proj complete (h final)
      CL_STAMP(0);
      load_x_norm<4, 4>(h, gr, a.eps, ssw, xr, warp, lane);
      CL_STAMP(1);
      const int nloc = consume_dynamic<4, 4, 4>(r, xr, part, ids, warp, lane);
      CL_STAMP(2);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int p = tid; p < nloc * 2; p += 256) {
        const float* pp = part + (size_t)(2 * p) * 4;
        const float v0 = (pp[0] + pp[1]) + (pp[2] + pp[3]);
        const float v1 = (pp[4] + pp[5]) + (pp[6] + pp[7]);
        const int gp = ids[p >> 1] * 2 + (p & 1), hh = gp / HALF, j = gp - hh * HALF;
        if (hh < a.n_heads + a.n_kv) {
          const float2 cs = rope[j];
          const float r0 = bf16_round(v0 * cs.x - v1 * cs.y), r1 = bf16_round(v1 * cs.x + v0 * cs.y);
          if (hh < a.n_heads) {
            qbuf[hh * HD + j] = r0;
            qbuf[hh * HD + j + HALF] = r1;
          } else {
            const size_t base = (((size_t)cur_pg * a.n_kv + (hh - a.n_heads)) * P + cur_off) * HD;
            L.kpool[base + j] = __float2bfloat16_rn(r0);
            L.kpool[base + j + HALF] = __float2bfloat16_rn(r1);
          }
        } else {
          const size_t base = (((size_t)cur_pg * a.n_kv + (hh - a.n_heads - a.n_kv)) * P + cur_off) * HD;
          L.vpool[base + j] = __float2bfloat16_rn(v0);
          L.vpool[base + j + HALF] = __float2bfloat16_rn(v1);
        }
      }
      grid_barrier(bars + 0, tid, pz);
      CL_STAMP(3);
    }
    // ------------------------------------------------------------------ P1: split-KV attention partials
    if (has_att) {
      // Tensor-core attention (mma.sync m16n8k16): one warp per KV page.  S[16 x 32] = Q[16 x 128] K^T with the
      // REP query heads in rows 0..REP-1 (rows above are zero padding), online softmax on the fragments,
      // O[16 x 128] += P V.  K/V tiles are 128B-swizzled TMA boxes -> conflict-free ldmatrix.
      const int rq = lane >> 2, cq = lane & 3;            // fragment row (head) / column pair
      uint32_t qf[HD / 16][4];
      {
        const float* q = qbuf + (size_t)g * REP * HD;
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
          qf[kk][1] = 0u; qf[kk][3] = 0u;                   // rows 8..15: padding
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
      float mrow = -INFINITY, lrow = 0.f;                   // row rq (valid for rq < REP)
      for (int t = 0; t < n_att_tiles; ++t) {
        const int st = r.slot();
        mbar_wait(&r.full[st], r.parity());
        const int npage = (pg0 + 2 * t + 1 < pg1) ? 2 : 1;
        for (int pgi = 0; pgi < npage; ++pgi) {
          if (((2 * t + pgi) & (NW - 1)) != warp) continue;  // page -> warp (round robin)
          const uint32_t kb = smem_u32(r.base + (size_t)st * SLOT + pgi * 16384), vb = kb + 8192;
          const int tok0 = (pg0 + 2 * t + pgi) * P;
          float sacc[4][4];
#pragma unroll
          for (int nj = 0; nj < 4; ++nj) { sacc[nj][0] = sacc[nj][1] = sacc[nj][2] = sacc[nj][3] = 0.f; }
          const int id = lane >> 3;
#pragma unroll
          for (int kk = 0; kk < HD / 16; ++kk) {
            const uint32_t kh = kb + (kk >> 2) * 4096;      // dims 0-63 | 64-127
#pragma unroll
            for (int np = 0; np < 2; ++np) {
              uint32_t kf[4];
              const int row = (2 * np + (id >> 1)) * 8 + (lane & 7), ch = (kk & 3) * 2 + (id & 1);
              ldsm_x4(kf, kh + row * 128 + ((ch ^ (row & 7)) << 4));
              mma_bf16(sacc[2 * np], qf[kk], kf[0], kf[1]);
              mma_bf16(sacc[2 * np + 1], qf[kk], kf[2], kf[3]);
            }
          }
          // online softmax for row rq (c0, c1 of every n-tile); tokens >= ctx are masked
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
          const float mn = fmaxf(mrow, mx);                  // finite: every page of a split holds >= 1 valid token
          const float corr = exp2f(mrow - mn);
          mrow = mn;
          float rs = 0.f;
          // P is split into two bf16 terms (hi + lo) so that P.V keeps ~fp32 accuracy: a single bf16 P would put a
          // 2^-9 relative error on every attention output, which the bf16 rounding points downstream amplify
          uint32_t pf[2][4], pl[2][4];
#pragma unroll
          for (int nj = 0; nj < 4; ++nj) {
            const float p0 = exp2f(sacc[nj][0] - mn), p1 = exp2f(sacc[nj][1] - mn);
            rs += p0 + p1;
            const float h0 = bf16_round(p0), h1 = bf16_round(p1);
            pf[nj >> 1][(nj & 1) * 2] = pack_bf16(h0, h1);
            pf[nj >> 1][(nj & 1) * 2 + 1] = 0u;             // rows 8..15
            pl[nj >> 1][(nj & 1) * 2] = pack_bf16(p0 - h0, p1 - h1);
            pl[nj >> 1][(nj & 1) * 2 + 1] = 0u;
          }
          lrow = lrow * corr + rs;
#pragma unroll
          for (int nd = 0; nd < HD / 8; ++nd) { o[nd][0] *= corr; o[nd][1] *= corr; }
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {                   // 16-token k-steps
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
        if (lane == 0) mbar_arrive(&r.empty[st]);
        ++r.git;
      }
      // row sums: the 4 lanes of a row hold partial sums
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
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float* pout = a.part + ((((size_t)slot * a.n_kv + g) * a.nsplit + sp) * REP) * (HD + 2);
      for (int t = tid; t < REP * HD; t += 256) {
        const int hh = t / HD, i = t % HD;
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < NW; ++w) M = fmaxf(M, red_m[w * REP + hh]);
        float Ls = 0.f, A = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
          const float mw = red_m[w * REP + hh];
          const float c = (mw == -INFINITY) ? 0.f : exp2f(mw - M);
          Ls = fmaf(red_l[w * REP + hh], c, Ls);
          A = fmaf(red_acc[(w * REP + hh) * HD + i], c, A);
        }
        float* ph = pout + (size_t)hh * (HD + 2);
        if (i == 0) { ph[0] = M; ph[1] = Ls; }
        ph[2 + i] = A;
      }
    }
    CL_STAMP(4);
    grid_barrier(bars + 1, tid, pz);
    CL_STAMP(5);
    // ------------------------------------------------------------------ P2: combine slice, then o-proj + residual
    {
      const int PS = HD + 2;
      const int c0 = (int)(((long long)a.q_dim * blockIdx.x) / gridDim.x), c1 = (int)(((long long)a.q_dim * (blockIdx.x + 1)) / gridDim.x);
      const float* pbase = a.part + (size_t)slot * a.n_kv * a.nsplit * REP * PS;
      constexpr int MAXR = 4;   // 4 rounds x 8 warps = 32 outputs >= ceil(4096 / 132)
      float mv[MAXR], lv[MAXR], av[MAXR];
#pragma unroll
      for (int q = 0; q < MAXR; ++q) {
        const int o = c0 + q * 8 + warp;
        mv[q] = -INFINITY; lv[q] = 0.f; av[q] = 0.f;
        if (o < c1 && lane < a.nsplit) {
          const int hg = o / HD, i = o - hg * HD;
          const float* p = pbase + (((size_t)(hg / REP) * a.nsplit + lane) * REP + (hg % REP)) * PS;
          mv[q] = __ldcg(p); lv[q] = __ldcg(p + 1); av[q] = __ldcg(p + 2 + i);
        }
      }
#pragma unroll
      for (int q = 0; q < MAXR; ++q) {
        const int o = c0 + q * 8 + warp;
        if (o < c1) {
          const float M = warp_max(mv[q]);
          const float w = (mv[q] == -INFINITY) ? 0.f : exp2f(mv[q] - M);
          const float Ls = warp_sum(lv[q] * w), A = warp_sum(av[q] * w);
          if (lane == 0) xatt[o] = bf16_round(A / Ls);
        }
      }
      grid_barrier(bars + 2, tid, pz);
      CL_STAMP(6);
      float xr[4][8];
      load_x<4, 4>(xatt, xr, warp, lane);
      const int nloc = consume_dynamic<4, 4, 4>(r, xr, part, ids, warp, lane);
      CL_STAMP(7);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int p = tid; p < nloc * 4; p += 256) {
        const int row = ids[p >> 2] * 4 + (p & 3);
        atomicAdd(h + row, (part[p * 4] + part[p * 4 + 1]) + (part[p * 4 + 2] + part[p * 4 + 3]));   // RED: exactly one add per row and phase
      }
      grid_barrier(bars + 3, tid, pz);
      CL_STAMP(8);
    }
    // ------------------------------------------------------------------ P3: norm + gate|up + SiLU*mul
    {
      float gr[4][8], xr[4][8];
      load_gain<4, 4>(L.ffn_norm, gr, warp, lane);
      load_x_norm<4, 4>(h, gr, a.eps, ssw, xr, warp, lane);
      CL_STAMP(9);
      const int nloc = consume_dynamic<4, 4, 4>(r, xr, part, ids, warp, lane);
      CL_STAMP(10);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int p = tid; p < nloc * 2; p += 256) {
        const float* pp = part + (size_t)(2 * p) * 4;
        const float gt = (pp[0] + pp[1]) + (pp[2] + pp[3]);
        const float up = (pp[4] + pp[5]) + (pp[6] + pp[7]);
        act[ids[p >> 1] * 2 + (p & 1)] = bf16_round(gt / (1.0f + __expf(-gt)) * up);
      }
      grid_barrier(bars + 4, tid, pz);
      CL_STAMP(11);
    }
    // ------------------------------------------------------------------ P4: down + residual
    {
      float xr[7][8];
      load_x<8, 7>(act, xr, warp, lane);
      CL_STAMP(12);
      const int nloc = consume_dynamic<1, 8, 7>(r, xr, part, ids, warp, lane);
      CL_STAMP(13);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int p = tid; p < nloc; p += 256) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) v += part[p * 8 + i];
        atomicAdd(h + ids[p], v);   // RED: exactly one add per row and phase (deterministic)
      }
      // the barrier that closes this phase is taken at the top of the next layer's P0 (after its gain prefetch);
      // after the last layer the kernel boundary does the job
      if (l + 1 < a.n_layers) { /* see P0 */ }
    }
  }
}

}  // namespace

bool mega_supported(int d, int d_ff, int head_dim, int n_heads, int n_kv, int page_size, int nsplit) {
  return d == D && d_ff == F && head_dim == HD && n_kv > 0 && n_heads == REP * n_kv && page_size == P && nsplit >= 1 &&
         nsplit <= MAXS && n_kv * nsplit <= sm_count() && (n_heads * HD + sm_count() - 1) / sm_count() <= 32 &&
         ((n_heads + 2 * n_kv) * HD) % 4 == 0;
}

static constexpr size_t kMegaSmem =
    (size_t)NS * SLOT + 2 * NS * 8 + (8 + CAP4 + 8 + CAP4 * 16 + 2 * NW * REP + NW * REP * HD + 2 * HALF) * 4 + 128 + 1024;

// The grid barriers need every CTA resident at once.  Per device: opt in to the shared-memory size once, and check
// that one CTA per SM fits (occupancy >= 1 with 288 threads + kMegaSmem); the engine falls back to the per-op path
// otherwise.  The launch is cooperative (cudaLaunchAttributeCooperative): the driver guarantees co-residency or fails
// the launch.  All in-kernel waits are bounded as well (clock64 -> __trap), so a protocol bug ends as a kernel error,
// never as a hung GPU.
static bool g_mega_ready[64] = {false}, g_mega_ok[64] = {false};
bool mega_prepare_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 63;
  if (!g_mega_ready[dev]) {
    g_mega_ready[dev] = true;
    int nb = 0;
    g_mega_ok[dev] = cudaFuncSetAttribute(decode_mega_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMegaSmem) == cudaSuccess &&
                     cudaFuncSetAttribute(decode_mega_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) == cudaSuccess &&
                     cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, decode_mega_kernel, 288, kMegaSmem) == cudaSuccess && nb >= 1;
    if (!g_mega_ok[dev]) cudaGetLastError();
  }
  return g_mega_ok[dev];
}

int launch_decode_mega(const MegaArgs& a, cudaStream_t st) {
  if (!mega_prepare_device()) return -1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(sm_count()); cfg.blockDim = dim3(288); cfg.dynamicSmemBytes = kMegaSmem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, decode_mega_kernel, a) == cudaSuccess ? 1 : -1;
}

}  // namespace cl
