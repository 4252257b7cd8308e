// kernels.h — host-side launch interface of the sm_90a kernels (internal to libclengine.so).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cl {

enum GemvEpi { EPI_STORE = 0, EPI_RESID = 1, EPI_GATEUP = 2, EPI_QKV = 3 };

// EPI_QKV: the q|k|v projection's rows are stored ROPE-PAIR-INTERLEAVED (within each head, row 2j holds
// dim j and row 2j+1 holds dim j + head_dim/2), so the row pair a GEMV thread owns is exactly one RoPE
// rotation pair: the epilogue rotates, rounds to bf16, writes q to y[slot][H*D] (natural dim order) and
// appends k / v straight into the paged cache.  The attention kernel then needs no RoPE and no append.
struct QkvEpi {
  const float2* rope = nullptr;       // [max_pos][head_dim/2]
  const int* pos = nullptr;           // [slot]
  const int* block_tables = nullptr;  // [slot][bt_stride]
  int bt_stride = 0;
  __nv_bfloat16* kpool = nullptr;     // this layer
  __nv_bfloat16* vpool = nullptr;
  int n_heads = 0, n_kv = 0, head_dim = 0, page_size = 0;
};

// y[slot] = epi(W * x[slot]).  Row pairs (2i, 2i+1) are always processed together so the
// gate/up interleaving (row 2i = gate_i, row 2i+1 = up_i) needs no special casing.
struct GemvArgs {
  const __nv_bfloat16* W = nullptr;  // [N][K] row-major
  int N = 0, K = 0;
  const float* x = nullptr;          // !norm: [slot][x_stride] bf16-rounded fp32 inputs
  const float* h = nullptr;          // norm: residual stream [slot][x_stride]
  const float* gain = nullptr;       // norm gains [K]
  float eps = 0.f;
  float* y = nullptr;                // [slot][y_stride]
  const float* resid = nullptr;      // EPI_RESID (may alias y)
  int x_stride = 0, y_stride = 0;
  const int* slots = nullptr;        // blockIdx.y = b -> slot (nullptr => identity)
  int batch = 1;
  int pdl_early = 1;                 // 1: trigger dependents at kernel start; 0: when this CTA has issued its last load
  QkvEpi qkv;                        // EPI_QKV only
  long long* tl = nullptr;           // debug timeline (CL_TIMELINE=1): 4 globaltimer stamps written by CTA 0
};

struct AttnDecodeArgs {
  const float* q = nullptr;          // [slot][q_stride] roped, bf16-rounded query of the current token
  int q_stride = 0;
  const __nv_bfloat16* kpool = nullptr;  // this layer: [n_pages][n_kv][page][head_dim]; holds tokens 0..pos
  const __nv_bfloat16* vpool = nullptr;
  const int* block_tables = nullptr; // [slot][bt_stride]
  int bt_stride = 0;
  const int* pos = nullptr;          // [slot] index of the current token (context = pos + 1 tokens)
  float* out = nullptr;              // [slot][out_stride] bf16-rounded fp32
  int out_stride = 0;
  __nv_bfloat16* out_bf16 = nullptr; // optional: the same values as bf16 [batch index][out_stride] (X operand of the batched o-projection)
  float* part = nullptr;             // [slot][n_kv][nsplit][rep][head_dim + 2]
  unsigned* counters = nullptr;      // [slot][n_kv]
  const int* slots = nullptr;
  int batch = 1;
  int n_heads = 0, n_kv = 0, head_dim = 0, page_size = 0, nsplit = 0;
  int pdl_early = 1;
  long long* tl = nullptr;
  int ring_bytes = 0;                // filled by the launcher
  int tc_small = 0;                  // attn_decode_tc: 4-warp CTAs, two per SM (attn_decode_tc_plan)
};

// ---- step tail: argmax or a seeded draw, then advance the sequence ----------------------------------
constexpr int kTailBlocks = 64;          // blocks per slot; each owns a contiguous slice of the vocabulary
constexpr int kSampleTopKMax = 128;      // device draws cover 1 <= top_k <= this
constexpr int kSampleHistMax = 256;      // ... and a repeat-penalty window of at most this many ids
constexpr int kSampleSliceMax = 2560;    // ... and vocab <= kTailBlocks * kSampleSliceMax (one slice's keys sit in shared memory)

struct SampleParams {                    // cl_sampling fields the draw reads
  float temperature = 0.f, top_p = 1.f, repeat_penalty = 1.f;
  int top_k = 0, repeat_last_n = 0;
  unsigned long long seed = 0;
};
// Per-slot sampler state of the step tail.  A slot whose mode is 1 draws exactly as the host sampler (host_util.cpp
// sample_token) would with history = its ring (+ the step's input token when push_input) and step = its draw counter.
struct SampleState {
  const int* mode = nullptr;             // [slot] 0: argmax, 1: draw (nullptr: argmax everywhere)
  const SampleParams* par = nullptr;     // [slot]
  unsigned long long* step = nullptr;    // [slot] RNG step of the next draw (+1 per draw)
  int* hist = nullptr;                   // [slot][kSampleHistMax] ring: id i of the history at i % kSampleHistMax
  int* hist_len = nullptr;               // [slot] ids in the history so far
  unsigned long long* cand = nullptr;    // [slot][kTailBlocks][kSampleTopKMax] per-block top-k keys (step tail)
  int push_input = 0;                   // 1 (decode steps): tok[slot], the step's input, joins the history before the draw
};

// Per-token log-probabilities of the step tail: natural-log log_softmax of the raw fp32 logits row (before the repeat
// penalty, temperature, top-k and top-p), whatever the sampler then does with it.  Every block of the row keys its slice
// (slice max, sum of expf(v - max), its top-n keys), the row's last block merges the kTailBlocks partials in fixed block
// order (lse in double) and writes lse and the top-n (value descending, id ascending); the block that makes the row's choice
// then writes the chosen id and logit[id] - lse.  Every logprob is (double)logit - lse rounded to fp32: an fp32 lse would
// carry half an ulp of the row's largest logits (5e-4 at 1e4).  A record thus depends on its logits row alone.
constexpr int kLogprobTopMax = 20;
struct LogprobRecord {                   // 184 bytes
  double lse;                            // log of the row's softmax denominator, max included
  int id;                                // the chosen id
  float logprob;                         // (double)logit[id] - lse, rounded to fp32
  int n_top;
  int top_ids[kLogprobTopMax];
  float top_logprobs[kLogprobTopMax];    // (double)logit - lse, rounded to fp32
};
struct LogprobState {
  const int* top_n = nullptr;            // [slot] -1: off, 0..kLogprobTopMax: on with that many alternatives (nullptr: off everywhere)
  float2* part = nullptr;                // [row][kTailBlocks] slice (max, sum of exp(v - max))
  unsigned long long* cand = nullptr;    // [row][kTailBlocks][kLogprobTopMax] slice top-n keys
  unsigned* counters = nullptr;          // [row], zero between launches
  LogprobRecord* last = nullptr;         // [row]: the row's latest record
  LogprobRecord* ring = nullptr;         // step tail only (may be nullptr): [ring_steps][ring_stride], parallel to the id ring
};

struct StepTailArgs {                // argmax (or a draw) over logits, advance the sequence
  const float* logits = nullptr;     // [slot][vocab]
  int vocab = 0;
  int* tok = nullptr;                // [slot] next input token (written)
  int* pos = nullptr;                // [slot] incremented
  int* ids_ring = nullptr;           // [ring_steps][max_batch] generated ids
  int* step_counter = nullptr;       // device scalar, incremented once per step
  unsigned* sync_counters = nullptr; // zeroed at the end of every step (MegaArgs: bars, tile_ctr, pf_ctr)
  int n_sync_counters = 0;
  int ring_steps = 0, ring_stride = 0;
  float* part_val = nullptr;         // [slot][nblk]
  int* part_idx = nullptr;
  unsigned* counters = nullptr;      // [slot]
  const int* slots = nullptr;
  int batch = 1;
  SampleState sample;
  LogprobState lp;                   // rows = slots
};

// Verify pass of speculative decoding for one slot (a segment of Engine::verify_batch): T = k + 1 rows with inputs x0, d1 .. dk.
// spec_tail_kernel makes row r's step-tail choice into choice[r] (the draw: history = ring + inputs[0..r], RNG step
// step[slot] + r); spec_accept_kernel then accepts the longest run of drafts equal to the choices and advances the slot.
struct SpecTailArgs {
  const float* logits = nullptr;     // [T][vocab]
  int vocab = 0, T = 0, slot = 0;
  int len = 0;                       // cached tokens of the sequence before the pass (x0 sits at position len)
  const int* inputs = nullptr;       // [T] x0, d1 .. dk
  int* choice = nullptr;             // [T] y_1 .. y_T
  float* part_val = nullptr;         // [T][kTailBlocks]
  int* part_idx = nullptr;
  unsigned* counters = nullptr;      // [T], zero between passes
  unsigned long long* cand = nullptr;   // [T][kTailBlocks][kSampleTopKMax]
  int* tok = nullptr;                // [slot] next input (written: y_{a+1})
  int* pos = nullptr;                // [slot] its position (written: len + a + 1)
  int* out = nullptr;                // [1 + T] a + 1, then y_1 .. y_{a+1}
  SampleState sample;                // mode / par / step / hist / hist_len of the slot (cand and push_input unused)
  LogprobState lp;                   // top_n of the slot; part / cand / counters / last per row of the pass (row r = y_{r+1}'s record)
};

// every launcher returns the number of kernels it enqueued (for cl_stats.kernel_launches)
int launch_gemv(int variant, int epi, bool norm, const GemvArgs& a, cudaStream_t st, bool pdl, int* n_ctas = nullptr);
int launch_attn_decode(const AttnDecodeArgs& a, cudaStream_t st, bool pdl);
// tensor-core variant for the batched step (attn_decode_tc.cu): head_dim 128, 4 q heads per kv head, page 32;
// kmap / vmap = pool-wide 2-D tensor maps (make_tmap_2d_bf16, box {64, 32}), layer_row0 = first row of this layer
bool attn_decode_tc_supported(int n_heads, int n_kv, int head_dim, int page_size, int nsplit);
void attn_decode_tc_plan(int n_kv, int batch, int nsplit_max, int cta_budget, int* nsplit, int* small);   // splits + kernel shape of a batched step
int launch_attn_decode_tc(const AttnDecodeArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st,
                          bool pdl);
int launch_embed(const __nv_bfloat16* table, int d, const int* tok, float* h, int h_stride, const int* slots,
                 int batch, cudaStream_t st);
int launch_step_tail(const StepTailArgs& a, cudaStream_t st);
int launch_spec_tail(const SpecTailArgs& a, cudaStream_t st, bool pdl);   // spec_tail_kernel + spec_accept_kernel (PDL)
// rope_hd > 0: rows are written rope-pair-interleaved per head of rope_hd rows (see QkvEpi)
int launch_synth_bf16(__nv_bfloat16* out, int64_t n_logical, int k_cols, int row_mult, int row_off, uint64_t seed,
                      int key, float scale, cudaStream_t st, int rope_hd = 0);
int launch_synth_gain(float* out, int n, uint64_t seed, int key, float scale, cudaStream_t st);
int launch_bf16_to_f32(const __nv_bfloat16* in, float* out, int64_t n, cudaStream_t st);
// parity aid: the oracle's oc_seq_fake_fill pattern into tokens 0..n_tokens-1 of one sequence, all layers
int launch_fake_fill_kv(__nv_bfloat16* kpool, __nv_bfloat16* vpool, size_t layer_elems, int n_layers, const int* block_table,
                        int page_size, int n_kv, int head_dim, int n_tokens, cudaStream_t st);

// Host tier of the prefix cache (kv_host.cu): copies of whole pages, every layer's K and V, between the pool and pinned,
// mapped host pages.  to_host: kv_spill_kernel (pool -> host), else kv_fill_kernel (host -> pool).  One launch copies
// n_moves pages; no page, device or host, may appear twice in one launch.  Never launched with PDL, and neither kernel
// triggers its dependents early.
struct KvMoveArgs {
  const int2* moves = nullptr;       // [n_moves] (device page, host page), device memory
  int n_moves = 0;
  __nv_bfloat16* kpool = nullptr;    // [n_layers][n_pages][n_kv][page][head_dim]
  __nv_bfloat16* vpool = nullptr;
  size_t layer_elems = 0;            // elements of one layer of the pool
  uint4* host = nullptr;             // device view of the host pages: [host page][K|V][n_layers][n_kv][page][head_dim]
  int n_layers = 0;
  int blk_vec = 0;                   // one page of one layer (n_kv * page * head_dim bf16) in 16-byte units
};
int launch_kv_move(bool to_host, const KvMoveArgs& a, cudaStream_t st);

int launch_gather_kv(const __nv_bfloat16* pool_layer, const int* block_table, int page_size, int n_kv, int head_dim, int t0, int n,
                     float* out, cudaStream_t st);

// ---- persistent whole-stack decode kernel (decode_mega.cu) ----------------------------------------
struct MegaLayer {
  const __nv_bfloat16* wqkv; const __nv_bfloat16* wo; const __nv_bfloat16* wgu; const __nv_bfloat16* wdown;
  const float* attn_norm; const float* ffn_norm;
  __nv_bfloat16* kpool; __nv_bfloat16* vpool;
};
struct MegaArgs {
  const MegaLayer* layers = nullptr;   // device array [n_layers]
  int n_layers = 0, q_dim = 0, qkv_dim = 0, n_heads = 0, n_kv = 0, nsplit = 0;
  float eps = 0.f;
  const float2* rope = nullptr;
  const int* pos = nullptr;
  const int* block_tables = nullptr;
  int bt_stride = 0;
  const int* slots = nullptr;          // slots[0] is the sequence slot
  float* h = nullptr;                  // [slot][d] residual stream (in: embedding, out: final hidden)
  float* q = nullptr;                  // [slot][q_dim]
  float* attn_x = nullptr;             // [slot][q_dim]
  float* act = nullptr;                // [slot][d_ff]
  float* part = nullptr;               // attention partials
  unsigned* bars = nullptr;            // [n_layers * 6] grid-barrier counters, zero at kernel start
  unsigned* tile_ctr = nullptr;        // [n_layers * 4] dynamic tile-scheduler counters, zero at kernel start
  unsigned* pf_ctr = nullptr;          // L2 lookahead frontier (one counter, zero at kernel start); nullptr = off
  int pause_in_barrier = 0;            // producer issues no new copies while the consumers sit in a grid barrier
  int max_flight = 6;                  // cap on bulk copies in flight per CTA (<= ring slots)
  int pf_min = 296, pf_budget = 0;     // lookahead window in tiles ahead of a CTA's own demand position
  long long* tl = nullptr;             // debug: [n_layers][16] globaltimer stamps of CTA tl_cta
  int tl_cta = 0;
  long long kv_layer_rows = 0;         // rows of one layer in the KV tensor maps (= n_pages * n_kv * page)
  alignas(64) CUtensorMap kmap;        // whole K pool as [L * n_pages * n_kv * page][head_dim], box {64, 32}, 128B swizzle
  alignas(64) CUtensorMap vmap;
};
bool make_tmap_2d_bf16(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_cols, uint32_t box_rows);
bool mega_supported(int d, int d_ff, int head_dim, int n_heads, int n_kv, int page_size, int nsplit);
bool mega_prepare_device();   // per device: shared-memory opt-in + "one CTA per SM fits" (call with the device current)
int launch_decode_mega(const MegaArgs& a, cudaStream_t st);

bool gemv_variant_supported(int variant, int N, int K);
int sm_count();
// "done once" flag per (call site, current device): function attributes (dynamic shared memory limit, carve-out) belong to a
// device's context, so a process that opens a second GPU must set them again (ADVICE r1)
struct PerDeviceOnce {
  bool done[64] = {};
  bool* slot() { int d = 0; cudaGetDevice(&d); return &done[d & 63]; }
  bool pending() { return !*slot(); }
  void mark() { *slot() = true; }
};

// ---- prefill path (prefill_kernels.cu / gemm_wgmma.cu) -----------------------------------------
// X bf16 [T][K] row-major, W bf16 [N][K] row-major -> Y fp32 [T][N] (+= resid when resid != nullptr)
// k_splits > 1: split-K, partial s is written to Y + s*T*N (no residual); the consumer sums the partials
int launch_gemm_bf16(const __nv_bfloat16* X, const __nv_bfloat16* W, float* Y, const float* resid, int T, int N, int K,
                     cudaStream_t st, int k_splits = 1, bool pdl = false);
bool gemm_tc_supported(int T, int N, int K);
bool gemm_splits_supported(int K, int k_splits);   // the split-K counts launch_gemm_bf16 takes (no residual)
// gate|up projection with the SiLU epilogue (gemm_wgmma.cu): W rows interleaved (2i gate, 2i+1 up) -> act[t][i] =
// bf16(silu(g) * u), act row stride ld_act; the fp32 result never leaves the SM
int launch_gemm_bf16_silu(const __nv_bfloat16* X, const __nv_bfloat16* W, int T, int N, int K, __nv_bfloat16* act, int ld_act, cudaStream_t st);
// xn[t] = bf16(rmsnorm(h[t]) * gain)
int launch_rmsnorm_bf16(const float* h, const float* gain, float eps, __nv_bfloat16* out, int T, int d, cudaStream_t st);
// rope q,k of T tokens starting at pos0; q -> bf16 [T][H][D]; k,v -> paged cache (bf16) and optional dense copies
// qkv columns arrive rope-pair-interleaved (the GEMM uses the same permuted wqkv rows)
struct RopeScatterArgs {
  const float* qkv; int qkv_stride; const float2* rope; int pos0; int T;
  __nv_bfloat16* q_out;              // [T][H*D]
  __nv_bfloat16* kpool; __nv_bfloat16* vpool; const int* block_table; int page_size;
  int n_heads, n_kv, head_dim;
  int n_split = 1; size_t split_stride = 0;   // qkv = sum of n_split split-K partials, split_stride floats apart (fixed order)
  // optional per-row (sequence, position) map of a pass over several sequences: row t goes to position row_pos[t] of
  // sequence row_seq[t], whose block table is block_table + row_seq[t] * bt_stride (pos0 unused).  nullptr: one sequence.
  const int* row_seq = nullptr; const int* row_pos = nullptr; int bt_stride = 0;
};
int launch_rope_scatter(const RopeScatterArgs& a, cudaStream_t st);
// causal attention of T new tokens (positions pos0..pos0+T-1) against the paged cache
struct AttnPrefillArgs {
  const __nv_bfloat16* q;            // [T][H*D] roped
  const __nv_bfloat16* kpool; const __nv_bfloat16* vpool; const int* block_table; int page_size;
  int pos0, T, n_heads, n_kv, head_dim;
  __nv_bfloat16* out;                // [T][H*D]
};
int launch_attn_prefill(const AttnPrefillArgs& a, cudaStream_t st);
// wgmma variant (attn_prefill_tc.cu): head_dim 128, page 32; kmap / vmap = pool-wide 2-D tensor maps (box {64, 32})
bool attn_prefill_tc_supported(int n_heads, int n_kv, int head_dim, int page_size, int pos0, int T);
int launch_attn_prefill_tc(const AttnPrefillArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st);
// multi-row split-KV attention (attn_verify_tc.cu): segment s holds len_s cached tokens and R_s <= kVerifyMaxRows new rows at
// positions len_s .. len_s + R_s - 1 (their K/V already in the pages); row r sees keys < len_s + r + 1
constexpr int kVerifyMaxRows = 16;
struct AttnVerifyArgs {
  const __nv_bfloat16* q = nullptr;      // [rows][q_stride] roped
  int q_stride = 0;
  const int* segs = nullptr;             // [n_segs][8]: block-table row, first row, rows R, cached len, partial offset (floats), splits, 0, 0
  const int* block_tables = nullptr;     // [seq][bt_stride]
  int bt_stride = 0;
  __nv_bfloat16* out = nullptr;          // [rows][out_stride]
  int out_stride = 0;
  float* part = nullptr;                 // per segment at its offset: [n_kv][splits][4 R][head_dim + 2]
  unsigned* counters = nullptr;          // [n_segs][n_kv], zero between launches (the kernel re-arms them)
  int n_segs = 0, n_heads = 0, n_kv = 0, head_dim = 0, page_size = 0;
  int nsplit = 1;                        // grid splits: the largest of the segments' split counts
  int split_pages = 0;                   // > 0: every split covers this many pages; 0: a segment's pages spread over its splits
};
bool attn_verify_tc_supported(int n_heads, int n_kv, int head_dim, int page_size);
int attn_verify_max_splits();
int launch_attn_verify_tc(const AttnVerifyArgs& a, const CUtensorMap& kmap, const CUtensorMap& vmap, long long layer_row0, cudaStream_t st);
// ---- batched decode glue (batch_kernels.cu) ------------------------------------------------------
int launch_batch_resid_norm(float* h, int d, const float* ypart, int n_split, int B, const float* gain, float eps, __nv_bfloat16* xn,
                            const int* slots, cudaStream_t st, bool pdl = false);
int launch_batch_rope_append(const float* ypart, int n_split, int B, const QkvEpi& e, float* q_out, int q_stride, const int* slots,
                             cudaStream_t st, bool pdl = false);
int launch_batch_silu(const float* ypart, int n_split, int B, int d_ff, __nv_bfloat16* act, cudaStream_t st, bool pdl = false);
int launch_batch_scatter_rows(const float* y, int n, float* out, int out_stride, const int* slots, int B, cudaStream_t st);
int launch_embed_rows(const __nv_bfloat16* table, int d, const int* ids_dev, float* h, int T, cudaStream_t st);

}  // namespace cl
