// prefill.cu — prompt (prefill) path of the engine.  Prompts of up to 256 tokens take the short-prompt path (split-K
// projections, prefill_small); longer ones go through the tile path: prefill_pass runs T rows through wgmma GEMMs
// (gemm_wgmma.cu) and the causal paged attention (prefill_kernels.cu / attn_prefill_tc.cu), once per chunk of up to
// prefill_chunk_tokens_ tokens (prefill_chunked) or once for several prompts (prefill_multi).  The last position's logits
// come from the decode LM head, so that prefill and decode share one logits/argmax tail.  Also: cl_op_gemm_bf16 /
// cl_op_gemm_bf16_epi / cl_op_attn_prefill*.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "engine.h"

namespace cl {

bool Engine::prefill_path_ok() const { return gemm_tc_supported(16, cfg.d_model, cfg.d_model); }

// split-K rule shared with the batched decode step (engine.cu)
int pick_splits_public(int n_rows, int K);

// A prefill workspace buffer: lives until the engine dies (allocs_).  Out of memory is reported, and the CUDA error state
// cleared, so that later launches do not see it.
template <typename T>
static int ws_alloc(std::vector<void*>& allocs, T*& p, size_t bytes) {
  void* v = nullptr;
  if (cudaMalloc(&v, bytes) != cudaSuccess) { cudaGetLastError(); set_last_error("prefill workspace: out of memory"); return CL_ERR_OOM; }
  allocs.push_back(v);
  p = reinterpret_cast<T*>(v);
  return CL_OK;
}

// Causal attention of one prefill segment in layer l: the wgmma kernel where it applies (head_dim 128, page 32, the pool's
// tensor maps), the mma.sync kernel otherwise.
int Engine::attn_prefill(const AttnPrefillArgs& a, int l, int& launches, LaunchProfiler& prof) {
  if (have_kv_maps_ && attn_prefill_tc_supported(a.n_heads, a.n_kv, a.head_dim, a.page_size, a.pos0, a.T))
    CL_LAUNCH(launch_attn_prefill_tc(a, kmap_, vmap_, (long long)l * n_pages_ * cfg.n_kv_heads * page_size_, stream_));
  else
    CL_LAUNCH(launch_attn_prefill(a, stream_));
  return CL_OK;
}

// Short prompts (prefill_min_tokens_ <= n <= 256, e.g. a 128-token chat): one token tile per W row tile means only
// N/128 CTAs stream the weights of a projection (48 for q|k|v, 32 for o and down), far below the
// machine's weight-streaming rate.  Same recipe as the batched decode step: split-K so that all SMs share every
// projection's weights, fp32 partials in a workspace, the per-row glue kernels (batch_kernels.cu) fold them in fixed
// order into the residual stream / RoPE / SiLU.  Rows are the prompt's tokens, attention is the causal prefill kernel.
int Engine::prefill_small(cl_seq_t s, const int32_t* ids, int n, float* logits_out) {
  auto& q = seqs_[s];
  int rc = ensure_capacity(s, q.len + n);
  if (rc) return rc;
  if ((rc = ensure_small_ws())) return rc;
  const int d = cfg.d_model;
  CL_CUDA_OK(cudaMemcpyAsync(d_prompt_, ids, (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
  int launches = 0;
  LaunchProfiler prof(stream_, "CL_PREFILL_PROFILE");
  const PrefillSegment seg{s, 0, n, q.len};
  if ((rc = small_pass(&seg, 1, d_prompt_, n, nullptr, nullptr, launches, prof))) return rc;
  // the last row -> the slot's residual row, then the shared tail (its own final norm + GEMV head)
  CL_CUDA_OK(cudaMemcpyAsync(d_h_ + (size_t)s * d, sws_->h + (size_t)(n - 1) * d, (size_t)d * 4, cudaMemcpyDeviceToDevice, stream_));
  const int last_pos = q.len + n - 1;
  CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &last_pos, 4, cudaMemcpyHostToDevice, stream_));
  rc = set_single_slot(s);
  if (rc) return rc;
  CL_LAUNCH(enqueue_lm_head(1, false));
  CL_LAUNCH(enqueue_step_tail(1, false));
  prof.report("prefill profile", 32, "short-prompt path, " + std::to_string(n) + " tokens");
  launches_ += launches;
  seq_advance(s, ids, n, n);
  if (logits_out) return read_logits(s, logits_out);
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  return CL_OK;
}

int Engine::ensure_small_ws() {
  if (sws_) return CL_OK;
  const int d = cfg.d_model, F = cfg.d_ff;
  const int s_qkv = pick_splits_public(qkv_dim_, d), s_o = pick_splits_public(d, q_dim_), s_gu = pick_splits_public(2 * F, d), s_dn = pick_splits_public(d, F);
  sws_.reset(new SmallPrefillWs());
  const size_t Tm = 256;
  size_t part = 0;
  part = std::max(part, (size_t)s_qkv * Tm * qkv_dim_);
  part = std::max(part, (size_t)s_o * Tm * d);
  part = std::max(part, (size_t)s_gu * Tm * 2 * F);
  part = std::max(part, (size_t)s_dn * Tm * d);
  int rc;
  if ((rc = ws_alloc(allocs_, sws_->part, part * 4)) || (rc = ws_alloc(allocs_, sws_->xn, Tm * d * 2)) ||
      (rc = ws_alloc(allocs_, sws_->q, Tm * q_dim_ * 2)) || (rc = ws_alloc(allocs_, sws_->attn, Tm * q_dim_ * 2)) ||
      (rc = ws_alloc(allocs_, sws_->h, Tm * d * 4)) || (rc = ws_alloc(allocs_, sws_->act, Tm * F * 2)) ||
      (rc = ws_alloc(allocs_, sws_->iota, Tm * 4))) { sws_.reset(); return rc; }
  std::vector<int> io(Tm);
  for (size_t i = 0; i < Tm; ++i) io[i] = (int)i;
  CL_CUDA_OK(cudaMemcpy(sws_->iota, io.data(), Tm * 4, cudaMemcpyHostToDevice));
  return CL_OK;
}

// One split-K pass over T <= 256 rows, token ids at ids (device): embedding, every layer (K/V written into the sequences'
// pages), and the final norm.  The rows are the segments' tokens, back to back.  Everything row-wise runs once over all
// rows; RoPE + cache scatter runs in one launch (through row_map when it is given).  The causal attention runs in one launch
// of the multi-row split-KV kernel (attn_verify_tc.cu) when seg_table is given and the shape is one it takes, else per
// segment (attn_prefill).  Leaves the final residual rows in sws_->h and their normalised bf16 rows, the LM head's input,
// in sws_->xn.  A row's results depend only on its own segment's rows before it.  prefill_small and the verify passes of
// speculative decoding (verify_batch; without the segment table: one segment, no map or table) run it.
int Engine::small_pass(const PrefillSegment* segs, int n_segs, const int* ids, int T, const int* row_map, const int* seg_table,
                       int& launches, LaunchProfiler& prof) {
  const int d = cfg.d_model, F = cfg.d_ff;
  const int s_qkv = pick_splits_public(qkv_dim_, d), s_o = pick_splits_public(d, q_dim_), s_gu = pick_splits_public(2 * F, d), s_dn = pick_splits_public(d, F);
  SmallPrefillWs& w = *sws_;
  int rc;
  AttnVerifyArgs va;
  const bool multi_row = seg_table && have_kv_maps_ && attn_verify_tc_supported(cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, page_size_);
  if (multi_row) {
    va.q = w.q; va.q_stride = q_dim_; va.segs = seg_table; va.block_tables = d_bt_; va.bt_stride = max_pages_per_seq_;
    va.out = w.attn; va.out_stride = q_dim_; va.part = spec_->attn_part; va.counters = spec_->attn_cnt;
    va.n_segs = n_segs; va.n_heads = cfg.n_heads; va.n_kv = cfg.n_kv_heads; va.head_dim = cfg.head_dim; va.page_size = page_size_;
    va.split_pages = verify_split_pages();
    va.nsplit = 1;
    for (int i = 0; i < n_segs; ++i)
      va.nsplit = std::max(va.nsplit, ((segs[i].pos0 + segs[i].n + page_size_ - 1) / page_size_ + va.split_pages - 1) / va.split_pages);
  }
  // programmatic dependent launch between the GEMMs and the per-row glue kernels, as in the batched decode step (the two
  // prefill kernels in between are launched normally and order the stream)
  const bool bp = use_pdl_;
  CL_LAUNCH(launch_embed_rows(embed_, d, ids, w.h, T, stream_));
  const float* pending = nullptr;   // split-K partials of the previous residual projection, folded in by the next norm
  int pending_s = 0;
  for (int l = 0; l < cfg.n_layers; ++l) {
    const auto& L = layers_[l];
    CL_LAUNCH(launch_batch_resid_norm(w.h, d, pending, pending_s, T, L.attn_norm, cfg.rms_eps, w.xn, w.iota, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.xn, L.wqkv, w.part, nullptr, T, qkv_dim_, d, stream_, s_qkv, bp));
    RopeScatterArgs ra{w.part, qkv_dim_, rope_, segs[0].pos0, T, w.q, kpool_ + (size_t)l * kv_layer_elems_, vpool_ + (size_t)l * kv_layer_elems_,
                       d_bt_ + (row_map ? 0 : (size_t)segs[0].seq * max_pages_per_seq_), page_size_, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim};
    ra.n_split = s_qkv; ra.split_stride = (size_t)T * qkv_dim_;
    if (row_map) { ra.row_seq = row_map; ra.row_pos = row_map + T; ra.bt_stride = max_pages_per_seq_; }
    CL_LAUNCH(launch_rope_scatter(ra, stream_));
    if (multi_row)
      CL_LAUNCH(launch_attn_verify_tc(va, kmap_, vmap_, (long long)l * n_pages_ * cfg.n_kv_heads * page_size_, stream_));
    for (int i = 0; i < n_segs && !multi_row; ++i) {
      const PrefillSegment& g = segs[i];
      AttnPrefillArgs aa{w.q + (size_t)g.row0 * q_dim_, kpool_ + (size_t)l * kv_layer_elems_, vpool_ + (size_t)l * kv_layer_elems_,
                         d_bt_ + (size_t)g.seq * max_pages_per_seq_, page_size_, g.pos0, g.n, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim,
                         w.attn + (size_t)g.row0 * q_dim_};
      if ((rc = attn_prefill(aa, l, launches, prof))) return rc;
    }
    CL_LAUNCH(launch_gemm_bf16(w.attn, L.wo, w.part, nullptr, T, d, q_dim_, stream_, s_o, bp));
    CL_LAUNCH(launch_batch_resid_norm(w.h, d, w.part, s_o, T, L.ffn_norm, cfg.rms_eps, w.xn, w.iota, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.xn, L.wgu, w.part, nullptr, T, 2 * F, d, stream_, s_gu, bp));
    CL_LAUNCH(launch_batch_silu(w.part, s_gu, T, F, w.act, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.act, L.wdown, w.part, nullptr, T, d, F, stream_, s_dn, bp));
    pending = w.part; pending_s = s_dn;
  }
  // fold the last down-projection into the residual rows; the final-norm rows it also writes feed the verify pass's head
  CL_LAUNCH(launch_batch_resid_norm(w.h, d, pending, pending_s, T, final_norm_, cfg.rms_eps, w.xn, w.iota, stream_, bp));
  return CL_OK;
}

int Engine::ensure_spec_ws() {
  if (spec_) return CL_OK;
  const size_t R = kSpecMaxRows, V = cfg.vocab_size;
  int rc;
  spec_.reset(new SpecWs());
  if ((rc = ws_alloc(allocs_, spec_->logits, R * V * 4)) || (rc = ws_alloc(allocs_, spec_->choice, R * 4)) ||
      (rc = ws_alloc(allocs_, spec_->part_val, R * kTailBlocks * 4)) || (rc = ws_alloc(allocs_, spec_->part_idx, R * kTailBlocks * 4)) ||
      (rc = ws_alloc(allocs_, spec_->counters, R * 4)) || (rc = ws_alloc(allocs_, spec_->cand, R * kTailBlocks * kSampleTopKMax * 8)) ||
      (rc = ws_alloc(allocs_, spec_->out, 2 * R * 4)) || (rc = ws_alloc(allocs_, spec_->row_map, 2 * R * 4)) ||
      (rc = ws_alloc(allocs_, spec_->segs, R * 8 * 4)) || (rc = ws_alloc(allocs_, spec_->attn_cnt, R * cfg.n_kv_heads * 4)) ||
      (rc = ws_alloc(allocs_, spec_->lp_part, R * kTailBlocks * sizeof(float2))) ||
      (rc = ws_alloc(allocs_, spec_->lp_cand, R * kTailBlocks * kLogprobTopMax * 8)) || (rc = ws_alloc(allocs_, spec_->lp_cnt, R * 4)) ||
      (rc = ws_alloc(allocs_, spec_->lp_rows, R * sizeof(LogprobRecord)))) { spec_.reset(); return rc; }
  // the multi-row attention's split partials: at most 4 query rows per pass row, per kv head and split
  if (attn_verify_tc_supported(cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, page_size_)) {
    const size_t max_splits = (max_pages_per_seq_ + verify_split_pages() - 1) / verify_split_pages();
    if ((rc = ws_alloc(allocs_, spec_->attn_part, R * 4 * cfg.n_kv_heads * max_splits * (cfg.head_dim + 2) * 4))) { spec_.reset(); return rc; }
  }
  CL_CUDA_OK(cudaMemsetAsync(spec_->counters, 0, R * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(spec_->lp_cnt, 0, R * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(spec_->attn_cnt, 0, R * cfg.n_kv_heads * 4, stream_));
  return CL_OK;
}

// Every split of the multi-row attention covers 8 pages (256 tokens at page 32), more only when a sequence of max_seq_len
// would need more than the kernel's 64 splits.  A segment's split plan thus depends on its own length alone, so a sequence's
// attention rows are the same bits whatever other sequences share the pass.
int Engine::verify_split_pages() const {
  return std::max(8, (max_pages_per_seq_ + attn_verify_max_splits() - 1) / attn_verify_max_splits());
}

// The spec tail of one segment of a verify pass: its rows' logits, inputs and tail buffers, and its 1 + n ints of output at
// out_off.  The segment's sequence is its slot; the sequence's cached length is g.pos0.
SpecTailArgs Engine::spec_tail_args(const PrefillSegment& g, int out_off) const {
  const size_t r0 = g.row0;
  SpecTailArgs t;
  t.logits = spec_->logits + r0 * cfg.vocab_size; t.vocab = cfg.vocab_size; t.T = g.n; t.slot = g.seq; t.len = g.pos0;
  t.inputs = d_prompt_ + r0; t.choice = spec_->choice + r0;
  t.part_val = spec_->part_val + r0 * kTailBlocks; t.part_idx = spec_->part_idx + r0 * kTailBlocks; t.counters = spec_->counters + r0;
  t.cand = spec_->cand + r0 * kTailBlocks * kSampleTopKMax;
  t.tok = d_tok_; t.pos = d_pos_; t.out = spec_->out + out_off;
  t.sample.mode = d_samp_mode_; t.sample.par = d_samp_par_; t.sample.step = d_samp_step_; t.sample.hist = d_samp_hist_;
  t.sample.hist_len = d_samp_hlen_;
  t.lp.top_n = d_lp_n_; t.lp.part = spec_->lp_part + r0 * kTailBlocks; t.lp.cand = spec_->lp_cand + r0 * kTailBlocks * kLogprobTopMax;
  t.lp.counters = spec_->lp_cnt + r0; t.lp.last = spec_->lp_rows + r0;
  return t;
}

bool Engine::spec_path_ok() const {
  return prefill_path_ok() && cfg.d_model <= 8192 && cfg.d_model % 4 == 0 && gemm_tc_supported(kSpecMaxDraft + 1, cfg.vocab_size, cfg.d_model);
}

// Verify pass of speculative decoding over n_seqs distinct sequences (include/clengine.h, cl_decode_verify and
// cl_decode_verify_batch): sequence i is segment i of one small_pass, rows x0[i], d_1 .. d_{k_i} at positions len_i ..
// len_i + k_i.  One GEMM computes the logits of all rows, then each segment runs the spec tail (row r's step-tail choice
// y_{r+1}) and the accept kernel (a = longest run with y_j == d_j; next input y_{a+1}; an armed slot's history and RNG step
// advanced as a + 1 steps would) on its own rows and slot.  Only {a + 1, y_1 .. y_{a+1}} of each sequence is read back.
// seg_table: small_pass gets the row map and the segment table, so the attention runs in the multi-row kernel where the
// shape allows it; without it (one sequence only) the segment goes through attn_prefill, as cl_decode_verify always has.
// Every row's computation is the one it has in a pass of its sequence alone, so each sequence's ids, logits and K/V equal
// verifying it alone.  Everything is checked before anything is enqueued; on an error no sequence's length changes.
// Rejected rows leave K/V at positions >= the new length, on the sequence's private pages.
int Engine::verify_batch(const cl_seq_t* ss, int n_seqs, const int32_t* x0, const int32_t* drafts, const int* ks, int32_t* ids_out,
                         int* n_out, float* logits_out, bool seg_table) {
  if (n_seqs < 1 || !ss || !x0 || !ks || !ids_out || !n_out) { set_last_error("verify_batch: bad arguments"); return CL_ERR_INVALID_ARG; }
  if (!spec_path_ok()) { set_last_error("verify: the model shape has no tensor-core split-K path"); return CL_ERR_INVALID_ARG; }
  const int V = cfg.vocab_size, d = cfg.d_model;
  std::vector<PrefillSegment> segs(n_seqs);
  std::vector<int32_t> in;
  int T = 0, n_drafted = 0;
  for (int i = 0; i < n_seqs; ++i) {
    const int s = ss[i];
    if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
    for (int j = 0; j < i; ++j) if (ss[j] == s) { set_last_error("duplicate sequence in batch"); return CL_ERR_INVALID_ARG; }
    if (ks[i] < 0 || ks[i] > kSpecMaxDraft || (ks[i] > 0 && !drafts)) { set_last_error("verify: k must be 0..15"); return CL_ERR_INVALID_ARG; }
    if (T + ks[i] + 1 > kSpecMaxRows) { set_last_error("verify: more than 128 rows in one pass"); return CL_ERR_INVALID_ARG; }
    segs[i] = PrefillSegment{s, T, ks[i] + 1, seqs_[s].len};
    in.push_back(x0[i]);
    in.insert(in.end(), drafts + n_drafted, drafts + n_drafted + ks[i]);
    T += ks[i] + 1;
    n_drafted += ks[i];
  }
  for (int t = 0; t < T; ++t)
    if (in[t] < 0 || in[t] >= V) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
  for (const auto& g : segs)
    if (g.pos0 + g.n > cfg.max_seq_len) { set_last_error("sequence exceeds max_seq_len"); return CL_ERR_TOO_LONG; }
  int rc;
  for (const auto& g : segs)
    if ((rc = ensure_capacity(g.seq, g.pos0 + g.n))) return rc;
  if ((rc = ensure_small_ws()) || (rc = ensure_spec_ws())) return rc;
  CL_CUDA_OK(cudaMemcpyAsync(d_prompt_, in.data(), (size_t)T * 4, cudaMemcpyHostToDevice, stream_));
  if (seg_table) {
    std::vector<int> row_map(2 * (size_t)T), table(8 * (size_t)n_seqs, 0);
    const int split_pages = verify_split_pages();
    long long part_off = 0;
    for (int i = 0; i < n_seqs; ++i) {
      const PrefillSegment& g = segs[i];
      for (int r = 0; r < g.n; ++r) { row_map[g.row0 + r] = g.seq; row_map[T + g.row0 + r] = g.pos0 + r; }
      const int pages = (g.pos0 + g.n + page_size_ - 1) / page_size_, ns = (pages + split_pages - 1) / split_pages;
      int* e = &table[8 * (size_t)i];
      e[0] = g.seq; e[1] = g.row0; e[2] = g.n; e[3] = g.pos0; e[4] = (int)part_off; e[5] = ns;
      if (ns > 1) part_off += (long long)cfg.n_kv_heads * ns * 4 * g.n * (cfg.head_dim + 2);
    }
    CL_CUDA_OK(cudaMemcpyAsync(spec_->row_map, row_map.data(), row_map.size() * 4, cudaMemcpyHostToDevice, stream_));
    CL_CUDA_OK(cudaMemcpyAsync(spec_->segs, table.data(), table.size() * 4, cudaMemcpyHostToDevice, stream_));
  }
  int launches = 0;
  LaunchProfiler prof(stream_, "CL_PREFILL_PROFILE");
  if ((rc = small_pass(segs.data(), n_seqs, d_prompt_, T, seg_table ? spec_->row_map : nullptr, seg_table ? spec_->segs : nullptr,
                       launches, prof)))
    return rc;
  CL_LAUNCH(launch_gemm_bf16(sws_->xn, lm_head_, spec_->logits, nullptr, T, V, d, stream_, 1, false));
  // segment i's output {n_i, ids} sits at out[row0_i + i]: one int more per segment than its rows
  for (int i = 0; i < n_seqs; ++i) CL_LAUNCH(launch_spec_tail(spec_tail_args(segs[i], segs[i].row0 + i), stream_, use_pdl_));
  CL_CUDA_OK(cudaMemcpyAsync(h_ids_pinned_, spec_->out, (size_t)(T + n_seqs) * 4, cudaMemcpyDeviceToHost, stream_));
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  prof.report("prefill profile", 32, "verify pass, " + std::to_string(n_seqs) + " sequences, " + std::to_string(T) + " rows");
  launches_ += launches;
  for (int i = 0; i < n_seqs; ++i) {
    const int n = h_ids_pinned_[segs[i].row0 + i];
    if (n < 1 || n > segs[i].n) { set_last_error("verify: accept kernel returned a bad count"); return CL_ERR_INTERNAL; }
  }
  // the records of a sequence's emitted ids y_1 .. y_{a+1} are those of its leading rows
  if (std::any_of(ss, ss + n_seqs, [&](cl_seq_t s) { return lp_n_[s] >= 0; }))
    CL_CUDA_OK(cudaMemcpy(h_lp_pinned_, spec_->lp_rows, (size_t)T * sizeof(LogprobRecord), cudaMemcpyDeviceToHost));
  int accepted = 0, emitted = 0;
  for (int i = 0; i < n_seqs; ++i) {
    const PrefillSegment& g = segs[i];
    const int n = h_ids_pinned_[g.row0 + i];
    if (lp_n_[g.seq] >= 0) seqs_[g.seq].lps.insert(seqs_[g.seq].lps.end(), h_lp_pinned_ + g.row0, h_lp_pinned_ + g.row0 + n);
    memcpy(ids_out + g.row0, h_ids_pinned_ + g.row0 + i + 1, (size_t)n * 4);
    n_out[i] = n;
    seq_advance(g.seq, in.data() + g.row0, n, n);   // x0, d1 .. da: only accepted tokens join the history and the prefix cache
    accepted += n - 1; emitted += n;
  }
  spec_passes_ += n_seqs; spec_drafted_ += n_drafted; spec_accepted_ += accepted; spec_emitted_ += emitted;
  if (n_seqs > 1) spec_multi_passes_++;
  if (logits_out) CL_CUDA_OK(cudaMemcpy(logits_out, spec_->logits, (size_t)T * V * 4, cudaMemcpyDeviceToHost));
  return CL_OK;
}

// cl_decode_verify: one sequence with 1..15 drafts, verified without the segment table
int Engine::decode_verify(cl_seq_t s, int32_t x0, const int32_t* draft, int k, const cl_sampling* sp, uint64_t step0, int32_t* ids_out,
                          int* n_out, float* logits_out) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (k < 1 || k > kSpecMaxDraft) { set_last_error("verify: k must be 1..15"); return CL_ERR_INVALID_ARG; }
  return decode_verify_batch(&s, 1, &x0, draft, &k, sp, &step0, ids_out, n_out, logits_out, false);
}

// cl_decode_verify_batch (seg_table = true) and cl_decode_verify: verify_batch with the device sampler armed for the pass
// on the sequences whose sp[i] draws
int Engine::decode_verify_batch(const cl_seq_t* ss, int n_seqs, const int32_t* x0, const int32_t* drafts, const int* ks,
                                const cl_sampling* sp, const uint64_t* step0, int32_t* ids_out, int* n_out, float* logits_out,
                                bool seg_table) {
  if (n_seqs < 1 || !ss) { set_last_error("verify_batch: bad arguments"); return CL_ERR_INVALID_ARG; }
  for (int i = 0; i < n_seqs; ++i) {
    if (ss[i] < 0 || ss[i] >= max_seqs_ || !seqs_[ss[i]].live) return CL_ERR_BAD_SEQ;
    if (sp && sp[i].temperature > 0.f && !device_sampling_ok(sp[i], cfg.vocab_size)) {
      set_last_error("sampling settings need the host sampler");
      return CL_ERR_INVALID_ARG;
    }
  }
  std::vector<cl_seq_t> armed;
  int rc = CL_OK;
  for (int i = 0; i < n_seqs && rc == CL_OK && sp; ++i) {
    if (!(sp[i].temperature > 0.f)) continue;
    const cl_seq_t s = ss[i];
    if (std::find(armed.begin(), armed.end(), s) != armed.end()) continue;   // a duplicate: verify_batch refuses it
    rc = arm_sampling(s, sp[i], step0 ? step0[i] : 0, seqs_[s].history.data(), (int)seqs_[s].history.size());
    if (rc == CL_OK) armed.push_back(s);
  }
  if (rc == CL_OK) rc = verify_batch(ss, n_seqs, x0, drafts, ks, ids_out, n_out, logits_out, seg_table);
  for (cl_seq_t s : armed) {
    const int r2 = disarm_sampling(s);
    if (rc == CL_OK) rc = r2;
  }
  return rc;
}

// (Re)allocate the tile-path workspace for passes of up to `tokens` rows; old buffers stay in allocs_ until the engine dies
// (grows at most once or twice).
int Engine::ensure_prefill_ws(int tokens) {
  const int d = cfg.d_model, F = cfg.d_ff;
  int rc;
  if (!pws_) pws_.reset(new PrefillWs());
  if (pws_->cap_tokens >= tokens) return CL_OK;
  const size_t T = (size_t)std::max(tokens, std::min(prefill_chunk_tokens_, cfg.max_seq_len));
  if ((rc = ws_alloc(allocs_, pws_->xn, T * d * 2)) || (rc = ws_alloc(allocs_, pws_->qkv, T * qkv_dim_ * 4)) ||
      (rc = ws_alloc(allocs_, pws_->q, T * q_dim_ * 2)) || (rc = ws_alloc(allocs_, pws_->attn, T * q_dim_ * 2)) ||
      (rc = ws_alloc(allocs_, pws_->h, T * d * 4)) || (rc = ws_alloc(allocs_, pws_->act, T * F * 2))) return rc;
  pws_->cap_tokens = (int)T;
  return CL_OK;
}

// One pass of the tile path over T rows whose token ids are at ids (device): embedding and every layer, leaving the final
// residual rows in pws_->h.  The rows are the segments' tokens, back to back.  Everything row-wise (RMSNorm, the four
// GEMMs, SiLU in the gate|up epilogue) runs once over all T rows; RoPE + cache scatter and the causal attention run per
// segment, at its sequence's positions and into its pages.  A row's results therefore do not depend on the other rows.
int Engine::prefill_pass(const PrefillSegment* segs, int n_segs, const int* ids, int T, int& launches, LaunchProfiler& prof) {
  const int d = cfg.d_model, F = cfg.d_ff;
  PrefillWs& w = *pws_;
  int rc;
  CL_LAUNCH(launch_embed_rows(embed_, d, ids, w.h, T, stream_));
  for (int l = 0; l < cfg.n_layers; ++l) {
    const auto& L = layers_[l];
    __nv_bfloat16* kp = kpool_ + (size_t)l * kv_layer_elems_;
    __nv_bfloat16* vp = vpool_ + (size_t)l * kv_layer_elems_;
    CL_LAUNCH(launch_rmsnorm_bf16(w.h, L.attn_norm, cfg.rms_eps, w.xn, T, d, stream_));
    CL_LAUNCH(launch_gemm_bf16(w.xn, L.wqkv, w.qkv, nullptr, T, qkv_dim_, d, stream_));
    for (int i = 0; i < n_segs; ++i) {
      const PrefillSegment& g = segs[i];
      RopeScatterArgs ra{w.qkv + (size_t)g.row0 * qkv_dim_, qkv_dim_, rope_, g.pos0, g.n, w.q + (size_t)g.row0 * q_dim_, kp, vp,
                         d_bt_ + (size_t)g.seq * max_pages_per_seq_, page_size_, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim};
      CL_LAUNCH(launch_rope_scatter(ra, stream_));
    }
    for (int i = 0; i < n_segs; ++i) {
      const PrefillSegment& g = segs[i];
      AttnPrefillArgs aa{w.q + (size_t)g.row0 * q_dim_, kp, vp, d_bt_ + (size_t)g.seq * max_pages_per_seq_, page_size_, g.pos0, g.n,
                         cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, w.attn + (size_t)g.row0 * q_dim_};
      if ((rc = attn_prefill(aa, l, launches, prof))) return rc;
    }
    CL_LAUNCH(launch_gemm_bf16(w.attn, L.wo, w.h, w.h, T, d, q_dim_, stream_));
    CL_LAUNCH(launch_rmsnorm_bf16(w.h, L.ffn_norm, cfg.rms_eps, w.xn, T, d, stream_));
    CL_LAUNCH(launch_gemm_bf16_silu(w.xn, L.wgu, T, 2 * F, d, w.act, F, stream_));
    CL_LAUNCH(launch_gemm_bf16(w.act, L.wdown, w.h, w.h, T, d, F, stream_));
  }
  return CL_OK;
}

int Engine::prefill_chunked(cl_seq_t s, const int32_t* ids, int n, float* logits_out) {
  auto& q = seqs_[s];
  int rc = ensure_capacity(s, q.len + n);
  if (rc) return rc;
  const int d = cfg.d_model;
  if ((rc = ensure_prefill_ws(std::min(n, prefill_chunk_tokens_)))) return rc;
  PrefillWs& w = *pws_;
  CL_CUDA_OK(cudaMemcpyAsync(d_prompt_, ids, (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
  int launches = 0;
  LaunchProfiler prof(stream_, "CL_PREFILL_PROFILE");
  int T = 0;
  for (int c0 = 0; c0 < n; c0 += T) {
    T = std::min(w.cap_tokens, n - c0);
    const PrefillSegment seg{s, 0, T, q.len + c0};
    if ((rc = prefill_pass(&seg, 1, d_prompt_ + c0, T, launches, prof))) return rc;
  }
  // last position -> slot residual row, then the shared decode tail (final norm + LM head + argmax)
  CL_CUDA_OK(cudaMemcpyAsync(d_h_ + (size_t)s * d, w.h + (size_t)(T - 1) * d, (size_t)d * 4, cudaMemcpyDeviceToDevice, stream_));
  const int last_pos = q.len + n - 1;
  CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &last_pos, 4, cudaMemcpyHostToDevice, stream_));
  rc = set_single_slot(s);
  if (rc) return rc;
  CL_LAUNCH(enqueue_lm_head(1, false));
  CL_LAUNCH(enqueue_step_tail(1, false));
  prof.report("prefill profile", 32, "tile path, " + std::to_string(n) + " tokens");
  launches_ += launches;
  seq_advance(s, ids, n, n);
  if (logits_out) return read_logits(s, logits_out);
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  return CL_OK;
}


// Several prompts in ONE pass of the tile path (admission of a burst of short chats): each prompt is a segment of the
// pass, so every projection streams its weights once for all of them and runs on full tiles (the split-K short-prompt
// path streams all weights once per prompt).  The last row of every sequence goes through the batched LM head of the
// decode step (final norm + wgmma GEMM + argmax), which leaves d_tok_ / d_pos_ of every slot ready for the first decode
// step.  Cache contents are bit-identical to prefill_chunked on each prompt alone; the logits differ from its GEMV head
// by the summation order only (tests/test_gpu_prefill.py).
int Engine::prefill_multi(int n_seqs, const cl_seq_t* ss, const int32_t* const* ids, const int* lens, float* logits_out) {
  if (n_seqs <= 0 || !ss || !ids || !lens) { set_last_error("prefill_multi: bad arguments"); return CL_ERR_INVALID_ARG; }
  if (!prefill_path_ok() || !bws_ || n_seqs > max_batch_) { set_last_error("prefill_multi: tensor-core paths unavailable or more sequences than max_batch"); return CL_ERR_INVALID_ARG; }
  const int d = cfg.d_model, V = cfg.vocab_size;
  int total = 0, rc;
  for (int i = 0; i < n_seqs; ++i) {
    const int s = ss[i];
    if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
    for (int c = 0; c < i; ++c) if (ss[c] == s) { set_last_error("duplicate sequence in batch"); return CL_ERR_INVALID_ARG; }
    if (lens[i] <= 0 || !ids[i]) { set_last_error("empty prompt"); return CL_ERR_INVALID_ARG; }
    for (int t = 0; t < lens[i]; ++t)
      if (ids[i][t] < 0 || ids[i][t] >= V) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
    if (seqs_[s].len + lens[i] > cfg.max_seq_len) { set_last_error("sequence exceeds max_seq_len"); return CL_ERR_TOO_LONG; }
    total += lens[i];
  }
  if (total > prefill_chunk_tokens_ || total > prompt_cap_) { set_last_error("prefill_multi: more rows than one pass holds"); return CL_ERR_TOO_LONG; }
  for (int i = 0; i < n_seqs; ++i)
    if ((rc = ensure_capacity(ss[i], seqs_[ss[i]].len + lens[i]))) return rc;
  if ((rc = ensure_prefill_ws(total))) return rc;
  PrefillWs& w = *pws_;
  BatchWs& bw = *bws_;
  std::vector<int32_t> all((size_t)total);
  std::vector<PrefillSegment> segs(n_seqs);
  for (int i = 0, r = 0; i < n_seqs; r += lens[i], ++i) {
    memcpy(all.data() + r, ids[i], (size_t)lens[i] * 4);
    segs[i] = PrefillSegment{ss[i], r, lens[i], seqs_[ss[i]].len};
  }
  CL_CUDA_OK(cudaMemcpyAsync(d_prompt_, all.data(), (size_t)total * 4, cudaMemcpyHostToDevice, stream_));
  int launches = 0;
  LaunchProfiler prof(stream_, "CL_PREFILL_PROFILE");
  if ((rc = prefill_pass(segs.data(), n_seqs, d_prompt_, total, launches, prof))) return rc;
  // last row of every sequence -> its slot's residual row and position, then the decode step's batched head
  std::vector<int> slots(n_seqs);
  for (int i = 0; i < n_seqs; ++i) {
    const PrefillSegment& g = segs[i];
    const int last_pos = g.pos0 + g.n - 1;
    slots[i] = g.seq;
    CL_CUDA_OK(cudaMemcpyAsync(d_h_ + (size_t)g.seq * d, w.h + (size_t)(g.row0 + g.n - 1) * d, (size_t)d * 4, cudaMemcpyDeviceToDevice, stream_));
    CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + g.seq, &last_pos, 4, cudaMemcpyHostToDevice, stream_));
  }
  CL_CUDA_OK(cudaMemcpyAsync(d_slots_, slots.data(), (size_t)n_seqs * 4, cudaMemcpyHostToDevice, stream_));
  slots_dirty_ = true;
  last_single_slot_ = n_seqs == 1 ? slots[0] : -1;
  CL_LAUNCH(launch_batch_resid_norm(d_h_, d, nullptr, 0, n_seqs, final_norm_, cfg.rms_eps, bw.xn, d_slots_, stream_, false));
  CL_LAUNCH(launch_gemm_bf16(bw.xn, lm_head_, bw.logits, nullptr, n_seqs, V, d, stream_, 1, false));
  CL_LAUNCH(launch_batch_scatter_rows(bw.logits, V, d_logits_, V, d_slots_, n_seqs, stream_));
  CL_LAUNCH(enqueue_step_tail(n_seqs, false));
  prof.report("prefill profile", 32, "multi-prompt tile path, " + std::to_string(total) + " tokens");
  launches_ += launches;
  for (int i = 0; i < n_seqs; ++i) seq_advance(ss[i], ids[i], lens[i], lens[i]);
  if ((rc = collect_logprobs(ss, n_seqs))) return rc;
  if (logits_out) {
    for (int i = 0; i < n_seqs; ++i)
      if ((rc = read_logits(ss[i], logits_out + (size_t)i * V))) return rc;
    return CL_OK;
  }
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  return CL_OK;
}

}  // namespace cl

// ================================================================================================
using namespace cl;

namespace {
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  template <typename T> T* as() { return reinterpret_cast<T*>(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 16); }
  cudaError_t upload(const void* h, size_t bytes) {
    cudaError_t e = alloc(bytes);
    return e != cudaSuccess ? e : cudaMemcpy(p, h, bytes, cudaMemcpyHostToDevice);
  }
};
int check_device(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) {
    cudaGetLastError();
    set_last_error("no CUDA device (libclengine has no CPU fallback)");
    return CL_ERR_NO_DEVICE;
  }
  CL_CUDA_OK(cudaSetDevice(device));
  return CL_OK;
}
struct Stream {
  cudaStream_t s = nullptr;
  ~Stream() { if (s) cudaStreamDestroy(s); }
};
}  // namespace

extern "C" {

// epi 0: y[k_splits][t][n] = the split-K partials (k_splits 0: the batched step's count, pick_splits_public); y == NULL only
//        reports that count through *k_splits_used.
// epi 1: y[t][n] = resid + x w^T, added in place (the tile path's o / down projections).
// epi 2: act[t][n/2] = bf16(silu(gate) * up) of the interleaved gate|up rows (launch_gemm_bf16_silu).
// The residual and SiLU epilogues run unsplit (k_splits 0 or 1), as in the tile path, and the SiLU launcher has no PDL launch.
// pdl = 1 launches with programmatic stream serialization, as the batched step does, so the kernel requests its first W tiles
// before griddepcontrol.wait.  Every output element starts as NaN.
int cl_op_gemm_bf16_epi(int device, int epi, int32_t k_splits, int pdl, const uint16_t* x, const uint16_t* w, const float* resid, float* y,
                        uint16_t* act, int32_t t, int32_t n, int32_t k, int32_t* k_splits_used) {
  if (!x || !w || t <= 0 || n <= 0 || k <= 0 || k_splits < 0 || epi < 0 || epi > 2 || (epi == 0 && !y && !k_splits_used) ||
      (epi == 1 && (!resid || !y)) || (epi == 2 && (!act || (n & 1) || pdl)))
    return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  if (!gemm_tc_supported(t, n, k)) { set_last_error("shape not supported by the wgmma GEMM (K % 8)"); return CL_ERR_INVALID_ARG; }
  const int ks = k_splits ? k_splits : epi == 0 ? pick_splits_public(n, k) : 1;
  if (k_splits_used) *k_splits_used = ks;
  if (epi == 0 && !y) return CL_OK;
  if (epi != 0 && ks != 1) { set_last_error("the residual and SiLU epilogues run unsplit"); return CL_ERR_INVALID_ARG; }
  if (!gemm_splits_supported(k, ks)) { set_last_error("launch_gemm_bf16 refuses this split count"); return CL_ERR_INVALID_ARG; }
  const size_t out_bytes = epi == 0 ? (size_t)ks * t * n * 4 : epi == 1 ? (size_t)t * n * 4 : (size_t)t * (n / 2) * 2;
  DevBuf dx, dw, dy;
  CL_CUDA_OK(dx.upload(x, (size_t)t * k * 2));
  CL_CUDA_OK(dw.upload(w, (size_t)n * k * 2));
  if (epi == 1) CL_CUDA_OK(dy.upload(resid, out_bytes));
  else {
    CL_CUDA_OK(dy.alloc(out_bytes));
    CL_CUDA_OK(cudaMemset(dy.p, 0xff, out_bytes));   // NaN pattern: every element must be written
  }
  // a pageable upload may return before its DMA lands and the fill is asynchronous: both must be done before the launch
  CL_CUDA_OK(cudaDeviceSynchronize());
  Stream st;
  CL_CUDA_OK(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
  const __nv_bfloat16 *X = dx.as<__nv_bfloat16>(), *W = dw.as<__nv_bfloat16>();
  const int r = epi == 2 ? launch_gemm_bf16_silu(X, W, t, n, k, dy.as<__nv_bfloat16>(), n / 2, st.s)
                         : launch_gemm_bf16(X, W, dy.as<float>(), epi == 1 ? dy.as<float>() : nullptr, t, n, k, st.s, ks, pdl != 0);
  if (r < 0) { CL_CUDA_OK(cudaGetLastError()); set_last_error("wgmma GEMM launch failed"); return CL_ERR_CUDA; }
  CL_CUDA_OK(cudaStreamSynchronize(st.s));
  CL_CUDA_OK(cudaMemcpy(epi == 2 ? (void*)act : (void*)y, dy.p, out_bytes, cudaMemcpyDeviceToHost));
  return CL_OK;
}

int cl_op_gemm_bf16(int device, const uint16_t* x, const uint16_t* w, float* y, int32_t t, int32_t n, int32_t k, int32_t iters,
                    float* ms) {
  if (!y) return CL_ERR_INVALID_ARG;
  const int rc = cl_op_gemm_bf16_epi(device, 0, 1, 0, x, w, nullptr, y, nullptr, t, n, k, nullptr);
  if (rc || iters <= 0 || !ms) return rc;
  DevBuf dx, dw, dy;
  CL_CUDA_OK(dx.upload(x, (size_t)t * k * 2));
  CL_CUDA_OK(dw.upload(w, (size_t)n * k * 2));
  CL_CUDA_OK(dy.alloc((size_t)t * n * 4));
  cudaEvent_t e0, e1;
  CL_CUDA_OK(cudaEventCreate(&e0));
  CL_CUDA_OK(cudaEventCreate(&e1));
  for (int i = 0; i < 3; ++i) launch_gemm_bf16(dx.as<__nv_bfloat16>(), dw.as<__nv_bfloat16>(), dy.as<float>(), nullptr, t, n, k, nullptr);
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaEventRecord(e0));
  for (int i = 0; i < iters; ++i) launch_gemm_bf16(dx.as<__nv_bfloat16>(), dw.as<__nv_bfloat16>(), dy.as<float>(), nullptr, t, n, k, nullptr);
  CL_CUDA_OK(cudaEventRecord(e1));
  CL_CUDA_OK(cudaDeviceSynchronize());
  float tm = 0.f;
  CL_CUDA_OK(cudaEventElapsedTime(&tm, e0, e1));
  *ms = tm / (float)iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return CL_OK;
}

// Causal attention of the queries at positions pos0 .. pos0 + t - 1 (q [t][n_heads * head_dim]) over keys 0 .. pos0 + t - 1
// (k, v [pos0 + t][n_kv][head_dim]), paged by op_build_kv_pool.  variant: -1 the engine's rule (Engine::attn_prefill: the wgmma
// kernel when it takes the shape), 0 mma.sync kernel, 1 wgmma kernel.  out [t][n_heads * head_dim] = the kernel's bf16 output.
static int attn_prefill_impl(int device, int variant, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t pos0, int32_t t,
                             int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, int iters, float* out, float* ms) {
  if (!q || !k || !v || !out || t <= 0 || pos0 < 0 || variant < -1 || variant > 1) return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  if ((head_dim != 64 && head_dim != 128) || n_kv <= 0 || n_heads % n_kv || (page_size != 16 && page_size != 32 && page_size != 64)) {
    set_last_error("unsupported attention shape");
    return CL_ERR_INVALID_ARG;
  }
  const int P = page_size, HD = head_dim, n_tok = pos0 + t;
  OpKvPool pool;
  op_build_kv_pool(k, v, &n_tok, 1, n_kv, HD, P, &pool);
  const size_t qd = (size_t)n_heads * HD;
  DevBuf dq, dk, dv, dbt, dout, dout32;
  CL_CUDA_OK(dq.upload(q, (size_t)t * qd * 2));
  CL_CUDA_OK(dk.upload(pool.k.data(), pool.k.size() * 2));
  CL_CUDA_OK(dv.upload(pool.v.data(), pool.v.size() * 2));
  CL_CUDA_OK(dbt.upload(pool.bt.data(), pool.bt.size() * 4));
  CL_CUDA_OK(dout.alloc((size_t)t * qd * 2));
  CL_CUDA_OK(cudaMemset(dout.p, 0xff, (size_t)t * qd * 2));   // NaN pattern: every output must be written
  CL_CUDA_OK(dout32.alloc((size_t)t * qd * 4));
  AttnPrefillArgs a{dq.as<__nv_bfloat16>(), dk.as<__nv_bfloat16>() + pool.layer_elems, dv.as<__nv_bfloat16>() + pool.layer_elems,
                    dbt.as<int>(), P, pos0, t, n_heads, n_kv, HD, dout.as<__nv_bfloat16>()};
  const long long pool_rows = 2LL * pool.n_pages * n_kv * P;
  CUtensorMap km, vm;
  bool tc = variant != 0 && attn_prefill_tc_supported(n_heads, n_kv, HD, P, pos0, t);
  if (tc) tc = make_tmap_2d_bf16(&km, dk.p, pool_rows, HD, 64, 32) && make_tmap_2d_bf16(&vm, dv.p, pool_rows, HD, 64, 32);
  if (variant == 1 && !tc) { set_last_error("wgmma prefill attention does not support this shape"); return CL_ERR_INVALID_ARG; }
  auto run = [&]() { return tc ? launch_attn_prefill_tc(a, km, vm, pool_rows / 2, nullptr) : launch_attn_prefill(a, nullptr); };
  if (run() < 0) { CL_CUDA_OK(cudaGetLastError()); set_last_error("prefill attention launch failed"); return CL_ERR_CUDA; }
  if (launch_bf16_to_f32(dout.as<__nv_bfloat16>(), dout32.as<float>(), (int64_t)t * qd, nullptr) < 0) return CL_ERR_CUDA;
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaMemcpy(out, dout32.p, (size_t)t * qd * 4, cudaMemcpyDeviceToHost));
  if (iters > 0 && ms) {
    cudaEvent_t e0, e1;
    CL_CUDA_OK(cudaEventCreate(&e0));
    CL_CUDA_OK(cudaEventCreate(&e1));
    for (int i = 0; i < 2; ++i) run();
    CL_CUDA_OK(cudaDeviceSynchronize());
    CL_CUDA_OK(cudaEventRecord(e0));
    for (int i = 0; i < iters; ++i) run();
    CL_CUDA_OK(cudaEventRecord(e1));
    CL_CUDA_OK(cudaDeviceSynchronize());
    float tm = 0.f;
    CL_CUDA_OK(cudaEventElapsedTime(&tm, e0, e1));
    *ms = tm / (float)iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  return CL_OK;
}

int cl_op_attn_prefill(int device, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t t, int32_t n_heads, int32_t n_kv,
                       int32_t head_dim, float* out) {
  return attn_prefill_impl(device, -1, q, k, v, 0, t, n_heads, n_kv, head_dim, 32, 0, out, nullptr);
}
int cl_op_attn_prefill_variant(int device, int variant, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t t, int32_t n_heads,
                               int32_t n_kv, int32_t head_dim, float* out, int32_t iters, float* ms) {
  return attn_prefill_impl(device, variant, q, k, v, 0, t, n_heads, n_kv, head_dim, 32, iters, out, ms);
}
int cl_op_attn_prefill_cached(int device, int variant, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t pos0, int32_t t,
                              int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, float* out) {
  return attn_prefill_impl(device, variant, q, k, v, pos0, t, n_heads, n_kv, head_dim, page_size, 0, out, nullptr);
}

}  // extern "C"
