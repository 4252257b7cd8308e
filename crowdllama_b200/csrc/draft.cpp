// draft.cpp — the draft model of speculative decoding: a second Engine inside the Engine, holding one mirror sequence per
// target sequence that drafts (contract in include/clengine.h, cl_engine_create_with_draft and cl_draft_model).
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>

#include <sys/stat.h>

#include "engine.h"

namespace cl {

static int64_t now_ns() {
  return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// The draft's engine config, before Engine::init fills in what it takes from the target: `draft` (preset / model /
// weights_path / weights_seed only), else env CL_DRAFT_MODEL (a preset name, or a model directory) with CL_DRAFT_SEED
// (default: the target's weights_seed).  Returns whether a draft model is configured.
bool draft_engine_config(const cl_engine_config& c, const cl_engine_config* draft, cl_engine_config* out) {
  cl_engine_config d;
  cl_default_engine_config(&d);
  d.model_name = "draft";
  if (draft) {
    d.preset = draft->preset;
    d.model = draft->model;
    d.weights_path = draft->weights_path;
    d.weights_seed = draft->weights_seed;
  } else {
    const char* m = getenv("CL_DRAFT_MODEL");
    if (!m || !*m) return false;
    struct stat st{};
    if (stat(m, &st) == 0 && S_ISDIR(st.st_mode)) d.weights_path = m;
    else d.preset = m;
    const char* seed = getenv("CL_DRAFT_SEED");
    d.weights_seed = seed && *seed ? strtoull(seed, nullptr, 0) : c.weights_seed;
  }
  *out = d;
  return true;
}

void Engine::seq_rewind(cl_seq_t s, int len) {
  SeqState& q = seqs_[s];
  q.len = len;
  q.history.resize((size_t)len);
  q.known = std::min(q.known, len);
}

int Engine::draft_tokens(const cl_seq_t* ss, int n, const int32_t* const* hists, const int* lens, const int* ks_in, const cl_sampling* sp,
                         const uint64_t* step0, int32_t* drafts, int* n_drafts) {
  if (!draft_) { set_last_error("no draft model (cl_engine_create_with_draft, env CL_DRAFT_MODEL)"); return CL_ERR_INVALID_ARG; }
  Engine& D = *draft_;
  if (n < 1 || n > D.max_batch_ || !ss || !hists || !lens || !ks_in || !drafts || !n_drafts) {
    set_last_error("draft: bad arguments (1 <= n_seqs <= min(max_batch, 32))");
    return CL_ERR_INVALID_ARG;
  }
  for (int i = 0; i < n; ++i) {
    const cl_seq_t s = ss[i];
    if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
    for (int j = 0; j < i; ++j) if (ss[j] == s) { set_last_error("duplicate sequence in batch"); return CL_ERR_INVALID_ARG; }
    if (ks_in[i] < 0 || ks_in[i] > kSpecMaxDraft) { set_last_error("draft: k must be 0..15"); return CL_ERR_INVALID_ARG; }
    if (ks_in[i] == 0) continue;
    if (lens[i] < 1 || !hists[i]) { set_last_error("draft: empty window"); return CL_ERR_INVALID_ARG; }
    if (lens[i] > cfg.max_seq_len) { set_last_error("draft: window exceeds max_seq_len"); return CL_ERR_TOO_LONG; }
    for (int t = 0; t < lens[i]; ++t)
      if (hists[i][t] < 0 || hists[i][t] >= cfg.vocab_size) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
    if (sp && sp[i].temperature > 0.f && !device_sampling_ok(sp[i], cfg.vocab_size, seqs_[s].ext)) {
      set_last_error("sampling settings need the host sampler");
      return CL_ERR_INVALID_ARG;
    }
  }
  const int64_t t0 = now_ns();
  std::vector<int> ks(ks_in, ks_in + n), m(n, -1);
  int rc = CL_OK;
  // 1. every mirror keeps the longest common prefix of what it holds and the window before x0, and gets pages for the window
  for (int i = 0; i < n; ++i) {
    if (ks[i] == 0) continue;
    int& ms = mirror_[ss[i]];
    if (ms < 0 && (rc = D.seq_create(&ms))) return rc;
    SeqState& q = D.seqs_[ms];
    q.ext = seqs_[ss[i]].ext;
    const int lim = std::min(q.len, lens[i] - 1);
    int c = 0;
    while (c < lim && q.history[(size_t)c] == hists[i][c]) ++c;
    D.seq_rewind(ms, c);
    rc = D.ensure_capacity(ms, lens[i]);
    if (rc == CL_ERR_OOM) { ks[i] = 0; continue; }
    if (rc) return rc;
    m[i] = ms;
  }
  // 2. the steps: max(ks) - 1 for every sequence with ks >= 2; one whose window leaves no room for them (or whose pages the
  // pool cannot give) drafts d1 only
  auto k_max = [&]() { return *std::max_element(ks.begin(), ks.end()); };
  for (bool changed = true; changed;) {
    changed = false;
    const int K = k_max();
    for (int i = 0; i < n; ++i) {
      if (ks[i] < 2) continue;
      rc = D.ensure_capacity(m[i], lens[i] + K - 1);
      if (rc == CL_ERR_OOM || rc == CL_ERR_TOO_LONG) { ks[i] = 1; changed = true; }
      else if (rc) return rc;
    }
  }
  // 3. catch-up: one prefill pass over the missing rows, whose tail chooses d1 (a sampled mirror draws it at step0)
  std::vector<cl_seq_t> ps;
  std::vector<const int32_t*> pids;
  std::vector<int> plens;
  int rows = 0;
  for (int i = 0; i < n; ++i) {
    if (ks[i] == 0) continue;
    const int c = D.seqs_[m[i]].len;
    rc = sp && sp[i].temperature > 0.f ? D.arm_sampling(m[i], sp[i], step0 ? step0[i] : 0, hists[i], lens[i]) : D.disarm_sampling(m[i]);
    if (rc) return rc;
    ps.push_back(m[i]); pids.push_back(hists[i] + c); plens.push_back(lens[i] - c);
    rows += lens[i] - c;
  }
  std::vector<int32_t> d1(n, 0), steps_out;
  int B = 0, K = 0;
  if (!ps.empty()) {
    if (ps.size() >= 2 && D.bws_ && D.prefill_path_ok() && rows <= std::min(D.prefill_chunk_tokens_, D.prompt_cap_)) {
      rc = D.prefill_multi((int)ps.size(), ps.data(), pids.data(), plens.data(), nullptr);
    } else {
      for (size_t j = 0; j < ps.size() && rc == CL_OK; ++j) rc = D.prefill(ps[j], pids[j], plens[j], nullptr);
    }
    if (rc) return rc;
    CL_CUDA_OK(cudaMemcpyAsync(D.h_ids_pinned_, D.d_tok_, (size_t)D.max_seqs_ * 4, cudaMemcpyDeviceToHost, D.stream_));
    CL_CUDA_OK(cudaStreamSynchronize(D.stream_));
    for (int i = 0; i < n; ++i) if (ks[i] > 0) d1[i] = D.h_ids_pinned_[m[i]];
    // 4. the draft steps, batched: draw j of a sampled mirror at step0 + j, with the window and d1 .. dj as its history
    K = k_max();
    std::vector<cl_seq_t> bs;
    std::vector<int32_t> first;
    std::vector<cl_sampling> bsp;
    std::vector<uint64_t> bst;
    cl_sampling greedy{};
    for (int i = 0; i < n; ++i) {
      if (ks[i] < 2) continue;
      bs.push_back(m[i]); first.push_back(d1[i]);
      bsp.push_back(sp ? sp[i] : greedy);
      bst.push_back((step0 ? step0[i] : 0) + 1);
    }
    B = (int)bs.size();
    if (B > 0) {
      steps_out.resize((size_t)(K - 1) * B);
      rc = D.decode_sample(bs.data(), B, first.data(), bsp.data(), bst.data(), K - 1, steps_out.data(), nullptr);
    }
    for (int i = 0; i < n; ++i) {   // a mirror that drafted d1 only is still armed from its prefill
      const int r2 = ks[i] > 0 ? D.disarm_sampling(m[i]) : CL_OK;
      if (rc == CL_OK) rc = r2;
    }
    if (rc) return rc;
  }
  // 5. the ids, at the offsets the caller's ks give
  for (int i = 0, off = 0, b = 0; i < n; off += ks_in[i], ++i) {
    n_drafts[i] = ks[i];
    if (ks[i] == 0) continue;
    drafts[off] = d1[i];
    if (ks[i] >= 2) {
      for (int j = 1; j < ks[i]; ++j) drafts[off + j] = steps_out[(size_t)(j - 1) * B + b];
      ++b;
    }
  }
  draft_rows_ += rows + (int64_t)B * std::max(0, K - 1);
  draft_ns_ += now_ns() - t0;
  draft_pages_ = D.pool_->used_pages();
  return CL_OK;
}

}  // namespace cl
