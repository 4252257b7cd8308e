// scheduler.cpp — request-level path: continuous-batching scheduler behind cl_generate().
//
// Replaces what the reference gets from the Ollama server's own scheduler (UPSTREAM of
// /root/reference/pkg/crowdllama/api.go:129-139).  Callers are the per-stream goroutines of
// Peer.handleInferenceRequest (/root/reference/pkg/peer/peer.go:190-256): many may block in
// cl_generate at once; the scheduler thread batches their decode steps (iteration-level
// scheduling) and preempts-by-recompute when the paged KV pool runs dry.
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>

#include "engine.h"

namespace cl {

static int64_t now_ns() {
  return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct Request {
  std::vector<int32_t> prompt;
  cl_sampling sp{};
  SamplerExt ext;                   // min_p and the presence / frequency penalties; the sequence carries them while admitted
  StopScan stop;                    // stop strings over the text of `out` (kept across preemptions and context shifts)
  std::vector<int32_t> out;
  cl_seq_t seq = -1;
  int max_new = 0;
  int n_preempted = 0;
  int status = CL_OK;
  std::string done_reason, err;
  bool done = false;
  bool sync = false;                // served by generate_sync (no scheduler thread)
  std::mutex m;
  std::condition_variable cv;
  // streaming: ids the scheduler has published to the waiting client thread (guarded by m); `out` itself is only
  // read by the client after `done`
  bool streaming = false;
  std::vector<int32_t> pub;
  std::atomic<bool> cancel{false};
  int64_t t_arrive = 0, prefill_ns = 0, decode_ns = 0, t_done = 0;
  uint64_t arrival = 0;
  std::vector<int32_t> full;        // prompt + out as of the last sync_full()
  size_t prefilled = 0;             // tokens of `full` already in the cache (chunked admission)
  bool dev_sample = false;          // sampled, and the step tail draws its tokens (device_sampling_ok, CL_DEVICE_SAMPLE)
  int top_n = -1;                   // logprobs: -1 off, else the alternatives per record (the sequence is armed with it)
  std::vector<LogprobRecord> lps;   // one record per id of `out` (kept across preemptions)
  std::vector<LogprobRecord> pub_lps;   // streaming: the records of `pub` (guarded by m)
  bool lp_mismatch = false;         // an id joined without its own record: the request fails with CL_ERR_INTERNAL
  int spec_backoff = 0;             // tokens to decode without drafting (after a verify pass that accepted nothing)
  bool ctx_shift = false;           // cl_engine_config.context_shift: the sequence shifts instead of ending at max_seq_len
  int keep = 0;                     // ... keeping its first `keep` ids
  int shifted = 0;                  // ids after the first `keep` that shifts have discarded so far
  bool greedy() const { return sp.temperature <= 0.f; }
  bool device_next() const { return greedy() || dev_sample; }   // the next id is d_tok_ after the step: no host sampler
  // prompt + out into `full`, reusing its storage: what an admission (re-)prefills, and the history a draft comes from.
  // After context shifts, the window the sequence holds: the first `keep` ids, then those after the discarded ones.
  const std::vector<int32_t>& sync_full() {
    full.assign(prompt.begin(), prompt.end());
    full.insert(full.end(), out.begin(), out.end());
    if (shifted) full.erase(full.begin() + keep, full.begin() + keep + shifted);
    return full;
  }
};

static void fill_result(const Request& r, cl_result* out, const Tokenizer* tok) {
  memset(out, 0, sizeof *out);
  out->n_prompt = (int32_t)r.prompt.size();
  out->n_generated = (int32_t)r.out.size();
  out->token_ids = (int32_t*)malloc(sizeof(int32_t) * std::max<size_t>(1, r.out.size()));
  if (!r.out.empty()) memcpy(out->token_ids, r.out.data(), r.out.size() * 4);
  std::string text;
  if (tok) text = r.stop.match() >= 0 ? Tokenizer::sanitize(tok->decode_bytes(r.out).substr(0, (size_t)r.stop.match())) : tok->decode(r.out);
  out->text = (char*)malloc(text.size() + 1);
  memcpy(out->text, text.c_str(), text.size() + 1);
  out->text_len = text.size();
  out->done_reason = strdup(r.done_reason.c_str());
  out->prefill_ns = r.prefill_ns;
  out->decode_ns = r.decode_ns;
  out->total_ns = r.t_done - r.t_arrive;
  out->n_preempted = r.n_preempted;
}

static bool finished(Request& r, const Tokenizer& tok, int max_seq_len) {
  if (r.cancel.load(std::memory_order_relaxed)) { r.done_reason = "cancelled"; return true; }
  if (r.stop.match() >= 0) { r.done_reason = "stop"; return true; }
  if (!r.out.empty() && !r.sp.ignore_eos && tok.is_stop(r.out.back())) { r.done_reason = "stop"; return true; }
  if ((int)r.out.size() >= r.max_new) { r.done_reason = "length"; return true; }
  if (!r.ctx_shift && (int)(r.prompt.size() + r.out.size()) >= max_seq_len) { r.done_reason = "length"; return true; }
  return false;
}

// ---- request transitions ---------------------------------------------------------------------------
// Join: ids[0..n) join r.out one at a time, each published to a streaming client, until r finishes.  Returns whether it did.
// Counting: tokens_generated_ (cl_stats; bench.py's mean batch divides it by sched_decode_steps) moves here and in retire()
// only, by one rule.  An id from a decode step or verify pass of the scheduler counts as it joins.  An id chosen at
// admission counts only when the request finishes with it: a request that goes on decoding never counts its admission id.
// The synchronous path counts r.out.size() when it retires successfully.
// With logprobs on, the i-th id takes the i-th record the calls since the last join left on r's sequence (the step tail's
// record of exactly that id); records of ids that did not join are dropped.  A missing record, or one of another id, is a
// defect: the request then fails when it retires instead of returning a wrong record.
bool Engine::join(Request& r, const int32_t* ids, int n, bool admission) {
  std::vector<LogprobRecord>* pending = r.top_n >= 0 ? &seqs_[r.seq].lps : nullptr;
  int joined = 0;
  bool fin = false;
  while (joined < n && !fin) {
    if (pending) {
      LogprobRecord rec{};
      rec.id = -1;
      if (joined < (int)pending->size()) rec = (*pending)[(size_t)joined];
      if (rec.id != ids[joined]) r.lp_mismatch = true;
      r.lps.push_back(rec);
    }
    r.out.push_back(ids[joined++]);
    if (r.stop.active()) r.stop.feed_id(*tok, r.out.back());
    if (r.streaming) {
      std::lock_guard<std::mutex> lk(r.m);
      r.pub.push_back(r.out.back());
      if (pending) r.pub_lps.push_back(r.lps.back());
      r.cv.notify_all();
    }
    fin = finished(r, *tok, cfg.max_seq_len);
  }
  if (pending) pending->clear();
  if (!r.sync && (!admission || fin)) tokens_generated_ += joined;
  return fin;
}

// Retire: r leaves the engine with `status` (CL_OK: finished or cancelled; else failed, with err): its sequence is freed, a
// successful request is counted, and the waiting client thread wakes.  requests_completed_ moves here only.
void Engine::retire(Request& r, int status, const std::string& err_in) {
  std::string err = err_in;
  if (status == CL_OK && r.lp_mismatch) {
    status = CL_ERR_INTERNAL;
    err = "logprobs: a generated id has no record of its own";
  }
  if (r.seq >= 0) seq_free(r.seq);
  r.seq = -1;
  if (status == CL_OK) {
    requests_completed_++;
    if (r.sync) tokens_generated_ += (int64_t)r.out.size();
  }
  std::lock_guard<std::mutex> lk(r.m);
  r.status = status;
  r.err = err;
  r.done = true;
  r.cv.notify_all();
}

// Pages admitting r takes out of free_pages(), with the prompt tokens it attaches from the prefix cache in *hit.  Attaching
// takes cached pages out of free_pages() too, so they count as needed (an upper bound when queued requests share pages):
// the check equals attaching first and comparing the missing pages with what is left, without attaching while r waits.
int Engine::admission_pages(Request& r, int* hit) {
  const std::vector<int32_t>& full = r.sync_full();
  int cached = 0;
  *hit = prefix_cache_ ? pool_->lookup(full.data(), (int)full.size(), &cached) : 0;
  return ((int)full.size() + 1 + page_size_ - 1) / page_size_ - *hit / page_size_ + cached;
}

// Preempt: r gives its pages back and waits at the queue's head; its next admission recomputes prompt + out (its window,
// after context shifts).  A window that would leave no position for the next token is shifted first, on the host only.
void Engine::preempt(std::shared_ptr<Request> r) {
  if (r->ctx_shift && (int)r->sync_full().size() >= cfg.max_seq_len) r->shifted += shift_discard(cfg.max_seq_len);
  seq_free(r->seq);
  r->seq = -1;
  r->n_preempted++;
  preemptions_++;
  std::lock_guard<std::mutex> lk(q_mu_);
  queue_.push_front(std::move(r));
}

// Context shift of a running request whose sequence holds max_seq_len tokens: the discard rule of cl_engine_config.context_shift
int Engine::shift_request(Request& r) {
  const int d = shift_discard(seqs_[r.seq].len);
  const int rc = seq_shift(r.seq, num_keep_, d);
  if (rc == CL_OK) r.shifted += d;
  return rc;
}

// Host next token: sample_token over the logits of r's slot (read back first with read_back, else already in `logits`), with
// hist[0..n_hist) as the repeat-penalty history and RNG step r.out.size().  The id of a host-sampled request then goes to
// d_tok_, the next step's input; a greedy request's step tail already put its choice there.
int Engine::host_next_token(Request& r, float* logits, bool read_back, const int32_t* hist, int n_hist, int32_t* next) {
  if (read_back) {
    const int rc = read_logits(r.seq, logits);
    if (rc) return rc;
  }
  *next = sample_token(logits, cfg.vocab_size, r.sp, hist, n_hist, (uint64_t)r.out.size(), r.ext);
  auto& pending = seqs_[r.seq].lps;
  if (r.top_n >= 0 && !pending.empty()) {   // lse and the top list are the device's; the host's id gets logit - lse as there
    LogprobRecord& rec = pending.back();
    rec.id = *next;
    rec.logprob = (float)((double)logits[*next] - rec.lse);
  }
  if (!r.device_next()) CL_CUDA_OK(cudaMemcpyAsync(d_tok_ + r.seq, next, 4, cudaMemcpyHostToDevice, stream_));
  return CL_OK;
}

// Speculative round of rs[0..n): a request decoding alone, or 2 .. speculate_batch running requests; every one must be
// greedy or device-sampled.  Each drafts from its prompt and output (the draft model's draft_tokens when the engine has one,
// else ngram_draft; nothing while backing off or without a match), clipped so that it passes neither max_new nor max_seq_len, and one verify pass checks all the drafts.  The pass
// holds at most kSpecMaxRows rows: every k is capped at the largest c with sum(min(k_i, c) + 1) <= kSpecMaxRows, so no
// request loses a drafted token while another keeps more than c.  A request the pool has no pages for drafts nothing this
// round.  A lone request keeps the per-segment attention of cl_decode_verify; several take the multi-row kernel.  Accepted
// ids join each request until it finishes.  Returns 1 after a pass, 0 when nobody drafted (the requests take a normal step
// instead), or an error status.
int Engine::spec_round(const std::shared_ptr<Request>* rs, int n) {
  if (speculate_ <= 0 || !std::all_of(rs, rs + n, [](const std::shared_ptr<Request>& r) { return r->device_next(); })) return 0;
  std::vector<int> ks(n, 0);
  std::vector<int32_t> drafts((size_t)n * kSpecMaxDraft);
  int cap = kSpecMaxDraft;
  auto rows = [&](int c) { int t = 0; for (int k : ks) t += std::min(k, c) + 1; return t; };
  for (int b = 0; b < n; ++b) {
    Request& r = *rs[b];
    if (r.spec_backoff > 0 || r.out.empty()) continue;
    const int k_max = std::min({speculate_, r.max_new - (int)r.out.size() - 1, cfg.max_seq_len - seqs_[r.seq].len - 1});
    if (k_max < 1) continue;
    const std::vector<int32_t>& hist = r.sync_full();   // ends with the next input x0
    ks[b] = draft_ ? k_max : ngram_draft(hist.data(), (int)hist.size(), k_max, drafts.data() + (size_t)b * kSpecMaxDraft);
  }
  if (draft_) {
    // the draft model drafts every id it is asked for, so the pass's row cap applies before it runs; a sampled request's
    // draft row i draws at the RNG step of its verify row i
    while (cap > 0 && rows(cap) > kSpecMaxRows) --cap;
    std::vector<cl_seq_t> ss(n);
    std::vector<const int32_t*> hists(n);
    std::vector<int> lens(n), got(n);
    std::vector<cl_sampling> sp(n);
    std::vector<uint64_t> step0(n);
    for (int b = 0; b < n; ++b) {
      Request& r = *rs[b];
      ks[b] = std::min(ks[b], cap);
      ss[b] = r.seq; hists[b] = r.full.data(); lens[b] = (int)r.full.size();   // r.full: synced above when ks[b] > 0
      sp[b] = r.sp; step0[b] = r.out.size();
    }
    std::vector<int32_t> packed((size_t)n * kSpecMaxDraft);
    if (const int rc = draft_tokens(ss.data(), n, hists.data(), lens.data(), ks.data(), sp.data(), step0.data(), packed.data(), got.data())) return rc;
    for (int b = 0, off = 0; b < n; off += ks[b], ++b) {
      std::copy(packed.begin() + off, packed.begin() + off + got[b], drafts.begin() + (size_t)b * kSpecMaxDraft);
    }
    for (int b = 0; b < n; ++b) ks[b] = got[b];
  }
  while (cap > 0 && rows(cap) > kSpecMaxRows) --cap;
  for (int b = 0; b < n; ++b) {
    ks[b] = std::min(ks[b], cap);
    if (ks[b] == 0) continue;
    // pages for the drafted rows (x0's are reserved already)
    const cl_seq_t s = rs[b]->seq;
    const int rc = ensure_capacity(s, seqs_[s].len + ks[b] + 1);
    if (rc == CL_ERR_OOM) ks[b] = 0;
    else if (rc) return rc;
  }
  if (std::all_of(ks.begin(), ks.end(), [](int k) { return k == 0; })) return 0;
  std::vector<cl_seq_t> ss(n);
  std::vector<int32_t> x0(n), packed, ids(kSpecMaxRows);
  std::vector<int> n_ids(n);
  for (int b = 0; b < n; ++b) {
    ss[b] = rs[b]->seq;
    x0[b] = rs[b]->out.back();
    packed.insert(packed.end(), drafts.begin() + (size_t)b * kSpecMaxDraft, drafts.begin() + (size_t)b * kSpecMaxDraft + ks[b]);
  }
  const int rc = verify_batch(ss.data(), n, x0.data(), packed.data(), ks.data(), ids.data(), n_ids.data(), nullptr, n > 1);
  if (rc) return rc;
  for (int b = 0, row0 = 0; b < n; row0 += ks[b] + 1, ++b) {
    Request& r = *rs[b];
    if (ks[b] > 0) r.spec_backoff = n_ids[b] == 1 ? kSpecBackoff : 0;
    else if (r.spec_backoff > 0) r.spec_backoff--;   // one token, as in a decode step
    join(r, ids.data() + row0, n_ids[b], false);
  }
  return 1;
}

// ---- synchronous path (no scheduler thread): one request at a time under the engine lock; the caller retires it --------
int Engine::generate_sync(const std::shared_ptr<Request>& rp, const TokenSink* sink) {
  Request& r = *rp;
  size_t emitted = 0;
  auto emit = [&]() {
    if (!sink || !sink->fn || r.out.size() <= emitted) return;
    const int n = (int)(r.out.size() - emitted);
    if (sink->lp_fn && r.top_n >= 0) {
      std::vector<cl_token_logprob> lp((size_t)n);
      for (int i = 0; i < n; ++i) lp[(size_t)i] = to_token_logprob(r.lps[emitted + (size_t)i]);
      if (sink->lp_fn(sink->user, lp.data(), n)) r.cancel = true;
    }
    if (sink->fn(sink->user, r.out.data() + emitted, n)) r.cancel = true;
    emitted = r.out.size();
  };
  int rc = seq_create(&r.seq);
  if (rc == CL_OK) seqs_[r.seq].ext = r.ext;
  if (rc == CL_OK && r.top_n >= 0) rc = set_logprobs(r.seq, r.top_n);
  if (rc) return rc;
  std::vector<float> logits(cfg.vocab_size);
  int64_t t0 = now_ns();
  // prefix cache: the prompt's cached pages are taken over, only the rest is prefilled (reused = 0 with the cache off)
  int reused = 0;
  rc = attach_prefix(r.seq, r.prompt.data(), (int)r.prompt.size(), &reused);
  // a device-sampled request is armed before the prefill, whose tail then draws the first token
  if (rc == CL_OK && r.dev_sample) rc = arm_sampling(r.seq, r.sp, 0, r.prompt.data(), (int)r.prompt.size());
  if (rc == CL_OK) rc = prefill(r.seq, r.prompt.data() + reused, (int)r.prompt.size() - reused, r.dev_sample ? nullptr : logits.data());
  r.prefill_ns = now_ns() - t0;
  if (rc) return rc;
  t0 = now_ns();
  int32_t next = 0;
  if (r.dev_sample) rc = read_next_token(r.seq, &next);
  else rc = host_next_token(r, logits.data(), false, r.prompt.data(), (int)r.prompt.size(), &next);
  if (rc) return rc;
  join(r, &next, 1, true);
  emit();
  while (!finished(r, *tok, cfg.max_seq_len)) {
    if (r.ctx_shift && seqs_[r.seq].len >= cfg.max_seq_len && (rc = shift_request(r))) break;
    const int spec = spec_round(&rp, 1);
    if (spec < 0) { rc = spec; break; }
    if (spec > 0) {
      next = r.out.back();
    } else if (r.device_next()) {   // greedy or device-sampled: the token loop stays on the device
      const int window = r.ctx_shift ? cfg.max_seq_len - seqs_[r.seq].len : cfg.max_seq_len - (int)(r.prompt.size() + r.out.size());
      int room = std::min(r.max_new - (int)r.out.size(), window);
      int chunk = std::min(room, sink ? 8 : 32);
      // speculating: back to drafting after the back-off, or after one step when the history had no match
      if (speculate_ > 0) chunk = std::min(chunk, std::max(1, r.spec_backoff));
      r.spec_backoff = std::max(0, r.spec_backoff - chunk);
      std::vector<int32_t> ids(chunk);
      rc = decode_greedy(&r.seq, 1, &next, chunk, ids.data(), nullptr);
      if (rc) break;
      join(r, ids.data(), chunk, false);
      next = r.out.back();
    } else {
      rc = decode_step(r.seq, next, logits.data(), nullptr);
      const std::vector<int32_t>& hist = seqs_[r.seq].history;   // prompt + out, the step's input included
      if (rc == CL_OK) rc = host_next_token(r, logits.data(), false, hist.data(), (int)hist.size(), &next);
      if (rc) break;
      join(r, &next, 1, false);
    }
    emit();
  }
  r.decode_ns = now_ns() - t0;
  return rc;
}

int Engine::generate_ids(const int32_t* prompt, int n_prompt, const cl_sampling& sp, cl_result* out, const TokenSink* sink, int top_n,
                         cl_token_logprob** lps, const SamplerExt* ext, const std::vector<std::string>* stop) {
  if (!prompt || n_prompt <= 0 || !out) { set_last_error("empty prompt"); return CL_ERR_INVALID_ARG; }
  std::vector<std::string> stops = stop ? *stop : std::vector<std::string>();
  const SamplerExt x = ext ? *ext : SamplerExt();
  if (int rc = check_sampling_ext(x, &stops)) return rc;
  if (top_n < -1 || top_n > kLogprobTopMax || (top_n >= 0 && cfg.vocab_size > kTailBlocks * kSampleSliceMax)) {
    set_last_error("logprobs: top_n must be -1..20 and the vocabulary at most 163840");
    return CL_ERR_INVALID_ARG;
  }
  if (n_prompt >= cfg.max_seq_len && !context_shift_) { set_last_error("prompt longer than max_seq_len"); return CL_ERR_TOO_LONG; }
  for (int i = 0; i < n_prompt; ++i)
    if (prompt[i] < 0 || prompt[i] >= cfg.vocab_size) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
  auto r = std::make_shared<Request>();
  r->ctx_shift = context_shift_;
  r->keep = num_keep_;
  if (n_prompt >= cfg.max_seq_len) {   // context shift: the first num_keep ids and the tail, one position left to generate
    r->prompt.assign(prompt, prompt + num_keep_);
    r->prompt.insert(r->prompt.end(), prompt + n_prompt - (cfg.max_seq_len - 1 - num_keep_), prompt + n_prompt);
    n_prompt = (int)r->prompt.size();
  } else {
    r->prompt.assign(prompt, prompt + n_prompt);
  }
  r->sp = sp;
  r->ext = x;
  r->stop = StopScan(std::move(stops));
  r->max_new = sp.max_new_tokens > 0 ? sp.max_new_tokens : cfg.max_seq_len - n_prompt;
  // num_predict <= 0 stays bounded by the window even with context shift: an unbounded request would hold a slot forever
  if (!r->ctx_shift || sp.max_new_tokens <= 0) r->max_new = std::min(r->max_new, cfg.max_seq_len - n_prompt);
  r->t_arrive = now_ns();
  r->sync = !sched_started_;
  r->streaming = !r->sync && sink && sink->fn;   // the synchronous path calls the sink itself
  r->dev_sample = device_sample_ && device_sampling_ok(sp, cfg.vocab_size, x);
  r->top_n = top_n;
  if (r->sync) {
    std::lock_guard<std::mutex> lk(mu_);
    const int rc = generate_sync(r, sink);
    retire(*r, rc, rc ? get_last_error() : "");
  } else {
    {
      std::lock_guard<std::mutex> lk(q_mu_);
      if (stop_) { set_last_error("engine shutting down"); return CL_ERR_SHUTDOWN; }
      static std::atomic<uint64_t> counter{0};
      r->arrival = counter++;
      queue_.push_back(r);
    }
    q_cv_.notify_all();
    std::unique_lock<std::mutex> lk(r->m);
    size_t seen = 0;
    std::vector<int32_t> fresh;
    std::vector<cl_token_logprob> fresh_lp;
    while (true) {
      r->cv.wait(lk, [&] { return r->done || r->pub.size() > seen; });
      if (r->pub.size() > seen) {
        fresh.assign(r->pub.begin() + seen, r->pub.end());
        fresh_lp.clear();
        for (size_t i = seen; i < r->pub_lps.size(); ++i) fresh_lp.push_back(to_token_logprob(r->pub_lps[i]));
        seen = r->pub.size();
        lk.unlock();                       // the callback runs on this (the caller's) thread, outside every lock
        if (sink->lp_fn && r->top_n >= 0 && sink->lp_fn(sink->user, fresh_lp.data(), (int)fresh_lp.size())) r->cancel = true;
        if (sink->fn(sink->user, fresh.data(), (int)fresh.size())) r->cancel = true;
        lk.lock();
        continue;
      }
      if (r->done) break;
    }
  }
  r->t_done = now_ns();
  if (r->status != CL_OK) {
    if (!r->err.empty()) set_last_error(r->err);
    return r->status;
  }
  fill_result(*r, out, tok.get());
  if (lps) {
    *lps = (cl_token_logprob*)malloc(sizeof(cl_token_logprob) * std::max<size_t>(1, r->lps.size()));
    for (size_t i = 0; i < r->lps.size(); ++i) (*lps)[i] = to_token_logprob(r->lps[i]);
  }
  return CL_OK;
}

void Engine::start_scheduler() {
  if (sched_started_) return;
  stop_ = false;
  sched_started_ = true;
  sched_thread_ = std::thread([this] { scheduler_main(); });
}

void Engine::stop_scheduler() {
  if (!sched_started_) return;
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    stop_ = true;
  }
  q_cv_.notify_all();
  if (sched_thread_.joinable()) sched_thread_.join();
  sched_started_ = false;
}

// ---- the scheduler thread ------------------------------------------------------------------------------
void Engine::scheduler_main() {
  cudaSetDevice(device_);
  {
    std::lock_guard<std::mutex> elk(mu_);
    const char* v = getenv("CL_SCHED_MULTI_PREFILL");
    sched_multi_prefill_ = v ? atoi(v) != 0 : kDefaultSchedMultiPrefill != 0;
    if (!step_done_ev_ && cudaEventCreateWithFlags(&step_done_ev_, cudaEventBlockingSync | cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      step_done_ev_ = nullptr;
    }
    sched_logits_.resize(cfg.vocab_size);
    sched_toks_.resize(max_seqs_);
    sched_slots_.clear();
    precapture_graphs(max_batch_);   // every batch size's step graph up front, not inside the first steps that meet it
    if (draft_) draft_->precapture_graphs(speculate_batch_);   // and the draft's, for the batches that draft together
  }
  while (wait_for_work()) {
    std::lock_guard<std::mutex> elk(mu_);
    // Admission.  A prompt is prefilled in chunks of sched_prefill_chunk_ tokens, ONE chunk per scheduler iteration,
    // interleaved with the decode steps of the running batch: an admit never stalls active sequences for more than one
    // chunk (a 4096-token prompt used to hold every running request for its whole prefill).  Several short prompts may be
    // admitted in one iteration as long as their tokens fit the same budget (a burst of 128-token chats fills the batch in
    // a few iterations instead of one request per decode step).
    const int budget = sched_prefill_chunk_ > 0 ? sched_prefill_chunk_ : (1 << 30);   // 0: unlimited = whole prompts
    if (!admit_group(budget)) admit_chunked(budget);
    make_room();
    if (active_.empty()) continue;
    if (speculate_running()) continue;
    if (const int rc = step_running()) fail_running(rc);
  }
  shutdown_requests();
}

// Waits until there is work; false once the engine stops.  Burst detection while nothing is running: requests of one wave
// reach the worker over a few milliseconds (one stream per request, pkg/peer/peer.go:177-182).  Waiting as long as new ones
// keep arriving within kSchedLingerUs of each other (at most 8x that in total) lets group admission take them in one
// pass instead of prefilling the first one alone; a lone request pays kSchedLingerUs once, against a prefill of several
// milliseconds.
bool Engine::wait_for_work() {
  std::unique_lock<std::mutex> lk(q_mu_);
  q_cv_.wait(lk, [&] { return stop_ || !queue_.empty() || !active_.empty() || prefilling_; });
  if (stop_) return false;
  if (sched_multi_prefill_ && active_.empty() && !prefilling_ && !queue_.empty()) {
    const auto t_end = std::chrono::steady_clock::now() + std::chrono::microseconds(8 * (int64_t)kSchedLingerUs);
    while ((int)queue_.size() < max_batch_ && std::chrono::steady_clock::now() < t_end) {
      const size_t n = queue_.size();
      if (!q_cv_.wait_for(lk, std::chrono::microseconds(kSchedLingerUs), [&] { return stop_ || queue_.size() != n; })) break;   // quiet: go
      if (stop_) break;
    }
  }
  return !stop_;
}

// Group admission: the prompts at the head of the queue that fit one pass go through the tile path TOGETHER
// (Engine::prefill_multi: one weight stream for all of them).  FIFO: the group is a prefix of the queue.  With running
// sequences the pass is bounded by the same token budget as a chunk; with none to stall, by the workspace (4096 rows).
// Returns true when a group of two or more went through, which is this iteration's whole admission.
bool Engine::admit_group(int budget) {
  if (!sched_multi_prefill_ || prefilling_ || (int)active_.size() >= max_batch_ || !bws_ || !prefill_path_ok()) return false;
  const int pass_rows = std::min(prefill_chunk_tokens_, prompt_cap_);   // what one prefill_multi pass holds
  const int cap_tokens = active_.empty() ? pass_rows : std::min(budget, pass_rows);
  std::vector<std::shared_ptr<Request>> group;
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    int tokens = 0, pages = 0;
    for (auto& r : queue_) {
      if ((int)(active_.size() + group.size()) >= max_batch_) break;
      int hit = 0;   // prefix cache: tokens the member will attach instead of computing
      const int need = admission_pages(*r, &hit), n = (int)r->full.size();
      if (r->cancel.load(std::memory_order_relaxed) || tokens + n - hit > cap_tokens || pages + need > pool_->free_pages()) break;
      group.push_back(r);
      tokens += n - hit;
      pages += need;
    }
    if (group.size() < 2) return false;
    queue_.erase(queue_.begin(), queue_.begin() + (long)group.size());
  }
  std::vector<cl_seq_t> ss;
  std::vector<const int32_t*> ptrs;
  std::vector<int> lens;
  int rc = CL_OK, total = 0;
  // every member attaches its cached prefix before any of them reserves: a reserve may evict cached pages
  for (auto& r : group) {
    rc = seq_create(&r->seq);
    if (rc == CL_OK) seqs_[r->seq].ext = r->ext;
    int reused = 0;
    if (rc == CL_OK) rc = attach_prefix(r->seq, r->full.data(), (int)r->full.size(), &reused);
    if (rc) break;
    r->prefilled = reused;
  }
  for (size_t i = 0; rc == CL_OK && i < group.size(); ++i) {
    auto& r = group[i];
    rc = ensure_capacity(r->seq, (int)r->full.size() + 1);
    if (rc == CL_OK && r->top_n >= 0) rc = set_logprobs(r->seq, r->top_n);
    // the pass's tail draws the next token of a device-sampled request (step = tokens generated before a preemption)
    if (rc == CL_OK && r->dev_sample) rc = arm_sampling(r->seq, r->sp, r->out.size(), r->full.data(), (int)r->full.size());
    if (rc) break;
    ss.push_back(r->seq); ptrs.push_back(r->full.data() + r->prefilled); lens.push_back((int)(r->full.size() - r->prefilled));
    total += lens.back();
  }
  const int64_t t0 = now_ns();
  if (rc == CL_OK) rc = prefill_multi((int)ss.size(), ss.data(), ptrs.data(), lens.data(), nullptr);
  const int64_t pdt = now_ns() - t0;
  if (rc == CL_OK && (cudaMemcpyAsync(sched_toks_.data(), d_tok_, (size_t)max_seqs_ * 4, cudaMemcpyDeviceToHost, stream_) != cudaSuccess ||
                      cudaStreamSynchronize(stream_) != cudaSuccess))
    rc = CL_ERR_CUDA;
  sched_prefill_calls_++; sched_prefill_tokens_ += total; sched_prefill_ns_ += pdt;
  slots_dirty_ = true;
  if (rc) {
    const std::string err = get_last_error();
    for (auto& r : group) retire(*r, rc, err);
    return true;
  }
  for (auto& r : group) {
    r->prefill_ns += pdt;
    r->prefilled = r->full.size();
    int32_t next = sched_toks_[r->seq];   // greedy / device-sampled: the pass's tail chose it
    if (!r->device_next() && (rc = host_next_token(*r, sched_logits_.data(), true, r->full.data(), (int)r->full.size(), &next))) {
      retire(*r, rc, get_last_error());
      continue;
    }
    admitted(r, next);
  }
  return true;
}

// Chunked admission of the request at the queue's head, one chunk of at most `budget` tokens per iteration (the whole rest
// of the prompt when nothing runs), and of further requests while the budget lasts.
void Engine::admit_chunked(int budget) {
  while (budget > 0) {
    if (!prefilling_ && (int)active_.size() < max_batch_) {
      std::shared_ptr<Request> r;
      {
        std::lock_guard<std::mutex> lk(q_mu_);
        if (!queue_.empty()) r = queue_.front();
      }
      if (r) {
        int hit = 0;
        if (admission_pages(*r, &hit) > pool_->free_pages()) {
          if (active_.empty()) {
            { std::lock_guard<std::mutex> lk(q_mu_); queue_.pop_front(); }
            retire(*r, CL_ERR_OOM, "prompt does not fit in the KV page pool");
            continue;
          }
          // else: wait for running requests to release pages
        } else {
          { std::lock_guard<std::mutex> lk(q_mu_); queue_.pop_front(); }
          int reused = 0;
          int rc = seq_create(&r->seq);
          if (rc == CL_OK) seqs_[r->seq].ext = r->ext;
          if (rc == CL_OK) rc = attach_prefix(r->seq, r->full.data(), (int)r->full.size(), &reused);   // takes `hit` tokens
          if (rc == CL_OK) rc = ensure_capacity(r->seq, (int)r->full.size() + 1);   // all pages up front: a later chunk cannot run dry
          if (rc) { retire(*r, rc, get_last_error()); continue; }
          r->prefilled = reused;
          prefilling_ = r;
        }
      }
    }
    if (!prefilling_) break;
    auto r = prefilling_;
    if (r->cancel.load(std::memory_order_relaxed)) {
      r->done_reason = "cancelled";
      prefilling_.reset();
      retire(*r, CL_OK, "");
      continue;
    }
    const size_t left = r->full.size() - r->prefilled;
    const size_t chunk = active_.empty() ? left : std::min(left, (size_t)budget);   // nobody to stall: the whole prompt at once
    const bool last = chunk == left;
    const int64_t t0 = now_ns();
    // only the last chunk's tail draws: earlier chunks run with the slot disarmed
    int rc = last && r->dev_sample ? arm_sampling(r->seq, r->sp, r->out.size(), r->full.data(), (int)r->full.size()) : CL_OK;
    if (rc == CL_OK && last && r->top_n >= 0) rc = set_logprobs(r->seq, r->top_n);
    if (rc == CL_OK) rc = prefill(r->seq, r->full.data() + r->prefilled, (int)chunk, last && !r->dev_sample ? sched_logits_.data() : nullptr);
    int32_t next = 0;
    if (rc == CL_OK && last && r->dev_sample) rc = read_next_token(r->seq, &next);
    const int64_t pdt = now_ns() - t0;
    r->prefill_ns += pdt;
    sched_prefill_calls_++; sched_prefill_tokens_ += (int64_t)chunk; sched_prefill_ns_ += pdt;
    slots_dirty_ = true;                // prefill rewrote d_slots_[0]
    budget -= (int)std::min(chunk, (size_t)budget);
    if (rc) { prefilling_.reset(); retire(*r, rc, get_last_error()); continue; }
    r->prefilled += chunk;
    if (!last) break;                   // budget used up in the middle of a prompt
    prefilling_.reset();
    if (!r->dev_sample && (rc = host_next_token(*r, sched_logits_.data(), false, r->full.data(), (int)r->full.size(), &next))) {
      retire(*r, rc, get_last_error());
      continue;
    }
    admitted(r, next);
  }
}

// r's (re-)prefill chose `next`: r joins the running batch, or retires when it finishes with that id
void Engine::admitted(const std::shared_ptr<Request>& r, int32_t next) {
  if (join(*r, &next, 1, true)) retire(*r, CL_OK, "");
  else active_.push_back(r);
}

// Makes room for one more token per running request, first shifting a request whose sequence fills max_seq_len (context
// shift).  On an empty pool the youngest request is preempted: the one still being admitted, else the running request that
// arrived last.  A request the pool cannot serve even alone fails.
void Engine::make_room() {
  for (size_t i = 0; i < active_.size();) {
    Request& r = *active_[i];
    int rc = r.ctx_shift && seqs_[r.seq].len >= cfg.max_seq_len ? shift_request(r) : CL_OK;
    if (rc == CL_OK) rc = ensure_capacity(r.seq, seqs_[r.seq].len + 1);
    if (rc == CL_ERR_OOM && prefilling_) {
      preempt(prefilling_);
      prefilling_.reset();
      continue;                         // retry this request's capacity
    }
    if (rc == CL_ERR_OOM && active_.size() > 1) {
      size_t victim = 0;
      for (size_t k = 1; k < active_.size(); ++k) if (active_[k]->arrival > active_[victim]->arrival) victim = k;
      auto v = active_[victim];
      active_.erase(active_.begin() + victim);
      preempt(v);
      i = 0;                            // restart the capacity pass
      continue;
    }
    if (rc) {
      auto dead = active_[i];
      active_.erase(active_.begin() + i);
      retire(*dead, rc, get_last_error());
      continue;
    }
    ++i;
  }
}

// Speculative decoding: 1 .. speculate_batch running requests with nothing to admit take one verify pass instead of a step
// (it counts as one decode step).  Returns true when the pass replaced this iteration's step.
bool Engine::speculate_running() {
  if (speculate_ <= 0 || (int)active_.size() > speculate_batch_ || prefilling_) return false;
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    if (!queue_.empty()) return false;
  }
  const int64_t t0 = now_ns();
  const int rc = spec_round(active_.data(), (int)active_.size());
  if (rc == 0) return false;
  if (rc < 0) { fail_running(rc); return true; }
  const int64_t dt = now_ns() - t0;
  for (auto& r : active_) r->decode_ns += dt;
  sched_decode_steps_++; sched_decode_ns_ += dt;
  retire_finished();
  return true;
}

// One batched decode step of every running request
int Engine::step_running() {
  const int B = (int)active_.size();
  // slots_dirty_: an admission-time prefill (or a token-level call) rewrote d_slots_[0] since the last upload — the
  // cached list would leave a finished request's slot in place and every later step would run on it
  bool same = !slots_dirty_ && (int)sched_slots_.size() == B;
  for (int b = 0; same && b < B; ++b) same = sched_slots_[b] == active_[b]->seq;
  if (!same) {
    sched_slots_.resize(B);
    for (int b = 0; b < B; ++b) sched_slots_[b] = active_[b]->seq;
    cudaMemcpyAsync(d_slots_, sched_slots_.data(), (size_t)B * 4, cudaMemcpyHostToDevice, stream_);
    slots_dirty_ = false;
    last_single_slot_ = B == 1 ? sched_slots_[0] : -1;
    if (B > 1) last_batch_slots_ = sched_slots_;
  }
  h_slots_ = sched_slots_;
  const int64_t t0 = now_ns();
  int rc = run_step_graph(B);
  if (rc) return rc;
  cudaMemcpyAsync(sched_toks_.data(), d_tok_, (size_t)max_seqs_ * 4, cudaMemcpyDeviceToHost, stream_);
  // Batched steps last milliseconds: wait on a blocking-sync event instead of spinning in cudaStreamSynchronize, so that
  // eight worker processes on one box do not burn eight host cores (the box's cgroup quota is 16) while their GPUs
  // work.  Single-sequence steps (latency matters) keep the spinning wait.
  if (B >= 2 && step_done_ev_) {
    if (cudaEventRecord(step_done_ev_, stream_) != cudaSuccess || cudaEventSynchronize(step_done_ev_) != cudaSuccess) return CL_ERR_CUDA;
  } else if (cudaStreamSynchronize(stream_) != cudaSuccess) {
    return CL_ERR_CUDA;
  }
  if ((rc = collect_logprobs(sched_slots_.data(), B))) return rc;
  for (auto& r : active_) {
    seq_advance(r->seq, &r->out.back(), 1, 1);
    const std::vector<int32_t>& hist = seqs_[r->seq].history;
    int32_t next = sched_toks_[r->seq];
    if (!r->device_next() && (rc = host_next_token(*r, sched_logits_.data(), true, hist.data(), (int)hist.size(), &next))) return rc;
    join(*r, &next, 1, false);
    if (r->spec_backoff > 0) r->spec_backoff--;
  }
  const int64_t dt = now_ns() - t0;
  for (auto& r : active_) r->decode_ns += dt;
  sched_decode_steps_++; sched_decode_ns_ += dt;
  const double tps = (double)max_batch_ / ((double)dt * 1e-9);   // capacity at the current step time (engine.cu, init)
  tok_per_sec_ewma_ = tok_per_sec_ewma_ == 0.0 ? tps : 0.9 * tok_per_sec_ewma_ + 0.1 * tps;
  retire_finished();
  return CL_OK;
}

void Engine::retire_finished() {
  for (size_t i = 0; i < active_.size();) {
    auto r = active_[i];
    if (finished(*r, *tok, cfg.max_seq_len)) {
      active_.erase(active_.begin() + i);
      retire(*r, CL_OK, "");
    } else {
      ++i;
    }
  }
}

void Engine::fail_running(int rc) {
  const std::string err = get_last_error();
  for (auto& r : active_) retire(*r, rc, err);
  active_.clear();
  sched_slots_.clear();
}

// shutdown: fail whatever is left
void Engine::shutdown_requests() {
  std::lock_guard<std::mutex> elk(mu_);
  for (auto& r : active_) retire(*r, CL_ERR_SHUTDOWN, "engine shutting down");
  active_.clear();
  if (prefilling_) { retire(*prefilling_, CL_ERR_SHUTDOWN, "engine shutting down"); prefilling_.reset(); }
  std::deque<std::shared_ptr<Request>> rest;
  { std::lock_guard<std::mutex> lk(q_mu_); rest.swap(queue_); }
  for (auto& r : rest) retire(*r, CL_ERR_SHUTDOWN, "engine shutting down");
}

}  // namespace cl
