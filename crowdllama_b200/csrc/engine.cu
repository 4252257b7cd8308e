// engine.cu — the worker-side decode engine: weights, paged KV cache, the token step (CUDA graph
// of hand-written sm_90a kernels), prefill, and the token-level entry points of the C-ABI.
//
// Replaces, behind crowdllama.UnifiedAPIHandler (/root/reference/pkg/crowdllama/api.go:19), the
// whole chain WorkerAPIHandler -> callOllamaAPI -> embedded Ollama server -> llama.cpp runner
// (api.go:45-160, /root/reference/cmd/crowdllama/main.go:283-297).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <set>

#include <sys/stat.h>

#include "common.cuh"
#include "engine.h"

namespace cl {

static int pick_splits(int n_rows, int K);   // batched-decode split-K rule (defined with the batched step)

enum { K_EMBED = 0, K_LM_HEAD = 1, K_FINAL_NORM = 2, K_ATTN_NORM = 3, K_WQ = 4, K_WK = 5, K_WV = 6, K_WO = 7,
       K_FFN_NORM = 8, K_WGATE = 9, K_WUP = 10, K_WDOWN = 11 };
static constexpr float kLinearScale = 1.35e-4f;
static constexpr float kNormScale = 1.0f / 4096.0f;

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}

Engine::~Engine() {
  stop_scheduler();
  if (stream_) cudaStreamSynchronize(stream_);
  for (auto& kv : graphs_) cudaGraphExecDestroy(kv.second);
  if (step_done_ev_) cudaEventDestroy(step_done_ev_);
  for (void* p : allocs_) cudaFree(p);
  if (h_logits_pinned_) cudaFreeHost(h_logits_pinned_);
  if (host_kv_) cudaFreeHost(host_kv_);
  if (h_ids_pinned_) cudaFreeHost(h_ids_pinned_);
  if (h_lp_pinned_) cudaFreeHost(h_lp_pinned_);
  if (ev0_) cudaEventDestroy(ev0_);
  if (ev1_) cudaEventDestroy(ev1_);
  if (stream_) cudaStreamDestroy(stream_);
}

#define DMALLOC(ptr, bytes)                                          \
  do {                                                               \
    void* _p = nullptr;                                              \
    cudaError_t _e = cudaMalloc(&_p, (bytes));                       \
    if (_e != cudaSuccess) {                                         \
      set_last_error(std::string("cudaMalloc(") + #ptr + ", " + std::to_string((size_t)(bytes)) + "): " + cudaGetErrorString(_e)); \
      return _e == cudaErrorMemoryAllocation ? CL_ERR_OOM : CL_ERR_CUDA; \
    }                                                                \
    allocs_.push_back(_p);                                           \
    ptr = reinterpret_cast<decltype(ptr)>(_p);                       \
  } while (0)

int64_t weight_bytes(const cl_model_config& m) {
  const int64_t d = m.d_model, F = m.d_ff, V = m.vocab_size, q = (int64_t)m.n_heads * m.head_dim, kv = (int64_t)m.n_kv_heads * m.head_dim;
  return 2 * (2 * V * d) + (int64_t)m.n_layers * 2 * ((q + 2 * kv) * d + d * q + 3 * F * d) + (int64_t)m.max_seq_len * m.head_dim * 4;
}

bool draft_engine_config(const cl_engine_config& c, const cl_engine_config* draft, cl_engine_config* out);   // draft.cpp

int Engine::init(const cl_engine_config& c, const cl_engine_config* draft) {
  if (c.abi_version != CL_ABI_VERSION) { set_last_error("abi_version mismatch"); return CL_ERR_INVALID_ARG; }
  const std::string wpath = c.weights_path ? c.weights_path : "";
  struct stat wst{};
  const bool wdir = !wpath.empty() && stat(wpath.c_str(), &wst) == 0 && S_ISDIR(wst.st_mode);
  int context_length = 0;
  const int rc0 = resolve_model_config(c, &cfg, &context_length);   // preset / config.json / c.model, the window, the num_keep check
  if (rc0) return rc0;
  model_name = c.model_name ? c.model_name : (c.preset ? c.preset : "model");
  const int rep = cfg.n_kv_heads > 0 ? cfg.n_heads / cfg.n_kv_heads : 0;
  if (cfg.n_layers <= 0 || cfg.d_model <= 0 || cfg.n_heads <= 0 || cfg.n_kv_heads <= 0 || cfg.d_ff <= 0 ||
      cfg.vocab_size <= 1 || cfg.max_seq_len <= 0 || (cfg.head_dim != 64 && cfg.head_dim != 128) ||
      cfg.n_heads % cfg.n_kv_heads || (rep != 1 && rep != 2 && rep != 4 && rep != 8) || cfg.d_model % 16 || cfg.d_ff % 16 ||
      (cfg.vocab_size & 1)) {
    set_last_error("unsupported model shape (need head_dim 64|128, heads/kv in {1,2,4,8}, d_model,d_ff %16==0, even vocab)");
    return CL_ERR_INVALID_ARG;
  }
  // the draft model: its config and the refusals that need no device (the rest follow once both engines exist)
  cl_engine_config dc{};
  cl_model_config dm{};
  const bool want_draft = !is_draft_ && draft_engine_config(c, draft, &dc);
  if (want_draft) {
    dc.context_length = cfg.max_seq_len;   // the target's window, which the draft must serve
    if (const int rc = resolve_model_config(dc, &dm, nullptr)) return rc;
    if (dm.vocab_size != cfg.vocab_size) {
      set_last_error("draft model: vocabulary of " + std::to_string(dm.vocab_size) + " ids, the target has " + std::to_string(cfg.vocab_size));
      return CL_ERR_INVALID_ARG;
    }
    if (env_int("CL_SPECULATE", c.speculate) == 0) { set_last_error("draft model: speculate is 0, so nothing would use it"); return CL_ERR_INVALID_ARG; }
  }
  // Deterministic mode runs every row through small_pass with the multi-row attention: its shapes (the split-K pass's
  // d_model <= 8192 included), and steps of at most one pass of rows.  Refused before the device is touched.  A draft
  // model's engine never runs it: drafts decide how many ids a pass accepts, not which ids.
  deterministic_ = !is_draft_ && env_int("CL_DETERMINISTIC", c.deterministic) != 0;
  if (deterministic_ && (!attn_verify_tc_supported(cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, c.page_size ? c.page_size : 32) ||
                         cfg.d_model > 8192)) {
    set_last_error("deterministic mode needs head_dim 128, 4 query heads per kv head and page_size 32");
    return CL_ERR_INVALID_ARG;
  }
  if (deterministic_ && c.max_batch > kSpecMaxRows) {
    set_last_error("deterministic mode takes max_batch up to " + std::to_string(kSpecMaxRows));
    return CL_ERR_INVALID_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    set_last_error("no CUDA device visible (libclengine has no CPU fallback)");
    return CL_ERR_NO_DEVICE;
  }
  device_ = c.device;
  if (device_ < 0 || device_ >= ndev) { set_last_error("bad device ordinal"); return CL_ERR_NO_DEVICE; }
  CL_CUDA_OK(cudaSetDevice(device_));
  cudaDeviceProp prop{};
  CL_CUDA_OK(cudaGetDeviceProperties(&prop, device_));
  if (prop.major != 9) {
    set_last_error(std::string("device is sm_") + std::to_string(prop.major * 10 + prop.minor) + ", kernels are built for sm_90a only");
    return CL_ERR_NO_DEVICE;
  }
  snprintf(gpu_name_, sizeof gpu_name_, "%s", prop.name);
  vram_gb_ = (int)(prop.totalGlobalMem >> 30);

  page_size_ = c.page_size ? c.page_size : 32;
  if (page_size_ != 16 && page_size_ != 32 && page_size_ != 64) { set_last_error("page_size must be 16, 32 or 64"); return CL_ERR_INVALID_ARG; }
  max_batch_ = c.max_batch > 0 ? c.max_batch : 8;
  max_seqs_ = c.max_seqs > 0 ? c.max_seqs : max_batch_;
  if (max_seqs_ < max_batch_) max_seqs_ = max_batch_;
  use_graph_ = c.use_cuda_graph >= 0 && env_int("CL_GRAPH", 1) != 0;
  use_pdl_ = env_int("CL_PDL", 1) != 0;
  want_timeline_ = env_int("CL_TIMELINE", 0) != 0;
  gemv_variant_ = c.decode_path == 1 ? 0 : 1;
  q_dim_ = cfg.n_heads * cfg.head_dim;
  kv_dim_ = cfg.n_kv_heads * cfg.head_dim;
  qkv_dim_ = q_dim_ + 2 * kv_dim_;
  nsplit_ = std::max(1, std::min(64, sm_count() / cfg.n_kv_heads));
  // decided AFTER nsplit_ is final: the persistent kernel's lane-parallel combine and part buffer are sized by it
  use_mega_ = !deterministic_ && env_int("CL_MEGA", 1) != 0 &&
              mega_supported(cfg.d_model, cfg.d_ff, cfg.head_dim, cfg.n_heads, cfg.n_kv_heads, page_size_, nsplit_);
  max_pages_per_seq_ = (cfg.max_seq_len + page_size_ - 1) / page_size_;

  const size_t kv_bytes_per_token = (size_t)2 * cfg.n_layers * kv_dim_ * 2;
  int64_t pool_bytes = c.kv_pool_bytes;
  if (pool_bytes <= 0) pool_bytes = (int64_t)max_seqs_ * max_pages_per_seq_ * page_size_ * (int64_t)kv_bytes_per_token;
  if (c.kv_pool_bytes <= 0 && context_length > 0) {
    // a long window: max_seqs full windows rarely fit, so the pool takes what is free after the weights (and the RoPE
    // table), less kPoolReserveBytes for the state and the lazily allocated prefill / verify workspaces.  With a draft model
    // both weight sets come off first, and the draft's pool, as many tokens as this one, takes its share of the rest.
    size_t free_b = 0, total_b = 0;
    CL_CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
    const int64_t weights = weight_bytes(cfg) + (want_draft ? weight_bytes(dm) : 0);
    const int64_t avail = (int64_t)free_b - weights - kPoolReserveBytes;
    pool_bytes = std::min(pool_bytes, target_pool_share(avail, (int64_t)kv_bytes_per_token, want_draft ? cl::kv_bytes_per_token(dm) : 0));
  }
  n_pages_ = (int)(pool_bytes / ((int64_t)page_size_ * (int64_t)kv_bytes_per_token));
  if (n_pages_ < 1) { set_last_error("kv_pool_bytes too small for one page"); return CL_ERR_INVALID_ARG; }

  CL_CUDA_OK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  CL_CUDA_OK(cudaEventCreate(&ev0_));
  CL_CUDA_OK(cudaEventCreate(&ev1_));
  int rc = alloc_weights();
  if (rc) return rc;
  // weights_path: HF llama-layout safetensors (file or model directory, weights_io.cpp); else seeded synthetic weights
  rc = wpath.empty() ? fill_synthetic(c.weights_seed) : load_safetensors(wpath);
  if (rc) return rc;
  rc = alloc_state();
  if (rc) return rc;
  if (cfg.head_dim == 128 && page_size_ == 32) {   // pool-wide KV tensor maps: persistent kernel + tensor-core batched attention
    const uint64_t rows = (uint64_t)cfg.n_layers * n_pages_ * cfg.n_kv_heads * page_size_;
    have_kv_maps_ = rows < (1ull << 31) && make_tmap_2d_bf16(&kmap_, kpool_, rows, cfg.head_dim, 64, 32) &&
                    make_tmap_2d_bf16(&vmap_, vpool_, rows, cfg.head_dim, 64, 32);
  }
  if (deterministic_) {
    if (!spec_path_ok()) { set_last_error("deterministic mode: the model shape has no tensor-core split-K path"); return CL_ERR_INVALID_ARG; }
    if (!have_kv_maps_) { set_last_error("deterministic mode: the KV pool is too large for its tensor maps"); return CL_ERR_INVALID_ARG; }
    if ((rc = ensure_small_ws()) || (rc = ensure_spec_ws())) return rc;
    DMALLOC(det_ids_, (size_t)kSpecMaxRows * 4);
    DMALLOC(det_xn_, (size_t)kSpecMaxRows * cfg.d_model * 2);
  }
  if (use_mega_ && !have_kv_maps_) {
    fprintf(stderr, "[clengine] KV tensor maps unavailable: using the per-op decode path\n");
    use_mega_ = false;
  }
  if (use_mega_ && !mega_prepare_device()) {
    fprintf(stderr, "[clengine] persistent decode kernel does not fit one CTA per SM on this device: using the per-op decode path\n");
    use_mega_ = false;
  }
  if (use_mega_) {
    std::vector<MegaLayer> ml(cfg.n_layers);
    for (int l = 0; l < cfg.n_layers; ++l)
      ml[l] = MegaLayer{layers_[l].wqkv, layers_[l].wo, layers_[l].wgu, layers_[l].wdown, layers_[l].attn_norm, layers_[l].ffn_norm,
                        kpool_ + (size_t)l * kv_layer_elems_, vpool_ + (size_t)l * kv_layer_elems_};
    DMALLOC(d_mega_layers_, ml.size() * sizeof(MegaLayer));
    CL_CUDA_OK(cudaMemcpy(d_mega_layers_, ml.data(), ml.size() * sizeof(MegaLayer), cudaMemcpyHostToDevice));
  }
  pool_.reset(new KvPool(n_pages_, page_size_));
  seqs_.assign(max_seqs_, SeqState());
  tok.reset(new ByteTokenizer(cfg.vocab_size));
  if (wdir) {   // a model directory brings its vocabulary: tokenizer.json replaces the byte-level fallback
    const std::string tj = wpath + "/tokenizer.json";
    if (stat(tj.c_str(), &wst) == 0) {
      std::string err;
      std::unique_ptr<Tokenizer> t = load_hf_tokenizer(tj, "", &err);
      if (!t) { set_last_error("tokenizer.json: " + err); return CL_ERR_IO; }
      if (t->vocab_size() > cfg.vocab_size) { set_last_error("tokenizer.json has more ids than the model's vocabulary"); return CL_ERR_IO; }
      tok = std::move(t);
      hf_tok_ = true;
    }
  }
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  {
    // Advertised throughput = CAPACITY, and load-INDEPENDENT: what this worker can deliver with a full batch, estimated
    // from the device's memory bandwidth and the model's bytes per token (70 % of the HBM roofline of one decode step x
    // max_batch).  Round 1 advertised the measured decode steps/s x max_batch; a step at B = 32 takes longer than at
    // B = 1, so busy workers advertised LESS than idle ones, crossed a half-octave bucket, and FindBestWorker's strict
    // maximum (manager.go:369-377) sent every request of a refresh interval to one idle worker.  Identical GPUs now advertise identical numbers and tie, which is what the reference's
    // constants (peer.go:319-343) did; the measured rate stays available as cl_stats.measured_tokens_per_sec.
    const double params = (double)cfg.n_layers * ((double)qkv_dim_ * cfg.d_model + (double)cfg.d_model * q_dim_ + 3.0 * cfg.d_ff * cfg.d_model) +
                          (double)cfg.vocab_size * cfg.d_model;
    double bw = 2.0 * (double)prop.memoryClockRate * 1e3 * (double)prop.memoryBusWidth / 8.0;   // bytes/s (DDR)
    if (!(bw > 1e11)) bw = 6.5e12;
    capacity_tok_per_sec_ = 0.7 * bw / (2.0 * params) * (double)max_batch_;
    tok_per_sec_ewma_ = 0.0;
  }
  // defaults of the round-2 features: see kDefault* in engine.h (flipped on once a GPU run has validated them)
  sched_prefill_chunk_ = env_int("CL_SCHED_PREFILL_CHUNK", kDefaultSchedPrefillChunk);
  if (sched_prefill_chunk_ > 0 && sched_prefill_chunk_ < 16) sched_prefill_chunk_ = 16;
  prefill_small_max_ = std::min(256, env_int("CL_PREFILL_SMALL_MAX", kDefaultPrefillSmallMax));
  device_sample_ = env_int("CL_DEVICE_SAMPLE", 1) != 0;
  verify_one_row_ = env_int("CL_VERIFY_ONE_ROW", 1) != 0;
  if (is_draft_) return CL_OK;   // a draft serves its target's drafter only: no prefix cache, shift, speculation or scheduler
  prefix_cache_ = env_int("CL_PREFIX_CACHE", c.prefix_cache) != 0;
  context_shift_ = env_int("CL_CONTEXT_SHIFT", c.context_shift) != 0;
  num_keep_ = env_int("CL_NUM_KEEP", c.num_keep);   // checked against the final window by resolve_model_config
  speculate_ = env_int("CL_SPECULATE", c.speculate);
  if (speculate_ < 0 || speculate_ > kSpecMaxDraft) { set_last_error("speculate must be 0..15"); return CL_ERR_INVALID_ARG; }
  if (want_draft && !spec_path_ok()) { set_last_error("draft model: the target's shape has no verify pass"); return CL_ERR_INVALID_ARG; }
  if (speculate_ > 0 && !spec_path_ok()) {
    fprintf(stderr, "[clengine] speculative decoding needs the tensor-core split-K path, which this model shape lacks: decoding normally\n");
    speculate_ = 0;
  }
  if (const char* v = getenv("CL_SPECULATE_BATCH")) {
    if (set_speculate_batch(atoi(v))) return CL_ERR_INVALID_ARG;
  }
  if (const char* v = getenv("CL_PREFIX_CACHE_HOST_MIB")) {
    const int rc = set_prefix_host_cache(atoll(v) * (1LL << 20));
    if (rc) return rc;
  }
  if (want_draft) {
    // same device and page size; one mirror per sequence handle; a pool of this pool's tokens; batches up to speculate_batch
    dc.device = device_;
    dc.page_size = page_size_;
    dc.max_seqs = max_seqs_;
    dc.max_batch = std::min(max_batch_, kSpecBatchMax);
    dc.use_cuda_graph = c.use_cuda_graph;
    dc.decode_path = c.decode_path;
    dc.kv_pool_bytes = (int64_t)n_pages_ * page_size_ * cl::kv_bytes_per_token(dm);
    draft_.reset(new Engine());
    draft_->is_draft_ = true;
    if (const int rc = draft_->init(dc)) return rc;
    bool same = draft_->cfg.max_seq_len == cfg.max_seq_len;
    if (hf_tok_ && draft_->hf_tok_) {
      same = same && tok->bos() == draft_->tok->bos() && tok->eos() == draft_->tok->eos();
      for (int id = 0; same && id < cfg.vocab_size; ++id) same = tok->is_stop(id) == draft_->tok->is_stop(id);
      if (!same) { set_last_error("draft model: bos / eos / stop ids differ from the target's"); return CL_ERR_INVALID_ARG; }
    }
    if (!same) { set_last_error("draft model: cannot serve the target's window"); return CL_ERR_INVALID_ARG; }
    mirror_.assign(max_seqs_, -1);
  }
  if (c.start_scheduler) start_scheduler();
  return CL_OK;
}

int Engine::alloc_weights() {
  const size_t d = cfg.d_model, F = cfg.d_ff, V = cfg.vocab_size;
  DMALLOC(embed_, V * d * 2);
  DMALLOC(lm_head_, V * d * 2);
  DMALLOC(final_norm_, d * 4);
  layers_.resize(cfg.n_layers);
  for (auto& L : layers_) {
    DMALLOC(L.attn_norm, d * 4);
    DMALLOC(L.ffn_norm, d * 4);
    DMALLOC(L.wqkv, (size_t)qkv_dim_ * d * 2);
    DMALLOC(L.wo, d * (size_t)q_dim_ * 2);
    DMALLOC(L.wgu, 2 * F * d * 2);
    DMALLOC(L.wdown, d * F * 2);
  }
  // RoPE table: computed on the host in double, rounded to fp32 — the same expression as
  // oracle/llama_oracle.c build_rope(), so both sides use bit-identical cos/sin.
  const int half = cfg.head_dim / 2;
  std::vector<float2> tab((size_t)cfg.max_seq_len * half);
  for (int p = 0; p < cfg.max_seq_len; ++p)
    for (int i = 0; i < half; ++i) {
      const double ang = (double)p * rope_inv_freq(cfg, i);
      tab[(size_t)p * half + i] = make_float2((float)cos(ang), (float)sin(ang));
    }
  DMALLOC(rope_, tab.size() * sizeof(float2));
  CL_CUDA_OK(cudaMemcpy(rope_, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice));
  kv_layer_elems_ = (size_t)n_pages_ * cfg.n_kv_heads * page_size_ * cfg.head_dim;
  DMALLOC(kpool_, kv_layer_elems_ * cfg.n_layers * 2);
  DMALLOC(vpool_, kv_layer_elems_ * cfg.n_layers * 2);
  CL_CUDA_OK(cudaMemsetAsync(kpool_, 0, kv_layer_elems_ * cfg.n_layers * 2, stream_));
  CL_CUDA_OK(cudaMemsetAsync(vpool_, 0, kv_layer_elems_ * cfg.n_layers * 2, stream_));
  return CL_OK;
}

int Engine::fill_synthetic(uint64_t seed) {
  const int d = cfg.d_model, F = cfg.d_ff, V = cfg.vocab_size;
  int n = 0;
  n += launch_synth_bf16(embed_, (int64_t)V * d, d, 1, 0, seed, K_EMBED, kLinearScale, stream_);
  n += launch_synth_bf16(lm_head_, (int64_t)V * d, d, 1, 0, seed, K_LM_HEAD, kLinearScale, stream_);
  n += launch_synth_gain(final_norm_, d, seed, K_FINAL_NORM, kNormScale, stream_);
  for (int l = 0; l < cfg.n_layers; ++l) {
    auto& L = layers_[l];
    const int b = l * 16;
    n += launch_synth_gain(L.attn_norm, d, seed, b + K_ATTN_NORM, kNormScale, stream_);
    n += launch_synth_gain(L.ffn_norm, d, seed, b + K_FFN_NORM, kNormScale, stream_);
    // q|k|v rows are stored rope-pair-interleaved per head (kernels.h: QkvEpi)
    n += launch_synth_bf16(L.wqkv, (int64_t)q_dim_ * d, d, 1, 0, seed, b + K_WQ, kLinearScale, stream_, cfg.head_dim);
    n += launch_synth_bf16(L.wqkv + (size_t)q_dim_ * d, (int64_t)kv_dim_ * d, d, 1, 0, seed, b + K_WK, kLinearScale, stream_, cfg.head_dim);
    n += launch_synth_bf16(L.wqkv + (size_t)(q_dim_ + kv_dim_) * d, (int64_t)kv_dim_ * d, d, 1, 0, seed, b + K_WV, kLinearScale, stream_, cfg.head_dim);
    n += launch_synth_bf16(L.wo, (int64_t)d * q_dim_, q_dim_, 1, 0, seed, b + K_WO, kLinearScale, stream_);
    n += launch_synth_bf16(L.wgu, (int64_t)F * d, d, 2, 0, seed, b + K_WGATE, kLinearScale, stream_);
    n += launch_synth_bf16(L.wgu, (int64_t)F * d, d, 2, 1, seed, b + K_WUP, kLinearScale, stream_);
    n += launch_synth_bf16(L.wdown, (int64_t)d * F, F, 1, 0, seed, b + K_WDOWN, kLinearScale, stream_);
  }
  launches_ += n;
  CL_CUDA_OK(cudaGetLastError());
  return CL_OK;
}

int Engine::set_tensor(int layer, int kind, const uint16_t* data, int64_t n) {
  const int64_t d = cfg.d_model, F = cfg.d_ff, V = cfg.vocab_size;
  auto copy16 = [&](__nv_bfloat16* dst, int64_t want) -> int {
    if (n != want) { set_last_error("set_tensor: wrong element count"); return CL_ERR_INVALID_ARG; }
    CL_CUDA_OK(cudaMemcpy(dst, data, (size_t)n * 2, cudaMemcpyHostToDevice));
    return CL_OK;
  };
  auto copy_gain = [&](float* dst, int64_t want) -> int {
    if (n != want) { set_last_error("set_tensor: wrong element count"); return CL_ERR_INVALID_ARG; }
    std::vector<float> f((size_t)n);
    for (int64_t i = 0; i < n; ++i) { uint32_t u = (uint32_t)data[i] << 16; memcpy(&f[i], &u, 4); }
    CL_CUDA_OK(cudaMemcpy(dst, f.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    return CL_OK;
  };
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  if (kind == K_EMBED) return copy16(embed_, V * d);
  if (kind == K_LM_HEAD) return copy16(lm_head_, V * d);
  if (kind == K_FINAL_NORM) return copy_gain(final_norm_, d);
  if (layer < 0 || layer >= cfg.n_layers) { set_last_error("set_tensor: bad layer"); return CL_ERR_INVALID_ARG; }
  auto& L = layers_[layer];
  switch (kind) {
    case K_ATTN_NORM: return copy_gain(L.attn_norm, d);
    case K_FFN_NORM: return copy_gain(L.ffn_norm, d);
    case K_WQ:
    case K_WK:
    case K_WV: {
      const int64_t rows = kind == K_WQ ? q_dim_ : kv_dim_;
      if (n != rows * d) { set_last_error("set_tensor: wrong element count"); return CL_ERR_INVALID_ARG; }
      __nv_bfloat16* dst = L.wqkv + (kind == K_WQ ? 0 : kind == K_WK ? (size_t)q_dim_ * d : (size_t)(q_dim_ + kv_dim_) * d);
      // rope-pair interleave per head: logical row (head, w) -> head*hd + (w < hd/2 ? 2w : 2(w - hd/2) + 1)
      std::vector<uint16_t> perm((size_t)n);
      const int hd = cfg.head_dim, half = hd / 2;
      for (int64_t r = 0; r < rows; ++r) {
        const int64_t head = r / hd;
        const int w = (int)(r % hd);
        const int64_t rr = head * hd + (w < half ? 2 * w : 2 * (w - half) + 1);
        memcpy(&perm[(size_t)rr * d], data + (size_t)r * d, (size_t)d * 2);
      }
      CL_CUDA_OK(cudaMemcpy(dst, perm.data(), (size_t)n * 2, cudaMemcpyHostToDevice));
      return CL_OK;
    }
    case K_WO: return copy16(L.wo, d * q_dim_);
    case K_WDOWN: return copy16(L.wdown, d * F);
    case K_WGATE:
    case K_WUP: {
      if (n != F * d) { set_last_error("set_tensor: wrong element count"); return CL_ERR_INVALID_ARG; }
      // interleave on the device side with a strided 2-D copy: row r -> row 2r (+1 for up)
      CL_CUDA_OK(cudaMemcpy2D(L.wgu + (kind == K_WUP ? d : 0), (size_t)2 * d * 2, data, (size_t)d * 2, (size_t)d * 2, (size_t)F,
                              cudaMemcpyHostToDevice));
      return CL_OK;
    }
    default: set_last_error("set_tensor: bad kind"); return CL_ERR_INVALID_ARG;
  }
}

int Engine::alloc_state() {
  const size_t S = max_seqs_, d = cfg.d_model;
  DMALLOC(d_tok_, S * 4);
  DMALLOC(d_pos_, S * 4);
  DMALLOC(d_bt_, S * max_pages_per_seq_ * 4);
  DMALLOC(d_shift_items_, ((size_t)max_pages_per_seq_ + 1) * sizeof(KvShiftItem));
  DMALLOC(d_slots_, (size_t)max_batch_ * 4);
  DMALLOC(d_h_, S * d * 4);
  DMALLOC(d_q_, S * q_dim_ * 4);
  DMALLOC(d_attn_, S * q_dim_ * 4);
  DMALLOC(d_act_, S * (size_t)cfg.d_ff * 4);
  DMALLOC(d_logits_, S * (size_t)cfg.vocab_size * 4);
  const int rep = cfg.n_heads / cfg.n_kv_heads;
  DMALLOC(d_attn_part_, S * cfg.n_kv_heads * nsplit_ * rep * (cfg.head_dim + 2) * 4);
  DMALLOC(d_attn_cnt_, S * cfg.n_kv_heads * 4);
  DMALLOC(d_tail_val_, S * kTailBlocks * 4);
  DMALLOC(d_tail_idx_, S * kTailBlocks * 4);
  DMALLOC(d_tail_cnt_, S * 4);
  DMALLOC(d_samp_mode_, S * 4);
  DMALLOC(d_samp_par_, S * sizeof(SampleParams));
  DMALLOC(d_samp_step_, S * 8);
  DMALLOC(d_samp_hist_, S * kSampleHistMax * 4);
  DMALLOC(d_samp_hlen_, S * 4);
  DMALLOC(d_samp_cand_, S * kTailBlocks * kSampleTopKMax * 8);
  CL_CUDA_OK(cudaMemsetAsync(d_samp_mode_, 0, S * 4, stream_));
  samp_hlen_.assign(S, -1);
  // logprobs: the captured step graphs point at these, so they exist from the start (the ring and its pinned mirror hold
  // ring_steps_ x max_batch_ records of 184 bytes: 24.1 MB each at max_batch 128)
  DMALLOC(d_lp_n_, S * 4);
  DMALLOC(d_lp_part_, S * kTailBlocks * sizeof(float2));
  DMALLOC(d_lp_cand_, S * kTailBlocks * kLogprobTopMax * 8);
  DMALLOC(d_lp_cnt_, S * 4);
  DMALLOC(d_lp_last_, S * sizeof(LogprobRecord));
  DMALLOC(d_lp_ring_, (size_t)ring_steps_ * max_batch_ * sizeof(LogprobRecord));
  CL_CUDA_OK(cudaMemsetAsync(d_lp_n_, 0xFF, S * 4, stream_));   // -1: off
  CL_CUDA_OK(cudaMemsetAsync(d_lp_cnt_, 0, S * 4, stream_));
  lp_n_.assign(S, -1);
  DMALLOC(d_ids_ring_, (size_t)ring_steps_ * max_batch_ * 4);
  DMALLOC(d_step_counter_, 4);
  n_sync_ = cfg.n_layers * 10 + 1;   // persistent kernel: 6 grid barriers + 4 tile counters per layer + the lookahead frontier
  DMALLOC(d_sync_, (size_t)n_sync_ * 4);
  CL_CUDA_OK(cudaMemsetAsync(d_sync_, 0, (size_t)n_sync_ * 4, stream_));
  if (want_timeline_) {
    DMALLOC(d_timeline_, (size_t)(cfg.n_layers * 5 + 1) * 4 * 8);   // >= n_layers * 16 stamps for the megakernel view
    CL_CUDA_OK(cudaMemsetAsync(d_timeline_, 0, (size_t)(cfg.n_layers * 5 + 1) * 4 * 8, stream_));
  }
  // token tile of the projections = 32 / 64 / 128 rows (gemm_wgmma.cu picks it from the step's batch size)
  use_batch_gemm_ = env_int("CL_BATCH_GEMM", 1) != 0 && max_batch_ >= 2 && gemm_tc_supported(max_batch_, cfg.d_model, cfg.d_model) &&
                    max_batch_ <= 128;
  if (use_batch_gemm_) {
    bws_.reset(new BatchWs());
    const size_t Bm = max_batch_, widest = std::max<size_t>((size_t)qkv_dim_, std::max<size_t>(2 * (size_t)cfg.d_ff, d));
    DMALLOC(bws_->xn, Bm * d * 2);
    DMALLOC(bws_->attn, Bm * q_dim_ * 2);
    DMALLOC(bws_->act, Bm * (size_t)cfg.d_ff * 2);
    CL_CUDA_OK(cudaMemsetAsync(bws_->xn, 0, Bm * d * 2, stream_));
    CL_CUDA_OK(cudaMemsetAsync(bws_->attn, 0, Bm * q_dim_ * 2, stream_));
    CL_CUDA_OK(cudaMemsetAsync(bws_->act, 0, Bm * (size_t)cfg.d_ff * 2, stream_));
    // split-K partial workspace of the four projections (pick_splits)
    size_t part_floats = 4 * Bm * widest;
    for (int nk : {0, 1, 2, 3}) {
      const int N = nk == 0 ? qkv_dim_ : nk == 2 ? 2 * cfg.d_ff : d, K = nk == 1 ? q_dim_ : nk == 3 ? cfg.d_ff : d;
      part_floats = std::max(part_floats, (size_t)pick_splits(N, K) * Bm * (size_t)N);
    }
    DMALLOC(bws_->part, part_floats * 4);
    DMALLOC(bws_->logits, Bm * (size_t)cfg.vocab_size * 4);
  }
  prompt_cap_ = cfg.max_seq_len;
  // also the input ids of a verify pass over several sequences, up to kSpecMaxRows even when max_seq_len is smaller
  DMALLOC(d_prompt_, (size_t)std::max(prompt_cap_, kSpecMaxRows) * 4);
  CL_CUDA_OK(cudaMemsetAsync(d_tok_, 0, S * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(d_pos_, 0, S * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(d_bt_, 0, S * max_pages_per_seq_ * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(d_slots_, 0, (size_t)max_batch_ * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(d_attn_cnt_, 0, S * cfg.n_kv_heads * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(d_tail_cnt_, 0, S * 4, stream_));
  CL_CUDA_OK(cudaMemsetAsync(d_step_counter_, 0, 4, stream_));
  CL_CUDA_OK(cudaMallocHost(&h_logits_pinned_, (size_t)cfg.vocab_size * 4));
  CL_CUDA_OK(cudaMallocHost(&h_ids_pinned_, (size_t)ring_steps_ * max_batch_ * 4));
  CL_CUDA_OK(cudaMallocHost(&h_lp_pinned_, (size_t)std::max(ring_steps_ * max_batch_, max_seqs_) * sizeof(LogprobRecord)));
  return CL_OK;
}

// ---- sequences ----------------------------------------------------------------------------------
int Engine::seq_create(cl_seq_t* out) {
  for (int i = 0; i < max_seqs_; ++i)
    if (!seqs_[i].live) {
      seqs_[i] = SeqState();
      seqs_[i].live = true;
      *out = i;
      const int rc = disarm_sampling(i);
      return rc ? rc : upload_logprobs(i, -1);
    }
  set_last_error("no free sequence slot (max_seqs)");
  return CL_ERR_OOM;
}
int Engine::seq_free(cl_seq_t s) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  pool_->release(s);
  seqs_[s] = SeqState();
  if (draft_ && mirror_[s] >= 0) {   // the draft's mirror of s goes with it
    const int rc = draft_->seq_free(mirror_[s]);
    mirror_[s] = -1;
    draft_pages_ = draft_->pool_->used_pages();
    if (rc) return rc;
  }
  const int rc = disarm_sampling(s);
  return rc ? rc : upload_logprobs(s, -1);
}

int Engine::set_logprobs(cl_seq_t s, int top_n) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (top_n < -1 || top_n > kLogprobTopMax) { set_last_error("logprobs: top_n must be -1..20"); return CL_ERR_INVALID_ARG; }
  if (top_n >= 0 && cfg.vocab_size > kTailBlocks * kSampleSliceMax) { set_last_error("logprobs: vocabulary above 163840"); return CL_ERR_INVALID_ARG; }
  seqs_[s].lps.clear();
  return upload_logprobs(s, top_n);
}

int Engine::upload_logprobs(cl_seq_t s, int top_n) {
  if (lp_n_[s] == top_n) return CL_OK;
  CL_CUDA_OK(cudaMemcpyAsync(d_lp_n_ + s, &top_n, 4, cudaMemcpyHostToDevice, stream_));
  lp_n_[s] = top_n;
  return CL_OK;
}

int Engine::take_logprobs(cl_seq_t s, cl_token_logprob* out, int cap, int* n_out) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  auto& q = seqs_[s].lps;
  if (!out) { *n_out = (int)q.size(); return CL_OK; }
  if (cap < 0) return CL_ERR_INVALID_ARG;
  const int n = std::min(cap, (int)q.size());
  for (int i = 0; i < n; ++i) out[i] = to_token_logprob(q[(size_t)i]);
  q.erase(q.begin(), q.begin() + n);
  *n_out = n;
  return CL_OK;
}

int Engine::collect_logprobs(const cl_seq_t* ss, int n) {
  bool any = false;
  for (int i = 0; i < n; ++i) any = any || lp_n_[ss[i]] >= 0;
  if (!any) return CL_OK;
  CL_CUDA_OK(cudaMemcpyAsync(h_lp_pinned_, d_lp_last_, (size_t)max_seqs_ * sizeof(LogprobRecord), cudaMemcpyDeviceToHost, stream_));
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  for (int i = 0; i < n; ++i)
    if (lp_n_[ss[i]] >= 0) seqs_[ss[i]].lps.push_back(h_lp_pinned_[ss[i]]);
  return CL_OK;
}

int Engine::set_sampling_ext(cl_seq_t s, const SamplerExt& ext) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (int rc = check_sampling_ext(ext, nullptr)) return rc;
  seqs_[s].ext = ext;
  return CL_OK;
}

int Engine::arm_sampling(cl_seq_t s, const cl_sampling& sp, uint64_t step0, const int32_t* hist, int n_hist) {
  const SamplerExt& ext = seqs_[s].ext;
  if (!device_sampling_ok(sp, cfg.vocab_size, ext)) { set_last_error("sampling settings need the host sampler"); return CL_ERR_INVALID_ARG; }
  const SampleParams par = sample_params(sp, ext);
  std::vector<int> ring(kSampleHistMax, 0);
  for (int i = std::max(0, n_hist - kSampleHistMax); i < n_hist; ++i) ring[i % kSampleHistMax] = hist[i];
  const int mode = 1;
  const unsigned long long st = step0;
  CL_CUDA_OK(cudaMemcpyAsync(d_samp_par_ + s, &par, sizeof par, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_samp_step_ + s, &st, 8, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_samp_hist_ + (size_t)s * kSampleHistMax, ring.data(), kSampleHistMax * 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_samp_hlen_ + s, &n_hist, 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_samp_mode_ + s, &mode, 4, cudaMemcpyHostToDevice, stream_));
  samp_hlen_[s] = n_hist;
  return CL_OK;
}

int Engine::disarm_sampling(cl_seq_t s) {
  if (samp_hlen_[s] < 0) return CL_OK;
  const int mode = 0;
  CL_CUDA_OK(cudaMemcpyAsync(d_samp_mode_ + s, &mode, 4, cudaMemcpyHostToDevice, stream_));
  samp_hlen_[s] = -1;
  return CL_OK;
}

int Engine::read_next_token(cl_seq_t s, int32_t* out) {
  CL_CUDA_OK(cudaMemcpyAsync(h_ids_pinned_, d_tok_ + s, 4, cudaMemcpyDeviceToHost, stream_));
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  *out = h_ids_pinned_[0];
  return CL_OK;
}

int Engine::ensure_capacity(cl_seq_t s, int n_tokens) {
  if (n_tokens > cfg.max_seq_len) { set_last_error("sequence exceeds max_seq_len"); return CL_ERR_TOO_LONG; }
  const size_t before = pool_->pages_of(s).size();
  const int rc = pool_->reserve(s, n_tokens);
  if (rc) { set_last_error("KV page pool exhausted"); return rc; }
  if (const int mrc = drain_kv_moves()) return mrc;
  const auto& pages = pool_->pages_of(s);
  if (pages.size() != before)
    CL_CUDA_OK(cudaMemcpyAsync(d_bt_ + (size_t)s * max_pages_per_seq_ + before, pages.data() + before,
                               (pages.size() - before) * 4, cudaMemcpyHostToDevice, stream_));
  return CL_OK;
}

void Engine::seq_advance(cl_seq_t s, const int32_t* ids, int n, int n_known) {
  auto& q = seqs_[s];
  if (q.known == (int)q.history.size()) q.known += n_known;
  q.len += n;
  q.history.insert(q.history.end(), ids, ids + n);
  if (prefix_cache_ && q.known >= page_size_) pool_->publish(s, q.history.data(), q.known);
}

// ---- prefix cache ---------------------------------------------------------------------------------
int Engine::attach_prefix(cl_seq_t s, const int32_t* ids, int n, int* reused) {
  *reused = 0;
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (!prefix_cache_) return CL_OK;
  auto& q = seqs_[s];
  if (q.len != 0 || !pool_->pages_of(s).empty()) { set_last_error("attach_prefix needs a new sequence (no tokens, no pages)"); return CL_ERR_INVALID_ARG; }
  const int r = pool_->attach(s, ids, std::min(n, cfg.max_seq_len));   // >= 0: the owner has no pages
  if (const int mrc = drain_kv_moves()) return mrc;
  prefix_lookups_++;
  prefix_tokens_looked_up_ += n;
  prefix_tokens_reused_ += r;
  if (r == 0) return CL_OK;
  const auto& pages = pool_->pages_of(s);
  CL_CUDA_OK(cudaMemcpyAsync(d_bt_ + (size_t)s * max_pages_per_seq_, pages.data(), pages.size() * 4, cudaMemcpyHostToDevice, stream_));
  q.len = r;
  q.known = r;
  q.history.assign(ids, ids + r);
  *reused = r;
  return CL_OK;
}

// ---- context shift --------------------------------------------------------------------------------
int Engine::seq_shift(cl_seq_t s, int n_keep, int n_discard) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  auto& q = seqs_[s];
  std::vector<KvShiftItem> items;
  const int rc = pool_->shift(s, q.len, n_keep, n_discard, &items);
  if (rc == CL_ERR_OOM) { set_last_error("context shift: no free page for a copy of a shared page"); return rc; }
  if (rc) { set_last_error("context shift: n_discard must be a positive multiple of page_size and n_keep + n_discard <= len"); return rc; }
  if (const int mrc = drain_kv_moves()) return mrc;   // a copy's page may have been spilled to the host tier first
  const auto& pages = pool_->pages_of(s);
  if (!pages.empty())
    CL_CUDA_OK(cudaMemcpyAsync(d_bt_ + (size_t)s * max_pages_per_seq_, pages.data(), pages.size() * 4, cudaMemcpyHostToDevice, stream_));
  if (!items.empty()) {
    CL_CUDA_OK(cudaMemcpyAsync(d_shift_items_, items.data(), items.size() * sizeof(KvShiftItem), cudaMemcpyHostToDevice, stream_));
    KvShiftArgs a;
    a.items = d_shift_items_; a.n_items = (int)items.size();
    a.kpool = kpool_; a.vpool = vpool_; a.layer_elems = kv_layer_elems_;
    a.n_layers = cfg.n_layers; a.n_kv = cfg.n_kv_heads; a.head_dim = cfg.head_dim; a.page_size = page_size_;
    a.rope_row = rope_ + (size_t)n_discard * (cfg.head_dim / 2);   // n_discard < len - n_keep <= max_seq_len when a row is kept
    int launches = 0;
    LaunchProfiler prof(stream_, nullptr);
    CL_LAUNCH(launch_kv_shift(a, stream_));
    launches_ += launches;
  }
  q.len -= n_discard;
  CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &q.len, 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  return CL_OK;
}

int Engine::prefix_stats(cl_prefix_stats* out) {
  memset(out, 0, sizeof *out);
  out->enabled = prefix_cache_ ? 1 : 0;
  out->cached_pages = pool_ ? pool_->cached_pages() : 0;
  out->lookups = prefix_lookups_;
  out->tokens_looked_up = prefix_tokens_looked_up_;
  out->tokens_reused = prefix_tokens_reused_;
  out->pages_evicted = pool_ ? pool_->evicted_pages() : 0;
  if (pool_) {
    out->host_pages = pool_->host_pages();
    out->host_pages_cached = pool_->host_cached_pages();
    out->pages_to_host = pool_->pages_to_host();
    out->pages_from_host = pool_->pages_from_host();
  }
  return CL_OK;
}

int Engine::set_prefix_host_cache(int64_t bytes) {
  const int64_t page_bytes = 2LL * (int64_t)kv_layer_elems_ / n_pages_ * cfg.n_layers * 2;   // K and V of every layer
  if (bytes < 0 || (bytes > 0 && bytes < page_bytes)) { set_last_error("prefix host cache: bytes must be 0 or at least one page"); return CL_ERR_INVALID_ARG; }
  if (!prefix_cache_) { set_last_error("prefix host cache needs the prefix cache"); return CL_ERR_INVALID_ARG; }
  bool busy = std::any_of(seqs_.begin(), seqs_.end(), [](const SeqState& q) { return q.live; });
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    busy = busy || !queue_.empty() || !active_.empty() || prefilling_;
  }
  if (busy) { set_last_error("prefix host cache can only be resized with no sequence live or queued"); return CL_ERR_INVALID_ARG; }
  const int64_t n = bytes / page_bytes;
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  pool_->set_host_pages(0);   // no moves are pending: every reserve and attach drains its own
  if (host_kv_) {
    CL_CUDA_OK(cudaFreeHost(host_kv_));
    host_kv_ = nullptr;
  }
  if (n == 0) return CL_OK;
  if (!d_moves_) DMALLOC(d_moves_, (size_t)2 * n_pages_ * sizeof(int2));
  void* h = nullptr;
  if (n > INT32_MAX || cudaHostAlloc(&h, (size_t)(n * page_bytes), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    set_last_error("prefix host cache: cannot pin " + std::to_string(n * page_bytes) + " bytes of host memory");
    return CL_ERR_OOM;
  }
  host_kv_ = static_cast<uint4*>(h);
  pool_->set_host_pages((int)n);
  return CL_OK;
}

int Engine::drain_kv_moves() {
  const auto& mv = pool_->moves();
  if (mv.empty()) return CL_OK;   // always so with the host tier off
  std::vector<int2> buf(mv.size());
  for (size_t i = 0; i < mv.size(); ++i) buf[i] = make_int2(mv[i].page, mv[i].host);
  CL_CUDA_OK(cudaMemcpyAsync(d_moves_, buf.data(), buf.size() * sizeof(int2), cudaMemcpyHostToDevice, stream_));
  KvMoveArgs a;
  a.kpool = kpool_; a.vpool = vpool_; a.layer_elems = kv_layer_elems_; a.host = host_kv_; a.n_layers = cfg.n_layers;
  a.blk_vec = (int)(kv_layer_elems_ / n_pages_ * 2 / 16);
  int launches = 0;
  LaunchProfiler prof(stream_, nullptr);
  // one launch per run of same-kind moves in which no device page and no host page repeats
  std::set<int> pages, hosts;
  size_t i0 = 0;
  for (size_t i = 0; i <= mv.size(); ++i) {
    if (i < mv.size() && mv[i].kind == mv[i0].kind && pages.insert(mv[i].page).second && hosts.insert(mv[i].host).second) continue;
    a.moves = d_moves_ + i0;
    a.n_moves = (int)(i - i0);
    CL_LAUNCH(launch_kv_move(mv[i0].kind == KvPool::kSpill, a, stream_));
    if (i == mv.size()) break;
    pages = {mv[i].page};
    hosts = {mv[i].host};
    i0 = i;
  }
  launches_ += launches;
  pool_->clear_moves();
  return CL_OK;
}

// ---- per-launch event profiler (CL_PREFILL_PROFILE, CL_STEP_PROFILE) ----------------------------
LaunchProfiler::LaunchProfiler(cudaStream_t st, const char* env) : st_(st) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  on_ = env && env_int(env, 0) != 0 && cap == cudaStreamCaptureStatusNone;
  mark("start");
}

void LaunchProfiler::mark(const char* call) {
  if (!on_) return;
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, st_);
  ev_.push_back(e);
  name_.push_back(call);
}

void LaunchProfiler::report(const char* tag, int key_width, const std::string& head) {
  if (!on_ || ev_.size() < 2) return;
  cudaStreamSynchronize(st_);
  std::map<std::string, std::pair<double, int>> acc;
  double total = 0.0;
  for (size_t i = 1; i < ev_.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_[i - 1], ev_[i]);
    const std::string full(name_[i]);
    std::string key = full.substr(0, full.find('('));
    auto has = [&](const char* arg) { return full.find(arg) != std::string::npos; };
    if (key == "launch_gemm_bf16")     // split by projection: the weight argument names it
      key += has("L.wqkv") ? ":qkv" : has("L.wo") ? ":o" : has("L.wgu") ? ":gate|up" : has("lm_head_") ? ":lm_head" : ":down";
    acc[key].first += ms; acc[key].second += 1;
    total += ms;
  }
  fprintf(stderr, "[%s] %s, %zu launches, %.3f ms on the device\n", tag, head.c_str(), ev_.size() - 1, total);
  for (auto& kv : acc)
    fprintf(stderr, "[%s]   %-*s n=%4d total %8.3f ms  mean %8.2f us\n", tag, key_width, kv.first.c_str(), kv.second.second, kv.second.first,
            1e3 * kv.second.first / kv.second.second);
  for (auto e : ev_) cudaEventDestroy(e);
  ev_.clear(); name_.clear();
}

// ---- one token step for the sequences listed in d_slots_[0..B) -----------------------------------
int Engine::enqueue_step(int B, int step_off) {
  if (deterministic_) return det_step(B, step_off);
  if (B >= 2 && use_batch_gemm_ && bws_) return enqueue_step_batched(B);   // from B = 2: faster than two GEMV passes
  const int d = cfg.d_model, F = cfg.d_ff, L_ = cfg.n_layers;
  int launches = 0;
  LaunchProfiler prof(stream_, nullptr);
  auto tl = [&](int l, int k) -> long long* { return d_timeline_ ? d_timeline_ + ((size_t)l * 5 + k) * 4 : nullptr; };
  CL_LAUNCH(launch_embed(embed_, d, d_tok_, d_h_, d, d_slots_, B, stream_));
  const bool mega = use_mega_ && B == 1 && d_mega_layers_ != nullptr;
  if (probe_ev_) cudaEventRecord(probe_ev_[probe_idx_], stream_);
  if (mega) {
    MegaArgs m;
    m.layers = d_mega_layers_; m.n_layers = L_; m.q_dim = q_dim_; m.qkv_dim = qkv_dim_; m.n_heads = cfg.n_heads; m.n_kv = cfg.n_kv_heads;
    m.nsplit = nsplit_; m.eps = cfg.rms_eps; m.rope = rope_; m.pos = d_pos_; m.block_tables = d_bt_; m.bt_stride = max_pages_per_seq_;
    m.slots = d_slots_; m.h = d_h_; m.q = d_q_; m.attn_x = d_attn_; m.act = d_act_; m.part = d_attn_part_; m.bars = d_sync_; m.tile_ctr = d_sync_ + (size_t)L_ * 6; m.pf_ctr = d_sync_ + (size_t)L_ * 10;
    m.tl = d_timeline_; m.tl_cta = env_int("CL_TIMELINE_CTA", 0);
    m.kv_layer_rows = (long long)n_pages_ * cfg.n_kv_heads * page_size_; m.kmap = kmap_; m.vmap = vmap_;
    CL_LAUNCH(launch_decode_mega(m, stream_));
  }
  for (int l = 0; l < (mega ? 0 : L_); ++l) {
    const auto& L = layers_[l];
    GemvArgs g;
    g.slots = d_slots_; g.batch = B;
    // (1) RMSNorm + fused q|k|v projection; epilogue: RoPE + bf16 round + q out + KV append into the paged cache
    g.W = L.wqkv; g.N = qkv_dim_; g.K = d; g.h = d_h_; g.gain = L.attn_norm; g.eps = cfg.rms_eps;
    g.y = d_q_; g.x_stride = d; g.y_stride = q_dim_;
    g.qkv.rope = rope_; g.qkv.pos = d_pos_; g.qkv.block_tables = d_bt_; g.qkv.bt_stride = max_pages_per_seq_;
    g.qkv.kpool = kpool_ + (size_t)l * kv_layer_elems_; g.qkv.vpool = vpool_ + (size_t)l * kv_layer_elems_;
    g.qkv.n_heads = cfg.n_heads; g.qkv.n_kv = cfg.n_kv_heads; g.qkv.head_dim = cfg.head_dim; g.qkv.page_size = page_size_;
    g.tl = tl(l, 0);
    CL_LAUNCH(launch_gemv(gemv_variant_, EPI_QKV, true, g, stream_, use_pdl_));
    // (2) paged GQA attention over tokens 0..pos
    AttnDecodeArgs a;
    a.q = d_q_; a.q_stride = q_dim_;
    a.kpool = kpool_ + (size_t)l * kv_layer_elems_; a.vpool = vpool_ + (size_t)l * kv_layer_elems_;
    a.block_tables = d_bt_; a.bt_stride = max_pages_per_seq_; a.pos = d_pos_;
    a.out = d_attn_; a.out_stride = q_dim_; a.part = d_attn_part_; a.counters = d_attn_cnt_;
    a.slots = d_slots_; a.batch = B; a.n_heads = cfg.n_heads; a.n_kv = cfg.n_kv_heads; a.head_dim = cfg.head_dim;
    a.page_size = page_size_; a.nsplit = nsplit_; a.tl = tl(l, 1);
    CL_LAUNCH(launch_attn_decode(a, stream_, use_pdl_));
    // (3) o projection + residual
    GemvArgs o;
    o.slots = d_slots_; o.batch = B;
    o.W = L.wo; o.N = d; o.K = q_dim_; o.x = d_attn_; o.x_stride = q_dim_; o.y = d_h_; o.resid = d_h_; o.y_stride = d; o.tl = tl(l, 2);
    CL_LAUNCH(launch_gemv(gemv_variant_, EPI_RESID, false, o, stream_, use_pdl_));
    // (4) RMSNorm + gate/up + SiLU*mul
    GemvArgs u;
    u.slots = d_slots_; u.batch = B;
    u.W = L.wgu; u.N = 2 * F; u.K = d; u.h = d_h_; u.gain = L.ffn_norm; u.eps = cfg.rms_eps; u.y = d_act_;
    u.x_stride = d; u.y_stride = F; u.tl = tl(l, 3);
    CL_LAUNCH(launch_gemv(gemv_variant_, EPI_GATEUP, true, u, stream_, use_pdl_));
    // (5) down projection + residual
    GemvArgs w;
    w.slots = d_slots_; w.batch = B;
    w.W = L.wdown; w.N = d; w.K = F; w.x = d_act_; w.x_stride = F; w.y = d_h_; w.resid = d_h_; w.y_stride = d; w.tl = tl(l, 4);
    CL_LAUNCH(launch_gemv(gemv_variant_, EPI_RESID, false, w, stream_, use_pdl_));
  }
  if (probe_ev_) cudaEventRecord(probe_ev_[probe_idx_ + 1], stream_);
  CL_LAUNCH(enqueue_lm_head(B, use_pdl_ && !mega));
  CL_LAUNCH(enqueue_step_tail(B, true));
  return launches;
}

// The LM head of a single-slot step or prefill: final RMSNorm + GEMV of d_h_ into d_logits_.
int Engine::enqueue_lm_head(int B, bool pdl) {
  GemvArgs lm;
  lm.slots = d_slots_; lm.batch = B;
  lm.W = lm_head_; lm.N = cfg.vocab_size; lm.K = cfg.d_model; lm.h = d_h_; lm.gain = final_norm_; lm.eps = cfg.rms_eps;
  lm.y = d_logits_; lm.x_stride = cfg.d_model; lm.y_stride = cfg.vocab_size;
  lm.tl = d_timeline_ ? d_timeline_ + (size_t)cfg.n_layers * 5 * 4 : nullptr;
  return launch_gemv(gemv_variant_, EPI_STORE, true, lm, stream_, pdl);
}

// The tail of every decode step and prefill: greedy id (or, on slots armed by arm_sampling, a draw) of d_logits_ for
// d_slots_[0..B) into d_tok_ and the id ring, d_pos_ += 1.  It also zeroes the persistent kernel's counters.  They are zero whenever no step is running, so the
// zeroing is needed only behind the persistent kernel and harmless everywhere else.
int Engine::enqueue_step_tail(int B, bool push_input) {
  StepTailArgs t;
  t.logits = d_logits_; t.vocab = cfg.vocab_size; t.tok = d_tok_; t.pos = d_pos_; t.ids_ring = d_ids_ring_;
  t.step_counter = d_step_counter_; t.ring_steps = ring_steps_; t.ring_stride = max_batch_;
  t.part_val = d_tail_val_; t.part_idx = d_tail_idx_; t.counters = d_tail_cnt_; t.slots = d_slots_; t.batch = B;
  t.sync_counters = d_sync_; t.n_sync_counters = n_sync_;
  SampleState& smp = t.sample;
  smp.mode = d_samp_mode_; smp.par = d_samp_par_; smp.step = d_samp_step_; smp.hist = d_samp_hist_; smp.hist_len = d_samp_hlen_;
  smp.cand = d_samp_cand_; smp.push_input = push_input ? 1 : 0;
  LogprobState& lp = t.lp;
  lp.top_n = d_lp_n_; lp.part = d_lp_part_; lp.cand = d_lp_cand_; lp.counters = d_lp_cnt_; lp.last = d_lp_last_; lp.ring = d_lp_ring_;
  return launch_step_tail(t, stream_);
}

// ---- batched token step (B >= 2): tensor-core projections (wgmma, split-K) + per-sequence glue -----
// split-K count of a batched-decode projection: the launch is as slow as its busiest CTA, i.e.
// rounds(= ceil(tiles * s / SMs)) x k-blocks per unit.  224 gate|up tiles on 132 SMs cost 2 x 64 k-blocks unsplit but
// 9 x 13 with 5 splits.  Among the counts within 10 % of the best the smallest wins
// (fewer partials for the consumer kernel to sum).
int pick_splits_public(int n_rows, int K) { return pick_splits(n_rows, K); }
static int pick_splits(int n_rows, int K) { return pick_splits_sms(n_rows, K, sm_count()); }
int pick_splits_sms(int n_rows, int K, int sms) {
  const int tiles = (n_rows + 127) / 128, nkb = (K + 63) / 64;
  int best_cost = 1 << 30;
  int cost_of[17];
  for (int s = 1; s <= 16; ++s) {
    const int kbp = (nkb + s - 1) / s;
    cost_of[s] = -1;
    if ((nkb + kbp - 1) / kbp != s) continue;                 // every split must own >= 1 k-block
    cost_of[s] = ((tiles * s + sms - 1) / sms) * kbp;
    best_cost = std::min(best_cost, cost_of[s]);
  }
  for (int s = 1; s <= 16; ++s)
    if (cost_of[s] >= 0 && cost_of[s] * 10 <= best_cost * 11) return s;
  return 1;
}

int Engine::enqueue_step_batched(int B) {
  const int d = cfg.d_model, F = cfg.d_ff, L_ = cfg.n_layers, V = cfg.vocab_size;
  int launches = 0;
  LaunchProfiler prof(stream_, "CL_STEP_PROFILE");   // eager launches only (CL_GRAPH=0)
  BatchWs& w = *bws_;
  const bool bp = use_pdl_;   // programmatic dependent launch between the kernels of the batched step
  const int s_qkv = pick_splits(qkv_dim_, d), s_o = pick_splits(d, q_dim_), s_gu = pick_splits(2 * F, d), s_dn = pick_splits(d, F);
  CL_LAUNCH(launch_embed(embed_, d, d_tok_, d_h_, d, d_slots_, B, stream_));
  const float* pending = nullptr;   // split-K partials of the previous residual projection, folded into the next norm
  int pending_s = 0;
  for (int l = 0; l < L_; ++l) {
    const auto& L = layers_[l];
    CL_LAUNCH(launch_batch_resid_norm(d_h_, d, pending, pending_s, B, L.attn_norm, cfg.rms_eps, w.xn, d_slots_, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.xn, L.wqkv, w.part, nullptr, B, qkv_dim_, d, stream_, s_qkv, bp));
    QkvEpi e;
    e.rope = rope_; e.pos = d_pos_; e.block_tables = d_bt_; e.bt_stride = max_pages_per_seq_;
    e.kpool = kpool_ + (size_t)l * kv_layer_elems_; e.vpool = vpool_ + (size_t)l * kv_layer_elems_;
    e.n_heads = cfg.n_heads; e.n_kv = cfg.n_kv_heads; e.head_dim = cfg.head_dim; e.page_size = page_size_;
    CL_LAUNCH(launch_batch_rope_append(w.part, s_qkv, B, e, d_q_, q_dim_, d_slots_, stream_, bp));
    AttnDecodeArgs a;
    a.q = d_q_; a.q_stride = q_dim_;
    a.kpool = e.kpool; a.vpool = e.vpool; a.block_tables = d_bt_; a.bt_stride = max_pages_per_seq_; a.pos = d_pos_;
    a.out = d_attn_; a.out_stride = q_dim_; a.out_bf16 = w.attn; a.part = d_attn_part_; a.counters = d_attn_cnt_;   // bf16 copy = X of the o-projection
    a.slots = d_slots_; a.batch = B; a.n_heads = cfg.n_heads; a.n_kv = cfg.n_kv_heads; a.head_dim = cfg.head_dim;
    // many sequences already fill the machine: fewer KV splits per sequence (cheaper combine, fewer CTAs)
    a.page_size = page_size_;
    attn_decode_tc_plan(cfg.n_kv_heads, B, nsplit_, sm_count(), &a.nsplit, &a.tc_small);
    if (have_kv_maps_ && attn_decode_tc_supported(cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, page_size_, a.nsplit))
      CL_LAUNCH(launch_attn_decode_tc(a, kmap_, vmap_, (long long)l * n_pages_ * cfg.n_kv_heads * page_size_, stream_, bp));
    else
      CL_LAUNCH(launch_attn_decode(a, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.attn, L.wo, w.part, nullptr, B, d, q_dim_, stream_, s_o, bp));
    CL_LAUNCH(launch_batch_resid_norm(d_h_, d, w.part, s_o, B, L.ffn_norm, cfg.rms_eps, w.xn, d_slots_, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.xn, L.wgu, w.part, nullptr, B, 2 * F, d, stream_, s_gu, bp));
    CL_LAUNCH(launch_batch_silu(w.part, s_gu, B, F, w.act, stream_, bp));
    CL_LAUNCH(launch_gemm_bf16(w.act, L.wdown, w.part, nullptr, B, d, F, stream_, s_dn, bp));
    pending = w.part; pending_s = s_dn;
  }
  CL_LAUNCH(launch_batch_resid_norm(d_h_, d, pending, pending_s, B, final_norm_, cfg.rms_eps, w.xn, d_slots_, stream_, bp));
  CL_LAUNCH(launch_gemm_bf16(w.xn, lm_head_, w.logits, nullptr, B, V, d, stream_, 1, bp));
  CL_LAUNCH(launch_batch_scatter_rows(w.logits, V, d_logits_, V, d_slots_, B, stream_));
  CL_LAUNCH(enqueue_step_tail(B, true));
  prof.report("step profile", 34, "B=" + std::to_string(B));
  return launches;
}

// Capture + instantiate + upload the step graph of batch size B (no launch).  Returns true if graphs_[B] exists afterwards.
bool Engine::ensure_graph(int B) {
  if (!use_graph_ || graph_failed_) return false;
  if (graphs_.count(B)) return true;
  for (int attempt = 0; attempt < 2; ++attempt) {
    cudaGraph_t g = nullptr;
    cudaGraphExec_t ex = nullptr;
    cudaError_t e = cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal);
    int n = e == cudaSuccess ? enqueue_step(B) : -1;
    cudaError_t e2 = cudaStreamEndCapture(stream_, &g);
    if (e == cudaSuccess && n > 0 && e2 == cudaSuccess && g) e = cudaGraphInstantiate(&ex, g, 0);
    else e = cudaErrorUnknown;
    if (g) cudaGraphDestroy(g);
    if (e == cudaSuccess && ex) {
      cudaGraphUpload(ex, stream_);
      graphs_[B] = ex;
      graph_nodes_[B] = n;
      return true;
    }
    cudaGetLastError();
    if (use_pdl_) {
      fprintf(stderr, "[clengine] graph capture with PDL failed (%s); retrying without PDL\n", cudaGetErrorString(e));
      use_pdl_ = false;
    } else {
      fprintf(stderr, "[clengine] graph capture failed (%s); falling back to eager launches\n", cudaGetErrorString(e));
      graph_failed_ = true;
      break;
    }
  }
  return false;
}

// A serving engine meets every batch size 1..max_batch as requests join and leave; capturing a 32-layer step graph
// costs tens of milliseconds, which would otherwise land inside 31 separate decode steps of the first minute of traffic
// (box benchmark, 64 concurrent chats: 16.6 req/s with lazy capture against 24.6 warm).  Called once when the
// scheduler thread starts.
void Engine::precapture_graphs(int max_b) {
  if (!use_graph_ || deterministic_) return;
  for (int B = 1; B <= max_b && !graph_failed_; ++B) ensure_graph(B);
  cudaStreamSynchronize(stream_);
}

int Engine::run_step_graph(int B, int step_off) {
  if (use_graph_ && !graph_failed_ && !deterministic_) {
    ensure_graph(B);
    auto it = graphs_.find(B);
    if (it != graphs_.end()) {
      CL_CUDA_OK(cudaGraphLaunch(it->second, stream_));
      launches_ += graph_nodes_[B];
      return CL_OK;
    }
  }
  const int n = enqueue_step(B, step_off);
  if (n < 0) return n;
  launches_ += n;
  return CL_OK;
}

int Engine::read_logits(int slot, float* out) {
  CL_CUDA_OK(cudaMemcpyAsync(h_logits_pinned_, d_logits_ + (size_t)slot * cfg.vocab_size, (size_t)cfg.vocab_size * 4,
                             cudaMemcpyDeviceToHost, stream_));
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  memcpy(out, h_logits_pinned_, (size_t)cfg.vocab_size * 4);
  return CL_OK;
}

int Engine::set_single_slot(cl_seq_t s) {
  h_slots_.assign(1, s);
  if (last_single_slot_ != s) {
    CL_CUDA_OK(cudaMemcpyAsync(d_slots_, &s, 4, cudaMemcpyHostToDevice, stream_));
    last_single_slot_ = s;
    slots_dirty_ = true;   // the scheduler's cached slot list no longer describes d_slots_
  }
  return CL_OK;
}

int Engine::decode_step(cl_seq_t s, int32_t id, float* logits_out, int32_t* argmax_out) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (id < 0 || id >= cfg.vocab_size) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
  auto& q = seqs_[s];
  int rc = ensure_capacity(s, q.len + 1);
  if (rc) return rc;
  const int hdr[2] = {id, q.len};
  CL_CUDA_OK(cudaMemcpyAsync(d_tok_ + s, &hdr[0], 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &hdr[1], 4, cudaMemcpyHostToDevice, stream_));
  rc = set_single_slot(s);
  if (rc) return rc;
  rc = run_step_graph(1);
  if (rc) return rc;
  seq_advance(s, &id, 1, 1);
  if ((rc = collect_logprobs(&s, 1))) return rc;
  if (logits_out) { rc = read_logits(s, logits_out); if (rc) return rc; }
  if (argmax_out) {
    CL_CUDA_OK(cudaMemcpyAsync(h_ids_pinned_, d_tok_ + s, 4, cudaMemcpyDeviceToHost, stream_));
    CL_CUDA_OK(cudaStreamSynchronize(stream_));
    *argmax_out = h_ids_pinned_[0];
  } else {
    CL_CUDA_OK(cudaStreamSynchronize(stream_));
  }
  return CL_OK;
}

int Engine::prefill_tokenwise(cl_seq_t s, const int32_t* ids, int n, float* logits_out) {
  auto& q = seqs_[s];
  pass_ = PassRecord{};   // decode steps, not a multi-row pass: debug_pass_rows must not offer an older pass's rows
  int rc = ensure_capacity(s, q.len + n);
  if (rc) return rc;
  CL_CUDA_OK(cudaMemcpyAsync(d_prompt_, ids, (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &q.len, 4, cudaMemcpyHostToDevice, stream_));
  rc = set_single_slot(s);
  if (rc) return rc;
  // An armed slot draws once, at the last prompt token.  The step graph's tail pushes its input, so the history length is
  // taken back by one first: the push then rewrites the ring entry that already holds that token.
  const int armed_hlen = samp_hlen_[s];
  const int off = 0, on = 1, hlen_before_last = std::max(0, armed_hlen - 1);
  if (armed_hlen >= 0 && n > 1) CL_CUDA_OK(cudaMemcpyAsync(d_samp_mode_ + s, &off, 4, cudaMemcpyHostToDevice, stream_));
  // likewise only the last token's tail records logprobs
  const int lp_off = -1, lp_on = lp_n_[s];
  if (lp_on >= 0 && n > 1) CL_CUDA_OK(cudaMemcpyAsync(d_lp_n_ + s, &lp_off, 4, cudaMemcpyHostToDevice, stream_));
  for (int i = 0; i < n; ++i) {
    CL_CUDA_OK(cudaMemcpyAsync(d_tok_ + s, d_prompt_ + i, 4, cudaMemcpyDeviceToDevice, stream_));
    if (armed_hlen >= 0 && i == n - 1) {
      CL_CUDA_OK(cudaMemcpyAsync(d_samp_mode_ + s, &on, 4, cudaMemcpyHostToDevice, stream_));
      CL_CUDA_OK(cudaMemcpyAsync(d_samp_hlen_ + s, &hlen_before_last, 4, cudaMemcpyHostToDevice, stream_));
    }
    if (lp_on >= 0 && n > 1 && i == n - 1) CL_CUDA_OK(cudaMemcpyAsync(d_lp_n_ + s, &lp_on, 4, cudaMemcpyHostToDevice, stream_));
    rc = run_step_graph(1);
    if (rc) return rc;
  }
  seq_advance(s, ids, n, n);
  if (logits_out) return read_logits(s, logits_out);
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  return CL_OK;
}

int Engine::prefill(cl_seq_t s, const int32_t* ids, int n, float* logits_out) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (n <= 0) { set_last_error("empty prompt"); return CL_ERR_INVALID_ARG; }
  for (int i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= cfg.vocab_size) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
  if (seqs_[s].len + n > cfg.max_seq_len) { set_last_error("sequence exceeds max_seq_len"); return CL_ERR_TOO_LONG; }
  int rc;
  if (deterministic_) {
    rc = det_prefill(1, &s, &ids, &n, logits_out);
  } else if (n >= prefill_min_tokens_ && prefill_path_ok()) {
    // short prompts: split-K projections so that every SM streams weights (d_model <= 8192: one 1024-thread CTA per row in the glue)
    if (n <= prefill_small_max_ && cfg.d_model <= 8192 && cfg.d_model % 4 == 0) rc = prefill_small(s, ids, n, logits_out);
    else rc = prefill_chunked(s, ids, n, logits_out);
  } else {
    rc = prefill_tokenwise(s, ids, n, logits_out);
  }
  return rc ? rc : collect_logprobs(&s, 1);
}

int Engine::decode_greedy(const cl_seq_t* ss, int B, const int32_t* first_ids, int n_steps, int32_t* ids_out, float* device_ms) {
  if (B <= 0 || B > max_batch_ || n_steps <= 0) { set_last_error("bad batch / steps"); return CL_ERR_INVALID_ARG; }
  for (int b = 0; b < B; ++b) {
    const int s = ss[b];
    if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
    for (int c = 0; c < b; ++c) if (ss[c] == s) { set_last_error("duplicate sequence in batch"); return CL_ERR_INVALID_ARG; }
    if (first_ids[b] < 0 || first_ids[b] >= cfg.vocab_size) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
    const int rc = ensure_capacity(s, seqs_[s].len + n_steps);
    if (rc) return rc;
  }
  for (int b = 0; b < B; ++b) {
    const int s = ss[b];
    CL_CUDA_OK(cudaMemcpyAsync(d_tok_ + s, &first_ids[b], 4, cudaMemcpyHostToDevice, stream_));
    CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &seqs_[s].len, 4, cudaMemcpyHostToDevice, stream_));
  }
  CL_CUDA_OK(cudaMemcpyAsync(d_slots_, ss, (size_t)B * 4, cudaMemcpyHostToDevice, stream_));
  h_slots_.assign(ss, ss + B);
  last_single_slot_ = B == 1 ? ss[0] : -1;
  if (B > 1) last_batch_slots_.assign(ss, ss + B);
  slots_dirty_ = true;
  float total_ms = 0.f;
  for (int done = 0; done < n_steps;) {
    const int chunk = std::min(ring_steps_, n_steps - done);
    CL_CUDA_OK(cudaMemsetAsync(d_step_counter_, 0, 4, stream_));
    CL_CUDA_OK(cudaEventRecord(ev0_, stream_));
    for (int i = 0; i < chunk; ++i) {
      const int rc = run_step_graph(B, done + i);
      if (rc) return rc;
    }
    CL_CUDA_OK(cudaEventRecord(ev1_, stream_));
    CL_CUDA_OK(cudaMemcpyAsync(h_ids_pinned_, d_ids_ring_, (size_t)chunk * max_batch_ * 4, cudaMemcpyDeviceToHost, stream_));
    CL_CUDA_OK(cudaStreamSynchronize(stream_));
    float ms = 0.f;
    CL_CUDA_OK(cudaEventElapsedTime(&ms, ev0_, ev1_));
    total_ms += ms;
    for (int i = 0; i < chunk; ++i)
      for (int b = 0; b < B; ++b) ids_out[(size_t)(done + i) * B + b] = h_ids_pinned_[(size_t)i * max_batch_ + b];
    if (std::any_of(ss, ss + B, [&](cl_seq_t s) { return lp_n_[s] >= 0; })) {   // the record ring, only when a slot records
      CL_CUDA_OK(cudaMemcpy(h_lp_pinned_, d_lp_ring_, (size_t)chunk * max_batch_ * sizeof(LogprobRecord), cudaMemcpyDeviceToHost));
      for (int i = 0; i < chunk; ++i)
        for (int b = 0; b < B; ++b)
          if (lp_n_[ss[b]] >= 0) seqs_[ss[b]].lps.push_back(h_lp_pinned_[(size_t)i * max_batch_ + b]);
    }
    done += chunk;
  }
  std::vector<int32_t> fed((size_t)n_steps);
  for (int b = 0; b < B; ++b) {   // step i was fed first_ids[b], then the id of step i - 1: all read back, all known
    fed[0] = first_ids[b];
    for (int i = 0; i + 1 < n_steps; ++i) fed[(size_t)i + 1] = ids_out[(size_t)i * B + b];
    seq_advance(ss[b], fed.data(), n_steps, n_steps);
  }
  tokens_generated_ += (int64_t)n_steps * B;
  if (total_ms > 0.f) {
    const double tps = (double)n_steps * max_batch_ / (total_ms * 1e-3);   // capacity: steps/s x max_batch
    tok_per_sec_ewma_ = tok_per_sec_ewma_ == 0.0 ? tps : 0.8 * tok_per_sec_ewma_ + 0.2 * tps;
  }
  if (device_ms) *device_ms = total_ms;
  return CL_OK;
}

int Engine::decode_sample(const cl_seq_t* ss, int B, const int32_t* first_ids, const cl_sampling* sp, const uint64_t* step0,
                          int n_steps, int32_t* ids_out, float* device_ms) {
  if (B <= 0 || B > max_batch_) { set_last_error("bad batch / steps"); return CL_ERR_INVALID_ARG; }
  for (int b = 0; b < B; ++b) {
    if (ss[b] < 0 || ss[b] >= max_seqs_ || !seqs_[ss[b]].live) return CL_ERR_BAD_SEQ;
    if (sp[b].temperature > 0.f && !device_sampling_ok(sp[b], cfg.vocab_size, seqs_[ss[b]].ext)) {
      set_last_error("sampling settings of sequence " + std::to_string(b) + " need the host sampler");
      return CL_ERR_INVALID_ARG;
    }
  }
  int rc = CL_OK;
  for (int b = 0; b < B && rc == CL_OK; ++b)
    if (sp[b].temperature > 0.f) {
      const auto& h = seqs_[ss[b]].history;
      rc = arm_sampling(ss[b], sp[b], step0 ? step0[b] : 0, h.data(), (int)h.size());
    }
  if (rc == CL_OK) rc = decode_greedy(ss, B, first_ids, n_steps, ids_out, device_ms);
  for (int b = 0; b < B; ++b) {
    const int r2 = disarm_sampling(ss[b]);
    if (rc == CL_OK) rc = r2;
  }
  return rc;
}

// ---- parity / benchmark aids ------------------------------------------------------------------------
int Engine::seq_fake_fill(cl_seq_t s, int n_tokens) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (n_tokens < 0) { set_last_error("fake_fill: negative length"); return CL_ERR_INVALID_ARG; }
  int rc = ensure_capacity(s, std::max(n_tokens, 1));
  if (rc) return rc;
  const int n = launch_fake_fill_kv(kpool_, vpool_, kv_layer_elems_, cfg.n_layers, d_bt_ + (size_t)s * max_pages_per_seq_, page_size_,
                                    cfg.n_kv_heads, cfg.head_dim, n_tokens, stream_);
  if (n < 0) { set_last_error(std::string("fake_fill: ") + cudaGetErrorString(cudaGetLastError())); return CL_ERR_CUDA; }
  launches_ += n;
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  seqs_[s].len = n_tokens;
  seqs_[s].history.assign((size_t)n_tokens, 0);   // placeholders under a synthetic cache: never published
  seqs_[s].known = 0;
  return CL_OK;
}

int Engine::debug_kv(cl_seq_t s, int layer, int which, int t0, int n, float* out) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  // which 2 / 3: K / V up to the end of the pages the sequence holds (a verify pass's rejected rows lie past its length)
  const long long end = which >= 2 ? (long long)pool_->pages_of(s).size() * page_size_ : seqs_[s].len;
  if (which < 0 || which > 3 || layer < 0 || layer >= cfg.n_layers || t0 < 0 || n <= 0 || t0 + n > end || !out) {
    set_last_error("debug_kv: bad selector or range");
    return CL_ERR_INVALID_ARG;
  }
  float* tmp = nullptr;
  const size_t bytes = (size_t)n * kv_dim_ * 4;
  CL_CUDA_OK(cudaMalloc(&tmp, bytes));
  const __nv_bfloat16* pool = (which & 1 ? vpool_ : kpool_) + (size_t)layer * kv_layer_elems_;
  int rc = CL_OK;
  if (launch_gather_kv(pool, d_bt_ + (size_t)s * max_pages_per_seq_, page_size_, cfg.n_kv_heads, cfg.head_dim, t0, n, tmp, stream_) < 0 ||
      cudaMemcpyAsync(out, tmp, bytes, cudaMemcpyDeviceToHost, stream_) != cudaSuccess || cudaStreamSynchronize(stream_) != cudaSuccess) {
    set_last_error(std::string("debug_kv: ") + cudaGetErrorString(cudaGetLastError()));
    rc = CL_ERR_CUDA;
  }
  cudaFree(tmp);
  return rc;
}

// one batched step with caller-chosen input tokens (teacher forcing); logits_out [n_seqs][vocab] (may be NULL)
int Engine::decode_step_batch(const cl_seq_t* ss, int B, const int32_t* ids, float* logits_out, int32_t* argmax_out) {
  if (B <= 0 || B > max_batch_) { set_last_error("bad batch"); return CL_ERR_INVALID_ARG; }
  for (int b = 0; b < B; ++b) {
    const int s = ss[b];
    if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
    for (int c = 0; c < b; ++c) if (ss[c] == s) { set_last_error("duplicate sequence in batch"); return CL_ERR_INVALID_ARG; }
    if (ids[b] < 0 || ids[b] >= cfg.vocab_size) { set_last_error("token id out of range"); return CL_ERR_INVALID_ARG; }
    const int rc = ensure_capacity(s, seqs_[s].len + 1);
    if (rc) return rc;
  }
  for (int b = 0; b < B; ++b) {
    const int s = ss[b];
    CL_CUDA_OK(cudaMemcpyAsync(d_tok_ + s, &ids[b], 4, cudaMemcpyHostToDevice, stream_));
    CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &seqs_[s].len, 4, cudaMemcpyHostToDevice, stream_));
  }
  CL_CUDA_OK(cudaMemcpyAsync(d_slots_, ss, (size_t)B * 4, cudaMemcpyHostToDevice, stream_));
  h_slots_.assign(ss, ss + B);
  last_single_slot_ = B == 1 ? ss[0] : -1;
  if (B > 1) last_batch_slots_.assign(ss, ss + B);
  slots_dirty_ = true;
  int rc = run_step_graph(B);
  if (rc) return rc;
  if ((rc = collect_logprobs(ss, B))) return rc;
  for (int b = 0; b < B; ++b) {
    seq_advance(ss[b], &ids[b], 1, 1);
    if (logits_out) { const int r2 = read_logits(ss[b], logits_out + (size_t)b * cfg.vocab_size); if (r2) return r2; }
  }
  if (argmax_out) {
    CL_CUDA_OK(cudaMemcpyAsync(h_ids_pinned_, d_tok_, (size_t)max_seqs_ * 4, cudaMemcpyDeviceToHost, stream_));
    CL_CUDA_OK(cudaStreamSynchronize(stream_));
    for (int b = 0; b < B; ++b) argmax_out[b] = h_ids_pinned_[ss[b]];
  } else {
    CL_CUDA_OK(cudaStreamSynchronize(stream_));
  }
  return CL_OK;
}

// bench.py's roofline.dominant_kernel: n_steps single-sequence greedy steps launched eagerly (the same kernels the
// CUDA graph holds), with a CUDA-event pair on the launching stream around the step's dominant kernel — the persistent
// whole-stack kernel (or, on the per-op path, the stack of per-layer kernels between the embedding and the LM head).
int Engine::time_dominant_kernel(cl_seq_t s, int32_t first_id, int n_steps, float* kernel_ms, float* step_ms) {
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  if (deterministic_) { set_last_error("time_dominant_kernel: deterministic mode has no step of the timed kernels"); return CL_ERR_INVALID_ARG; }
  if (n_steps <= 0 || n_steps > 4096 || first_id < 0 || first_id >= cfg.vocab_size) { set_last_error("bad steps / token"); return CL_ERR_INVALID_ARG; }
  int rc = ensure_capacity(s, seqs_[s].len + n_steps);
  if (rc) return rc;
  CL_CUDA_OK(cudaMemcpyAsync(d_tok_ + s, &first_id, 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_pos_ + s, &seqs_[s].len, 4, cudaMemcpyHostToDevice, stream_));
  CL_CUDA_OK(cudaMemcpyAsync(d_slots_, &s, 4, cudaMemcpyHostToDevice, stream_));
  last_single_slot_ = s;
  slots_dirty_ = true;
  CL_CUDA_OK(cudaMemsetAsync(d_step_counter_, 0, 4, stream_));
  std::vector<cudaEvent_t> ev((size_t)2 * n_steps + 2);
  for (auto& e : ev) CL_CUDA_OK(cudaEventCreate(&e));
  probe_ev_ = ev.data();
  CL_CUDA_OK(cudaEventRecord(ev[2 * n_steps], stream_));
  for (int i = 0; i < n_steps && rc == CL_OK; ++i) {
    probe_idx_ = 2 * i;
    const int n = enqueue_step(1);
    if (n < 0) rc = n; else launches_ += n;
  }
  probe_ev_ = nullptr;
  if (rc == CL_OK && cudaEventRecord(ev[2 * n_steps + 1], stream_) != cudaSuccess) rc = CL_ERR_CUDA;
  if (rc == CL_OK && cudaStreamSynchronize(stream_) != cudaSuccess) { set_last_error(cudaGetErrorString(cudaGetLastError())); rc = CL_ERR_CUDA; }
  double k = 0.0;
  float ms = 0.f;
  if (rc == CL_OK) {
    for (int i = 0; i < n_steps; ++i) { cudaEventElapsedTime(&ms, ev[2 * i], ev[2 * i + 1]); k += ms; }
    cudaEventElapsedTime(&ms, ev[2 * n_steps], ev[2 * n_steps + 1]);
    if (kernel_ms) *kernel_ms = (float)(k / n_steps);
    if (step_ms) *step_ms = ms / n_steps;
    // the device advanced tok/pos itself; mirror it on the host
    CL_CUDA_OK(cudaMemcpy(h_ids_pinned_, d_ids_ring_, (size_t)std::min(n_steps, ring_steps_) * max_batch_ * 4, cudaMemcpyDeviceToHost));
    // The id ring holds the last ring_steps_ ids: with more steps, step i's id was overwritten by step i + ring_steps_'s
    // and the ids after the ring are zeros.  Only first_id is known then, and nothing after it is ever published.
    std::vector<int32_t> fed((size_t)n_steps, 0);
    fed[0] = first_id;
    for (int i = 0; i + 1 < n_steps && i < ring_steps_; ++i) fed[(size_t)i + 1] = h_ids_pinned_[(size_t)i * max_batch_];
    seq_advance(s, fed.data(), n_steps, n_steps <= ring_steps_ ? n_steps : 1);
    tokens_generated_ += n_steps;
  }
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

int Engine::debug_timeline(long long* out, int n) {
  const int want = (cfg.n_layers * 5 + 1) * 4;
  if (!d_timeline_ || n < want) return CL_ERR_INVALID_ARG;
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  CL_CUDA_OK(cudaMemcpy(out, d_timeline_, (size_t)want * 8, cudaMemcpyDeviceToHost));
  return want;
}

int Engine::debug_hidden(float* out, int n) {
  if (last_single_slot_ < 0) return CL_ERR_INVALID_ARG;
  // negative n selects a last-layer intermediate of the most recent single-sequence step (diagnostics):
  // -1 = q (roped), -2 = attention output, -3 = SwiGLU activation
  if (n < 0 && n >= -3) return debug_seq_hidden(last_single_slot_, -n, out, n == -3 ? cfg.d_ff : q_dim_, nullptr);
  return debug_seq_hidden(last_single_slot_, 0, out, n, nullptr);
}

int Engine::debug_seq_hidden(cl_seq_t s, int what, float* out, int n, int32_t* mega_out) {
  if (mega_out) *mega_out = use_mega_ && d_mega_layers_ != nullptr ? 1 : 0;
  if (!out && n == 0) return CL_OK;   // only the flag was asked for
  if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ;
  const int want = what == 0 ? cfg.d_model : what == 3 || what == 5 ? cfg.d_ff : q_dim_;
  if (what < 0 || what > 5 || n != want || !out) { set_last_error("debug_seq_hidden: bad buffer selector or element count"); return CL_ERR_INVALID_ARG; }
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  if (what <= 3) {   // per-slot fp32 state: written by every step that contains the sequence
    const float* src = what == 0 ? d_h_ + (size_t)s * cfg.d_model : what == 1 ? d_q_ + (size_t)s * q_dim_
                     : what == 2 ? d_attn_ + (size_t)s * q_dim_ : d_act_ + (size_t)s * cfg.d_ff;
    CL_CUDA_OK(cudaMemcpy(out, src, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return CL_OK;
  }
  // bf16 operands of the batched step's GEMMs: rows in batch order
  int b = -1;
  for (size_t i = 0; i < last_batch_slots_.size(); ++i) if (last_batch_slots_[i] == s) b = (int)i;
  if (b < 0 || !bws_) { set_last_error("debug_seq_hidden: the sequence was not part of the latest batched step"); return CL_ERR_INVALID_ARG; }
  std::vector<uint16_t> tmp((size_t)n);
  CL_CUDA_OK(cudaMemcpy(tmp.data(), (what == 4 ? bws_->attn : bws_->act) + (size_t)b * n, (size_t)n * 2, cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; ++i) { const uint32_t u = (uint32_t)tmp[(size_t)i] << 16; memcpy(&out[i], &u, 4); }
  return CL_OK;
}

int Engine::debug_pass_info(int32_t* info, int32_t* segs, int max_segs) {
  if (pass_.T == 0) { set_last_error("debug_pass_info: no multi-row pass since the last token-wise prefill or failed pass"); return CL_ERR_INVALID_ARG; }
  if (!info || max_segs < 0 || (max_segs > 0 && !segs)) { set_last_error("debug_pass_info: bad arguments"); return CL_ERR_INVALID_ARG; }
  info[0] = pass_.path; info[1] = pass_.attn; info[2] = pass_.T; info[3] = (int32_t)pass_.segs.size();
  for (int i = 0; i < max_segs && i < (int)pass_.segs.size(); ++i) {
    const PrefillSegment& g = pass_.segs[(size_t)i];
    segs[4 * i] = g.seq; segs[4 * i + 1] = g.row0; segs[4 * i + 2] = g.n; segs[4 * i + 3] = g.pos0;
  }
  return CL_OK;
}

int Engine::debug_pass_rows(int what, int row0, int n, float* out) {
  if (pass_.T == 0) { set_last_error("debug_pass_rows: no multi-row pass since the last token-wise prefill or failed pass"); return CL_ERR_INVALID_ARG; }
  if (what < 0 || what > 3 || row0 < 0 || n <= 0 || row0 + n > pass_.T || !out) { set_last_error("debug_pass_rows: bad selector or range"); return CL_ERR_INVALID_ARG; }
  const bool small = pass_.path == kPassSplitK;
  CL_CUDA_OK(cudaStreamSynchronize(stream_));
  if (what == 0) {
    const size_t w = cfg.d_model;
    CL_CUDA_OK(cudaMemcpy(out, (small ? sws_->h : pws_->h) + (size_t)row0 * w, (size_t)n * w * 4, cudaMemcpyDeviceToHost));
    return CL_OK;
  }
  const size_t w = what == 3 ? cfg.d_ff : q_dim_, cnt = (size_t)n * w;
  const __nv_bfloat16* src = what == 1 ? (small ? sws_->q : pws_->q) : what == 2 ? (small ? sws_->attn : pws_->attn) : (small ? sws_->act : pws_->act);
  std::vector<uint16_t> tmp(cnt);
  CL_CUDA_OK(cudaMemcpy(tmp.data(), src + (size_t)row0 * w, cnt * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < cnt; ++i) { const uint32_t u = (uint32_t)tmp[i] << 16; memcpy(&out[i], &u, 4); }
  return CL_OK;
}

int Engine::spec_stats(cl_spec_stats* out) {
  memset(out, 0, sizeof *out);
  out->enabled = speculate_ > 0 ? 1 : 0;
  out->max_draft = speculate_;
  out->verify_passes = spec_passes_;
  out->tokens_drafted = spec_drafted_;
  out->tokens_accepted = spec_accepted_;
  out->tokens_emitted = spec_emitted_;
  out->multi_passes = spec_multi_passes_;
  out->draft_rows = draft_rows_;
  out->draft_ns = draft_ns_;
  out->draft_pages_used = draft_pages_;
  return CL_OK;
}

int Engine::set_speculate_batch(int n) {
  if (n < 1 || n > std::min(max_batch_, kSpecBatchMax)) {
    set_last_error("speculate_batch must be 1..min(max_batch, 32)");
    return CL_ERR_INVALID_ARG;
  }
  speculate_batch_ = n;
  return CL_OK;
}

int Engine::stats(cl_stats* out) {
  memset(out, 0, sizeof *out);
  out->tokens_per_sec = capacity_tok_per_sec_;
  out->measured_tokens_per_sec = tok_per_sec_ewma_;
  int active = 0;
  for (auto& s : seqs_) active += s.live ? 1 : 0;
  out->active_seqs = active;
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    out->queue_depth = (int)queue_.size();
  }
  out->load = (double)(active + out->queue_depth) / (double)max_batch_;   // queued requests count as load: > 1 = requests are waiting
  out->kv_pages_total = n_pages_;
  out->kv_pages_used = pool_ ? pool_->used_pages() : 0;
  out->tokens_generated = tokens_generated_;
  out->requests_completed = requests_completed_;
  out->preemptions = preemptions_;
  out->sched_decode_steps = sched_decode_steps_;
  out->sched_decode_ns = sched_decode_ns_;
  out->sched_prefill_calls = sched_prefill_calls_;
  out->sched_prefill_tokens = sched_prefill_tokens_;
  out->sched_prefill_ns = sched_prefill_ns_;
  out->vram_gb = vram_gb_;
  memcpy(out->gpu_model, gpu_name_, sizeof out->gpu_model);
  out->kernel_launches = launches_;
  return CL_OK;
}

}  // namespace cl
