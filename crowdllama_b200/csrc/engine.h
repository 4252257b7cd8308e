// engine.h — internal C++ interface of libclengine.so (the C-ABI lives in include/clengine.h).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <deque>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/clengine.h"
#include "kernels.h"

namespace cl {

// Defaults of the features added in round 2.  Each has an environment switch; the default is turned on only after a GPU run
// of the parity tests and the benchmark with it.
constexpr int kDefaultSchedPrefillChunk = 1024; // CL_SCHED_PREFILL_CHUNK: admission token budget per scheduler iteration (0 = whole prompts); validated r2e
constexpr int kDefaultPrefillSmallMax = 256;    // CL_PREFILL_SMALL_MAX: prompts up to this many tokens take the split-K path (0 = off)
constexpr int kDefaultSchedMultiPrefill = 1;    // CL_SCHED_MULTI_PREFILL: scheduler admits the prompts at the head of the queue in one tile-path pass (Engine::prefill_multi)
constexpr int kSchedLingerUs = 1000;  // burst detection before a group admission into an empty batch (Engine::wait_for_work)

constexpr int kMaxContext = 131072;   // longest window cl_engine_config.context_length may ask for (Llama-3.1 / 3.2's 128K)
// Prefill segments that end past this many tokens (the longest window served before context_length) run the split-KV
// prefill attention; shorter ones keep their kernels and bits (Engine::attn_prefill)
constexpr int kLongPrefillFrom = 32768;
// the attention kernel of a multi-row pass (cl_debug_pass_info; Engine::prefill_attn_kind)
enum { kPassAttnMma = 0, kPassAttnWgmma = 1, kPassAttnVerify = 2, kPassAttnMixed = 3, kPassAttnLong = 4 };
// Device memory a context_length > 0 engine leaves outside its KV pool when it sizes the pool itself: the per-slot state,
// the tile-path prefill workspace at its chunk size, the verify pass's logits (128 rows x vocab fp32) and split partials,
// and the CUDA context's own growth; 4 GiB covers them for the 8B shapes at max_batch 8 with room to spare
constexpr int64_t kPoolReserveBytes = 4LL << 30;
// Speculative decoding (cl_engine_config.speculate, Engine::verify_batch, ngram_draft): the constants of the drafter.
constexpr int kSpecMaxDraft = 15;     // drafted tokens per verify pass at most (its rows: x0 + drafts <= 16)
constexpr int kDraftNgramMax = 3;     // the drafter matches the history's last 3 ids, then its last 2
constexpr int kDraftNgramMin = 2;
constexpr int kSpecBackoff = 8;       // tokens a request decodes without drafting after a verify pass that accepted nothing
constexpr int kSpecMaxRows = 128;     // rows of one verify pass over several sequences (Engine::verify_batch) at most
constexpr int kSpecBatchMax = 32;     // sequences the scheduler verifies in one pass at most (cl_engine_set_speculate_batch)
// Deterministic mode (cl_engine_config.deterministic): split-K counts are pick_splits' at this many SMs (an H100 SXM's)
// whatever the device has, so a card with fewer SMs computes the same bits
constexpr int kDetSms = 132;

// split-K count of an n_rows x K projection on sms SMs (engine.cu: the batched step's and the split-K pass's rule)
int pick_splits_sms(int n_rows, int K, int sms);

// Prompt-lookup drafter: the longest suffix of hist[0..n) of length kDraftNgramMax .. kDraftNgramMin that also occurs
// earlier in hist; from its most recent earlier occurrence, the up to k ids that followed it (stopping at the end of
// hist) go to out.  Returns how many (0: no match).
int ngram_draft(const int32_t* hist, int n, int k, int32_t* out);

// the C-ABI view of a step tail record (lse stays internal)
inline cl_token_logprob to_token_logprob(const LogprobRecord& r) {
  cl_token_logprob o{};
  o.id = r.id; o.logprob = r.logprob; o.n_top = r.n_top;
  for (int j = 0; j < r.n_top && j < kLogprobTopMax; ++j) { o.top_ids[j] = r.top_ids[j]; o.top_logprobs[j] = r.top_logprobs[j]; }
  return o;
}
static_assert(sizeof(cl_token_logprob) == 172, "cl_token_logprob is 172 bytes");
static_assert(kLogprobTopMax == CL_MAX_TOP_LOGPROBS, "one top-n limit");

void set_last_error(const std::string& s);
const char* get_last_error();

// KV pool of the single-op entry points that take paged attention (cl_op_attn_decode_batch, cl_op_attn_prefill*): the token
// rows of several sequences paged the way a long-running engine leaves them (ops_api.cu, op_build_kv_pool).
struct OpKvPool {
  std::vector<uint16_t> k, v;   // bf16 [2 layers][n_pages][n_kv][page][head_dim]; the tokens sit in layer 1
  std::vector<int> bt;          // [sequence][bt_stride]
  int n_pages = 0, bt_stride = 0;
  int pad_page = 0;             // token-less page named by the block-table entries past a sequence's last page
  size_t layer_elems = 0;       // n_pages * n_kv * page * head_dim
};
void op_build_kv_pool(const uint16_t* k, const uint16_t* v, const int* lens, int n_seqs, int n_kv, int head_dim, int page_size,
                      OpKvPool* pool);

#define CL_CUDA_OK(expr)                                                                          \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::cl::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                   \
      return CL_ERR_CUDA;                                                                         \
    }                                                                                             \
  } while (0)

// CL_PREFILL_PROFILE / CL_STEP_PROFILE = 1 (eager launches only): a CUDA event after every launch; report() prints the
// device time per kernel class, gap before each kernel included, to stderr.  Off while the stream is being captured.
class LaunchProfiler {
 public:
  LaunchProfiler(cudaStream_t st, const char* env);   // env == nullptr: never on
  void mark(const char* call);                        // call: the launcher expression, its name up to '(' is the class
  void report(const char* tag, int key_width, const std::string& head);   // "[tag] head, N launches, T ms on the device"

 private:
  bool on_ = false;
  cudaStream_t st_ = nullptr;
  std::vector<cudaEvent_t> ev_;
  std::vector<const char*> name_;
};

// Enqueue one launcher call (kernels.h) inside an Engine member that keeps `int launches` and `LaunchProfiler prof`.
#define CL_LAUNCH(call)                                                                                     \
  do {                                                                                                      \
    const int r_ = (call);                                                                                  \
    if (r_ < 0) {                                                                                           \
      ::cl::set_last_error(std::string(#call) + ": " + cudaGetErrorString(cudaGetLastError()));             \
      return CL_ERR_CUDA;                                                                                   \
    }                                                                                                       \
    launches += r_;                                                                                         \
    prof.mark(#call);                                                                                       \
  } while (0)

// ---- paged-KV allocator: host-side free list + per-owner page lists (no GPU needed) -----------
// Prefix sharing: a full page whose P tokens are known can be published into an index keyed by (entry uid of the previous
// page of the chain, the page's P token ids), compared exactly.  Chains start at kRootUid.  A page is then free, referenced
// by one or more owners (refcount), or cached: refcount 0 but still indexed, on an LRU list that reserve() evicts from
// once the free list is empty.  Attached pages are read-only for their owners: every kernel writes K/V only at positions
// >= the sequence's length, and attach() leaves at least one token of the prompt to compute.  Without attach / publish
// the allocator hands out exactly the pages it always did.
//
// Host tier (set_host_pages(H), H > 0): an index entry lives on a device page or on one of H host pages, each holding one
// device page's K and V of every layer.  Evicting a cached device page then moves its entry to a free host page (a spill)
// instead of erasing it; with no host page free, the host LRU front is dropped first (deepest page of a chain first, as
// release orders them).  attach() walks the chain as before and gives every host entry on it a device page, from the free
// list or by evicting the device LRU (which may spill in turn), and frees the host page (a fill).  Before making room it
// references the chain's device entries and takes its host entries off the host LRU, so it never evicts or drops its own
// chain; it takes the longest prefix whose host entries can all get a device page now.  Every spill and fill is recorded
// as a Move, in decision order, and the caller must execute the moves in exactly that order before anything reads or
// writes the pages involved: a device page may be spilled and then filled in one call, and a host page freed by a fill
// may be reused by a later spill of the same call.  A spill run may also name one host page twice (the entry spilled
// first was dropped again to make room), so moves of one kind run concurrently only while no page repeats.
class KvPool {
 public:
  static constexpr uint64_t kRootUid = 0;
  enum MoveKind { kSpill = 0, kFill = 1 };
  struct Move { int kind, page, host; };   // kSpill: device page -> host page; kFill: host page -> device page
  KvPool(int n_pages, int page_size);
  int reserve(int owner, int n_tokens);  // CL_OK / CL_ERR_OOM (atomic: nothing taken on failure); evicts cached pages last
  int release(int owner);                // published pages whose refcount drops to 0 become cached, the rest free
  // Only on an owner without pages: takes the longest indexed chain matching ids[0..n), at most P * floor((n - 1) / P)
  // tokens (host-tier entries only as far as device pages can be found for them).  Returns the tokens reused (>= 0) or
  // CL_ERR_INVALID_ARG.
  int attach(int owner, const int32_t* ids, int n);
  // Tokens attach() would reuse, without taking anything; *cached_pages (may be nullptr): how many of the matching pages
  // are cached on the device or held by the host tier (attaching either takes a page out of free_pages()).
  int lookup(const int32_t* ids, int n, int* cached_pages) const;
  // Index the owner's full pages covering ids[0..n_known) not published yet.  A page whose key is already indexed stays private.
  int publish(int owner, const int32_t* ids, int n_known);
  // Context shift of an owner holding len tokens: tokens [n_keep, n_keep + n_discard) go, n_discard a positive multiple of
  // the page size and n_keep + n_discard <= len.  With k0 = n_keep / P and d = n_discard / P, entries k0 + 1 .. k0 + d are
  // released (k0 .. k0 + d - 1 when n_keep % P == 0) and the row is compacted; *items get the kernel's work (kv_shift.cu):
  // rows [n_keep % P, P) of old entry k0 + d into entry k0, and every later page holding tokens rotated in place.  A page
  // the shift writes (entry k0 and after) that another owner holds or the index keys is first replaced by a private page
  // (copy-on-write: its item reads the original and writes the copy, rows [0, n_keep % P) of entry k0 copied unrotated),
  // so the index and other owners never see the shifted rows; the original keeps its entry or goes to the cache.  The owner
  // publishes nothing more.  CL_ERR_INVALID_ARG / CL_ERR_OOM (copies need free pages) change nothing.
  int shift(int owner, int len, int n_keep, int n_discard, std::vector<KvShiftItem>* items);
  const std::vector<int>& pages_of(int owner);
  int free_pages() const { return (int)free_.size() + (int)lru_.size(); }   // allocatable: free + cached
  int used_pages() const { return n_pages_ - free_pages(); }                // referenced by some owner
  int cached_pages() const { return (int)lru_.size(); }
  int64_t evicted_pages() const { return evicted_; }
  int n_pages() const { return n_pages_; }
  int page_size() const { return page_size_; }
  // Host tier of n pages (0: off).  Drops every entry the tier held.  CL_ERR_INVALID_ARG for n < 0 or while moves are pending.
  int set_host_pages(int n);
  int host_pages() const { return host_n_; }
  int host_cached_pages() const { return host_n_ - (int)host_free_.size(); }
  int64_t pages_to_host() const { return to_host_; }
  int64_t pages_from_host() const { return from_host_; }
  const std::vector<Move>& moves() const { return moves_; }   // recorded since the last clear_moves(), in order
  void clear_moves() { moves_.clear(); }

 private:
  struct Key {
    uint64_t parent;
    std::vector<int32_t> ids;
    bool operator<(const Key& o) const { return parent != o.parent ? parent < o.parent : ids < o.ids; }
  };
  struct Entry { int loc; uint64_t uid; };   // loc >= 0: device page; loc < 0: host page ~loc
  using Index = std::map<Key, Entry>;
  struct Chain { int published = 0; uint64_t tail = kRootUid; bool shifted = false; };   // leading pages indexed (or matched), uid of the last
  void unref(int p);      // one owner fewer: at 0 an indexed page becomes cached, any other free
  int walk(const int32_t* ids, int n, std::vector<int>* locs) const;   // the chain's entry locations
  int take_page();        // a free page, else the device LRU front, evicted (spilled when a host page can be had)
  int take_host_page();   // a free host page, else the host LRU front, dropped; -1 when there is none
  int n_pages_, page_size_;
  std::vector<int> free_;  // stack; low page ids are handed out first
  std::map<int, std::vector<int>> owned_;
  std::vector<int> empty_;
  // prefix sharing
  Index index_;
  std::vector<Index::iterator> entry_;             // page -> its index entry (index_.end(): not published)
  std::vector<int> ref_;                           // page -> owners holding it
  std::list<int> lru_;                             // cached pages, evicted from the front
  std::vector<std::list<int>::iterator> lru_pos_;
  std::map<int, Chain> chain_;
  uint64_t next_uid_ = kRootUid + 1;
  int64_t evicted_ = 0;
  // host tier
  int host_n_ = 0;
  std::vector<int> host_free_;                     // stack; low host page ids first
  std::vector<Index::iterator> host_entry_;        // host page -> its index entry (index_.end(): free)
  std::list<int> host_lru_;                        // host pages holding an entry, dropped from the front
  std::vector<std::list<int>::iterator> host_lru_pos_;
  std::vector<Move> moves_;
  int64_t to_host_ = 0, from_host_ = 0;
};

// ---- tokenizers ---------------------------------------------------------------------------------
class Tokenizer {
 public:
  virtual ~Tokenizer() {}
  virtual std::vector<int32_t> encode(const std::string& text, bool add_bos) const = 0;
  virtual std::string decode_bytes(const std::vector<int32_t>& ids) const = 0;   // raw surface bytes (may cut a UTF-8 sequence)
  // What id adds to decode_bytes of a sequence when appended to it; at_start: nothing before it rendered any byte
  virtual std::string piece_bytes(int32_t id, bool at_start) const { (void)at_start; return decode_bytes({id}); }
  std::string decode(const std::vector<int32_t>& ids) const { return sanitize(decode_bytes(ids)); }
  static std::string sanitize(const std::string& raw);              // invalid UTF-8 / control bytes -> U+FFFD
  virtual int bos() const = 0;
  virtual int eos() const = 0;
  virtual bool is_stop(int id) const { return id == eos(); }        // Llama-3 also stops on <|eot_id|>
  // chat framing the Ollama server applies upstream of the model (role forced to "user", api.go:111-116)
  virtual std::string apply_chat_template(const std::string& user_prompt) const = 0;
  virtual int vocab_size() const = 0;
};

// byte-level fallback (no vocab files exist offline; SURVEY.md §8f row 2): ids 0..2 = <pad>, <bos>, <eos>;
// byte b -> 3 + b.  Needs vocab >= 259.  A neutral, documented chat framing is used.
class ByteTokenizer : public Tokenizer {
 public:
  explicit ByteTokenizer(int vocab_size) : vocab_(vocab_size) {}
  std::vector<int32_t> encode(const std::string& text, bool add_bos) const override;
  std::string decode_bytes(const std::vector<int32_t>& ids) const override;
  int bos() const override { return 1; }
  int eos() const override { return 2; }
  std::string apply_chat_template(const std::string& user_prompt) const override;
  int vocab_size() const override { return vocab_; }

 private:
  int vocab_;
};

// HF tokenizer.json (BPE: SentencePiece-style and byte-level) — tokenizer.cpp.  chat_family: "llama3" | "mistral" |
// "zephyr" | "chatml" | "" (auto-detect from the added tokens).  nullptr + *err on failure.
std::unique_ptr<Tokenizer> load_hf_tokenizer(const std::string& path, const std::string& chat_family, std::string* err);

// HF config.json of a model directory -> cl_model_config (weights_io.cpp)
int model_config_from_dir(const std::string& dir, cl_model_config* out, double* limits);
int resolve_model_config(const cl_engine_config& c, cl_model_config* out, int* context_length);   // cl_resolve_model_config

// ---- sampler (host; mirrors oracle oc_sample) ---------------------------------------------------
// inverse rotary frequency of dimension pair i: theta^(-2i/head_dim), with the "llama3" scaling of cl_model_config when
// rope_factor > 1 — the same expression as oracle/llama_oracle.c rope_inv_freq(), so both sides build bit-identical tables
double rope_inv_freq(const cl_model_config& c, int i);
// The sampler options of cl_sampling_ext (include/clengine.h) that the draw reads; all zero: cl_sampling alone
struct SamplerExt {
  float min_p = 0.f, presence_penalty = 0.f, frequency_penalty = 0.f;
};
constexpr int kMaxStops = 16;           // stop strings of one request at most
constexpr int kMaxStopBytes = 256;      // ... each at most this long
// Validates a caller's options: min_p in [0, 1], finite penalties, and when stop is not nullptr at most kMaxStops strings
// of at most kMaxStopBytes each (empty ones are dropped from *stop).  CL_OK, or CL_ERR_INVALID_ARG with the last error set.
int check_sampling_ext(const SamplerExt& x, std::vector<std::string>* stop);
// ext == nullptr: all zero; the stop strings go to *stop when it is not nullptr (checked as check_sampling_ext does)
int read_sampling_ext(const cl_sampling_ext* ext, SamplerExt* x, std::vector<std::string>* stop);
int32_t sample_token(const float* logits, int32_t vocab, const cl_sampling& sp, const int32_t* history, int32_t n_history,
                     uint64_t step, const SamplerExt& ext = SamplerExt());
// True when the step tail's device sampler draws exactly what sample_token draws for these settings: temperature > 0,
// 1 <= top_k <= kSampleTopKMax with top_k < vocab, vocab <= kTailBlocks * kSampleSliceMax, and the penalty stage (repeat,
// presence and frequency penalties) off or over a window of 1..kSampleHistMax ids.  Everything else (top_k 0,
// repeat_last_n -1, ...) stays on the host sampler.  min_p and the penalties' values need no more (check_sampling_ext).
inline bool device_sampling_ok(const cl_sampling& sp, int vocab, const SamplerExt& ext = SamplerExt()) {
  if (!(sp.temperature > 0.f)) return false;
  if (sp.top_k < 1 || sp.top_k > kSampleTopKMax || sp.top_k >= vocab || vocab > kTailBlocks * kSampleSliceMax) return false;
  const bool penalty = sp.repeat_last_n != 0 && (sp.repeat_penalty != 1.0f || ext.presence_penalty != 0.f || ext.frequency_penalty != 0.f);
  return !penalty || (sp.repeat_last_n > 0 && sp.repeat_last_n <= kSampleHistMax);
}
inline SampleParams sample_params(const cl_sampling& sp, const SamplerExt& ext) {
  SampleParams p;
  p.temperature = sp.temperature; p.top_p = sp.top_p; p.repeat_penalty = sp.repeat_penalty;
  p.min_p = ext.min_p; p.presence_penalty = ext.presence_penalty; p.frequency_penalty = ext.frequency_penalty;
  p.top_k = sp.top_k; p.repeat_last_n = sp.repeat_last_n; p.seed = sp.seed;
  return p;
}

// Stop sequences (Ollama's `stop`): the one place that decides where a response's text ends.  The generated text's bytes
// are fed in order; the first time one of the stop strings occurs in them, match() is the offset of the earliest such
// occurrence and the text is cut there.  safe() is how many leading bytes no later byte can cut: everything before the
// longest tail that could still begin a stop string (match() once matched).  Each feed costs O(stops x (longest stop +
// bytes fed)), whatever the text's length.
class StopScan {
 public:
  StopScan() = default;
  explicit StopScan(std::vector<std::string> stops);
  bool active() const { return !stops_.empty(); }
  void feed(const std::string& bytes);                                 // a no-op once matched
  void feed_id(const Tokenizer& tok, int32_t id);                      // the id's bytes as they appear in decode_bytes
  int64_t match() const { return match_; }                             // -1: no match yet
  int64_t safe() const { return match_ >= 0 ? match_ : n_ - hold_; }
  int64_t size() const { return n_; }

 private:
  std::vector<std::string> stops_;
  size_t keep_ = 0;        // longest stop string - 1: the bytes a later match can start in
  std::string tail_;       // the last keep_ bytes fed
  int64_t n_ = 0, match_ = -1, hold_ = 0;
};

// ---- minimal protobuf codec for llama.v1.BaseMessage (pbmsg.cpp) -------------------------------
// GenerateOptions: the proto extension SURVEY.md §8f row 3 asks for (seed / temperature / num_predict ... are
// inexpressible on the reference's wire, api.go:193-197).  Every field has explicit presence: temperature 0
// (greedy) must be distinguishable from "not set".
struct PbGenerateOptions {
  uint32_t has = 0;   // bit i set <=> field number i present
  uint64_t seed = 0; float temperature = 0.f; int32_t top_k = 0; float top_p = 0.f; float repeat_penalty = 0.f;
  int32_t repeat_last_n = 0; int32_t num_predict = 0; bool raw = false;
  bool logprobs = false; int32_t top_logprobs = 0;   // Ollama's top-level logprobs / top_logprobs (fields 9, 10)
  std::vector<std::string> stop;                      // fields 11 - 14: stop, min_p, presence_penalty, frequency_penalty
  SamplerExt ext;
};
struct PbGenerateRequest { std::string model, prompt; bool stream = false; PbGenerateOptions opt; };
// request options override the caller's default sampling field by field
void apply_options(const PbGenerateOptions& o, cl_sampling* sp, SamplerExt* ext);
struct PbTokenLogprob { std::string token, bytes; float logprob = 0.f; std::vector<PbTokenLogprob> top; };
struct PbGenerateResponse {
  std::string model, response, done_reason, worker_id;
  int64_t created_at_sec = 0; int32_t created_at_nanos = 0;
  bool done = false; int64_t total_duration = 0;
  std::vector<PbTokenLogprob> logprobs;   // field 8: the records of this frame's tokens
};
bool pb_decode_request(const uint8_t* data, size_t len, PbGenerateRequest* out);  // false: not a GenerateRequest
std::vector<uint8_t> pb_encode_response(const PbGenerateResponse& r);

struct LayerWeights {
  float* attn_norm = nullptr;
  float* ffn_norm = nullptr;
  __nv_bfloat16* wqkv = nullptr;   // [(H + 2 KV) * D][d]   rows: q | k | v
  __nv_bfloat16* wo = nullptr;     // [d][H * D]
  __nv_bfloat16* wgu = nullptr;    // [2 F][d]             row 2i = gate_i, row 2i+1 = up_i
  __nv_bfloat16* wdown = nullptr;  // [d][F]
};

struct SeqState {
  bool live = false;
  int len = 0;            // tokens whose K/V are in the cache
  int known = 0;          // leading history ids that are the real tokens of the cached K/V (seq_fake_fill's are not)
  std::vector<int32_t> history;
  std::vector<LogprobRecord> lps;   // records of the ids the step tail chose while logprobs were on, not taken yet
  SamplerExt ext;                   // cl_seq_set_sampling_ext: merged into every cl_sampling the sequence draws with
};

struct Request;  // scheduler.cpp

// Device bytes of a model's weights and RoPE table, as Engine::alloc_weights allocates them
int64_t weight_bytes(const cl_model_config& m);
// KV bytes per token of a model: K and V of every layer, bf16
inline int64_t kv_bytes_per_token(const cl_model_config& m) { return 2LL * m.n_layers * m.n_kv_heads * m.head_dim * 2; }
// The target's share of `avail` bytes of KV pool when a draft model's pool must hold as many tokens as the target's: the
// bytes are split in proportion to bytes per token (draft_tok = 0: all of it)
inline int64_t target_pool_share(int64_t avail, int64_t target_tok, int64_t draft_tok) {
  if (avail <= 0) return 0;
  return draft_tok > 0 ? avail / (target_tok + draft_tok) * target_tok : avail;
}

class Engine {
 public:
  Engine() = default;
  ~Engine();
  // draft (may be nullptr: CL_DRAFT_MODEL / CL_DRAFT_SEED decide): the draft model of speculative decoding
  int init(const cl_engine_config& cfg, const cl_engine_config* draft = nullptr);

  // token-level API (callers hold mu_)
  int seq_create(cl_seq_t* out);
  int seq_free(cl_seq_t s);
  int seq_len(cl_seq_t s, int32_t* out) { if (s < 0 || s >= max_seqs_ || !seqs_[s].live) return CL_ERR_BAD_SEQ; *out = seqs_[s].len; return CL_OK; }
  // Prefix cache (CL_PREFIX_CACHE / cl_engine_config.prefix_cache): a live sequence with len 0 takes the cached pages of
  // the longest page-aligned prefix of ids[0..n), at most n - 1 tokens; len = *reused.  A no-op (0) with the cache off.
  int attach_prefix(cl_seq_t s, const int32_t* ids, int n, int* reused);
  // Context shift (contract in include/clengine.h, cl_seq_shift): tokens [n_keep, n_keep + n_discard) leave the cache, the
  // kept K after them is rotated to its new position (kv_shift.cu), len and the device pos drop by n_discard.
  int seq_shift(cl_seq_t s, int n_keep, int n_discard);
  // the request-level switch (cl_engine_config.context_shift / num_keep) and its discard rule at length len
  bool context_shift() const { return context_shift_; }
  int shift_discard(int len) const { return page_size_ * ((len - num_keep_) / (2 * page_size_)); }
  bool prefix_cache() const { return prefix_cache_; }
  int prefix_stats(cl_prefix_stats* out);
  // Host tier of the prefix cache (contract in include/clengine.h, cl_engine_set_prefix_host_cache); callers hold mu_
  int set_prefix_host_cache(int64_t bytes);
  int prefill(cl_seq_t s, const int32_t* ids, int n, float* logits_out);
  // several prompts in one pass of the tile path (prefill.cu); logits_out: [n_seqs][vocab] or nullptr
  int prefill_multi(int n_seqs, const cl_seq_t* ss, const int32_t* const* ids, const int* lens, float* logits_out);
  int decode_step(cl_seq_t s, int32_t id, float* logits_out, int32_t* argmax_out);
  int decode_greedy(const cl_seq_t* seqs, int n_seqs, const int32_t* first_ids, int n_steps, int32_t* ids_out,
                    float* device_ms);
  // decode_greedy with the device sampler on the slots whose sp[b].temperature > 0 (every one must pass
  // device_sampling_ok); draw i of sequence b uses RNG step step0[b] + i (step0 may be nullptr: 0)
  int decode_sample(const cl_seq_t* seqs, int n_seqs, const int32_t* first_ids, const cl_sampling* sp, const uint64_t* step0,
                    int n_steps, int32_t* ids_out, float* device_ms);
  // Device sampler of one slot: every later step tail of `s` draws with `sp`, the first draw at RNG step `step0`, with the
  // last kSampleHistMax ids of hist[0..n_hist) as its history.  seq_create / seq_free disarm.
  // The sequence's SamplerExt (set_sampling_ext) joins sp.
  int arm_sampling(cl_seq_t s, const cl_sampling& sp, uint64_t step0, const int32_t* hist, int n_hist);
  int set_sampling_ext(cl_seq_t s, const SamplerExt& ext);   // seq_create / seq_free reset it to all zero
  int disarm_sampling(cl_seq_t s);
  int read_next_token(cl_seq_t s, int32_t* out);   // d_tok_[s]: what the last step tail of `s` chose
  // Log-probabilities (contract in include/clengine.h, cl_seq_set_logprobs): top_n -1 = off, 0..kLogprobTopMax = every
  // later step tail of `s` leaves a record, which the call that ran it appends to seqs_[s].lps.  seq_create / seq_free disarm.
  int set_logprobs(cl_seq_t s, int top_n);
  int take_logprobs(cl_seq_t s, cl_token_logprob* out, int cap, int* n_out);
  bool logprobs_on(cl_seq_t s) const { return lp_n_[s] >= 0; }
  // Speculative decoding: one verify pass over n_seqs distinct sequences (prefill.cu; contract in include/clengine.h,
  // cl_decode_verify_batch): sequence i verifies x0[i] and ks[i] (0..15) drafts, taken back to back from drafts.  Its ids
  // land at ids_out + its first row (the sum of k_j + 1 over the sequences before it), n_out[i] = a + 1 of them; logits_out
  // (may be nullptr): [rows][vocab].  seg_table: the attention takes the multi-row kernel (small_pass); false only with
  // one sequence, whose attention then runs per segment as in cl_decode_verify.
  int verify_batch(const cl_seq_t* ss, int n_seqs, const int32_t* x0, const int32_t* drafts, const int* ks, int32_t* ids_out,
                   int* n_out, float* logits_out, bool seg_table);
  // verify_batch with the device sampler armed for the pass on every sequence whose sp[i] draws (sp, step0 may be nullptr)
  int decode_verify_batch(const cl_seq_t* ss, int n_seqs, const int32_t* x0, const int32_t* drafts, const int* ks, const cl_sampling* sp,
                          const uint64_t* step0, int32_t* ids_out, int* n_out, float* logits_out, bool seg_table);
  // cl_decode_verify: decode_verify_batch of one sequence with k in 1..15, without the segment table (sp nullptr or
  // temperature <= 0: greedy)
  int decode_verify(cl_seq_t s, int32_t x0, const int32_t* draft, int k, const cl_sampling* sp, uint64_t step0, int32_t* ids_out,
                    int* n_out, float* logits_out);
  bool spec_path_ok() const;          // the verify pass runs on this model shape
  // The draft model's drafter (contract in include/clengine.h, cl_draft_model): for each target sequence ss[i], its mirror in
  // the draft engine catches up with hists[i][0..lens[i]) (the window ending with the next input x0) and drafts ks[i] ids
  // (0..15) with sp[i] / step0[i] (both may be nullptr: greedy, step 0).  The ids of sequence i land back to back at drafts +
  // the sum of ks[j] over j < i; n_drafts[i] = ks[i], or 0 when the draft pool has no pages for its mirror.
  int draft_tokens(const cl_seq_t* ss, int n, const int32_t* const* hists, const int* lens, const int* ks, const cl_sampling* sp,
                   const uint64_t* step0, int32_t* drafts, int* n_drafts);
  bool has_draft() const { return draft_ != nullptr; }
  int speculate() const { return speculate_; }
  int speculate_batch() const { return speculate_batch_; }
  int set_speculate_batch(int n);     // 1..min(max_batch, kSpecBatchMax), else CL_ERR_INVALID_ARG
  int64_t spec_multi_passes() const { return spec_multi_passes_; }
  int spec_stats(cl_spec_stats* out);
  bool device_sample() const { return device_sample_; }
  bool deterministic() const { return deterministic_; }
  int set_tensor(int layer, int kind, const uint16_t* data, int64_t n);
  int load_safetensors(const std::string& path);   // HF llama-layout checkpoint (file or directory) -> set_tensor (weights_io.cpp)
  // parity / benchmark aids (token level)
  int debug_kv(cl_seq_t s, int layer, int which, int t0, int n, float* out);   // cached K/V rows -> host [n][n_kv*head_dim]
  int seq_fake_fill(cl_seq_t s, int n_tokens);     // oracle oc_seq_fake_fill pattern into the paged cache of every layer
  int decode_step_batch(const cl_seq_t* seqs, int n_seqs, const int32_t* ids, float* logits_out, int32_t* argmax_out);
  int time_dominant_kernel(cl_seq_t s, int32_t first_id, int n_steps, float* kernel_ms, float* step_ms);
  int debug_hidden(float* out, int n);
  int debug_seq_hidden(cl_seq_t s, int what, float* out, int n, int32_t* mega_out);   // contract in include/clengine.h
  int debug_pass_info(int32_t* info, int32_t* segs, int max_segs);                  // the latest multi-row pass (clengine.h)
  int debug_pass_rows(int what, int row0, int n, float* out);                        // rows of its workspace (clengine.h)
  int debug_timeline(long long* out, int n);   // CL_TIMELINE=1: globaltimer stamps of the last step (CTA 0 of every node)
  int stats(cl_stats* out);

  // request-level (scheduler.cpp)
  // sink (optional): called on the CALLING thread with every batch of newly generated ids; nonzero return cancels
  // lp_fn (optional, with logprobs on): called just before fn with the records of the same ids
  struct TokenSink {
    int (*fn)(void* user, const int32_t* ids, int n) = nullptr; void* user = nullptr;
    int (*lp_fn)(void* user, const cl_token_logprob* lps, int n) = nullptr;
  };
  // top_n >= 0: logprobs on for the request; *lps (malloc'd, one record per generated id) when lps is not nullptr.
  // ext / stop (may be nullptr: none): checked by check_sampling_ext; a stop ends the request as StopScan decides.
  int generate_ids(const int32_t* prompt, int n_prompt, const cl_sampling& sp, cl_result* out, const TokenSink* sink = nullptr,
                   int top_n = -1, cl_token_logprob** lps = nullptr, const SamplerExt* ext = nullptr,
                   const std::vector<std::string>* stop = nullptr);
  void scheduler_main();
  void start_scheduler();
  void stop_scheduler();

  cl_model_config cfg{};
  std::string model_name;
  std::mutex mu_;               // serialises every GPU-touching call
  std::unique_ptr<Tokenizer> tok;

 private:
  int alloc_weights();
  int fill_synthetic(uint64_t seed);
  int alloc_state();
  int ensure_capacity(cl_seq_t s, int n_tokens);  // reserve pages + upload block table row
  // Enqueue the KvPool's pending spills and fills on stream_, in the order the pool decided them, and clear them.  Every
  // call that reserves or attaches pages ends here, so the copies sit on the stream ahead of any kernel that writes an
  // evicted page or reads an attached one.  Eager launches: never inside a captured graph.
  int drain_kv_moves();
  // Every call that appends K/V to sequence s ends here: len += n, ids join the history, and with the prefix cache on the
  // full pages whose tokens are all known are published.  The first n_known ids are real tokens; a placeholder stops
  // publishing for the rest of the sequence.  The work that wrote the pages is already on stream_, ahead of any reader.
  void seq_advance(cl_seq_t s, const int32_t* ids, int n, int n_known);
  // kernels of one token step for d_slots_[0..B); step_off: steps already enqueued since the sequences' lengths were last
  // advanced on the host (a device loop's step index), which deterministic mode needs for its segment table
  int enqueue_step(int B, int step_off = 0);
  int enqueue_step_batched(int B);                 // B >= 2: wgmma projections + per-sequence glue kernels
  int enqueue_lm_head(int B, bool pdl);            // final norm + LM-head GEMV of d_h_ -> d_logits_ for d_slots_[0..B)
  // argmax (or, on armed slots, a draw) of d_logits_, advance tok / pos, id ring (step_tail_kernel); push_input: decode
  // steps, whose input token joins an armed slot's history.  Prefill tails do not push: the armed history holds the prompt.
  int enqueue_step_tail(int B, bool push_input);
  int run_step_graph(int B, int step_off = 0);    // deterministic mode: enqueue_step, eagerly
  // Deterministic mode (prefill.cu).  det_step: the step of B sequences as B one-row segments of small_pass, its LM head the
  // pass's wgmma GEMM, then the step tail.  det_prefill: prompts of n_seqs distinct sequences as passes of at most
  // kSpecMaxRows rows, each prompt cut into segments of at most kVerifyMaxRows rows; the last rows' logits from the same
  // GEMM head, then the step tail without pushing its input (collect_logprobs is the caller's).
  int det_step(int B, int step_off);
  int det_prefill(int n_seqs, const cl_seq_t* ss, const int32_t* const* ids, const int* lens, float* logits_out);
  int proj_splits(int N, int K) const;            // split-K count of the split-K pass's projections (kDetSms in deterministic mode)
  bool ensure_graph(int B);
  void precapture_graphs(int max_b);              // the step graphs of batch sizes 1..max_b
  int read_logits(int slot, float* out);
  // After a call whose step tail ran once for the sequences ss[0..n): each one with logprobs on appends its record
  // (d_lp_last_) to its pending list.  Nothing is copied when none is on.  Synchronises the stream.
  int collect_logprobs(const cl_seq_t* ss, int n);
  int upload_logprobs(cl_seq_t s, int top_n);     // d_lp_n_[s] = top_n unless it holds it already
  int prefill_tokenwise(cl_seq_t s, const int32_t* ids, int n, float* logits_out);
  int prefill_chunked(cl_seq_t s, const int32_t* ids, int n, float* logits_out);
  int ensure_prefill_ws(int tokens);  // tensor-core path (prefill.cu)
  struct PrefillSegment { int seq, row0, n, pos0; };   // rows row0 .. row0 + n - 1 of a pass: sequence seq from position pos0
  // one tile-path pass of T rows made of n_segs segments; leaves the final residual rows in pws_->h
  int prefill_pass(const PrefillSegment* segs, int n_segs, const int* ids, int T, int& launches, LaunchProfiler& prof);
  int attn_prefill(const AttnPrefillArgs& a, int layer, int& launches, LaunchProfiler& prof);   // the one choice of prefill attention kernel
  int prefill_attn_kind(int pos0, int n) const;   // the kernel attn_prefill runs for n rows from pos0: kPassAttnMma / Wgmma / Verify / Long
  int ensure_long_attn_ws();                      // the split workspace of the segments that end past kLongPrefillFrom
  // What the latest multi-row pass was, on the host (debug_pass_info / debug_pass_rows); T == 0: no pass whose rows the
  // workspace holds (none yet, a token-wise prefill since, or a failed pass).  Recording adds no device work.
  enum { kPassSplitK = 0, kPassTile = 1 };
  struct PassRecord { int path = -1, attn = -1, T = 0; std::vector<PrefillSegment> segs; };
  void record_pass(int path, bool multi_row, const PrefillSegment* segs, int n_segs, int T);
  PassRecord pass_;
  int prefill_small(cl_seq_t s, const int32_t* ids, int n, float* logits_out);    // short prompts: split-K projections (prefill.cu)
  int ensure_small_ws();
  // the split-K pass of prefill_small and verify_batch: T rows made of n_segs segments; leaves sws_->h and the
  // final-norm rows sws_->xn.  row_map (device, or nullptr with one segment): [2][T] the sequence, then the position of every
  // row; seg_table (device, may be nullptr): the segments as AttnVerifyArgs::segs, which selects the multi-row attention
  // kernel where the shape allows it.
  int small_pass(const PrefillSegment* segs, int n_segs, const int* ids, int T, const int* row_map, const int* seg_table, int& launches,
                 LaunchProfiler& prof);
  // row map and segment table of a small_pass over segs into spec_->row_map / spec_->segs (the multi-row attention's plan)
  int upload_pass_tables(const PrefillSegment* segs, int n_segs, int T);
  int ensure_spec_ws();
  SpecTailArgs spec_tail_args(const PrefillSegment& g, int out_off) const;   // the spec tail of one verify segment
  bool prefill_path_ok() const;
  int set_single_slot(cl_seq_t s);

  // request-level transitions and scheduler phases (scheduler.cpp); callers hold mu_
  bool join(Request& r, const int32_t* ids, int n, bool admission);
  void retire(Request& r, int status, const std::string& err);
  void preempt(std::shared_ptr<Request> r);
  int shift_request(Request& r);
  int host_next_token(Request& r, float* logits, bool read_back, const int32_t* hist, int n_hist, int32_t* next);
  int spec_round(const std::shared_ptr<Request>* rs, int n);
  int generate_sync(const std::shared_ptr<Request>& r, const TokenSink* sink);
  int admission_pages(Request& r, int* hit);
  bool wait_for_work();
  bool admit_group(int budget);
  void admit_chunked(int budget);
  void admitted(const std::shared_ptr<Request>& r, int32_t next);
  void make_room();
  bool speculate_running();
  int step_running();
  void retire_finished();
  void fail_running(int rc);
  void shutdown_requests();

  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
  cudaEvent_t step_done_ev_ = nullptr;     // scheduler: blocking-sync event behind every batched step (scheduler.cpp)
  bool sched_multi_prefill_ = false;       // group admission through prefill_multi (CL_SCHED_MULTI_PREFILL)
  int page_size_ = 32, max_batch_ = 8, max_seqs_ = 8, n_pages_ = 0, max_pages_per_seq_ = 0;
  int gemv_variant_ = 1, nsplit_ = 16;
  bool use_graph_ = true, use_pdl_ = true;
  bool want_timeline_ = false, use_mega_ = false;
  MegaLayer* d_mega_layers_ = nullptr;
  CUtensorMap kmap_{}, vmap_{};
  bool have_kv_maps_ = false;
  long long* d_timeline_ = nullptr;
  unsigned* d_sync_ = nullptr;             // the persistent kernel's counters (MegaArgs: bars, tile_ctr, pf_ctr)
  int n_sync_ = 0;
  int qkv_dim_ = 0, q_dim_ = 0, kv_dim_ = 0;

  // weights
  std::vector<void*> allocs_;
  __nv_bfloat16* embed_ = nullptr;
  __nv_bfloat16* lm_head_ = nullptr;
  float* final_norm_ = nullptr;
  std::vector<LayerWeights> layers_;
  float2* rope_ = nullptr;
  __nv_bfloat16* kpool_ = nullptr;  // [L][n_pages][KV][P][D]
  __nv_bfloat16* vpool_ = nullptr;
  size_t kv_layer_elems_ = 0;

  // per-slot state
  int* d_tok_ = nullptr; int* d_pos_ = nullptr; int* d_bt_ = nullptr; int* d_slots_ = nullptr;
  float* d_h_ = nullptr; float* d_q_ = nullptr; float* d_attn_ = nullptr; float* d_act_ = nullptr;
  float* d_logits_ = nullptr; float* d_attn_part_ = nullptr; unsigned* d_attn_cnt_ = nullptr;
  float* d_tail_val_ = nullptr; int* d_tail_idx_ = nullptr; unsigned* d_tail_cnt_ = nullptr;
  int* d_ids_ring_ = nullptr; int* d_step_counter_ = nullptr; int* d_prompt_ = nullptr;
  int ring_steps_ = 1024, prompt_cap_ = 0;
  float* h_logits_pinned_ = nullptr; int* h_ids_pinned_ = nullptr;
  // device sampler (kernels.h SampleState), indexed by sequence handle
  int* d_samp_mode_ = nullptr; SampleParams* d_samp_par_ = nullptr; unsigned long long* d_samp_step_ = nullptr;
  int* d_samp_hist_ = nullptr; int* d_samp_hlen_ = nullptr; unsigned long long* d_samp_cand_ = nullptr;
  std::vector<int> samp_hlen_;        // host: history length uploaded by arm_sampling, -1 = disarmed
  // log-probabilities (kernels.h LogprobState), indexed by sequence handle; the ring runs parallel to the id ring
  int* d_lp_n_ = nullptr; float2* d_lp_part_ = nullptr; unsigned long long* d_lp_cand_ = nullptr; unsigned* d_lp_cnt_ = nullptr;
  LogprobRecord* d_lp_last_ = nullptr; LogprobRecord* d_lp_ring_ = nullptr; LogprobRecord* h_lp_pinned_ = nullptr;
  std::vector<int> lp_n_;             // host mirror of d_lp_n_
  bool device_sample_ = true;         // CL_DEVICE_SAMPLE: the scheduler and the synchronous path draw on the device where they can
  bool deterministic_ = false;        // CL_DETERMINISTIC / cl_engine_config.deterministic (det_step, det_prefill)
  bool verify_one_row_ = true;        // CL_VERIFY_ONE_ROW: passes of one-row segments run the one-warp multi-row attention
  std::vector<int> h_slots_;          // host copy of d_slots_[0..B) as its last upload left it (det_step's segment table)
  int* det_ids_ = nullptr;            // det_step: the step's input ids, row order [kSpecMaxRows]
  __nv_bfloat16* det_xn_ = nullptr;   // det_prefill: final-norm rows of the prompts' last tokens [kSpecMaxRows][d]

  // prefill workspace (allocated lazily)
  struct PrefillWs {
    int cap_tokens = 0;
    __nv_bfloat16* xn = nullptr;    // [T][d]
    float* qkv = nullptr;           // [T][qkv_dim]
    __nv_bfloat16* q = nullptr;     // [T][q_dim]
    __nv_bfloat16* attn = nullptr;  // [T][q_dim]
    float* h = nullptr;             // [T][d]
    __nv_bfloat16* act = nullptr;   // [T][F]
  };
  std::unique_ptr<PrefillWs> pws_;
  struct SmallPrefillWs { float* part = nullptr; __nv_bfloat16* xn = nullptr; __nv_bfloat16* q = nullptr; __nv_bfloat16* attn = nullptr;
                          float* h = nullptr; __nv_bfloat16* act = nullptr; int* iota = nullptr; };
  std::unique_ptr<SmallPrefillWs> sws_;
  float* long_part_ = nullptr;        // split-KV partials of the long-context prefill kernel (lazily, attn_prefill)
  unsigned* long_cnt_ = nullptr;      // its arrival counters, zero between launches
  int* long_seg_ = nullptr;           // the one-segment table of a long segment run by the multi-row verify kernel
  // verify passes (allocated lazily): rows of at most kSpecMaxRows; out holds 1 + T ints per sequence, row_map [2][rows];
  // segs [rows][8], attn_part and attn_cnt: the multi-row attention's segment table, split partials and counters
  struct SpecWs { float* logits = nullptr; int* choice = nullptr; float* part_val = nullptr; int* part_idx = nullptr;
                  unsigned* counters = nullptr; unsigned long long* cand = nullptr; int* out = nullptr; int* row_map = nullptr;
                  int* segs = nullptr; float* attn_part = nullptr; unsigned* attn_cnt = nullptr;
                  float2* lp_part = nullptr; unsigned long long* lp_cand = nullptr; unsigned* lp_cnt = nullptr; LogprobRecord* lp_rows = nullptr; };
  int verify_split_pages() const;     // pages per split of the multi-row attention (a function of max_seq_len only)
  std::unique_ptr<SpecWs> spec_;
  int speculate_ = 0;                 // most drafted tokens per verify pass in the scheduler / synchronous path (0 = off)
  std::atomic<int> speculate_batch_{1};   // most sequences the scheduler verifies in one pass (1: only a request running alone)
  std::atomic<int64_t> spec_passes_{0}, spec_drafted_{0}, spec_accepted_{0}, spec_emitted_{0}, spec_multi_passes_{0};
  // Draft model (draft.cpp): an engine of its own on the same device, with no scheduler, prefix cache or speculation, whose
  // pool holds as many tokens as this one's.  mirror_[s]: the draft sequence that mirrors target sequence s (-1: none).
  std::unique_ptr<Engine> draft_;
  bool is_draft_ = false;             // this engine is another engine's draft: the env switches of serving features stay off
  bool hf_tok_ = false;               // the tokenizer came from the model directory's tokenizer.json
  std::vector<int> mirror_;
  std::atomic<int64_t> draft_rows_{0}, draft_ns_{0}, draft_pages_{0};   // cl_spec_stats.draft_*; draft_pages_: the draft pool's used pages
  void seq_rewind(cl_seq_t s, int len);  // a draft mirror: len drops to `len` (history with it), its pages stay
  int prefill_small_max_ = 0;         // prompts up to this many tokens take the split-K path (CL_PREFILL_SMALL_MAX, 0 = off)
  struct BatchWs { __nv_bfloat16* xn = nullptr; __nv_bfloat16* attn = nullptr; __nv_bfloat16* act = nullptr; float* part = nullptr; float* logits = nullptr; };
  std::unique_ptr<BatchWs> bws_;
  bool use_batch_gemm_ = false;
  int prefill_chunk_tokens_ = 4096;

  std::unique_ptr<KvPool> pool_;
  uint4* host_kv_ = nullptr;          // host tier of the prefix cache: pinned, mapped pages (KvMoveArgs::host)
  int2* d_moves_ = nullptr;           // the moves of one drain (at most 2 per pool page), uploaded for the transfer kernels
  std::vector<SeqState> seqs_;
  bool prefix_cache_ = false;         // share full KV pages across sequences with the same prefix (CL_PREFIX_CACHE)
  bool context_shift_ = false;        // requests shift their sequence instead of stopping at max_seq_len (CL_CONTEXT_SHIFT)
  int num_keep_ = 0;                  // leading tokens a request's shift never discards (CL_NUM_KEEP)
  KvShiftItem* d_shift_items_ = nullptr;   // one shift's work list (at most max_pages_per_seq_ + 1 items)
  std::atomic<int64_t> prefix_lookups_{0}, prefix_tokens_looked_up_{0}, prefix_tokens_reused_{0};
  std::map<int, cudaGraphExec_t> graphs_;
  std::map<int, int> graph_nodes_;
  int prefill_min_tokens_ = 16;
  bool graph_failed_ = false;
  int last_single_slot_ = -1;
  std::vector<int> last_batch_slots_;  // sequences of the latest step over two or more sequences, in batch order (debug_seq_hidden)
  bool slots_dirty_ = false;          // d_slots_ was rewritten outside the scheduler loop: its cached copy is stale
  cudaEvent_t* probe_ev_ = nullptr;   // time_dominant_kernel: event pair recorded around the dominant kernel of an eager step
  int probe_idx_ = 0;

  // stats
  std::atomic<int64_t> launches_{0}, tokens_generated_{0}, requests_completed_{0}, preemptions_{0};
  // scheduler accounting (cl_stats.sched_*): where the scheduler thread's time goes
  std::atomic<int64_t> sched_decode_steps_{0}, sched_decode_ns_{0}, sched_prefill_calls_{0}, sched_prefill_tokens_{0}, sched_prefill_ns_{0};
  double tok_per_sec_ewma_ = 0.0;          // measured: EWMA of decode steps/s x max_batch (diagnostic)
  double capacity_tok_per_sec_ = 0.0;      // advertised: load-independent capacity estimate (engine.cu init)
  char gpu_name_[64] = {0};
  int vram_gb_ = 0;

  // scheduler
  std::thread sched_thread_;
  std::mutex q_mu_;
  std::condition_variable q_cv_;
  std::deque<std::shared_ptr<Request>> queue_;
  std::vector<std::shared_ptr<Request>> active_;
  std::shared_ptr<Request> prefilling_;   // the one request whose prompt is being prefilled chunk by chunk (scheduler.cpp)
  int sched_prefill_chunk_ = 0;           // admission token budget per iteration while other sequences are decoding (CL_SCHED_PREFILL_CHUNK; 0 = unlimited)
  // the scheduler thread's host buffers: a host-sampled request's logits, d_tok_ read back, the slot list last uploaded to d_slots_
  std::vector<float> sched_logits_;
  std::vector<int32_t> sched_toks_;
  std::vector<int> sched_slots_;
  std::atomic<bool> stop_{false};
  bool sched_started_ = false;
  friend struct Request;
};

}  // namespace cl

struct cl_engine {
  cl::Engine impl;
};
struct cl_kvpool {
  cl::KvPool pool;
  std::mutex mu;
  cl_kvpool(int n, int p) : pool(n, p) {}
};
