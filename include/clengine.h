/*
 * clengine.h — C-ABI of the H100-native (sm_90a) CrowdLlama worker decode engine (libclengine.so).
 *
 * This is the drop-in boundary for the ONE hot path this repository accelerates: the
 * worker-side model step that the reference reaches through
 *     crowdllama.UnifiedAPIHandler            /root/reference/pkg/crowdllama/api.go:19
 *     crowdllama.WorkerAPIHandler             /root/reference/pkg/crowdllama/api.go:45-96
 *     callOllamaAPI (HTTP POST /api/chat)     /root/reference/pkg/crowdllama/api.go:108-160
 * and, behind that HTTP call, the un-vendored github.com/ollama/ollama v0.9.6
 * (/root/reference/go.mod:12) llama.cpp decode loop.  A Go cgo shim (go/b200handler/handler.go,
 * shown in INTEGRATION.md) builds a UnifiedAPIHandler closure over cl_generate(); Python tests
 * and bench.py bind the same symbols with ctypes.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - every function returns 0 (CL_OK) or a negative cl_status; nothing throws across the ABI.
 *   - the library never retains caller pointers after a call returns (cgo rule); strings and
 *     id arrays handed back in cl_result are malloc()'d by the library and released with
 *     cl_result_free().
 *   - cl_generate(), cl_generate_ids(), cl_engine_stats() are thread-safe and re-entrant (one goroutine per inbound
 *     libp2p stream calls the handler concurrently: /root/reference/pkg/peer/peer.go:177-182).
 *     The token-level cl_seq_* / cl_prefill / cl_decode_step calls are serialised internally by one engine lock.
 *   - there is NO CPU fallback: if no sm_90 (compute capability 9.x) device is present cl_engine_create fails with
 *     CL_ERR_NO_DEVICE.
 */
#ifndef CLENGINE_H_
#define CLENGINE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CL_ABI_VERSION 2

typedef enum cl_status {
  CL_OK = 0,
  CL_ERR_INVALID_ARG = -1,
  CL_ERR_NO_DEVICE = -2,     /* no CUDA device / not sm_90 */
  CL_ERR_CUDA = -3,          /* CUDA runtime error; see cl_last_error() */
  CL_ERR_OOM = -4,           /* device memory or KV pages exhausted */
  CL_ERR_UNKNOWN_MODEL = -5, /* model name not served by this engine */
  CL_ERR_TOO_LONG = -6,      /* prompt + generation exceeds max_seq_len */
  CL_ERR_BAD_SEQ = -7,       /* unknown / freed sequence handle */
  CL_ERR_SHUTDOWN = -8,      /* engine is being destroyed */
  CL_ERR_IO = -9,            /* weight / tokenizer file error */
  CL_ERR_INTERNAL = -10,
  CL_ERR_BAD_MESSAGE = -11   /* cl_handle_message: not a GenerateRequest (api.go:48-51) */
} cl_status;

/* Llama-family architecture description (public architecture facts; SURVEY.md §8). */
typedef struct cl_model_config {
  int32_t n_layers;
  int32_t d_model;
  int32_t n_heads;
  int32_t n_kv_heads;
  int32_t head_dim;
  int32_t d_ff;
  int32_t vocab_size;
  int32_t max_seq_len;   /* positions covered by the RoPE table and block tables */
  float rope_theta;
  float rms_eps;
  /* "llama3" rotary scaling (Llama-3.1 / 3.2 checkpoints; HF config.json rope_scaling / rope_parameters with
   * rope_type "llama3").  rope_factor <= 1 (e.g. 0): plain rotary embeddings.  Otherwise the inverse frequency of
   * dimension pair i is divided by rope_factor where its wavelength exceeds rope_original_max_pos / rope_low_freq_factor,
   * kept where it is below rope_original_max_pos / rope_high_freq_factor, and blended linearly in between. */
  float rope_factor;
  float rope_low_freq_factor;
  float rope_high_freq_factor;
  int32_t rope_original_max_pos;
} cl_model_config;

typedef struct cl_engine_config {
  int32_t abi_version;     /* must be CL_ABI_VERSION */
  int32_t device;          /* CUDA ordinal (one engine process per GPU) */
  const char* model_name;  /* name advertised / matched exactly, like Resource.SupportedModels
                              (/root/reference/pkg/peermanager/manager.go:349-354) */
  const char* preset;      /* "llama3-8b" | "mistral-7b" | "tinyllama-1.1b" | "tiny-test" | NULL
                              (NULL => take `model` below) */
  cl_model_config model;   /* used when preset == NULL */
  const char* weights_path;/* HF llama-layout checkpoint: a .safetensors file, or a model directory with *.safetensors shards
                              (+ config.json, used when preset == NULL and model.n_layers == 0, + tokenizer.json, loaded
                              when present); BF16 / F16 / F32 tensors -> bf16.  NULL => synthetic seeded weights */
  uint64_t weights_seed;   /* seed of the counter-based synthetic weight generator */
  int64_t kv_pool_bytes;   /* bytes of HBM for the paged KV pool; 0 => derive from max_seqs */
  int32_t page_size;       /* tokens per KV page: 16, 32 or 64 (0 => 32) */
  int32_t max_batch;       /* max concurrently decoding sequences (0 => 8); the tensor-core batched step serves 2..128,
                              larger values fall back to per-sequence GEMV kernels */
  int32_t max_seqs;        /* max live sequence handles (0 => max_batch) */
  int32_t use_cuda_graph;  /* 1 => capture the token step in a CUDA graph (default 1; -1 => 0) */
  int32_t decode_path;     /* 0 auto, 1 = generic LDG GEMV kernels, 2 = TMA-ring streaming GEMV */
  int32_t start_scheduler; /* 1 => start the continuous-batching thread behind cl_generate */
  int32_t prefix_cache;    /* 1 => reuse the cached KV pages of earlier requests that share a prompt prefix (default 0;
                              env CL_PREFIX_CACHE=0|1 overrides).  Full pages of known tokens stay indexed after their
                              sequence is freed and are evicted least recently used first when the pool runs dry, so a
                              request whose prompt starts with an earlier prompt (or a preempted request coming back)
                              prefills only the rest.  See cl_seq_attach_prefix / cl_engine_prefix_stats, and
                              cl_engine_set_prefix_host_cache for a host-memory tier behind the pool. */
  int32_t speculate;       /* speculative decoding: 0 => off (default), 1..15 => the most drafted tokens per verify pass
                              (env CL_SPECULATE overrides; other values make cl_engine_create fail with CL_ERR_INVALID_ARG).
                              While exactly one request is running and nothing waits, a greedy or device-sampled request
                              drafts the ids that followed the latest earlier occurrence of its last 3 (or 2) ids in its
                              prompt and output (cl_draft_ngram) and checks them in one pass over the weights
                              (cl_decode_verify).  The ids are the ones single steps would produce, up to near-tie flips
                              between the two kernel paths (none in deterministic mode, where they are the same bits).  Model shapes without the verify path decode normally.  With a
                              draft model (cl_engine_create_with_draft, env CL_DRAFT_MODEL) the drafts come from it instead. */
  int32_t context_shift;   /* 1 => a request whose sequence fills max_seq_len shifts it (cl_seq_shift) and goes on generating
                              instead of ending with done_reason "length"; 0 => off (default; env CL_CONTEXT_SHIFT=0|1
                              overrides).  Ollama's rule, as its documentation states it (its source cannot be checked
                              here, like the sampler order and the templates): keep the first num_keep tokens and discard
                              half of the rest.  Here the half is rounded down to whole KV pages: before a decode step or a
                              verify pass would write position max_seq_len, the request's sequence discards
                                  delta = page_size * floor((max_seq_len - num_keep) / (2 * page_size))
                              tokens after its first num_keep.  With the switch on:
                              - num_predict > 0 may exceed max_seq_len - n_prompt.  num_predict <= 0 keeps its meaning,
                                "until EOS or max_seq_len - n_prompt tokens", on purpose: an unbounded request would hold
                                a slot of a shared worker forever.
                              - A prompt of max_seq_len tokens or more keeps its first num_keep ids and its last
                                max_seq_len - 1 - num_keep ids instead of failing with CL_ERR_TOO_LONG; cl_result.n_prompt
                                counts what was prefilled.
                              - A shifted request that is preempted comes back by prefilling its current window (first
                                num_keep ids, then the ids after the discarded ones).  Those K/V are computed without the
                                discarded context in view, so they differ from the shifted cache they replace.
                              - Speculative rounds still draft only up to max_seq_len; the shift runs before the next round.
                              The device loops (cl_decode_greedy*, cl_decode_sample_batch) never shift. */
  int32_t num_keep;        /* leading tokens a context shift never discards (env CL_NUM_KEEP overrides).
                              cl_default_engine_config leaves it 0, like the reserved ints it came from; the Python Engine
                              and worker.py pass 4, Ollama's documented default.  A C caller that turns context_shift on
                              should set num_keep too (4 to match Ollama): with 0, the first shift discards the BOS token
                              and the start of the prompt.  With context_shift on, cl_engine_create
                              fails with CL_ERR_INVALID_ARG unless 0 <= num_keep <= max_seq_len - 2 * page_size (a
                              shift must discard at least one page). */
  int32_t context_length;  /* the served context window in tokens (env CL_CONTEXT_LENGTH overrides).  0 (the default) keeps
                              the model's own: a preset's or cl_model_config's max_seq_len, and for a model directory
                              min(max_position_embeddings, 32768), capped by sliding_window.  > 0 sets max_seq_len to it,
                              from 2 pages up to 131072 tokens (Llama-3.1 / 3.2's 128K window); a model directory refuses
                              it above max_position_embeddings or sliding_window.  A window cl_engine_create does not
                              accept fails it with CL_ERR_INVALID_ARG; cl_resolve_model_config applies the same rule on the
                              host.  With kv_pool_bytes == 0 and context_length > 0, the KV pool takes the device memory
                              that is free after the weights, less a 4 GiB reserve for the engine's state and prefill /
                              verify workspaces, capped at max_seqs x the window: at 131072 tokens a full batch of
                              windows rarely fits, and a prompt whose pages exceed the whole pool fails with CL_ERR_OOM.
                              Prefill segments that end past 32768 tokens run split-KV attention kernels for head_dim
                              128 / page 32 (up to 16 rows: the multi-row verify kernel); shorter segments run what they
                              always have. */
  int32_t deterministic;   /* 1 => deterministic mode (env CL_DETERMINISTIC=0|1 overrides; 0, the default, changes nothing).
                              Every token path runs one row-invariant pass: each decode step is one-row segments of the
                              split-K pass of verify passes, every prefill is passes of at most 128 rows cut into segments of
                              at most 16 rows, all with the multi-row split-KV attention and the pass's wgmma LM head, and
                              the split-K counts are those of a 132-SM card whatever the device has (cl_gemm_split_plan).
                              With the switch on, a sequence's logits, K/V, ids and logprob records are the same bits
                                - whatever other sequences share its steps and passes (batch size, neighbours' lengths);
                                - however its prompt is split: one call, scheduler chunks, cl_prefill_batch groups, pages
                                  of the prefix cache or its host tier, recompute after preemption;
                                - whether its ids come from single steps or verify passes (n-gram or draft-model drafter);
                                - on any sm_90 GPU, for the same model, weights, page size and context_length.
                              The one exception is context_shift's: a shifted request that is preempted recomputes its
                              window without the discarded context.  The persistent kernel, the GEMV path, the batched step
                              and step graphs are not used.  cl_engine_create fails with CL_ERR_INVALID_ARG for shapes the
                              pass does not take (head_dim 128, 4 query heads per kv head and page 32 only: Llama-3 /
                              3.1-8B, Mistral-7B) and for max_batch > 128. */
  int32_t reserved[2];
} cl_engine_config;

/* Sampler.  The reference sends no options (api.go:109-118), so Ollama defaults apply upstream:
 * temperature 0.8, top_k 40, top_p 0.9, repeat_penalty 1.1 over the last 64 tokens, random seed.
 * temperature <= 0 selects greedy argmax with lowest-index tie-break (the parity mode) and ignores every stage below.
 * The stages, in order (cl_sampling_ext adds the presence / frequency penalties and min_p):
 *   1. penalty stage over the last repeat_last_n ids of the history (out-of-range ids skipped): an id occurring c > 0
 *      times there gets v / repeat_penalty (v > 0) or v * repeat_penalty, then v -= c * frequency_penalty +
 *      presence_penalty (llama.cpp's formula, in fp32);
 *   2. top-k (value descending, id ascending);  3. softmax at `temperature` (p_i = exp((v_i - v_0) / T) in double);
 *   4. top-p: the shortest leading run whose normalised mass reaches top_p;
 *   5. min_p: of those, the leading candidates with p_i >= min_p * p_0 (the top candidate always stays);
 *   6. one draw from the counter-based generator at (seed, step).
 * This order follows Ollama's own sampler (top-k, temperature, softmax, top-p, min-p).  Like the rest of the chain it is
 * unpinned: it was not checked draw for draw against Ollama's binary.
 * Where the draw runs: with temperature > 0, 1 <= top_k <= 128, top_k < vocab_size, vocab_size <= 163840, and the penalty
 * stage off (repeat_penalty 1 and both other penalties 0, or repeat_last_n 0) or over 1..256 ids, the decode step's last
 * kernel draws the token on the GPU, so the token loop never waits for the host (Ollama's defaults qualify, and so does
 * any min_p and any finite presence / frequency penalty).  Other settings (top_k 0, repeat_last_n -1, ...) run the host
 * sampler on the step's logits.  Both draw the same id for the same logits, history, seed and step (cl_sample_token[_ext]
 * is the host one; env CL_DEVICE_SAMPLE=0 sends every request to it). */
typedef struct cl_sampling {
  float temperature;
  int32_t top_k;
  float top_p;
  float repeat_penalty;
  int32_t repeat_last_n;
  uint64_t seed;
  int32_t max_new_tokens;  /* num_predict; <= 0 => until EOS or context full */
  int32_t ignore_eos;      /* 1 => never stop on EOS (benchmarks) */
} cl_sampling;

/* Ollama's other generation options, kept out of cl_sampling so that its layout stays what callers compiled against.  All
 * zero is exactly the behaviour of cl_sampling alone; every entry point that takes only a cl_sampling runs with all zero.
 *   min_p: 0..1 (0 off), stage 5 above.  presence_penalty, frequency_penalty: any finite value (0 off), stage 1 above.
 *   stop / n_stop: request level only (cl_generate_ids_ext).  Generation ends as soon as the response text contains one of
 *   the strings: done_reason "stop" (over "length" on the same token), cl_result.text ends just before the earliest
 *   occurrence.  Matched against the raw bytes of the generated ids (cl_tokenizer_decode of them, never the prompt), so a
 *   match may span tokens and start or end inside one token's bytes.  token_ids / n_generated keep every generated id up to
 *   and including the one that completed the match, and logprob records stay one per id: only the text is cut.  Streamed
 *   deltas hold back any text that could still begin a stop string, so they never carry a byte of one and concatenate to
 *   cl_result.text.  At most 16 non-empty strings (empty ones are dropped) of at most 256 bytes each.
 * CL_ERR_INVALID_ARG, with cl_last_error set, for min_p outside [0, 1], a NaN or infinite penalty, or stops past the limits.
 * The token-level calls know nothing of text and ignore stop / n_stop. */
typedef struct cl_sampling_ext {
  float min_p;
  float presence_penalty;
  float frequency_penalty;
  int32_t n_stop;
  const char* const* stop;   /* n_stop NUL-terminated strings */
  int32_t reserved[8];
} cl_sampling_ext;

typedef struct cl_result {
  char* text;            /* NUL-terminated UTF-8, malloc'd */
  size_t text_len;
  char* done_reason;     /* "stop" | "length", malloc'd (GenerateResponse.DoneReason, api.go:82) */
  int32_t* token_ids;    /* generated ids, malloc'd */
  int32_t n_prompt;
  int32_t n_generated;
  int64_t prefill_ns;
  int64_t decode_ns;
  int64_t total_ns;
  int32_t n_preempted;   /* times this request was evicted and recomputed */
} cl_result;

typedef struct cl_stats {
  double tokens_per_sec;     /* capacity, load-independent: 70 % of the HBM roofline of one decode step x max_batch, from the
                                device's memory bandwidth and the model's bytes per token -> Resource.TokensThroughput (types.go:33) */
  double load;               /* (active + queued) / max_batch; > 1: requests are waiting for a batch slot -> Resource.Load
                                (types.go:35) through the two-level rule of INTEGRATION.md "What to advertise" */
  int32_t queue_depth;
  int32_t active_seqs;
  int32_t kv_pages_total;
  int32_t kv_pages_used;
  int64_t tokens_generated;
  int64_t requests_completed;
  int64_t preemptions;
  int32_t vram_gb;           /* -> Resource.VRAMGB */
  char gpu_model[64];        /* -> Resource.GPUModel */
  int64_t kernel_launches;   /* kernels of this library launched so far (graph nodes counted) */
  double measured_tokens_per_sec; /* EWMA of decode steps/s x max_batch at the CURRENT batch sizes (diagnostic; not for routing) */
  /* scheduler accounting since engine creation: batched decode steps (tokens_generated / sched_decode_steps = mean batch)
     and admission-time prefill calls, with the scheduler thread's wall time inside each */
  int64_t sched_decode_steps, sched_decode_ns;
  int64_t sched_prefill_calls, sched_prefill_tokens, sched_prefill_ns;
} cl_stats;

/* Prefix cache accounting since engine creation (all zero with the cache off). */
typedef struct cl_prefix_stats {
  int32_t enabled;
  int32_t cached_pages;      /* now: pages no sequence holds that are kept for reuse (counted as free in cl_stats) */
  int64_t lookups;           /* sequences that looked their prompt up (cl_seq_attach_prefix, every request admission) */
  int64_t tokens_looked_up;  /* prompt tokens of those lookups */
  int64_t tokens_reused;     /* of which found in the cache: their prefill was skipped */
  int64_t pages_evicted;     /* cached pages handed out again because the pool ran dry */
  /* host tier (cl_engine_set_prefix_host_cache); pages dropped from it = pages_to_host - pages_from_host - host_pages_cached */
  int64_t host_pages;        /* capacity in pages (0: off) */
  int64_t host_pages_cached; /* now: host pages holding an evicted page that stays indexed */
  int64_t pages_to_host;     /* evicted pages copied to the host tier (spills) */
  int64_t pages_from_host;   /* of which copied back to HBM because a sequence attached them (fills) */
} cl_prefix_stats;

/* Speculative decoding accounting since engine creation (cl_engine_config.speculate). */
typedef struct cl_spec_stats {
  int32_t enabled;           /* the scheduler and the synchronous path speculate */
  int32_t max_draft;         /* most drafted tokens per verify pass */
  int64_t verify_passes;     /* sequences verified: a pass over n sequences counts n (cl_decode_verify[_batch] calls included) */
  int64_t tokens_drafted;    /* drafted tokens they checked */
  int64_t tokens_accepted;   /* of which accepted */
  int64_t tokens_emitted;    /* tokens they emitted: tokens_accepted + verify_passes */
  int64_t multi_passes;      /* passes that verified two or more sequences at once (cl_engine_set_speculate_batch) */
  /* draft model (cl_engine_create_with_draft; all zero without one) */
  int64_t draft_rows;        /* rows the draft computed: catch-up rows of its prefill passes plus its decode steps */
  int64_t draft_ns;          /* host wall time inside draft calls (cl_draft_model and the scheduler's rounds) */
  int64_t draft_pages_used;  /* now: pages of the draft's KV pool that mirrors hold */
} cl_spec_stats;

typedef struct cl_engine cl_engine;
typedef int32_t cl_seq_t;

/* ---- lifecycle -------------------------------------------------------------------------- */
int cl_abi_version(void);
const char* cl_strerror(int status);
/* thread-local description of the last failing call on this thread ("" if none) */
const char* cl_last_error(void);
void cl_default_engine_config(cl_engine_config* cfg);
void cl_default_sampling(cl_sampling* s);        /* Ollama defaults listed above */
void cl_greedy_sampling(cl_sampling* s, int32_t max_new_tokens);
/* The engine's host-side sampler on caller-provided logits (no GPU involved): repeat penalty over the last repeat_last_n
 * ids of `history` -> top-k -> softmax at `temperature` -> top-p -> one draw from the counter-based generator at
 * (seed, step).  Exposed so that each stage can be checked against an independent implementation
 * (tests/test_host_logic.py pins it to the HF transformers logits processors). */
int cl_sample_token(const float* logits, int32_t vocab, const cl_sampling* s, const int32_t* history, int32_t n_history,
                    uint64_t step, int32_t* id);
/* cl_sample_token with the stages of cl_sampling_ext (ext may be NULL: all zero; its stop strings are ignored). */
int cl_sample_token_ext(const float* logits, int32_t vocab, const cl_sampling* s, const cl_sampling_ext* ext, const int32_t* history,
                        int32_t n_history, uint64_t step, int32_t* id);
int cl_model_preset(const char* name, cl_model_config* out);
/* Host only (no GPU needed): the model config cl_engine_create derives from cfg — the preset, the model directory's
 * config.json or cfg->model — with the served window of cfg->context_length (and CL_CONTEXT_LENGTH) in max_seq_len, and
 * the same checks: CL_ERR_INVALID_ARG for a window it refuses or a num_keep that leaves no room to shift (context_shift on),
 * CL_ERR_UNKNOWN_MODEL / CL_ERR_IO as cl_engine_create.  cl_checkpoint_info keeps the default window. */
int cl_resolve_model_config(const cl_engine_config* cfg, cl_model_config* out);
/* The prompt-lookup drafter of speculative decoding (host only, no GPU involved): the longest suffix of hist[0..n) of
 * length 3, else 2, that also occurs earlier in hist; from its most recent earlier occurrence, the up to k ids that
 * followed it, stopping at the end of hist, go to out.  *n_out = their count (0: no match).  k: 1..15. */
int cl_draft_ngram(const int32_t* hist, int32_t n, int32_t k, int32_t* out, int32_t* n_out);

/* replaces: embedded Ollama server start, /root/reference/cmd/crowdllama/main.go:283-297 */
int cl_engine_create(const cl_engine_config* cfg, cl_engine** out);
/* cl_engine_create with a draft model for speculative decoding: a small model of the same vocabulary drafts, the served
 * model verifies the drafts in one pass (cl_engine_config.speculate), in place of the prompt-lookup drafter.  Only
 * draft->preset / model / weights_path / weights_seed are read; the draft runs on the target's device with the target's
 * page size and window (max_seq_len), a KV pool of as many tokens as the target's, no scheduler, no prefix cache and no
 * speculation of its own.  Every emitted id stays the served model's own greedy choice or seeded draw, so output does not
 * depend on the draft; only how many ids a pass accepts does.
 *   - Memory: with context_length > 0 and kv_pool_bytes == 0, both weight sets come off the free memory first, and the rest
 *     (less the 4 GiB reserve) is split in proportion to KV bytes per token, so the target's pool is smaller than it would be
 *     alone: 128 KiB against 32 KiB per token for Llama-3-8B with Llama-3.2-1B leaves the target 4/5 of it.  Otherwise the
 *     target's pool is what it would be alone, and the draft's pool takes as many tokens on top.
 *   - Drafting: each target sequence that drafts has a mirror sequence in the draft, freed with it.  A round gives the
 *     mirror the window ending with the next input x0; the mirror keeps the longest common prefix of what it holds and that
 *     window before x0, prefills the rest in one pass (1 or 2 rows after an accepted round; the whole window on first use or
 *     after a context shift or preemption), and takes k - 1 steps.  A greedy request drafts the draft's argmax; a
 *     device-sampled one draws with its own settings, penalty history and RNG step, so draft row i uses the same
 *     (seed, step) as verify row i.  A sequence whose mirror gets no pages from the draft pool drafts nothing that round.
 * CL_ERR_INVALID_ARG, with cl_last_error set, when the vocabularies differ, both models have a tokenizer.json and their
 * bos / eos / stop ids differ, the target shape has no verify pass, speculate is 0, or the draft cannot serve the target's
 * window; otherwise the errors of cl_engine_create.  cl_engine_create itself takes a draft from env CL_DRAFT_MODEL (a preset
 * name or a model directory) with the synthetic-weight seed CL_DRAFT_SEED (default: the target's weights_seed). */
int cl_engine_create_with_draft(const cl_engine_config* cfg, const cl_engine_config* draft, cl_engine** out);
void cl_engine_destroy(cl_engine* e);
int cl_engine_model_config(const cl_engine* e, cl_model_config* out);
int cl_engine_stats(cl_engine* e, cl_stats* out);
int cl_engine_prefix_stats(cl_engine* e, cl_prefix_stats* out);
int cl_engine_spec_stats(cl_engine* e, cl_spec_stats* out);
/* How many running requests the scheduler may verify in one pass (speculative decoding, cl_engine_config.speculate > 0).
 * n = 1 (the default): a request speculates only while it runs alone.  n >= 2: while 2 .. n requests are running, nothing
 * waits or is being prefilled, every one of them is greedy or device-sampled and at least one has a draft, each drafts as
 * it would alone and one pass over the weights verifies all of them (cl_decode_verify_batch); otherwise they take batched
 * steps.  n: 1 .. min(max_batch, 32), else CL_ERR_INVALID_ARG.  Env CL_SPECULATE_BATCH sets it at cl_engine_create (an
 * invalid value makes the create fail with CL_ERR_INVALID_ARG). */
int cl_engine_set_speculate_batch(cl_engine* e, int32_t n);
/* Host tier of the prefix cache: `bytes` of pinned, mapped host memory (rounded down to whole pages; a page holds one pool
 * page's K and V of every layer) behind the HBM page pool.  A cached page the pool evicts is copied there and stays
 * indexed instead of being forgotten (the least recently evicted one is dropped when the tier is full), and a sequence
 * whose prompt reaches it copies it back into a free pool page instead of prefilling it again.  Reuse stays bit-identical:
 * a restored page holds the bytes that were evicted.  Off by default; 0 frees the tier.  Copies run on the engine's
 * stream inside the calls that reserve or attach pages (cl_seq_attach_prefix, prefill, decode, request admission).
 * CL_ERR_INVALID_ARG while any sequence is live or a request is queued, with the prefix cache off, for bytes < 0 and
 * for 0 < bytes < one page; CL_ERR_OOM when the memory cannot be pinned (the tier is then off).  Env
 * CL_PREFIX_CACHE_HOST_MIB sets it at cl_engine_create (a failure there makes the create fail with that status). */
int cl_engine_set_prefix_host_cache(cl_engine* e, int64_t bytes);
/* Overwrite one weight tensor from host memory (bf16 bits, logical [out][in] row-major; norm
 * gains as bf16 too).  kind: 0 embed, 1 lm_head, 2 final_norm, 3 attn_norm, 4 wq, 5 wk, 6 wv,
 * 7 wo, 8 ffn_norm, 9 w_gate, 10 w_up, 11 w_down (same numbering as the synthetic generator).
 * Used to load real checkpoints tensor by tensor and by the HF golden-vector parity tests. */
int cl_engine_set_tensor(cl_engine* e, int32_t layer, int32_t kind, const uint16_t* data, int64_t n);

/* Host-only check of a checkpoint (no GPU needed): parses config.json (when cfg_io->n_layers == 0 and path is a model
 * directory; the result is written back) and every safetensors header, validating tensor names, dtypes, shapes and
 * offsets against the architecture exactly as cl_engine_create does.  n_tensors / n_params (may be NULL): what the
 * engine would load. */
int cl_checkpoint_info(const char* path, cl_model_config* cfg_io, int32_t* n_tensors, int64_t* n_params);

/* ---- request level (what the Go shim calls) --------------------------------------------- */
/* replaces: callOllamaAPI, api.go:108-160.  Blocking; enqueues into the continuous-batching
 * scheduler.  `model` must equal the engine's model_name (else CL_ERR_UNKNOWN_MODEL).  The
 * prompt is raw user text (api.go:111-116 forces role "user"); it is copied before return. */
int cl_generate(cl_engine* e, const char* model, const char* prompt, size_t prompt_len,
                const cl_sampling* s, cl_result* out);
/* token-id variant of the same path (tokenizer bypass; used by parity tests and bench.py) */
int cl_generate_ids(cl_engine* e, const int32_t* prompt_ids, int32_t n_prompt,
                    const cl_sampling* s, cl_result* out);
void cl_result_free(cl_result* r);

/* Streaming variant of cl_generate (SURVEY.md §8f row 4; the reference rejects stream:true, api.go:155).
 * cb runs on the CALLING thread (cgo-safe) with each batch of new tokens: text = UTF-8 delta that later tokens
 * cannot change (an incomplete multi-byte tail is held back), ids/n_ids = the new token ids (NULL/0 for the final
 * flush).  A nonzero return cancels the request (done_reason "cancelled").  out receives the whole result. */
typedef int (*cl_token_cb)(void* user, const char* text, size_t text_len, const int32_t* ids, int32_t n_ids);
int cl_generate_stream(cl_engine* e, const char* model, const char* prompt, size_t prompt_len,
                       const cl_sampling* s, cl_token_cb cb, void* user, cl_result* out);
/* Byte-level streaming handler: like cl_handle_message, but when GenerateRequest.stream is set the answer is a
 * sequence of serialised BaseMessage{GenerateResponse} frames — Done=false frames carrying text deltas, then one
 * Done=true frame with done_reason — each handed to cb (the host writes them length-prefixed to the stream,
 * pbwire.go:14-33).  Without stream: exactly one Done=true frame.  GenerateRequest.options (field 4, the proto
 * extension of §8f row 3: seed, temperature, top_k, top_p, repeat_penalty, repeat_last_n, num_predict, raw, and
 * stop, min_p, presence_penalty, frequency_penalty as in cl_sampling_ext) override `s` field by field in both entry points. */
typedef int (*cl_frame_cb)(void* user, const uint8_t* msg, size_t len);
int cl_handle_message_stream(cl_engine* e, const uint8_t* req, size_t req_len, const cl_sampling* s,
                             cl_frame_cb cb, void* user);
/* replaces: WorkerAPIHandler, api.go:45-96, at the byte level.  `req`/`req_len` is a serialised
 * llama.v1.BaseMessage (the payload pbwire.go:14-41 length-prefixes); on success *resp is a
 * malloc'd serialised BaseMessage{GenerateResponse} (free with cl_buffer_free).  A request that
 * is not a GenerateRequest returns CL_ERR_BAD_MESSAGE (api.go:48-51). */
int cl_handle_message(cl_engine* e, const uint8_t* req, size_t req_len, const cl_sampling* s,
                      uint8_t** resp, size_t* resp_len);
void cl_buffer_free(void* p);

/* tokenizer of the served model (byte-level fallback when no vocab file is configured) */
int cl_tokenize(cl_engine* e, const char* text, size_t len, int32_t* ids, int32_t cap, int32_t* n_out);
int cl_detokenize(cl_engine* e, const int32_t* ids, int32_t n, char* buf, size_t cap, size_t* len_out);

/* ---- token level (parity tests, benchmarks) --------------------------------------------- */
int cl_seq_create(cl_engine* e, cl_seq_t* out);
int cl_seq_free(cl_engine* e, cl_seq_t seq);
int cl_seq_len(cl_engine* e, cl_seq_t seq, int32_t* len_out);
/* Prefix cache, token level: on a new sequence (length 0), take the cached K/V of the longest page-aligned prefix of
 * ids[0..n) that an earlier sequence computed, at most n - 1 tokens (the last position is always computed, so the
 * caller gets its logits).  *n_reused = the sequence's length afterwards; the caller then cl_prefills ids[n_reused..n).
 * Shared pages are read-only: every later write lands at positions >= the sequence's length, on pages of its own.
 * With the cache off *n_reused = 0 and nothing changes. */
int cl_seq_attach_prefix(cl_engine* e, cl_seq_t seq, const int32_t* ids, int32_t n, int32_t* n_reused);
/* Append n prompt tokens to the sequence.  logits_out (host, may be NULL) receives the
 * vocab_size fp32 logits of the LAST position. */
int cl_prefill(cl_engine* e, cl_seq_t seq, const int32_t* ids, int32_t n, float* logits_out);
/* The prompts of n_seqs sequences in ONE pass of the tensor-core path (the scheduler's admission of a burst of short
 * chats): ids = the prompts back to back, lens[i] tokens for seqs[i]; at most 4096 rows in total and n_seqs <= max_batch.
 * logits_out (host, may be NULL): [n_seqs][vocab_size] logits of every prompt's last position.  Results are
 * bit-identical to cl_prefill on each prompt alone through the same (tile) path. */
int cl_prefill_batch(cl_engine* e, const cl_seq_t* seqs, int32_t n_seqs, const int32_t* ids, const int32_t* lens, float* logits_out);
/* Append one token and compute the next-token logits (host, may be NULL);
 * argmax_out (may be NULL) receives the greedy next id (lowest index on ties). */
int cl_decode_step(cl_engine* e, cl_seq_t seq, int32_t id, float* logits_out, int32_t* argmax_out);
/* Run n_steps greedy decode steps entirely on the device (each step feeds its argmax to the
 * next); ids_out receives the n_steps generated ids.  device_ms (may be NULL) receives the
 * CUDA-event time of the loop.  This is the timed region of bench.py's `value`. */
int cl_decode_greedy(cl_engine* e, cl_seq_t seq, int32_t first_id, int32_t n_steps,
                     int32_t* ids_out, float* device_ms);
/* Batched greedy decode: n_seqs sequences advance together for n_steps (continuous-batching
 * inner loop without the scheduler).  first_ids[n_seqs]; ids_out[n_steps * n_seqs]. */
int cl_decode_greedy_batch(cl_engine* e, const cl_seq_t* seqs, int32_t n_seqs,
                           const int32_t* first_ids, int32_t n_steps, int32_t* ids_out,
                           float* device_ms);
/* cl_decode_greedy_batch with the device sampler: sequence b draws with sp[b] (temperature <= 0: greedy argmax, so greedy
 * and sampled sequences may share the batch); draw i of sequence b uses RNG step step0[b] + i (step0 may be NULL: 0)
 * and the repeat-penalty window of the sequence's history plus the tokens fed.  The ids are the ones cl_sample_token
 * draws on the logits of cl_decode_step_batch fed the same tokens.  CL_ERR_INVALID_ARG if some sp[b] needs the host
 * sampler (see cl_sampling).  Kernel launches per step are those of cl_decode_greedy_batch. */
int cl_decode_sample_batch(cl_engine* e, const cl_seq_t* seqs, int32_t n_seqs, const int32_t* first_ids,
                           const cl_sampling* sp, const uint64_t* step0, int32_t n_steps, int32_t* ids_out,
                           float* device_ms);
/* One batched decode step with caller-chosen input tokens (teacher forcing for the parity tests of the batched
 * path): ids[n_seqs]; logits_out (host, may be NULL) receives [n_seqs][vocab_size] fp32; argmax_out (may be NULL)
 * the greedy next ids. */
int cl_decode_step_batch(cl_engine* e, const cl_seq_t* seqs, int32_t n_seqs, const int32_t* ids, float* logits_out,
                         int32_t* argmax_out);
/* Speculative decoding, token level: one verify pass.  The sequence has len cached tokens and the next input input_id
 * (x0: the last generated id, not cached yet); draft[0..k) = d1 .. dk, 1 <= k <= 15, are the guessed ids after it.
 *   - The pass runs x0, d1 .. dk at positions len .. len + k through every layer (their K/V are written) and computes the
 *     logits of all k + 1 rows.  Row r makes the decode step tail's choice y_{r+1}: greedy argmax (lowest index on ties),
 *     or with a sampled sp the draw of cl_sample_token with history = the sequence's history + x0, d1 .. dr and RNG step
 *     step0 + r.
 *   - a = the largest count with y_j == d_j for every j <= a.  ids_out receives y_1 .. y_{a+1}, *n_out = a + 1.
 *   - Afterwards len += a + 1 (x0, d1 .. da are cached) and the next input is y_{a+1}: exactly the state a + 1
 *     cl_decode_step calls would leave, so the ids equal sequential decoding's up to logit differences between the two
 *     kernel paths (near-tie flips).  K/V of rejected rows lies at positions >= the new length: nothing reads it, the
 *     next writes overwrite it, and pages attached from the prefix cache are never written.
 * sp may be NULL, or have temperature <= 0, for greedy; a sampled sp arms the device sampler for the pass and disarms it
 * afterwards, like cl_decode_sample_batch.  logits_out (host, may be NULL): [k + 1][vocab_size].  Works whatever
 * cl_engine_config.speculate is.  CL_ERR_INVALID_ARG for k outside 1..15, settings that need the host sampler, or a
 * model shape without the verify path; CL_ERR_TOO_LONG past max_seq_len. */
int cl_decode_verify(cl_engine* e, cl_seq_t seq, int32_t input_id, const int32_t* draft, int32_t k, const cl_sampling* sp,
                     uint64_t step0, int32_t* ids_out, int32_t* n_out, float* logits_out);
/* Speculative decoding, token level: one verify pass over n_seqs distinct sequences, so that one pass over the weights
 * checks the drafts of all of them.  Sequence seqs[i] has the contract of cl_decode_verify with input_ids[i], its ks[i]
 * drafts (0 <= ks[i] <= 15; the drafts of all sequences back to back in `drafts`), sp[i] and step0[i] (sp and step0 may be
 * NULL: greedy, step 0).  ks[i] = 0 is allowed: the sequence then advances by exactly the one id a decode step would choose.
 * Its rows are r0_i .. r0_i + ks[i], r0_i = the sum of ks[j] + 1 over j < i, at most 128 rows in all:
 *   - ids_out [rows]: the emitted ids of sequence i start at ids_out + r0_i; n_out[i] = their count (a_i + 1).
 *   - logits_out (host, may be NULL): [rows][vocab_size].
 * Each sequence's ids, logits and K/V are those of the same call with that sequence alone.  CL_ERR_INVALID_ARG for a
 * duplicate sequence, k outside 0..15, more than 128 rows, an id out of range, settings that need the host sampler or a
 * model shape without the verify path; CL_ERR_TOO_LONG if a sequence would pass max_seq_len.  On an error no sequence's
 * length changes. */
int cl_decode_verify_batch(cl_engine* e, const cl_seq_t* seqs, int32_t n_seqs, const int32_t* input_ids, const int32_t* drafts,
                           const int32_t* ks, const cl_sampling* sp, const uint64_t* step0, int32_t* ids_out, int32_t* n_out,
                           float* logits_out);
/* Speculative decoding, token level: the draft model's drafter (cl_engine_create_with_draft), the counterpart of
 * cl_draft_ngram.  For each i < n_seqs, the mirror of target sequence seqs[i] (a live handle; its own K/V are not touched)
 * catches up with hists[i][0..hist_lens[i]), the window whose last id is the next input x0, and drafts ks[i] ids (0..15)
 * after it: one prefill pass over the catch-up rows of every sequence (its tail chooses d1; several sequences share one
 * tile-path pass when their rows fit it), then max(ks) - 1 batched draft steps for the sequences with ks[i] >= 2.  Draft row
 * j of sequence i is the draft's greedy argmax, or with a sampled sp[i] the draft's device draw at RNG step step0[i] + j
 * with the window (plus d1 .. dj) as its penalty history; sp and step0 may be NULL (greedy, step 0).  The ids of sequence i
 * land back to back in `drafts` after those of the sequences before it (sum of ks[j], j < i); n_drafts[i] = ks[i], 1 when its
 * window (or the draft pool) leaves no room for the max(ks) - 1 steps, or 0 when the draft pool has no pages for that
 * mirror.  Afterwards the mirror holds the window plus the drafts it fed (hist_lens[i] + max(ks) - 1 tokens when it took
 * the steps).  CL_ERR_INVALID_ARG without a draft model, for a duplicate sequence, k
 * outside 0..15, an empty window, an id out of range or settings that need the host sampler; CL_ERR_TOO_LONG past max_seq_len. */
int cl_draft_model(cl_engine* e, const cl_seq_t* seqs, int32_t n_seqs, const int32_t* const* hists, const int32_t* hist_lens,
                   const int32_t* ks, const cl_sampling* sp, const uint64_t* step0, int32_t* drafts, int32_t* n_drafts);

/* Context shift, token level: the cached tokens [n_keep, n_keep + n_discard) of the sequence leave its cache.  Afterwards:
 *   - position p < n_keep holds exactly what it held;
 *   - position p >= n_keep holds what position p + n_discard held: V bit-identical, K = bf16(R(-n_discard) K_old), rotated
 *     in fp32 (a c + b s, b c - a s, each product and sum rounded, for the pair of dims j and j + head_dim/2) with row
 *     n_discard of the engine's own cos/sin table, the one prefill and decode use ("llama3" scaling included);
 *   - len and the slot's device position drop by n_discard.  The next input id, the id history, an armed sampler's RNG step
 *     and penalty window, and logprobs are unchanged.
 * The kept K/V were computed with the discarded tokens in view: they are not what a prefill of the kept ids would give.
 * Pages the shift writes that another sequence or the prefix cache holds are copied first (copy-on-write), so neither ever
 * sees a shifted row; the sequence publishes no page to the prefix cache afterwards.  Works whatever
 * cl_engine_config.context_shift is.  CL_ERR_INVALID_ARG unless n_discard is a positive multiple of page_size and
 * 0 <= n_keep, n_keep + n_discard <= len; CL_ERR_OOM when a copy-on-write finds no free page.  On these errors nothing
 * changes.  CL_ERR_CUDA (a failed copy or launch after the page list was rewritten) leaves the sequence's pages and K/V
 * undefined, like any CUDA failure: free the sequence. */
int cl_seq_shift(cl_engine* e, cl_seq_t seq, int32_t n_keep, int32_t n_discard);

/* ---- per-token log-probabilities (Ollama's `logprobs` / `top_logprobs`) -----------------------------------------------
 * What is computed: the natural-log log_softmax of the logits row the step tail chose the id from, taken over the raw fp32
 * logits, i.e. BEFORE the repeat penalty, temperature, top-k and top-p: the model's distribution, whatever the sampler
 * then does with it.  (Which distribution Ollama reports could not be pinned against its source; this is the choice.)
 * The step tail kernel computes it on the device: lse = M + log(sum_b s_b exp(m_b - M)) over its 64 vocabulary slices
 * (slice max m_b, slice sum s_b of expf(v - m_b); the merge in double, in fixed slice order), logprob(id) = logit[id] - lse
 * in double rounded to fp32, and the top n_top ids by logit (value descending, id ascending, the greedy tie rule).  A record depends on its
 * logits row alone: it is the same bits run to run, whatever other sequences share the step, and whether the id was
 * chosen greedily or drawn.  A sequence without logprobs runs exactly the step tail it ran before. */
#define CL_MAX_TOP_LOGPROBS 20
typedef struct cl_token_logprob {  /* 172 bytes */
  int32_t id;          /* the chosen id */
  float logprob;       /* its log-probability (<= 0) */
  int32_t n_top;       /* entries of top_ids / top_logprobs in use */
  int32_t top_ids[CL_MAX_TOP_LOGPROBS];
  float top_logprobs[CL_MAX_TOP_LOGPROBS];
} cl_token_logprob;
/* top_n -1: off (the default of a new sequence; cl_seq_free disarms too), 0..20: every later id the step tail chooses for
 * the sequence leaves a record with top_n alternatives.  Pending records are dropped.  CL_ERR_INVALID_ARG for top_n outside
 * -1..20, and for arming a model whose vocabulary exceeds 163 840 (64 slices of 2 560, the device sampler's limit). */
int cl_seq_set_logprobs(cl_engine* e, cl_seq_t seq, int32_t top_n);
/* The records of the ids the step tail chose for the sequence since the last take, in order: one per id chosen by
 * cl_prefill (its last token), cl_prefill_batch, cl_decode_step[_batch], cl_decode_greedy[_batch], cl_decode_sample_batch
 * and cl_decode_verify[_batch] (the emitted ids).  Up to cap records go to out and are removed; *n_out = how many.
 * out == NULL: *n_out = the count pending, nothing is removed. */
int cl_seq_take_logprobs(cl_engine* e, cl_seq_t seq, cl_token_logprob* out, int32_t cap, int32_t* n_out);
/* Arms the sequence with min_p and the presence / frequency penalties of ext (NULL: all zero; stop strings are ignored):
 * every later token-level call that draws for it with a cl_sampling (cl_decode_sample_batch, cl_decode_verify[_batch])
 * applies them too, on the device, and so does the prefill tail of an armed sampler.  cl_seq_create / cl_seq_free reset
 * it to all zero.  CL_ERR_INVALID_ARG as cl_sampling_ext states. */
int cl_seq_set_sampling_ext(cl_engine* e, cl_seq_t seq, const cl_sampling_ext* ext);
/* cl_generate_ids with logprobs on (top_n 0..20): *lps (malloc'd, free with cl_buffer_free) = one record per generated id,
 * out->n_generated of them.  The ids equal those of the same request through cl_generate_ids.  A host-sampled request
 * (settings the device sampler does not cover) takes lse and the top list from the device and sets logprob = logit[id] - lse
 * with the same double subtraction and fp32 rounding. */
int cl_generate_ids_logprobs(cl_engine* e, const int32_t* prompt_ids, int32_t n_prompt, const cl_sampling* s, int32_t top_n,
                             cl_result* out, cl_token_logprob** lps);
/* cl_generate_ids with Ollama's remaining options: ext (may be NULL: all zero) adds min_p, the presence / frequency penalties
 * and stop strings (cl_sampling_ext); top_n -1 = logprobs off, 0..20 = on as cl_generate_ids_logprobs (*lps then one record
 * per generated id; lps may be NULL with top_n -1); cb (may be NULL) streams text deltas as cl_generate_stream does, the
 * last flush with ids NULL.  With an all-zero ext the ids are those of cl_generate_ids. */
int cl_generate_ids_ext(cl_engine* e, const int32_t* prompt_ids, int32_t n_prompt, const cl_sampling* s, const cl_sampling_ext* ext,
                        int32_t top_n, cl_token_cb cb, void* user, cl_result* out, cl_token_logprob** lps);
/* Parity aid: make the sequence hold n_tokens cached tokens whose K/V, in every layer, are the CPU oracle's
 * synthetic cache pattern (oracle/llama_oracle.c oc_seq_fake_fill: k[i] = (((i * 2654435761) >> 24 & 255) - 128) / 128,
 * v[i] = (((i * 40503) >> 8 & 255) - 128) / 128 with i = token * n_kv * head_dim + head * head_dim + dim; exact in
 * bf16).  Lets the long-context decode kernels be compared with the oracle without a long CPU prefill. */
int cl_seq_fake_fill(cl_engine* e, cl_seq_t seq, int32_t n_tokens);
/* Parity aid: cached K (which = 0) / V (which = 1) rows of `layer`, tokens t0..t0+n-1 of the sequence, gathered from
 * the paged pool: out[n][n_kv_heads*head_dim] fp32 (the bf16 cache values).  Checks EVERY position of a long prefill.
 * which = 2 (K) / 3 (V) read up to the end of the pages the sequence holds rather than its length: there a verify pass
 * (cl_decode_verify*) leaves the K/V of its rejected rows.  Those rows are valid only until the sequence's next pass or
 * step, which writes the same positions.  CL_ERR_INVALID_ARG for another `which` or a range past that end. */
int cl_debug_kv(cl_engine* e, cl_seq_t seq, int32_t layer, int32_t which, int32_t t0, int32_t n, float* out);
/* bench.py's roofline.dominant_kernel: n_steps greedy single-sequence steps launched eagerly with a CUDA-event pair
 * (on the launching stream) around the step's dominant kernel — decode_mega_kernel, or the per-layer kernel stack
 * on the per-op path.  kernel_ms / step_ms (may be NULL): mean per step.  CL_ERR_INVALID_ARG in deterministic mode,
 * whose steps run neither. */
int cl_time_dominant_kernel(cl_engine* e, cl_seq_t seq, int32_t first_id, int32_t n_steps, float* kernel_ms, float* step_ms);
/* debugging / parity: copy the residual stream after `layer` (or the final norm input when
 * layer == n_layers) of the most recent single-sequence step to host (d_model floats). */
int cl_debug_hidden(cl_engine* e, float* out, int32_t n);
/* The same buffers for any live sequence, after the latest decode step (single or batched) that contained it; the stream is
 * synchronised first.  what: 0 = the residual stream after the last layer (d_model floats); 1 = the last layer's roped q
 * (n_heads * head_dim); 2 = its attention output, fp32 (n_heads * head_dim); 3 = its SwiGLU activation as a single-sequence
 * step leaves it (d_ff; a batched step does not write this buffer).  After a step over two or more sequences, until the next
 * such step or multi-prompt prefill: 4 = the bf16 attention row the o-projection GEMM read, 5 = the bf16 activation row
 * the down-projection GEMM read (as floats).  n must be the buffer's element count.  *mega_out (may be NULL): 1 when this
 * engine's single-sequence steps run decode_mega_kernel, 0 when they run the per-op kernels (the shape, CL_MEGA=0 or the
 * device ruled the persistent kernel out); out == NULL with n == 0 reports only that.  cl_debug_hidden(out, n) is this call
 * on the sequence of the most recent single-sequence step.  CL_ERR_INVALID_ARG for a wrong n or `what`, and for 4 / 5 when
 * the sequence was not in the latest batched step. */
int cl_debug_seq_hidden(cl_engine* e, cl_seq_t seq, int32_t what, float* out, int32_t n, int32_t* mega_out);
/* Parity aid: the latest multi-row pass — a split-K pass (prompts of 16 .. 256 tokens, every cl_decode_verify /
 * cl_decode_verify_batch) or a tile-path pass (longer prompts, one per chunk; cl_prefill_batch).  info[4] = {path (0 split-K,
 * 1 tile), attention kernel (0 mma.sync prefill, 1 wgmma prefill, 2 multi-row verify, 3 segments with different prefill
 * kernels, 4 split-KV wgmma prefill: segments of more than 16 rows that end past 32768 tokens; up to 16 rows run the
 * multi-row verify kernel there, 2), T (rows), n_segs}; segs[min(n_segs, max_segs)][4] = {sequence, first row, rows, position of the first row}.  A
 * prefill longer than one chunk leaves its last chunk's pass.  CL_ERR_INVALID_ARG when no pass is recorded: none yet, or a
 * token-wise prefill (fewer than 16 tokens) or a failed pass since. */
int cl_debug_pass_info(cl_engine* e, int32_t* info, int32_t* segs, int32_t max_segs);
/* Rows row0 .. row0+n-1 of that pass's workspace after its last layer, as fp32; the stream is synchronised first.  what:
 * 0 = the fp32 residual stream (d_model; for a split-K pass after its final fold), 1 = roped q (n_heads * head_dim, bf16),
 * 2 = attention output (n_heads * head_dim, bf16), 3 = SwiGLU activation (d_ff, bf16).  Valid until the next pass.
 * CL_ERR_INVALID_ARG for a wrong `what`, a range outside 0 .. T - 1, or no recorded pass (cl_debug_pass_info). */
int cl_debug_pass_rows(cl_engine* e, int32_t what, int32_t row0, int32_t n, float* out);
/* profiling aid (engine created with env CL_TIMELINE=1): %globaltimer stamps [node][4] = {CTA start,
 * dependency satisfied, inputs loaded / pages consumed, outputs written} of CTA 0 of every kernel node of
 * the most recent token step; nodes = n_layers * {qkv, attn, o, gate|up, down} + lm_head.  Returns the
 * number of int64 values written (or a negative status). */
int cl_debug_timeline(cl_engine* e, int64_t* out, int32_t n);

/* ---- single-op entry points (host buffers in/out; kernel parity tests and microbenches) --
 * Each runs exactly the CUDA kernel the token step uses.  bf16 data is passed as uint16_t.
 * `variant`: 0 = generic LDG kernel, 1 = TMA-ring streaming kernel.  iters>0 => repeat and
 * report the average device time (ms) through *ms (may be NULL). */
int cl_op_gemv(int device, int variant, const uint16_t* w, const float* x, float* y,
               int32_t n_rows, int32_t k, int32_t iters, float* ms);
/* y = resid + W x */
int cl_op_gemv_residual(int device, int variant, const uint16_t* w, const float* x,
                        const float* resid, float* y, int32_t n_rows, int32_t k);
/* xn = bf16round(rmsnorm(h) * gain); y = W xn (norm fused in the GEMV prologue) */
int cl_op_rmsnorm_gemv(int device, int variant, const uint16_t* w, const float* h,
                       const float* gain, float eps, float* y, int32_t n_rows, int32_t k);
/* w_gu interleaved rows (2i = gate_i, 2i+1 = up_i); act_i = bf16round(silu(g_i) * u_i) */
int cl_op_rmsnorm_gateup(int device, int variant, const uint16_t* w_gu, const float* h,
                         const float* gain, float eps, float* act, int32_t d_ff, int32_t k);
/* fused q|k|v projection of ONE token, exactly as the token step runs it: xn = bf16(rmsnorm(h)*gain);
 * [q|k|v] = W xn (w_qkv: logical rows q | k | v in natural dim order; the wrapper applies the engine's
 * rope-pair row interleave); RoPE at `pos`; bf16 rounding.  q_out [n_heads*head_dim] fp32 (roped),
 * k_out / v_out [n_kv*head_dim] bf16 as appended to the paged cache. */
int cl_op_qkv_rope_append(int device, int variant, const uint16_t* w_qkv, const float* h, const float* gain,
                          float eps, int32_t d_model, int32_t n_heads, int32_t n_kv, int32_t head_dim,
                          int32_t pos, float rope_theta, float* q_out, uint16_t* k_out, uint16_t* v_out);
/* paged GQA decode attention for one sequence: q [n_heads*head_dim] fp32 (roped, bf16-rounded);
 * k_cache/v_cache [ctx_len][n_kv][head_dim] bf16 = tokens 0..ctx_len-1 (the current token included);
 * out [n_heads*head_dim] bf16-rounded fp32.  The wrapper scatters the cache into scrambled pages. */
int cl_op_attn_decode(int device, const float* q, const uint16_t* k_cache, const uint16_t* v_cache,
                      int32_t ctx_len, int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size,
                      float* out);
/* decode attention of the batched step for `batch` sequences at once.  q [batch][n_heads*head_dim] fp32; k_cache/v_cache
 * [sum of ctx_lens][n_kv][head_dim] bf16 = the sequences' tokens back to back (each one's current token last); slots[batch]
 * (NULL: 0..batch-1) distinct and < n_slots; out [n_slots][n_heads*head_dim] fp32 is read and written: rows of the slots
 * outside the batch come back unchanged; out_bf16 [batch][n_heads*head_dim] (may be NULL) = the bf16 copy the o-projection
 * reads.  variant 0: CUDA-core kernel (decode_kernels.cu), 1: tensor-core kernel (attn_decode_tc.cu), -1: the step's choice.
 * nsplit 0 / tc_small -1: the step's plan (attn_decode_tc_plan); other values are used as given.  *nsplit_used and
 * *tc_small_used (-1: the CUDA-core kernel ran) report what ran.  The kernel runs twice without resetting its split counters;
 * CL_ERR_INTERNAL when the two outputs differ in any bit. */
int cl_op_attn_decode_batch(int device, int variant, int32_t nsplit, int32_t tc_small, const float* q, const uint16_t* k_cache,
                            const uint16_t* v_cache, const int32_t* ctx_lens, const int32_t* slots, int32_t batch, int32_t n_slots,
                            int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, float* out, uint16_t* out_bf16,
                            int32_t* nsplit_used, int32_t* tc_small_used);
/* The multi-row split-KV attention of a verify pass over several sequences (cl_decode_verify_batch): segment s has
 * ctx_lens[s] cached tokens and rows[s] (1..16) new query rows at positions ctx_lens[s] .. ctx_lens[s] + rows[s] - 1; row r
 * sees keys < ctx_lens[s] + r + 1.  q [sum(rows)][n_heads * head_dim] bf16 (roped), the segments' rows back to back;
 * k/v caches [sum(ctx_lens + rows)][n_kv][head_dim] bf16, the segments back to back, paged by the engine's rules into a
 * scrambled pool.  out [sum(rows)][n_heads * head_dim] bf16.  nsplit 0: the engine's split plan (every split 8 pages),
 * else every segment spreads its pages over nsplit (1..64) splits; *nsplit_used (may be NULL) = the grid's splits.  The
 * kernel launches twice without re-arming its split counters and the call fails with CL_ERR_INTERNAL if the two outputs
 * differ in any bit.  Shapes: head_dim 128, 4 query heads per kv head, page 32; others return CL_ERR_INVALID_ARG.  Eight or
 * more segments of one row each run the kernel's one-warp instantiation, as the engine's steps do; its rows are the
 * 4-warp kernel's bits. */
int cl_op_attn_verify(int device, const uint16_t* q, const uint16_t* k_cache, const uint16_t* v_cache, const int32_t* ctx_lens,
                      const int32_t* rows, int32_t n_segs, int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t nsplit,
                      uint16_t* out, int32_t* nsplit_used);
/* The host tier's transfer kernels (cl_engine_set_prefix_host_cache): a pool of n_layers layers and 2 n_moves + 2 pages,
 * scattered, in which n_moves pages hold random bits and every other element the largest finite bf16 (+ K, - V).  One
 * kv_spill_kernel launch copies the n_moves pages to pinned, mapped host pages, one kv_fill_kernel launch copies those
 * into the n_moves other pages.  CL_ERR_INTERNAL unless every destination and every host page holds exactly the source's
 * bytes and every other page is unchanged.  iters > 0: ms[0] / ms[1] = CUDA-event time of one spill / fill launch, the
 * mean over iters launches of each.  head_dim 64 or 128, page_size 16, 32 or 64. */
int cl_op_kv_host_roundtrip(int device, int32_t n_layers, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t n_moves,
                            int32_t iters, float* ms);
/* The context shift's kernel (kv_shift_kernel, cl_seq_shift): k, v [n_layers][len][n_kv][head_dim] bf16 are the rows of a
 * sequence paged into a scattered pool whose other pages hold the largest finite bf16 (+ K, - V).  The allocator's shift
 * (cl_kvpool_shift, no page shared) plans the work and one launch runs it with rope_row [head_dim / 2][2] (cos, sin) as
 * row n_discard of the RoPE table.  k_out, v_out [n_layers][len - n_discard][n_kv][head_dim] = the sequence's rows
 * afterwards.  CL_ERR_INTERNAL if any element of the pool outside those rows changed.  iters > 0: *ms = CUDA-event time of
 * one launch, the mean over iters more launches of the same work (rotating again).  head_dim 64 or 128, page_size 16, 32 or
 * 64; the cl_seq_shift argument rules otherwise (CL_ERR_INVALID_ARG). */
int cl_op_kv_shift(int device, int32_t n_layers, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t len, int32_t n_keep,
                   int32_t n_discard, const float* rope_row, const uint16_t* k, const uint16_t* v, uint16_t* k_out, uint16_t* v_out,
                   int32_t iters, float* ms);
/* prefill GEMM on the tensor cores (wgmma): Y[t][n] = sum_k X[t][k] W[n][k]; X,W bf16, Y fp32 */
int cl_op_gemm_bf16(int device, const uint16_t* x, const uint16_t* w, float* y, int32_t t,
                    int32_t n, int32_t k, int32_t iters, float* ms);
/* the same GEMM with the epilogues and launches of the engine.  epi 0: y [k_splits][t][n] = the split-K partials (split s
 * sums k-blocks of 64 s*ceil(nkb/k_splits) ..), k_splits 0 = the batched step's count; y == NULL only reports the count.
 * epi 1: y [t][n] = resid + X W^T.  epi 2: act [t][n/2] bf16 = bf16(silu(gate) * up) of interleaved gate|up rows.  Epilogues
 * 1 and 2 run unsplit (k_splits 0 or 1) and epi 2 without PDL.  pdl 1: programmatic dependent launch, as in the batched
 * step.  *k_splits_used (may be NULL) reports the count; CL_ERR_INVALID_ARG for a count the GEMM refuses. */
int cl_op_gemm_bf16_epi(int device, int epi, int32_t k_splits, int pdl, const uint16_t* x, const uint16_t* w, const float* resid,
                        float* y, uint16_t* act, int32_t t, int32_t n, int32_t k, int32_t* k_splits_used);
/* causal prefill attention: q [t][n_heads][d], k,v [t][n_kv][d] bf16 (roped), out bf16-rounded fp32 */
int cl_op_attn_prefill(int device, const uint16_t* q, const uint16_t* k, const uint16_t* v,
                       int32_t t, int32_t n_heads, int32_t n_kv, int32_t head_dim, float* out);
/* the same with the kernel chosen explicitly — variant 0: mma.sync kernel (prefill_kernels.cu, any head_dim 64|128),
 * 1: wgmma kernel (attn_prefill_tc.cu, head_dim 128, up to 10240 tokens), 2: split-KV wgmma kernel (attn_prefill_tc.cu,
 * head_dim 128, page 32, any length; its own split plan), -1: what the engine would pick — and an optional timing loop */
int cl_op_attn_prefill_variant(int device, int variant, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t t,
                               int32_t n_heads, int32_t n_kv, int32_t head_dim, float* out, int32_t iters, float* ms);
/* the same behind a cached prefix: q [t][n_heads][d] for positions pos0 .. pos0+t-1, k,v [pos0+t][n_kv][d]; page_size 16,
 * 32 or 64.  CL_ERR_INVALID_ARG when variant 1 does not take the shape. */
int cl_op_attn_prefill_cached(int device, int variant, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t pos0,
                              int32_t t, int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, float* out);
/* cl_op_attn_prefill_cached with the split count of variant 2 and a timing loop.  nsplit: 0 = the kernel's own plan (what
 * the engine runs), > 0 = that many KV splits per (128-row tile, head), clamped to 1 .. the KV blocks (64 tokens) of the
 * first tile.  *nsplit_used (may be NULL): the splits that ran (1 for variants 0 and 1); *kind_used (may be NULL): the kernel
 * that ran, numbered as cl_debug_pass_info's attention kernels (0 mma.sync, 1 wgmma, 2 multi-row verify, 4 split-KV
 * wgmma), which for variant -1 is the engine's rule: segments that end within 32768 tokens keep the kernels they ran before;
 * past it, up to 16 rows run the multi-row verify kernel (every split over max(8, ceil(pages / 64)) pages) and more rows
 * the split-KV wgmma kernel.  The split kernels launch twice without re-arming their counters and the call fails with
 * CL_ERR_INTERNAL if the two outputs differ in any bit.  iters > 0: *ms = CUDA-event time of one launch over iters launches. */
int cl_op_attn_prefill_long(int device, int variant, const uint16_t* q, const uint16_t* k, const uint16_t* v, int32_t pos0,
                            int32_t t, int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t nsplit,
                            int32_t iters, float* out, float* ms, int32_t* nsplit_used, int32_t* kind_used);
/* Host-only: the split plan of the split-KV prefill attention for t rows from pos0 over n_heads query heads on sms SMs
 * (nsplit as above), and *part_floats (may be NULL) = the fp32 workspace the engine gives it, which bounds every automatic
 * plan's partials (tiles x n_heads x splits x 128 rows x (head_dim + 2)). */
int cl_attn_prefill_long_plan(int32_t pos0, int32_t t, int32_t n_heads, int32_t sms, int32_t nsplit, int32_t* nsplit_used,
                              int64_t* part_floats);
/* Host-only: the split-K count of the projections of the split-K pass and the batched step for an N x K weight on sms SMs
 * (*k_splits), the count cl_op_gemm_bf16_epi's k_splits 0 picks on such a card.  deterministic 1: the count deterministic
 * mode uses, the same for every sms (it is evaluated at 132 SMs, an H100 SXM's). */
int cl_gemm_split_plan(int32_t n, int32_t k, int32_t sms, int32_t deterministic, int32_t* k_splits);
/* the decode step's device sampler (the step tail kernel) on host logits [n_rows][vocab]: row r draws with sp[r] at RNG
 * step step[r], with history row r = history + r * hist_stride, n_history[r] ids (history may be NULL when every
 * n_history[r] is 0).  ids_out[n_rows].  CL_ERR_INVALID_ARG for settings the device sampler does not cover. */
int cl_op_sample(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const int32_t* history,
                 const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t* ids_out);
/* cl_op_sample with every row's logprobs on (top_n 0..20): the same step tail kernel; lp_out[n_rows] = the records.  A row
 * whose sp[r].temperature <= 0 takes the greedy choice instead of a draw.  vocab <= 163 840. */
int cl_op_sample_logprobs(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const int32_t* history,
                          const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t top_n, int32_t* ids_out,
                          cl_token_logprob* lp_out);
/* cl_op_sample with ext[n_rows] (may be NULL: all zero; stop strings ignored): row r also applies ext[r]'s stages. */
int cl_op_sample_ext(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const cl_sampling_ext* ext,
                     const int32_t* history, const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t* ids_out);
/* synthetic weight generator (device kernel) -> host copy, for known-answer tests */
int cl_op_synth_weights(int device, uint64_t seed, int32_t tensor_key, int64_t n, float scale,
                        uint16_t* out_bf16);

/* ---- tokenizer (host logic; usable without a GPU) --------------------------------------------
 * Loader for HF `tokenizer.json` BPE tokenizers — SentencePiece-style (Llama-2 / Mistral / TinyLlama) and byte-level
 * (Llama-3) — replacing what the Ollama server does upstream of the reference's handler (api.go:108-160; SURVEY.md
 * §8f row 2).  chat_family: "llama3" | "mistral" | "zephyr" | "chatml" | NULL (auto from the added tokens). */
typedef struct cl_tokenizer cl_tokenizer;
int cl_tokenizer_load(const char* tokenizer_json_path, const char* chat_family, cl_tokenizer** out);
void cl_tokenizer_free(cl_tokenizer* t);
/* chat != 0: wrap text as one user turn + generation prompt first.  ids may be NULL to query *n_out. */
int cl_tokenizer_encode(const cl_tokenizer* t, const char* text, size_t len, int32_t add_bos, int32_t chat,
                        int32_t* ids, int32_t cap, int32_t* n_out);
/* raw surface bytes, special tokens skipped (may end inside a UTF-8 sequence); buf may be NULL to query *len_out */
int cl_tokenizer_decode(const cl_tokenizer* t, const int32_t* ids, int32_t n, char* buf, size_t cap, size_t* len_out);
int cl_tokenizer_info(const cl_tokenizer* t, int32_t* vocab_size, int32_t* bos, int32_t* eos);
/* install a tokenizer.json into an engine (replaces the byte-level fallback behind cl_generate*, cl_tokenize).
 * Call it before the engine serves requests: in-flight cl_generate calls tokenise without a lock. */
int cl_engine_load_tokenizer(cl_engine* e, const char* tokenizer_json_path, const char* chat_family);

/* ---- paged-KV allocator (host logic; usable without a GPU) ------------------------------ */
typedef struct cl_kvpool cl_kvpool;
int cl_kvpool_create(int32_t n_pages, int32_t page_size, cl_kvpool** out);
void cl_kvpool_destroy(cl_kvpool* p);
/* grow `owner`'s page list so it covers n_tokens; CL_ERR_OOM if the free list runs dry
 * (nothing is allocated in that case). */
int cl_kvpool_reserve(cl_kvpool* p, int32_t owner, int32_t n_tokens);
int cl_kvpool_release(cl_kvpool* p, int32_t owner);
int cl_kvpool_pages_of(cl_kvpool* p, int32_t owner, int32_t* pages, int32_t cap, int32_t* n_out);
int cl_kvpool_free_pages(cl_kvpool* p);   /* allocatable: free + cached */
int cl_kvpool_used_pages(cl_kvpool* p);   /* held by some owner */
/* Prefix sharing (what the engine's prefix cache runs on).  attach: only on an owner without pages; takes the longest
 * published page chain matching ids[0..n), at most page_size * floor((n - 1) / page_size) tokens, into the owner's page
 * list (*n_reused tokens).  publish: index the owner's full pages covering ids[0..n_known) (incremental; a page whose
 * tokens and prefix are already indexed stays private).  Published pages outlive their owners as cached pages, which
 * reserve hands out (least recently released first, deepest page of a chain first) once no free page is left. */
int cl_kvpool_attach(cl_kvpool* p, int32_t owner, const int32_t* ids, int32_t n, int32_t* n_reused);
int cl_kvpool_publish(cl_kvpool* p, int32_t owner, const int32_t* ids, int32_t n_known);
int cl_kvpool_cached_pages(cl_kvpool* p);
/* Host tier (what cl_engine_set_prefix_host_cache runs on).  set_host_pages: n host pages (0: off), dropping every entry
 * the tier held; CL_ERR_INVALID_ARG for n < 0 or while moves are pending.  With the tier on, reserve and attach record
 * moves: kind 0 (spill) copies a cached device page that reserve or attach evicts to a host page, which keeps its index
 * entry; kind 1 (fill) copies a host page back into a device page when attach takes its entry.  With no host page free, the
 * least recently spilled entry is dropped.  The moves must be executed in the order given: a device page can be spilled and
 * then filled, and a host page freed by a fill reused by a later spill, within one call.  take_moves: *n_out = the moves
 * pending; with moves != NULL (cap >= *n_out, else CL_ERR_INVALID_ARG) they are written as [n][3] (kind, device page,
 * host page) and cleared.  host_cached_pages: host pages holding an entry now. */
int cl_kvpool_set_host_pages(cl_kvpool* p, int32_t n);
int cl_kvpool_take_moves(cl_kvpool* p, int32_t* moves, int32_t cap, int32_t* n_out);
int cl_kvpool_host_cached_pages(cl_kvpool* p);
/* Context shift (what cl_seq_shift runs on): `owner` holds len tokens; tokens [n_keep, n_keep + n_discard) go.  With
 * P = page_size, k0 = n_keep / P and d = n_discard / P, entries k0 + 1 .. k0 + d of the owner's page list are released
 * (k0 .. k0 + d - 1 when n_keep % P == 0) and the list is compacted.  The pages the shift writes are the new entry k0 and
 * every later one holding tokens; each that another owner holds or the index keys is first replaced by a fresh page
 * (copy-on-write) and the original keeps its index entry or becomes cached.  The owner publishes nothing afterwards.
 * items (cap >= the owner's page count + 1, else CL_ERR_INVALID_ARG before anything changes) receive the kernel's work as
 * [n][5] (source page, destination page, first row, end row, rotate): rotate 1 moves rows [first, end) with K rotated by
 * -n_discard and V copied unless source == destination; rotate 0 copies K and V unchanged (rows [0, n_keep % P) of a
 * copied entry k0).  *n_out = n.  CL_ERR_INVALID_ARG for the cl_seq_shift argument rules or a list covering fewer than len
 * tokens; CL_ERR_OOM when the copies find no page (free or cached).  On an error nothing changes. */
int cl_kvpool_shift(cl_kvpool* p, int32_t owner, int32_t len, int32_t n_keep, int32_t n_discard, int32_t* items, int32_t cap,
                    int32_t* n_out);

#ifdef __cplusplus
}
#endif
#endif /* CLENGINE_H_ */
