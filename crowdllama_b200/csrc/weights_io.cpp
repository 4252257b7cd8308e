// weights_io.cpp — checkpoint loading behind cl_engine_config.weights_path.
//
// The reference worker serves real checkpoints by name through the embedded Ollama server
// (/root/reference/cmd/crowdllama/main.go:283-297; names advertised at /root/reference/pkg/peer/peer.go:319-343).
// This engine reads the HF llama-family layout instead: a `.safetensors` file, or a model directory holding
// `*.safetensors` shards (+ optional `config.json` for the architecture — incl. the "llama3" rotary scaling of
// Llama-3.1 / 3.2 — and `tokenizer.json` for the vocabulary).
//
// safetensors container: u64 little-endian header length N | N bytes of JSON
//   { "<tensor name>": {"dtype": "BF16"|"F16"|"F32", "shape": [...], "data_offsets": [begin, end]}, "__metadata__": {...} }
// | raw tensor bytes (offsets relative to the end of the header).  Tensors are [out][in] row-major, which is the
// engine's logical layout; Engine::set_tensor applies the device-side row interleaves (rope pairs for q|k|v,
// gate/up pairs) of DESIGN.md §4.  F16 / F32 sources are rounded to bf16 (round-to-nearest-even).
#include <dirent.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <functional>
#include <sstream>

#include "engine.h"
#include "json_min.h"

namespace cl {

namespace {
using jsonmin::JParser;
using jsonmin::JVal;

enum { K_EMBED = 0, K_LM_HEAD = 1, K_FINAL_NORM = 2, K_ATTN_NORM = 3, K_WQ = 4, K_WK = 5, K_WV = 6, K_WO = 7, K_FFN_NORM = 8,
       K_WGATE = 9, K_WUP = 10, K_WDOWN = 11 };

struct Mapped {
  const uint8_t* p = nullptr;
  size_t n = 0;
  ~Mapped() { if (p) munmap(const_cast<uint8_t*>(p), n); }
  bool open(const std::string& path, std::string* err) {
    const int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) { *err = "cannot open " + path; return false; }
    struct stat st{};
    if (fstat(fd, &st) != 0 || st.st_size < 8) { ::close(fd); *err = path + ": not a safetensors file"; return false; }
    n = (size_t)st.st_size;
    void* m = mmap(nullptr, n, PROT_READ, MAP_PRIVATE, fd, 0);
    ::close(fd);
    if (m == MAP_FAILED) { *err = "mmap failed for " + path; return false; }
    p = static_cast<const uint8_t*>(m);
    return true;
  }
};

bool is_dir(const std::string& p) { struct stat st{}; return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode); }
bool is_file(const std::string& p) { struct stat st{}; return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode); }

uint16_t bf16_from_f32_bits(uint32_t u) {
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
uint32_t f32_bits_from_f16(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1fu, man = h & 0x3ffu;
  if (exp == 0) {
    if (man == 0) return sign;
    exp = 113;                                   // subnormal: normalise
    while (!(man & 0x400u)) { man <<= 1; --exp; }
    man &= 0x3ffu;
    return sign | (exp << 23) | (man << 13);
  }
  if (exp == 31) return sign | 0x7f800000u | (man << 13);
  return sign | ((exp + 112) << 23) | (man << 13);
}

// "model.layers.12.self_attn.q_proj.weight" -> (12, K_WQ); false for tensors the engine does not use (rotary inv_freq ...)
bool map_name(const std::string& name, int* layer, int* kind) {
  *layer = 0;
  if (name == "model.embed_tokens.weight") { *kind = K_EMBED; return true; }
  if (name == "lm_head.weight") { *kind = K_LM_HEAD; return true; }
  if (name == "model.norm.weight") { *kind = K_FINAL_NORM; return true; }
  const char* pre = "model.layers.";
  if (name.compare(0, strlen(pre), pre) != 0) return false;
  size_t i = strlen(pre), j = i;
  while (j < name.size() && name[j] >= '0' && name[j] <= '9') ++j;
  if (j == i || j >= name.size() || name[j] != '.' || j - i > 6) return false;
  *layer = atoi(name.substr(i, j - i).c_str());
  const std::string rest = name.substr(j + 1);
  static const struct { const char* n; int k; } tab[] = {
      {"input_layernorm.weight", K_ATTN_NORM},        {"post_attention_layernorm.weight", K_FFN_NORM},
      {"self_attn.q_proj.weight", K_WQ},              {"self_attn.k_proj.weight", K_WK},
      {"self_attn.v_proj.weight", K_WV},              {"self_attn.o_proj.weight", K_WO},
      {"mlp.gate_proj.weight", K_WGATE},              {"mlp.up_proj.weight", K_WUP},
      {"mlp.down_proj.weight", K_WDOWN}};
  for (const auto& t : tab)
    if (rest == t.n) { *kind = t.k; return true; }
  return false;
}

bool read_text(const std::string& path, std::string* out) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  std::ostringstream ss;
  ss << f.rdbuf();
  *out = ss.str();
  return true;
}
}  // namespace

// HF config.json -> cl_model_config (LlamaConfig / MistralConfig field names).  limits (may be NULL): the longest window
// the checkpoint allows, {max_position_embeddings, sliding_window or 0}.
int model_config_from_dir(const std::string& dir, cl_model_config* out, double* limits) {
  std::string text;
  if (!read_text(dir + "/config.json", &text)) { set_last_error("weights_path: no config.json in " + dir + " (pass a preset or a model config)"); return CL_ERR_IO; }
  JParser jp{text.data(), text.data() + text.size(), {}};
  JVal root;
  if (!jp.value(&root) || root.type != JVal::Obj) { set_last_error("config.json: " + (jp.err.empty() ? std::string("not an object") : jp.err)); return CL_ERR_IO; }
  auto num = [&](const char* k, double dflt) { const JVal* v = root.get(k); return v && v->type == JVal::Num ? v->n : dflt; };
  cl_model_config c{};
  c.n_layers = (int)num("num_hidden_layers", 0);
  c.d_model = (int)num("hidden_size", 0);
  c.n_heads = (int)num("num_attention_heads", 0);
  c.n_kv_heads = (int)num("num_key_value_heads", c.n_heads);
  c.head_dim = (int)num("head_dim", c.n_heads > 0 ? c.d_model / c.n_heads : 0);
  c.d_ff = (int)num("intermediate_size", 0);
  c.vocab_size = (int)num("vocab_size", 0);
  c.max_seq_len = (int)std::min(num("max_position_embeddings", 8192), 32768.0);
  double theta = num("rope_theta", 0.0);
  if (theta <= 0.0) {                         // transformers >= 5 nests it: "rope_parameters": {"rope_theta": ...}
    const JVal* rp = root.get("rope_parameters");
    const JVal* rt = rp ? rp->get("rope_theta") : nullptr;
    theta = rt && rt->type == JVal::Num ? rt->n : 10000.0;
  }
  c.rope_theta = (float)theta;
  c.rms_eps = (float)num("rms_norm_eps", 1e-5);
  // What the engine does NOT implement must fail here, not produce different tokens quietly:
  //  * scaled rotary embeddings other than "llama3" ("linear", "dynamic", "yarn" ...) change inv_freq at EVERY position;
  //  * an activation other than SiLU, attention / MLP biases.
  // A sliding attention window (Mistral-7B-v0.1: 4096) is honoured by never serving a context beyond it: inside the
  // window, sliding-window attention IS full attention.
  auto rope_type_of = [](const JVal* o) -> std::string {
    if (!o || o->type != JVal::Obj) return "";
    std::string t = o->str("rope_type", "");
    if (t.empty()) t = o->str("type", "");
    return t;
  };
  for (const char* key : {"rope_scaling", "rope_parameters"}) {
    const JVal* o = root.get(key);
    const std::string t = rope_type_of(o);
    if (t.empty() || t == "default") continue;
    if (t != "llama3") { set_last_error(std::string("config.json: ") + key + " type \"" + t + "\" is not supported (default and llama3 rotary embeddings only)"); return CL_ERR_IO; }
    auto f = [&](const char* k) { const JVal* v = o->get(k); return v && v->type == JVal::Num ? v->n : 0.0; };
    c.rope_factor = (float)f("factor");
    c.rope_low_freq_factor = (float)f("low_freq_factor");
    c.rope_high_freq_factor = (float)f("high_freq_factor");
    c.rope_original_max_pos = (int)f("original_max_position_embeddings");
    if (!(c.rope_factor >= 1.f) || !(c.rope_low_freq_factor > 0.f) || !(c.rope_high_freq_factor > c.rope_low_freq_factor) || c.rope_original_max_pos <= 0) {
      set_last_error(std::string("config.json: ") + key + " llama3 needs factor >= 1, 0 < low_freq_factor < high_freq_factor, original_max_position_embeddings > 0");
      return CL_ERR_IO;
    }
  }
  const std::string act = root.str("hidden_act", "silu");
  if (act != "silu") { set_last_error("config.json: hidden_act \"" + act + "\" is not supported (silu)"); return CL_ERR_IO; }
  for (const char* key : {"attention_bias", "mlp_bias"}) {
    const JVal* v = root.get(key);
    if (v && v->type == JVal::Bool && v->b) { set_last_error(std::string("config.json: ") + key + " = true is not supported"); return CL_ERR_IO; }
  }
  const double window = num("sliding_window", 0.0);
  if (window >= 1.0 && window < (double)c.max_seq_len) c.max_seq_len = (int)window;
  if (limits) { limits[0] = num("max_position_embeddings", 8192); limits[1] = window >= 1.0 ? window : 0.0; }
  if (c.n_layers <= 0 || c.d_model <= 0 || c.n_heads <= 0 || c.d_ff <= 0 || c.vocab_size <= 0) {
    set_last_error("config.json: missing llama-family fields (num_hidden_layers, hidden_size, num_attention_heads, intermediate_size, vocab_size)");
    return CL_ERR_IO;
  }
  *out = c;
  return CL_OK;
}

// Walk every tensor of the checkpoint that the engine uses, validated against `cfg`, as bf16 bits in the logical
// [out][in] layout.  Host-only (no CUDA): Engine::load_safetensors feeds set_tensor, cl_checkpoint_info just counts.
int visit_checkpoint(const std::string& path, const cl_model_config& cfg,
                     const std::function<int(int layer, int kind, const uint16_t* bf16, int64_t n)>& fn) {
  const int64_t q_dim_ = (int64_t)cfg.n_heads * cfg.head_dim, kv_dim_ = (int64_t)cfg.n_kv_heads * cfg.head_dim;
  std::vector<std::string> files;
  if (is_dir(path)) {
    if (DIR* d = opendir(path.c_str())) {
      while (dirent* e = readdir(d)) {
        const std::string n = e->d_name;
        if (n.size() > 12 && n.compare(n.size() - 12, 12, ".safetensors") == 0) files.push_back(path + "/" + n);
      }
      closedir(d);
    }
    std::sort(files.begin(), files.end());
  } else if (is_file(path)) {
    files.push_back(path);
  }
  if (files.empty()) { set_last_error("weights_path: no .safetensors file at " + path); return CL_ERR_IO; }

  const int64_t d = cfg.d_model, F = cfg.d_ff, V = cfg.vocab_size;
  auto expect = [&](int kind, int64_t* rows, int64_t* cols) {
    switch (kind) {
      case K_EMBED: case K_LM_HEAD: *rows = V; *cols = d; break;
      case K_FINAL_NORM: case K_ATTN_NORM: case K_FFN_NORM: *rows = d; *cols = 1; break;
      case K_WQ: *rows = q_dim_; *cols = d; break;
      case K_WK: case K_WV: *rows = kv_dim_; *cols = d; break;
      case K_WO: *rows = d; *cols = q_dim_; break;
      case K_WGATE: case K_WUP: *rows = F; *cols = d; break;
      default: *rows = d; *cols = F; break;   // K_WDOWN
    }
  };
  std::vector<char> seen((size_t)cfg.n_layers * 16 + 16, 0);
  const uint8_t* embed_src = nullptr; std::string embed_dtype; int64_t embed_n = 0;
  std::vector<uint16_t> conv;
  std::vector<std::unique_ptr<Mapped>> maps;   // keep every shard mapped until the tie fallback below has run
  for (const auto& file : files) {
    std::string err;
    maps.emplace_back(new Mapped());
    Mapped& m = *maps.back();
    if (!m.open(file, &err)) { set_last_error(err); return CL_ERR_IO; }
    uint64_t hlen = 0;
    memcpy(&hlen, m.p, 8);
    if (hlen < 2 || hlen > m.n - 8 || hlen > (100u << 20)) { set_last_error(file + ": bad safetensors header length"); return CL_ERR_IO; }
    JParser jp{reinterpret_cast<const char*>(m.p) + 8, reinterpret_cast<const char*>(m.p) + 8 + hlen, {}};
    JVal root;
    if (!jp.value(&root) || root.type != JVal::Obj) { set_last_error(file + ": header is not JSON (" + jp.err + ")"); return CL_ERR_IO; }
    const uint8_t* data = m.p + 8 + hlen;
    const size_t data_len = m.n - 8 - hlen;
    for (const auto& kv : root.o) {
      int layer = 0, kind = 0;
      if (kv.first == "__metadata__") continue;
      if (kv.first.size() > 5 && kv.first.compare(kv.first.size() - 5, 5, ".bias") == 0 && kv.first.compare(0, 6, "model.") == 0) {
        set_last_error(kv.first + ": projection biases are not supported by this engine"); return CL_ERR_IO;
      }
      if (!map_name(kv.first, &layer, &kind)) continue;
      if (layer >= cfg.n_layers) { set_last_error(kv.first + ": layer index beyond n_layers"); return CL_ERR_IO; }
      const JVal& t = kv.second;
      const JVal* shape = t.get("shape");
      const JVal* offs = t.get("data_offsets");
      const std::string dtype = t.str("dtype", "");
      if (!shape || shape->type != JVal::Arr || !offs || offs->type != JVal::Arr || offs->a.size() != 2) { set_last_error(kv.first + ": malformed entry"); return CL_ERR_IO; }
      int64_t n = 1;
      bool nums_ok = offs->a[0].type == JVal::Num && offs->a[1].type == JVal::Num && offs->a[0].n >= 0 && offs->a[1].n >= 0 &&
                     offs->a[0].n < 9e15 && offs->a[1].n < 9e15 && shape->a.size() <= 2;
      for (const auto& s : shape->a) {
        if (s.type != JVal::Num || s.n < 0 || s.n > 2147483647.0) { nums_ok = false; break; }
        n *= (int64_t)s.n;
      }
      if (!nums_ok) { set_last_error(kv.first + ": malformed shape / data_offsets"); return CL_ERR_IO; }
      int64_t rows = 0, cols = 0;
      expect(kind, &rows, &cols);
      const bool shape_ok = cols == 1 ? (shape->a.size() == 1 && (int64_t)shape->a[0].n == rows)
                                      : (shape->a.size() == 2 && (int64_t)shape->a[0].n == rows && (int64_t)shape->a[1].n == cols);
      if (!shape_ok) { set_last_error(kv.first + ": shape does not match the model config"); return CL_ERR_IO; }
      const size_t esz = dtype == "F32" ? 4 : (dtype == "BF16" || dtype == "F16") ? 2 : 0;
      if (!esz) { set_last_error(kv.first + ": unsupported dtype " + dtype + " (BF16, F16, F32)"); return CL_ERR_IO; }
      const uint64_t b0 = (uint64_t)offs->a[0].n, b1 = (uint64_t)offs->a[1].n;
      if (b1 < b0 || b1 > data_len || b1 - b0 != (uint64_t)n * esz) { set_last_error(kv.first + ": data_offsets out of range"); return CL_ERR_IO; }
      const uint8_t* src = data + b0;
      const uint16_t* bf = nullptr;
      if (dtype == "BF16") {
        bf = reinterpret_cast<const uint16_t*>(src);
      } else {
        conv.resize((size_t)n);
        if (dtype == "F32") {
          for (int64_t i = 0; i < n; ++i) { uint32_t u; memcpy(&u, src + (size_t)i * 4, 4); conv[(size_t)i] = bf16_from_f32_bits(u); }
        } else {
          for (int64_t i = 0; i < n; ++i) { uint16_t h; memcpy(&h, src + (size_t)i * 2, 2); conv[(size_t)i] = bf16_from_f32_bits(f32_bits_from_f16(h)); }
        }
        bf = conv.data();
      }
      const int rc = fn(layer, kind, bf, n);
      if (rc) return rc;
      seen[(size_t)(kind <= K_FINAL_NORM ? 0 : layer + 1) * 16 + kind] = 1;
      if (kind == K_EMBED) { embed_src = src; embed_dtype = dtype; embed_n = n; }
    }
  }
  if (!seen[K_LM_HEAD] && seen[K_EMBED]) {
    // tie_word_embeddings: the checkpoint stores one matrix for both ends
    const uint16_t* bf = reinterpret_cast<const uint16_t*>(embed_src);
    if (embed_dtype != "BF16") {
      conv.resize((size_t)embed_n);
      for (int64_t i = 0; i < embed_n; ++i) {
        if (embed_dtype == "F32") { uint32_t u; memcpy(&u, embed_src + (size_t)i * 4, 4); conv[(size_t)i] = bf16_from_f32_bits(u); }
        else { uint16_t h; memcpy(&h, embed_src + (size_t)i * 2, 2); conv[(size_t)i] = bf16_from_f32_bits(f32_bits_from_f16(h)); }
      }
      bf = conv.data();
    }
    const int rc = fn(0, K_LM_HEAD, bf, embed_n);
    if (rc) return rc;
    seen[K_LM_HEAD] = 1;
  }
  std::string missing;
  for (int k : {K_EMBED, K_LM_HEAD, K_FINAL_NORM}) if (!seen[k]) missing += " global:" + std::to_string(k);
  for (int l = 0; l < cfg.n_layers; ++l)
    for (int k = K_ATTN_NORM; k <= K_WDOWN; ++k)
      if (!seen[(size_t)(l + 1) * 16 + k]) missing += " L" + std::to_string(l) + ":" + std::to_string(k);
  if (!missing.empty()) { set_last_error("checkpoint misses tensors (layer:kind)" + missing.substr(0, 200)); return CL_ERR_IO; }
  return CL_OK;
}

int Engine::load_safetensors(const std::string& path) {
  return visit_checkpoint(path, cfg, [this](int layer, int kind, const uint16_t* bf, int64_t n) { return set_tensor(layer, kind, bf, n); });
}

// The model config and served window of an engine config (cl_engine_create / cl_resolve_model_config): the one place that
// reads context_length and CL_CONTEXT_LENGTH.  *context_length (may be NULL): the value applied, 0 for the model's window.
int resolve_model_config(const cl_engine_config& c, cl_model_config* out, int* context_length) {
  cl_model_config cfg{};
  double limits[2] = {0.0, 0.0};   // a model directory's max_position_embeddings and sliding window; 0: no limit
  const std::string wpath = c.weights_path ? c.weights_path : "";
  struct stat wst{};
  const bool wdir = !wpath.empty() && stat(wpath.c_str(), &wst) == 0 && S_ISDIR(wst.st_mode);
  if (c.preset) {
    if (cl_model_preset(c.preset, &cfg) != CL_OK) { set_last_error("unknown preset"); return CL_ERR_UNKNOWN_MODEL; }
  } else if (c.model.n_layers == 0 && wdir) {
    // a model directory describes itself: config.json (HF LlamaConfig / MistralConfig field names)
    const int rc = model_config_from_dir(wpath, &cfg, limits);
    if (rc) return rc;
  } else {
    cfg = c.model;
  }
  const char* env = getenv("CL_CONTEXT_LENGTH");
  const int ctx = env && *env ? atoi(env) : c.context_length;
  const int page = c.page_size ? c.page_size : 32;
  if (ctx != 0) {
    if (ctx < 2 * page || ctx > kMaxContext) {
      set_last_error("context_length " + std::to_string(ctx) + " is outside " + std::to_string(2 * page) + " .. " + std::to_string(kMaxContext));
      return CL_ERR_INVALID_ARG;
    }
    if (limits[0] > 0.0 && ctx > limits[0]) {
      set_last_error("context_length " + std::to_string(ctx) + " exceeds the model's max_position_embeddings (" + std::to_string((long long)limits[0]) + ")");
      return CL_ERR_INVALID_ARG;
    }
    if (limits[1] > 0.0 && ctx > limits[1]) {
      set_last_error("context_length " + std::to_string(ctx) + " exceeds the model's sliding_window (" + std::to_string((long long)limits[1]) + ")");
      return CL_ERR_INVALID_ARG;
    }
    cfg.max_seq_len = ctx;
  }
  const char* shift = getenv("CL_CONTEXT_SHIFT");
  const char* keep = getenv("CL_NUM_KEEP");
  const bool context_shift = (shift && *shift ? atoi(shift) : c.context_shift) != 0;
  const int num_keep = keep && *keep ? atoi(keep) : c.num_keep;
  if (context_shift && (num_keep < 0 || cfg.max_seq_len - num_keep < 2 * page)) {
    set_last_error("num_keep must leave at least two pages of max_seq_len to shift");
    return CL_ERR_INVALID_ARG;
  }
  *out = cfg;
  if (context_length) *context_length = ctx;
  return CL_OK;
}

}  // namespace cl

extern "C" int cl_resolve_model_config(const cl_engine_config* c, cl_model_config* out) {
  if (!c || !out) return CL_ERR_INVALID_ARG;
  if (c->abi_version != CL_ABI_VERSION) { cl::set_last_error("abi_version mismatch"); return CL_ERR_INVALID_ARG; }
  try {
    return cl::resolve_model_config(*c, out, nullptr);
  } catch (const std::exception& ex) {
    cl::set_last_error(ex.what());
    return CL_ERR_INTERNAL;
  }
}

extern "C" int cl_checkpoint_info(const char* path, cl_model_config* cfg_io, int32_t* n_tensors, int64_t* n_params) {
  using namespace cl;
  if (!path || !cfg_io) return CL_ERR_INVALID_ARG;
  try {
    struct stat st{};
    if (cfg_io->n_layers == 0) {
      if (stat(path, &st) != 0 || !S_ISDIR(st.st_mode)) { set_last_error("cl_checkpoint_info: a model config is needed unless path is a model directory"); return CL_ERR_INVALID_ARG; }
      const int rc = model_config_from_dir(path, cfg_io, nullptr);
      if (rc) return rc;
    }
    int32_t nt = 0;
    int64_t np = 0;
    const int rc = visit_checkpoint(path, *cfg_io, [&](int, int, const uint16_t*, int64_t n) { ++nt; np += n; return (int)CL_OK; });
    if (n_tensors) *n_tensors = nt;
    if (n_params) *n_params = np;
    return rc;
  } catch (const std::exception& ex) {
    set_last_error(ex.what());
    return CL_ERR_INTERNAL;
  }
}
