// ops_api.cu — cl_op_*: single-kernel entry points of the C-ABI with HOST buffers in and out.
// Each runs exactly the kernel the token step uses (parity tests per kernel, microbenchmarks).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <random>
#include <vector>

#include "common.cuh"
#include "engine.h"

namespace cl {

// Pages of all sequences interleaved (page i of every sequence, then page i + 1) and scattered by a fixed pseudo-random
// permutation; one filler page that block-table entries past a sequence's last page (and the rows of slots outside a batch)
// name, and one page that nothing references.  Every pool element that holds no token (layer 0, the tails of last pages, the
// two token-less pages) is set to the largest finite bf16: + for K, - for V.  Reading any of them puts an enormous term into
// the output, while a masked probability of exactly 0 leaves it untouched (0 x finite = 0; a NaN filler would not, in the
// tensor-core P.V).
void op_build_kv_pool(const uint16_t* k, const uint16_t* v, const int* lens, int n_seqs, int n_kv, int head_dim, int page_size,
                      OpKvPool* pool) {
  const int P = page_size, HD = head_dim;
  std::vector<int> npg(n_seqs);
  int used = 0, maxp = 1;
  for (int b = 0; b < n_seqs; ++b) {
    npg[b] = (lens[b] + P - 1) / P;
    used += npg[b];
    maxp = std::max(maxp, npg[b]);
  }
  pool->n_pages = used + 2;                    // + the padding page (perm[used]) and the unreferenced one (perm[used + 1])
  std::vector<int> perm(pool->n_pages);
  std::iota(perm.begin(), perm.end(), 0);
  std::shuffle(perm.begin(), perm.end(), std::mt19937(0x5eed));
  pool->pad_page = perm[used];
  pool->bt_stride = maxp;
  pool->bt.assign((size_t)n_seqs * maxp, pool->pad_page);
  for (int i = 0, r = 0; i < maxp; ++i)
    for (int b = 0; b < n_seqs; ++b)
      if (i < npg[b]) pool->bt[(size_t)b * maxp + i] = perm[r++];
  pool->layer_elems = (size_t)pool->n_pages * n_kv * P * HD;
  pool->k.assign(2 * pool->layer_elems, 0x7F7F);
  pool->v.assign(2 * pool->layer_elems, 0xFF7F);
  size_t row0 = 0;
  for (int b = 0; b < n_seqs; ++b) {
    const int* bt = pool->bt.data() + (size_t)b * maxp;
    for (int t = 0; t < lens[b]; ++t)
      for (int g = 0; g < n_kv; ++g) {
        const size_t dst = pool->layer_elems + (((size_t)bt[t / P] * n_kv + g) * P + t % P) * HD;
        const size_t src = ((row0 + t) * n_kv + g) * HD;
        memcpy(&pool->k[dst], k + src, (size_t)HD * 2);
        memcpy(&pool->v[dst], v + src, (size_t)HD * 2);
      }
    row0 += lens[b];
  }
}

}  // namespace cl

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

int run_gemv(int device, int variant, int epi, bool norm, const uint16_t* w, const float* x_or_h, const float* gain, float eps,
             const float* resid, float* y, int n_rows, int k, int out_n, int iters, float* ms) {
  int rc = check_device(device);
  if (rc) return rc;
  if (!gemv_variant_supported(variant, n_rows, k)) {
    set_last_error("gemv variant does not support this shape");
    return CL_ERR_INVALID_ARG;
  }
  DevBuf dw, dx, dg, dy;
  CL_CUDA_OK(dw.upload(w, (size_t)n_rows * k * 2));
  CL_CUDA_OK(dx.upload(x_or_h, (size_t)k * 4));
  if (gain) CL_CUDA_OK(dg.upload(gain, (size_t)k * 4));
  CL_CUDA_OK(dy.alloc((size_t)std::max(out_n, n_rows) * 4));
  if (resid) CL_CUDA_OK(cudaMemcpy(dy.p, resid, (size_t)out_n * 4, cudaMemcpyHostToDevice));
  else CL_CUDA_OK(cudaMemset(dy.p, 0, (size_t)out_n * 4));
  GemvArgs a;
  a.W = dw.as<__nv_bfloat16>(); a.N = n_rows; a.K = k;
  if (norm) { a.h = dx.as<float>(); a.gain = dg.as<float>(); a.eps = eps; } else { a.x = dx.as<float>(); }
  a.y = dy.as<float>(); a.resid = resid ? dy.as<float>() : nullptr; a.x_stride = k; a.y_stride = out_n; a.batch = 1;
  cudaStream_t st = nullptr;
  if (launch_gemv(variant, epi, norm, a, st, false) < 0) { CL_CUDA_OK(cudaGetLastError()); return CL_ERR_CUDA; }
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaMemcpy(y, dy.p, (size_t)out_n * 4, cudaMemcpyDeviceToHost));
  if (iters > 0 && ms && epi != EPI_RESID) {
    // timing loop: rotate over enough weight copies (256 MB) to exceed the L2 (50 MB on H100)
    const size_t wbytes = (size_t)n_rows * k * 2;
    int copies = (int)std::min<size_t>(16, (256ull << 20) / wbytes + 1);
    std::vector<DevBuf> extra(copies > 1 ? copies - 1 : 0);
    std::vector<const __nv_bfloat16*> ws{dw.as<__nv_bfloat16>()};
    for (auto& b : extra) {
      CL_CUDA_OK(b.alloc(wbytes));
      CL_CUDA_OK(cudaMemcpy(b.p, dw.p, wbytes, cudaMemcpyDeviceToDevice));
      ws.push_back(b.as<__nv_bfloat16>());
    }
    cudaEvent_t e0, e1;
    CL_CUDA_OK(cudaEventCreate(&e0));
    CL_CUDA_OK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) { a.W = ws[i % ws.size()]; launch_gemv(variant, epi, norm, a, st, false); }
    CL_CUDA_OK(cudaDeviceSynchronize());
    CL_CUDA_OK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i) { a.W = ws[i % ws.size()]; launch_gemv(variant, epi, norm, a, st, false); }
    CL_CUDA_OK(cudaEventRecord(e1, st));
    CL_CUDA_OK(cudaDeviceSynchronize());
    float t = 0.f;
    CL_CUDA_OK(cudaEventElapsedTime(&t, e0, e1));
    *ms = t / (float)iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  return CL_OK;
}

}  // namespace

extern "C" {

int cl_op_gemv(int device, int variant, const uint16_t* w, const float* x, float* y, int32_t n_rows, int32_t k, int32_t iters,
               float* ms) {
  if (!w || !x || !y) return CL_ERR_INVALID_ARG;
  return run_gemv(device, variant, EPI_STORE, false, w, x, nullptr, 0.f, nullptr, y, n_rows, k, n_rows, iters, ms);
}
int cl_op_gemv_residual(int device, int variant, const uint16_t* w, const float* x, const float* resid, float* y, int32_t n_rows,
                        int32_t k) {
  if (!w || !x || !y || !resid) return CL_ERR_INVALID_ARG;
  return run_gemv(device, variant, EPI_RESID, false, w, x, nullptr, 0.f, resid, y, n_rows, k, n_rows, 0, nullptr);
}
int cl_op_rmsnorm_gemv(int device, int variant, const uint16_t* w, const float* h, const float* gain, float eps, float* y,
                       int32_t n_rows, int32_t k) {
  if (!w || !h || !y || !gain) return CL_ERR_INVALID_ARG;
  return run_gemv(device, variant, EPI_STORE, true, w, h, gain, eps, nullptr, y, n_rows, k, n_rows, 0, nullptr);
}
int cl_op_rmsnorm_gateup(int device, int variant, const uint16_t* w_gu, const float* h, const float* gain, float eps, float* act,
                         int32_t d_ff, int32_t k) {
  if (!w_gu || !h || !act || !gain) return CL_ERR_INVALID_ARG;
  return run_gemv(device, variant, EPI_GATEUP, true, w_gu, h, gain, eps, nullptr, act, 2 * d_ff, k, d_ff, 0, nullptr);
}

int cl_op_attn_decode(int device, const float* q, const uint16_t* k_cache, const uint16_t* v_cache, int32_t ctx_len, int32_t n_heads,
                      int32_t n_kv, int32_t head_dim, int32_t page_size, float* out) {
  if (!q || !out || ctx_len <= 0 || !k_cache || !v_cache) return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  const int rep = n_kv > 0 ? n_heads / n_kv : 0;
  if ((head_dim != 64 && head_dim != 128) || (rep != 1 && rep != 2 && rep != 4 && rep != 8) || n_heads % n_kv ||
      (page_size != 16 && page_size != 32 && page_size != 64)) {
    set_last_error("unsupported attention shape");
    return CL_ERR_INVALID_ARG;
  }
  const int P = page_size, HD = head_dim;
  const int n_pages = (ctx_len + P - 1) / P;
  // scatter the dense cache into pages in a scrambled page order (exercises the block table)
  std::vector<int> bt(n_pages);
  for (int i = 0; i < n_pages; ++i) bt[i] = (int)(((long long)i * 7 + 3) % n_pages);
  if (n_pages % 7 == 0) for (int i = 0; i < n_pages; ++i) bt[i] = n_pages - 1 - i;
  const size_t pool_elems = (size_t)n_pages * n_kv * P * HD;
  std::vector<uint16_t> kp(pool_elems, 0x7fc0), vp(pool_elems, 0x7fc0);   // NaN fill: slots past ctx must never be read into the result
  for (int t = 0; t < ctx_len; ++t)
    for (int g = 0; g < n_kv; ++g) {
      const size_t dst = (((size_t)bt[t / P] * n_kv + g) * P + t % P) * HD;
      memcpy(&kp[dst], k_cache + ((size_t)t * n_kv + g) * HD, (size_t)HD * 2);
      memcpy(&vp[dst], v_cache + ((size_t)t * n_kv + g) * HD, (size_t)HD * 2);
    }
  const int qd = n_heads * HD;
  const int pos = ctx_len - 1;
  const int nsplit = std::max(1, std::min(64, sm_count() / n_kv));
  DevBuf dq, dk, dv, dbt, dpos, dout, dpart, dcnt;
  CL_CUDA_OK(dq.upload(q, (size_t)qd * 4));
  CL_CUDA_OK(dk.upload(kp.data(), pool_elems * 2));
  CL_CUDA_OK(dv.upload(vp.data(), pool_elems * 2));
  CL_CUDA_OK(dbt.upload(bt.data(), bt.size() * 4));
  CL_CUDA_OK(dpos.upload(&pos, 4));
  CL_CUDA_OK(dout.alloc((size_t)qd * 4));
  CL_CUDA_OK(dpart.alloc((size_t)n_kv * nsplit * rep * (HD + 2) * 4));
  CL_CUDA_OK(dcnt.alloc((size_t)n_kv * 4));
  CL_CUDA_OK(cudaMemset(dcnt.p, 0, (size_t)n_kv * 4));
  AttnDecodeArgs a;
  a.q = dq.as<float>(); a.q_stride = qd;
  a.kpool = dk.as<__nv_bfloat16>(); a.vpool = dv.as<__nv_bfloat16>(); a.block_tables = dbt.as<int>(); a.bt_stride = n_pages;
  a.pos = dpos.as<int>(); a.out = dout.as<float>(); a.out_stride = qd; a.part = dpart.as<float>(); a.counters = dcnt.as<unsigned>();
  a.batch = 1; a.n_heads = n_heads; a.n_kv = n_kv; a.head_dim = HD; a.page_size = P; a.nsplit = nsplit;
  // run twice: the second launch checks that the split counters re-arm (graph replay safety)
  for (int i = 0; i < 2; ++i)
    if (launch_attn_decode(a, nullptr, false) < 0) { CL_CUDA_OK(cudaGetLastError()); set_last_error("launch_attn_decode failed"); return CL_ERR_CUDA; }
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaMemcpy(out, dout.p, (size_t)qd * 4, cudaMemcpyDeviceToHost));
  return CL_OK;
}

int cl_op_attn_decode_batch(int device, int variant, int32_t nsplit, int32_t tc_small, const float* q, const uint16_t* k_cache,
                            const uint16_t* v_cache, const int32_t* ctx_lens, const int32_t* slots, int32_t batch, int32_t n_slots,
                            int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, float* out, uint16_t* out_bf16,
                            int32_t* nsplit_used, int32_t* tc_small_used) {
  if (!q || !k_cache || !v_cache || !ctx_lens || !out || batch <= 0 || n_slots < batch || variant < -1 || variant > 1 || nsplit < 0 ||
      tc_small < -1 || tc_small > 1)
    return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  const int rep = n_kv > 0 ? n_heads / n_kv : 0;
  if ((head_dim != 64 && head_dim != 128) || (rep != 1 && rep != 2 && rep != 4 && rep != 8) || n_heads % n_kv ||
      (page_size != 16 && page_size != 32 && page_size != 64)) {
    set_last_error("unsupported attention shape");
    return CL_ERR_INVALID_ARG;
  }
  const int P = page_size, HD = head_dim;
  const size_t qd = (size_t)n_heads * HD;
  std::vector<int> slot(batch), taken(n_slots, 0);
  for (int b = 0; b < batch; ++b) {
    slot[b] = slots ? slots[b] : b;
    if (ctx_lens[b] <= 0 || slot[b] < 0 || slot[b] >= n_slots || taken[slot[b]]++) {
      set_last_error("cl_op_attn_decode_batch: every context needs >= 1 token and a distinct slot < n_slots");
      return CL_ERR_INVALID_ARG;
    }
  }
  // the batched step's plan (Engine::enqueue_step_batched); explicit choices override it
  int ns = 0, small = 0;
  attn_decode_tc_plan(n_kv, batch, std::max(1, std::min(64, sm_count() / n_kv)), sm_count(), &ns, &small);
  if (nsplit > 0) ns = nsplit;
  if (tc_small >= 0) small = tc_small;
  OpKvPool pool;
  op_build_kv_pool(k_cache, v_cache, ctx_lens, batch, n_kv, HD, P, &pool);
  // q, pos, the block tables, out, the partials and the counters are indexed by slot, as in the engine; q rows of the slots
  // outside the batch are NaN
  std::vector<float> qs((size_t)n_slots * qd, NAN);
  std::vector<int> pos(n_slots, 0), bts((size_t)n_slots * pool.bt_stride, pool.pad_page);
  for (int b = 0; b < batch; ++b) {
    memcpy(&qs[(size_t)slot[b] * qd], q + (size_t)b * qd, qd * 4);
    pos[slot[b]] = ctx_lens[b] - 1;
    memcpy(&bts[(size_t)slot[b] * pool.bt_stride], &pool.bt[(size_t)b * pool.bt_stride], (size_t)pool.bt_stride * 4);
  }
  DevBuf dq, dk, dv, dbt, dpos, dslots, dout, dob, dpart, dcnt;
  CL_CUDA_OK(dq.upload(qs.data(), qs.size() * 4));
  CL_CUDA_OK(dk.upload(pool.k.data(), pool.k.size() * 2));
  CL_CUDA_OK(dv.upload(pool.v.data(), pool.v.size() * 2));
  CL_CUDA_OK(dbt.upload(bts.data(), bts.size() * 4));
  CL_CUDA_OK(dpos.upload(pos.data(), pos.size() * 4));
  CL_CUDA_OK(dslots.upload(slot.data(), slot.size() * 4));
  CL_CUDA_OK(dout.alloc((size_t)n_slots * qd * 4));
  CL_CUDA_OK(dob.alloc((size_t)batch * qd * 2));
  CL_CUDA_OK(dpart.alloc((size_t)n_slots * n_kv * ns * rep * (HD + 2) * 4));
  CL_CUDA_OK(dcnt.alloc((size_t)n_slots * n_kv * 4));
  CL_CUDA_OK(cudaMemset(dcnt.p, 0, (size_t)n_slots * n_kv * 4));
  AttnDecodeArgs a;
  a.q = dq.as<float>(); a.q_stride = (int)qd;
  a.kpool = dk.as<__nv_bfloat16>() + pool.layer_elems; a.vpool = dv.as<__nv_bfloat16>() + pool.layer_elems;
  a.block_tables = dbt.as<int>(); a.bt_stride = pool.bt_stride; a.pos = dpos.as<int>();
  a.out = dout.as<float>(); a.out_stride = (int)qd; a.out_bf16 = out_bf16 ? dob.as<__nv_bfloat16>() : nullptr;
  a.part = dpart.as<float>(); a.counters = dcnt.as<unsigned>(); a.slots = dslots.as<int>(); a.batch = batch;
  a.n_heads = n_heads; a.n_kv = n_kv; a.head_dim = HD; a.page_size = P; a.nsplit = ns; a.tc_small = small;
  // variant -1: the tensor-core kernel where it takes the shape and the pool's tensor maps exist, as in the engine
  const long long pool_rows = 2LL * pool.n_pages * n_kv * P;
  CUtensorMap km, vm;
  bool tc = variant != 0 && attn_decode_tc_supported(n_heads, n_kv, HD, P, ns);
  if (tc) tc = make_tmap_2d_bf16(&km, dk.p, pool_rows, HD, 64, 32) && make_tmap_2d_bf16(&vm, dv.p, pool_rows, HD, 64, 32);
  if ((variant == 1 && !tc) || (!tc && ns > 64)) {
    set_last_error("the decode attention kernel does not take this shape or split count");
    return CL_ERR_INVALID_ARG;
  }
  // two launches without re-arming the split counters in between must give the same bits
  std::vector<float> out1((size_t)n_slots * qd);
  std::vector<uint16_t> ob1((size_t)batch * qd), ob2(ob1.size());
  for (int run = 0; run < 2; ++run) {
    CL_CUDA_OK(cudaMemcpy(dout.p, out, (size_t)n_slots * qd * 4, cudaMemcpyHostToDevice));
    CL_CUDA_OK(cudaMemset(dob.p, 0xff, (size_t)batch * qd * 2));   // NaN: every element must be written
    const int r = tc ? launch_attn_decode_tc(a, km, vm, pool_rows / 2, nullptr, false) : launch_attn_decode(a, nullptr, false);
    if (r < 0) { CL_CUDA_OK(cudaGetLastError()); set_last_error("decode attention launch failed"); return CL_ERR_CUDA; }
    CL_CUDA_OK(cudaDeviceSynchronize());
    CL_CUDA_OK(cudaMemcpy(run ? out : out1.data(), dout.p, (size_t)n_slots * qd * 4, cudaMemcpyDeviceToHost));
    CL_CUDA_OK(cudaMemcpy(run ? ob2.data() : ob1.data(), dob.p, ob1.size() * 2, cudaMemcpyDeviceToHost));
  }
  if (nsplit_used) *nsplit_used = ns;
  if (tc_small_used) *tc_small_used = tc ? small : -1;
  if (out_bf16) memcpy(out_bf16, ob2.data(), ob2.size() * 2);
  if (memcmp(out, out1.data(), out1.size() * 4) || memcmp(ob1.data(), ob2.data(), ob1.size() * 2)) {
    set_last_error("cl_op_attn_decode_batch: the second launch (split counters not reset) changed the output");
    return CL_ERR_INTERNAL;
  }
  return CL_OK;
}

int cl_op_kv_host_roundtrip(int device, int32_t n_layers, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t n_moves,
                            int32_t iters, float* ms) {
  if (n_layers <= 0 || n_kv <= 0 || n_moves <= 0 || iters < 0 || (head_dim != 64 && head_dim != 128) ||
      (page_size != 16 && page_size != 32 && page_size != 64)) {
    set_last_error("cl_op_kv_host_roundtrip: unsupported shape");
    return CL_ERR_INVALID_ARG;
  }
  int rc = check_device(device);
  if (rc) return rc;
  // pool of 2 n + 2 pages, scattered: the n spilled pages hold random bits, their n destinations and two pages nothing
  // names the largest finite bf16 (+ for K, - for V), so a block copied short, to the wrong place or not at all shows
  const int n = n_moves, n_pages = 2 * n + 2;
  const size_t blk = (size_t)n_kv * page_size * head_dim, layer_elems = (size_t)n_pages * blk;
  std::vector<int> perm(n_pages);
  std::iota(perm.begin(), perm.end(), 0);
  std::shuffle(perm.begin(), perm.end(), std::mt19937(0x5eed));
  std::vector<int2> spill(n), fill(n);
  for (int i = 0; i < n; ++i) {
    spill[i] = make_int2(perm[2 * i], n - 1 - i);   // host pages in the other order
    fill[i] = make_int2(perm[2 * i + 1], n - 1 - i);
  }
  const size_t pool_elems = (size_t)n_layers * layer_elems;
  std::vector<uint16_t> k(pool_elems, 0x7F7F), v(pool_elems, 0xFF7F);
  std::mt19937 rng(0xc0ffee);
  for (int i = 0; i < n; ++i)
    for (int l = 0; l < n_layers; ++l)
      for (size_t e = 0; e < blk; ++e) {
        const size_t at = l * layer_elems + (size_t)spill[i].x * blk + e;
        k[at] = (uint16_t)rng();
        v[at] = (uint16_t)rng();
      }
  DevBuf dk, dv, dmv;
  CL_CUDA_OK(dk.upload(k.data(), pool_elems * 2));
  CL_CUDA_OK(dv.upload(v.data(), pool_elems * 2));
  std::vector<int2> moves(spill);
  moves.insert(moves.end(), fill.begin(), fill.end());
  CL_CUDA_OK(dmv.upload(moves.data(), moves.size() * sizeof(int2)));
  const size_t host_bytes = (size_t)n * 2 * n_layers * blk * 2;
  void* host = nullptr;
  CL_CUDA_OK(cudaHostAlloc(&host, host_bytes, cudaHostAllocMapped | cudaHostAllocPortable));
  struct HostFree { void* p; ~HostFree() { cudaFreeHost(p); } } host_guard{host};
  memset(host, 0xff, host_bytes);
  KvMoveArgs a;
  a.n_moves = n; a.kpool = dk.as<__nv_bfloat16>(); a.vpool = dv.as<__nv_bfloat16>(); a.layer_elems = layer_elems;
  a.host = static_cast<uint4*>(host); a.n_layers = n_layers; a.blk_vec = (int)(blk * 2 / 16);
  KvMoveArgs f = a;
  a.moves = dmv.as<int2>();
  f.moves = dmv.as<int2>() + n;
  if (launch_kv_move(true, a, nullptr) < 0 || launch_kv_move(false, f, nullptr) < 0) {
    CL_CUDA_OK(cudaGetLastError());
    return CL_ERR_CUDA;
  }
  CL_CUDA_OK(cudaDeviceSynchronize());
  std::vector<uint16_t> k2(pool_elems), v2(pool_elems);
  CL_CUDA_OK(cudaMemcpy(k2.data(), dk.p, pool_elems * 2, cudaMemcpyDeviceToHost));
  CL_CUDA_OK(cudaMemcpy(v2.data(), dv.p, pool_elems * 2, cudaMemcpyDeviceToHost));
  // expected: every destination page equals its source, every other page is unchanged, host page h = [K|V][layer] blocks
  std::vector<uint16_t> kw(k), vw(v);
  const uint16_t* hp = static_cast<const uint16_t*>(host);
  bool host_ok = true;
  for (int i = 0; i < n; ++i)
    for (int l = 0; l < n_layers; ++l) {
      const size_t src = l * layer_elems + (size_t)spill[i].x * blk, dst = l * layer_elems + (size_t)fill[i].x * blk;
      memcpy(&kw[dst], &k[src], blk * 2);
      memcpy(&vw[dst], &v[src], blk * 2);
      const size_t h = (size_t)spill[i].y * 2 * n_layers;
      host_ok = host_ok && !memcmp(hp + (h + l) * blk, &k[src], blk * 2) && !memcmp(hp + (h + n_layers + l) * blk, &v[src], blk * 2);
    }
  if (!host_ok || k2 != kw || v2 != vw) {
    set_last_error(std::string("cl_op_kv_host_roundtrip: ") + (host_ok ? "the pool" : "a host page") + " differs from the expected bytes");
    return CL_ERR_INTERNAL;
  }
  if (iters > 0 && ms) {
    cudaEvent_t e0, e1, e2;
    CL_CUDA_OK(cudaEventCreate(&e0));
    CL_CUDA_OK(cudaEventCreate(&e1));
    CL_CUDA_OK(cudaEventCreate(&e2));
    CL_CUDA_OK(cudaEventRecord(e0, nullptr));
    for (int i = 0; i < iters; ++i) launch_kv_move(true, a, nullptr);
    CL_CUDA_OK(cudaEventRecord(e1, nullptr));
    for (int i = 0; i < iters; ++i) launch_kv_move(false, f, nullptr);
    CL_CUDA_OK(cudaEventRecord(e2, nullptr));
    CL_CUDA_OK(cudaEventSynchronize(e2));
    CL_CUDA_OK(cudaGetLastError());
    float t0 = 0.f, t1 = 0.f;
    CL_CUDA_OK(cudaEventElapsedTime(&t0, e0, e1));
    CL_CUDA_OK(cudaEventElapsedTime(&t1, e1, e2));
    ms[0] = t0 / (float)iters;
    ms[1] = t1 / (float)iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaEventDestroy(e2);
  }
  return CL_OK;
}

int cl_op_kv_shift(int device, int32_t n_layers, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t len, int32_t n_keep,
                   int32_t n_discard, const float* rope_row, const uint16_t* k, const uint16_t* v, uint16_t* k_out, uint16_t* v_out,
                   int32_t iters, float* ms) {
  if (n_layers <= 0 || n_kv <= 0 || len <= 0 || iters < 0 || !rope_row || !k || !v || !k_out || !v_out ||
      (head_dim != 64 && head_dim != 128) || (page_size != 16 && page_size != 32 && page_size != 64)) {
    set_last_error("cl_op_kv_shift: unsupported shape");
    return CL_ERR_INVALID_ARG;
  }
  int rc = check_device(device);
  if (rc) return rc;
  // the sequence's pages (one more than its tokens need, as after a reserve for the next token) scattered among 0..2 filler
  // pages each, seeded; every page the sequence does not hold names the largest finite bf16 (+ K, - V)
  const int P = page_size, np = (len + P - 1) / P + 1, n_pages = 3 * np + 2;
  KvPool pool(n_pages, P);
  std::mt19937 rng(0x5417);
  int fill = 0;
  for (int i = 0; i < np; ++i) {
    fill += (int)(rng() % 3);
    pool.reserve(1, fill * P);
    pool.reserve(0, (i + 1) * P);
  }
  const std::vector<int> before = pool.pages_of(0);
  const size_t blk = (size_t)n_kv * P * head_dim, layer_elems = (size_t)n_pages * blk, pool_elems = (size_t)n_layers * layer_elems;
  const size_t row = (size_t)n_kv * head_dim;
  auto at = [&](const std::vector<int>& pages, int l, int t, int g) {
    return (size_t)l * layer_elems + (size_t)pages[(size_t)t / P] * blk + ((size_t)g * P + t % P) * head_dim;
  };
  std::vector<uint16_t> kp(pool_elems, 0x7F7F), vp(pool_elems, 0xFF7F);
  for (int l = 0; l < n_layers; ++l)
    for (int t = 0; t < len; ++t)
      for (int g = 0; g < n_kv; ++g) {
        memcpy(&kp[at(before, l, t, g)], k + ((size_t)l * len + t) * row + (size_t)g * head_dim, (size_t)head_dim * 2);
        memcpy(&vp[at(before, l, t, g)], v + ((size_t)l * len + t) * row + (size_t)g * head_dim, (size_t)head_dim * 2);
      }
  std::vector<KvShiftItem> items;
  if ((rc = pool.shift(0, len, n_keep, n_discard, &items))) {
    set_last_error("cl_op_kv_shift: n_discard must be a positive multiple of page_size and n_keep + n_discard <= len");
    return rc;
  }
  const std::vector<int> after = pool.pages_of(0);
  DevBuf dk, dv, di, dr;
  CL_CUDA_OK(dk.upload(kp.data(), pool_elems * 2));
  CL_CUDA_OK(dv.upload(vp.data(), pool_elems * 2));
  CL_CUDA_OK(di.upload(items.data(), items.size() * sizeof(KvShiftItem)));
  CL_CUDA_OK(dr.upload(rope_row, (size_t)head_dim / 2 * sizeof(float2)));
  KvShiftArgs a;
  a.items = di.as<KvShiftItem>(); a.n_items = (int)items.size();
  a.kpool = dk.as<__nv_bfloat16>(); a.vpool = dv.as<__nv_bfloat16>(); a.layer_elems = layer_elems;
  a.n_layers = n_layers; a.n_kv = n_kv; a.head_dim = head_dim; a.page_size = P; a.rope_row = dr.as<float2>();
  if (launch_kv_shift(a, nullptr) < 0) {
    CL_CUDA_OK(cudaGetLastError());
    return CL_ERR_CUDA;
  }
  CL_CUDA_OK(cudaDeviceSynchronize());
  std::vector<uint16_t> k2(pool_elems), v2(pool_elems);
  CL_CUDA_OK(cudaMemcpy(k2.data(), dk.p, pool_elems * 2, cudaMemcpyDeviceToHost));
  CL_CUDA_OK(cudaMemcpy(v2.data(), dv.p, pool_elems * 2, cudaMemcpyDeviceToHost));
  // the sequence's rows out, then zeroed on both sides: everything else must be the bytes it was
  const int len2 = len - n_discard;
  for (int l = 0; l < n_layers; ++l)
    for (int t = 0; t < len2; ++t)
      for (int g = 0; g < n_kv; ++g) {
        const size_t e = at(after, l, t, g), o = ((size_t)l * len2 + t) * row + (size_t)g * head_dim;
        memcpy(k_out + o, &k2[e], (size_t)head_dim * 2);
        memcpy(v_out + o, &v2[e], (size_t)head_dim * 2);
        std::fill_n(&k2[e], head_dim, 0); std::fill_n(&v2[e], head_dim, 0);
        std::fill_n(&kp[e], head_dim, 0); std::fill_n(&vp[e], head_dim, 0);
      }
  if (k2 != kp || v2 != vp) {
    set_last_error("cl_op_kv_shift: an element outside the sequence's rows changed");
    return CL_ERR_INTERNAL;
  }
  if (iters > 0 && ms && !items.empty()) {
    cudaEvent_t e0, e1;
    CL_CUDA_OK(cudaEventCreate(&e0));
    CL_CUDA_OK(cudaEventCreate(&e1));
    launch_kv_shift(a, nullptr);   // warm-up
    CL_CUDA_OK(cudaEventRecord(e0, nullptr));
    for (int i = 0; i < iters; ++i) launch_kv_shift(a, nullptr);
    CL_CUDA_OK(cudaEventRecord(e1, nullptr));
    CL_CUDA_OK(cudaEventSynchronize(e1));
    CL_CUDA_OK(cudaGetLastError());
    float t = 0.f;
    CL_CUDA_OK(cudaEventElapsedTime(&t, e0, e1));
    *ms = t / (float)iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  return CL_OK;
}

int cl_op_attn_verify(int device, const uint16_t* q, const uint16_t* k_cache, const uint16_t* v_cache, const int32_t* ctx_lens,
                      const int32_t* rows, int32_t n_segs, int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t page_size, int32_t nsplit,
                      uint16_t* out, int32_t* nsplit_used) {
  if (!q || !k_cache || !v_cache || !ctx_lens || !rows || !out || n_segs <= 0 || nsplit < 0) return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  if (!attn_verify_tc_supported(n_heads, n_kv, head_dim, page_size) || nsplit > attn_verify_max_splits()) {
    set_last_error("the multi-row attention kernel does not take this shape or split count");
    return CL_ERR_INVALID_ARG;
  }
  const int P = page_size, HD = head_dim;
  const size_t qd = (size_t)n_heads * HD;
  std::vector<int> toks(n_segs);
  int T = 0, max_pages = 0;
  for (int s = 0; s < n_segs; ++s) {
    if (ctx_lens[s] < 0 || rows[s] < 1 || rows[s] > kVerifyMaxRows) {
      set_last_error("cl_op_attn_verify: every segment needs 1..16 rows and a cached length >= 0");
      return CL_ERR_INVALID_ARG;
    }
    toks[s] = ctx_lens[s] + rows[s];
    T += rows[s];
    max_pages = std::max(max_pages, (toks[s] + P - 1) / P);
  }
  OpKvPool pool;
  op_build_kv_pool(k_cache, v_cache, toks.data(), n_segs, n_kv, HD, P, &pool);
  // the engine's plan (Engine::verify_split_pages) unless nsplit is given: then every segment spreads its pages over nsplit
  const int split_pages = nsplit ? 0 : std::max(8, (max_pages + attn_verify_max_splits() - 1) / attn_verify_max_splits());
  std::vector<int> table(8 * (size_t)n_segs, 0);
  long long part = 0;
  int grid_splits = 1;
  for (int s = 0, r0 = 0; s < n_segs; r0 += rows[s], ++s) {
    const int pages = (toks[s] + P - 1) / P, ns = nsplit ? nsplit : (pages + split_pages - 1) / split_pages;
    int* e = &table[8 * (size_t)s];
    e[0] = s; e[1] = r0; e[2] = rows[s]; e[3] = ctx_lens[s]; e[4] = (int)part; e[5] = ns;
    if (ns > 1) part += (long long)n_kv * ns * 4 * rows[s] * (HD + 2);
    grid_splits = std::max(grid_splits, ns);
  }
  DevBuf dq, dk, dv, dbt, dseg, dout, dpart, dcnt;
  CL_CUDA_OK(dq.upload(q, (size_t)T * qd * 2));
  CL_CUDA_OK(dk.upload(pool.k.data(), pool.k.size() * 2));
  CL_CUDA_OK(dv.upload(pool.v.data(), pool.v.size() * 2));
  CL_CUDA_OK(dbt.upload(pool.bt.data(), pool.bt.size() * 4));
  CL_CUDA_OK(dseg.upload(table.data(), table.size() * 4));
  CL_CUDA_OK(dout.alloc((size_t)T * qd * 2));
  CL_CUDA_OK(dpart.alloc((size_t)part * 4));
  CL_CUDA_OK(dcnt.alloc((size_t)n_segs * n_kv * 4));
  CL_CUDA_OK(cudaMemset(dcnt.p, 0, (size_t)n_segs * n_kv * 4));
  const long long pool_rows = 2LL * pool.n_pages * n_kv * P;
  CUtensorMap km, vm;
  if (!make_tmap_2d_bf16(&km, dk.p, pool_rows, HD, 64, 32) || !make_tmap_2d_bf16(&vm, dv.p, pool_rows, HD, 64, 32)) {
    set_last_error("cl_op_attn_verify: tensor map creation failed");
    return CL_ERR_CUDA;
  }
  AttnVerifyArgs a;
  a.q = dq.as<__nv_bfloat16>(); a.q_stride = (int)qd; a.segs = dseg.as<int>(); a.block_tables = dbt.as<int>(); a.bt_stride = pool.bt_stride;
  a.out = dout.as<__nv_bfloat16>(); a.out_stride = (int)qd; a.part = dpart.as<float>(); a.counters = dcnt.as<unsigned>();
  a.n_segs = n_segs; a.n_heads = n_heads; a.n_kv = n_kv; a.head_dim = HD; a.page_size = P; a.nsplit = grid_splits; a.split_pages = split_pages;
  a.max_rows = *std::max_element(rows, rows + n_segs);
  // two launches without re-arming the split counters in between must give the same bits
  std::vector<uint16_t> first((size_t)T * qd);
  for (int run = 0; run < 2; ++run) {
    CL_CUDA_OK(cudaMemset(dout.p, 0xff, (size_t)T * qd * 2));   // NaN: every element must be written
    CL_CUDA_OK(cudaDeviceSynchronize());
    if (launch_attn_verify_tc(a, km, vm, pool_rows / 2, nullptr) < 0) {
      CL_CUDA_OK(cudaGetLastError());
      set_last_error("multi-row attention launch failed");
      return CL_ERR_CUDA;
    }
    CL_CUDA_OK(cudaDeviceSynchronize());
    CL_CUDA_OK(cudaMemcpy(run ? out : first.data(), dout.p, (size_t)T * qd * 2, cudaMemcpyDeviceToHost));
  }
  if (nsplit_used) *nsplit_used = grid_splits;
  if (memcmp(out, first.data(), first.size() * 2)) {
    set_last_error("cl_op_attn_verify: the second launch (split counters not reset) changed the output");
    return CL_ERR_INTERNAL;
  }
  return CL_OK;
}

int cl_op_qkv_rope_append(int device, int variant, const uint16_t* w_qkv, const float* h, const float* gain, float eps, int32_t d_model,
                          int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t pos, float rope_theta, float* q_out,
                          uint16_t* k_out, uint16_t* v_out) {
  if (!w_qkv || !h || !gain || !q_out || !k_out || !v_out || pos < 0) return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  const int HD = head_dim, half = HD / 2, P = 32;
  const int qd = n_heads * HD, kvd = n_kv * HD, rows = qd + 2 * kvd;
  if (!gemv_variant_supported(variant, rows, d_model) || (HD != 64 && HD != 128)) { set_last_error("unsupported shape"); return CL_ERR_INVALID_ARG; }
  // the engine stores q|k|v rows rope-pair-interleaved per head
  std::vector<uint16_t> wp((size_t)rows * d_model);
  for (int r = 0; r < rows; ++r) {
    const int head = r / HD, w = r % HD;
    const int rr = head * HD + (w < half ? 2 * w : 2 * (w - half) + 1);
    memcpy(&wp[(size_t)rr * d_model], w_qkv + (size_t)r * d_model, (size_t)d_model * 2);
  }
  std::vector<float2> rope((size_t)(pos + 1) * half);
  for (int p = 0; p <= pos; ++p)
    for (int i = 0; i < half; ++i) {
      const double inv = pow((double)rope_theta, -2.0 * (double)i / (double)HD);
      rope[(size_t)p * half + i] = make_float2((float)cos((double)p * inv), (float)sin((double)p * inv));
    }
  const int n_pages = pos / P + 1;
  std::vector<int> bt(n_pages);
  for (int i = 0; i < n_pages; ++i) bt[i] = n_pages - 1 - i;
  const size_t pool_elems = (size_t)n_pages * n_kv * P * HD;
  DevBuf dw, dh, dg, dr, dbt, dpos, dq, dk, dv;
  CL_CUDA_OK(dw.upload(wp.data(), wp.size() * 2));
  CL_CUDA_OK(dh.upload(h, (size_t)d_model * 4));
  CL_CUDA_OK(dg.upload(gain, (size_t)d_model * 4));
  CL_CUDA_OK(dr.upload(rope.data(), rope.size() * sizeof(float2)));
  CL_CUDA_OK(dbt.upload(bt.data(), bt.size() * 4));
  CL_CUDA_OK(dpos.upload(&pos, 4));
  CL_CUDA_OK(dq.alloc((size_t)qd * 4));
  CL_CUDA_OK(dk.alloc(pool_elems * 2));
  CL_CUDA_OK(dv.alloc(pool_elems * 2));
  GemvArgs a;
  a.W = dw.as<__nv_bfloat16>(); a.N = rows; a.K = d_model; a.h = dh.as<float>(); a.gain = dg.as<float>(); a.eps = eps;
  a.y = dq.as<float>(); a.x_stride = d_model; a.y_stride = qd; a.batch = 1;
  a.qkv.rope = dr.as<float2>(); a.qkv.pos = dpos.as<int>(); a.qkv.block_tables = dbt.as<int>(); a.qkv.bt_stride = n_pages;
  a.qkv.kpool = dk.as<__nv_bfloat16>(); a.qkv.vpool = dv.as<__nv_bfloat16>();
  a.qkv.n_heads = n_heads; a.qkv.n_kv = n_kv; a.qkv.head_dim = HD; a.qkv.page_size = P;
  if (launch_gemv(variant, EPI_QKV, true, a, nullptr, false) < 0) { CL_CUDA_OK(cudaGetLastError()); return CL_ERR_CUDA; }
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaMemcpy(q_out, dq.p, (size_t)qd * 4, cudaMemcpyDeviceToHost));
  const int page = bt[pos / P], off = pos % P;
  for (int g = 0; g < n_kv; ++g) {
    const size_t src = (((size_t)page * n_kv + g) * P + off) * HD;
    CL_CUDA_OK(cudaMemcpy(k_out + (size_t)g * HD, dk.as<uint16_t>() + src, (size_t)HD * 2, cudaMemcpyDeviceToHost));
    CL_CUDA_OK(cudaMemcpy(v_out + (size_t)g * HD, dv.as<uint16_t>() + src, (size_t)HD * 2, cudaMemcpyDeviceToHost));
  }
  return CL_OK;
}

// cl_op_sample, cl_op_sample_ext (ext: [n_rows], may be nullptr) and with top_n >= 0 cl_op_sample_logprobs (rows with
// temperature <= 0 then take the greedy choice)
static int op_sample(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const cl_sampling_ext* ext,
                     const int32_t* history, const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t top_n,
                     int32_t* ids_out, cl_token_logprob* lp_out) {
  if (!logits || n_rows <= 0 || vocab <= 1 || !sp || !n_history || !step || !ids_out) return CL_ERR_INVALID_ARG;
  if (top_n >= 0 && (top_n > kLogprobTopMax || !lp_out || vocab > kTailBlocks * kSampleSliceMax)) return CL_ERR_INVALID_ARG;
  const size_t R = (size_t)n_rows;
  std::vector<SampleParams> par(R);
  std::vector<int> ring(R * kSampleHistMax, 0), hlen(R), mode(R, 1);
  for (size_t r = 0; r < R; ++r) {
    SamplerExt x;
    if (int rc = read_sampling_ext(ext ? ext + r : nullptr, &x, nullptr)) return rc;
    if (top_n >= 0 && !(sp[r].temperature > 0.f)) mode[r] = 0;
    else if (!device_sampling_ok(sp[r], vocab, x)) { set_last_error("cl_op_sample: settings the device sampler does not cover"); return CL_ERR_INVALID_ARG; }
    const int n = n_history[r];
    if (n < 0 || (n > 0 && (!history || n > hist_stride))) return CL_ERR_INVALID_ARG;
    par[r] = sample_params(sp[r], x);
    for (int i = std::max(0, n - kSampleHistMax); i < n; ++i) ring[r * kSampleHistMax + i % kSampleHistMax] = history[r * hist_stride + i];
    hlen[r] = n;
  }
  int rc = check_device(device);
  if (rc) return rc;
  DevBuf dl, dpar, dstep, dhist, dhlen, dmode, dcand, dtok, dpos, dring, dsc, dval, didx, dcnt;
  CL_CUDA_OK(dl.upload(logits, R * vocab * 4));
  CL_CUDA_OK(dpar.upload(par.data(), R * sizeof(SampleParams)));
  CL_CUDA_OK(dstep.upload(step, R * 8));
  CL_CUDA_OK(dhist.upload(ring.data(), ring.size() * 4));
  CL_CUDA_OK(dhlen.upload(hlen.data(), R * 4));
  CL_CUDA_OK(dmode.upload(mode.data(), R * 4));
  CL_CUDA_OK(dcand.alloc(R * kTailBlocks * kSampleTopKMax * 8));
  CL_CUDA_OK(dtok.alloc(R * 4));
  CL_CUDA_OK(dpos.alloc(R * 4));
  CL_CUDA_OK(dring.alloc(R * 4));
  CL_CUDA_OK(dsc.alloc(4));
  CL_CUDA_OK(dval.alloc(R * kTailBlocks * 4));
  CL_CUDA_OK(didx.alloc(R * kTailBlocks * 4));
  CL_CUDA_OK(dcnt.alloc(R * 4));
  CL_CUDA_OK(cudaMemset(dtok.p, 0, R * 4));
  CL_CUDA_OK(cudaMemset(dpos.p, 0, R * 4));
  CL_CUDA_OK(cudaMemset(dsc.p, 0, 4));
  CL_CUDA_OK(cudaMemset(dcnt.p, 0, R * 4));
  StepTailArgs t;
  t.logits = dl.as<float>(); t.vocab = vocab; t.tok = dtok.as<int>(); t.pos = dpos.as<int>(); t.ids_ring = dring.as<int>();
  t.step_counter = dsc.as<int>(); t.ring_steps = 1; t.ring_stride = n_rows;
  t.part_val = dval.as<float>(); t.part_idx = didx.as<int>(); t.counters = dcnt.as<unsigned>(); t.batch = n_rows;
  t.sample.mode = dmode.as<int>(); t.sample.par = dpar.as<SampleParams>(); t.sample.step = dstep.as<unsigned long long>();
  t.sample.hist = dhist.as<int>(); t.sample.hist_len = dhlen.as<int>(); t.sample.cand = dcand.as<unsigned long long>();
  t.sample.push_input = 0;
  DevBuf dlpn, dlpart, dlcand, dlcnt, dlrec;
  if (top_n >= 0) {
    const std::vector<int> lpn(R, top_n);
    CL_CUDA_OK(dlpn.upload(lpn.data(), R * 4));
    CL_CUDA_OK(dlpart.alloc(R * kTailBlocks * sizeof(float2)));
    CL_CUDA_OK(dlcand.alloc(R * kTailBlocks * kLogprobTopMax * 8));
    CL_CUDA_OK(dlcnt.alloc(R * 4));
    CL_CUDA_OK(dlrec.alloc(R * sizeof(LogprobRecord)));
    CL_CUDA_OK(cudaMemset(dlcnt.p, 0, R * 4));
    t.lp.top_n = dlpn.as<int>(); t.lp.part = dlpart.as<float2>(); t.lp.cand = dlcand.as<unsigned long long>();
    t.lp.counters = dlcnt.as<unsigned>(); t.lp.last = dlrec.as<LogprobRecord>();
  }
  if (launch_step_tail(t, nullptr) < 0) { CL_CUDA_OK(cudaGetLastError()); set_last_error("launch_step_tail failed"); return CL_ERR_CUDA; }
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaMemcpy(ids_out, dtok.p, R * 4, cudaMemcpyDeviceToHost));
  if (top_n >= 0) {
    std::vector<LogprobRecord> rec(R);
    CL_CUDA_OK(cudaMemcpy(rec.data(), dlrec.p, R * sizeof(LogprobRecord), cudaMemcpyDeviceToHost));
    for (size_t r = 0; r < R; ++r) lp_out[r] = to_token_logprob(rec[r]);
  }
  return CL_OK;
}

int cl_op_sample(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const int32_t* history,
                 const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t* ids_out) {
  return op_sample(device, logits, n_rows, vocab, sp, nullptr, history, n_history, hist_stride, step, -1, ids_out, nullptr);
}

int cl_op_sample_ext(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const cl_sampling_ext* ext,
                     const int32_t* history, const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t* ids_out) {
  return op_sample(device, logits, n_rows, vocab, sp, ext, history, n_history, hist_stride, step, -1, ids_out, nullptr);
}

int cl_op_sample_logprobs(int device, const float* logits, int32_t n_rows, int32_t vocab, const cl_sampling* sp, const int32_t* history,
                          const int32_t* n_history, int32_t hist_stride, const uint64_t* step, int32_t top_n, int32_t* ids_out,
                          cl_token_logprob* lp_out) {
  if (top_n < 0) return CL_ERR_INVALID_ARG;
  return op_sample(device, logits, n_rows, vocab, sp, nullptr, history, n_history, hist_stride, step, top_n, ids_out, lp_out);
}

int cl_op_synth_weights(int device, uint64_t seed, int32_t tensor_key, int64_t n, float scale, uint16_t* out_bf16) {
  if (!out_bf16 || n <= 0) return CL_ERR_INVALID_ARG;
  int rc = check_device(device);
  if (rc) return rc;
  DevBuf d;
  CL_CUDA_OK(d.alloc((size_t)n * 2));
  if (launch_synth_bf16(d.as<__nv_bfloat16>(), n, (int)std::min<int64_t>(n, 4096), 1, 0, seed, tensor_key, scale, nullptr) < 0) return CL_ERR_CUDA;
  CL_CUDA_OK(cudaDeviceSynchronize());
  CL_CUDA_OK(cudaMemcpy(out_bf16, d.p, (size_t)n * 2, cudaMemcpyDeviceToHost));
  return CL_OK;
}

}  // extern "C"
