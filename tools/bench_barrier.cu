// Stand-alone microbenchmark: cost of one grid-wide barrier among persistent CTAs (one per SM, sm_90a), idle and
// under a saturating background stream (a producer warp per CTA pulling 32 KB bulk copies, like the decode
// megakernel).  Variants of the arrive/poll protocol are compared.  Build + run: tools/bench_barrier.sh
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e_), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_volatile(const unsigned* p) { unsigned v; asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ long long gtime() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

struct Args {
  unsigned* cnt;        // [iters] one counter per barrier (variant 0/1/2) ; hierarchical: [iters][1 + NG]
  unsigned* flags;      // [grid] per-CTA generation flags (variant 3)
  const uint8_t* stream; size_t stream_bytes;
  float* sink; long long* t_out; unsigned long long* tiles_out;
  int iters, variant, bg, work;
};

constexpr int NG = 12;   // groups for the hierarchical variant

__device__ __forceinline__ void barrier(const Args& a, int it, int tid) {
  const unsigned G = gridDim.x;
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (a.variant == 0) {          // red.release + ld.acquire poll (what the decode kernel does)
    if (tid == 0) {
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.cnt + it) : "memory");
      while (ld_acquire(a.cnt + it) < G) {}
    }
  } else if (a.variant == 1) {   // fence + relaxed red, relaxed poll, fence
    if (tid == 0) {
      __threadfence();
      asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(a.cnt + it) : "memory");
      while (ld_relaxed(a.cnt + it) < G) {}
      __threadfence();
    }
  } else if (a.variant == 2) {   // hierarchical: NG group counters, last arriver bumps the top counter
    if (tid == 0) {
      unsigned* base = a.cnt + (size_t)it * (1 + NG);
      const unsigned grp = blockIdx.x % NG;
      const unsigned gsize = (G - grp + NG - 1) / NG;
      unsigned old;
      asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(base + 1 + grp) : "memory");
      if (old + 1 == gsize) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(base) : "memory");
      while (ld_acquire(base) < NG) {}
    }
  } else if (a.variant == 3) {   // flag array: every CTA publishes its generation, warp 0 polls all flags
    if (tid == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.flags + blockIdx.x), "r"((unsigned)(it + 1)) : "memory");
    if (tid < 32) {
      bool done;
      do {
        done = true;
        for (unsigned i = tid; i < G; i += 32) done &= ld_relaxed(a.flags + i) >= (unsigned)(it + 1);
        done = __all_sync(0xffffffffu, done);
      } while (!done);
      __threadfence();
    }
  } else if (a.variant == 4) {   // all 32 lanes of warp 0 poll the same counter (more polls in flight)
    if (tid == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.cnt + it) : "memory");
    if (tid < 32) {
      while (ld_acquire(a.cnt + it) < G) {}
    }
  } else if (a.variant == 5) {   // 8 warps' lane 0 poll staggered
    if (tid == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.cnt + it) : "memory");
    if ((tid & 31) == 0) { while (ld_volatile(a.cnt + it) < G) {} }
    __threadfence();
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

__global__ void __launch_bounds__(288, 1) bench_kernel(const Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t bar[6];
  __shared__ volatile int stop;
  const int tid = threadIdx.x;
  if (tid == 0) {
    stop = 0;
    for (int i = 0; i < 6; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar[i])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid >= 256) {
    // background stream: keep 6 x 32 KB bulk copies in flight until the consumers are done
    if (tid != 256 || !a.bg) return;
    uint32_t ph[6] = {0, 0, 0, 0, 0, 0};
    size_t off = (size_t)blockIdx.x * 32768;
    const int NF = a.bg;
    unsigned long long ntiles = 0;
    for (int i = 0; i < NF; ++i) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[i])), "r"(32768) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem + i * 32768)), "l"(a.stream + off), "r"(32768), "r"(smem_u32(&bar[i])) : "memory");
      off = (off + (size_t)gridDim.x * 32768) % a.stream_bytes;
    }
    int i = 0;
    while (!stop) {
      ++ntiles;
      uint32_t ok = 0;
      while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(&bar[i])), "r"(ph[i]) : "memory");
      ph[i] ^= 1u;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[i])), "r"(32768) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem + i * 32768)), "l"(a.stream + off), "r"(32768), "r"(smem_u32(&bar[i])) : "memory");
      off = (off + (size_t)gridDim.x * 32768) % a.stream_bytes;
      i = (i + 1) % NF;
    }
    a.tiles_out[blockIdx.x] = ntiles;
    // drain
    for (int k = 0; k < NF; ++k) {
      uint32_t ok = 0;
      while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(&bar[(i + k) % NF])), "r"(ph[(i + k) % NF]) : "memory");
    }
    return;
  }
  float acc = 0.f;
  long long t0 = 0;
  for (int it = 0; it < a.iters; ++it) {
    if (it == a.iters / 4 && tid == 0) t0 = gtime();
    // a little "phase work": each thread writes one float (like an epilogue) and spins `work` iterations
    a.sink[(size_t)blockIdx.x * 256 + tid] = acc;
    for (int w = 0; w < a.work; ++w) acc = fmaf(acc, 1.0001f, 0.5f);
    barrier(a, it, tid);
  }
  if (tid == 0) {
    a.t_out[blockIdx.x] = gtime() - t0;
    stop = 1;
  }
  a.sink[(size_t)blockIdx.x * 256 + tid] = acc;
}

int main() {
  int dev = 0;
  CK(cudaSetDevice(dev));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, dev));
  const int G = prop.multiProcessorCount, iters = 4000;
  unsigned *cnt, *flags;
  uint8_t* stream;
  float* sink;
  long long* t_out;
  unsigned long long* tiles_out;
  const size_t stream_bytes = (size_t)4 << 30;
  CK(cudaMalloc(&cnt, (size_t)iters * (1 + NG) * 4));
  CK(cudaMalloc(&flags, (size_t)G * 4));
  CK(cudaMalloc(&stream, stream_bytes));
  CK(cudaMemset(stream, 1, stream_bytes));
  CK(cudaMalloc(&sink, (size_t)G * 256 * 4));
  CK(cudaMalloc(&t_out, (size_t)G * 8));
  CK(cudaMalloc(&tiles_out, (size_t)G * 8));
  const size_t smem = 6 * 32768 + 1024;
  CK(cudaFuncSetAttribute(bench_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const char* names[] = {"red.release + ld.acquire poll", "fence + relaxed red/poll", "hierarchical (12 groups)", "flag array + warp poll",
                         "red.release + 32-lane acquire poll", "red.release + 8 volatile pollers", "no grid barrier (bar.sync only)"};
  for (int bg = 0; bg <= 6; ++bg)
    for (int variant = 0; variant < 7; variant += 6)
      for (int work = 2000; work <= 2000; work += 2000) {
        CK(cudaMemset(cnt, 0, (size_t)iters * (1 + NG) * 4));
        CK(cudaMemset(flags, 0, (size_t)G * 4));
        CK(cudaMemset(tiles_out, 0, (size_t)G * 8));
        Args a{cnt, flags, stream, stream_bytes, sink, t_out, tiles_out, iters, variant, bg, work};
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        CK(cudaEventRecord(e0));
        bench_kernel<<<G, 288, smem>>>(a);
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        long long t[256];
        CK(cudaMemcpy(t, t_out, (size_t)G * 8, cudaMemcpyDeviceToHost));
        const double per = (double)t[0] / (iters - iters / 4) / 1e3;
        unsigned long long tl[256]; double tot = 0;
        CK(cudaMemcpy(tl, tiles_out, (size_t)G * 8, cudaMemcpyDeviceToHost));
        for (int q = 0; q < G; ++q) tot += (double)tl[q];
        const double gbs = tot * 32768.0 / (ms * 1e-3) / 1e9;
        printf("{\"bench\": \"grid_barrier\", \"bg_stream\": %d, \"variant\": \"%s\", \"work_iters\": %d, \"us_per_iter\": %.3f, \"kernel_ms\": %.2f, \"stream_GBs\": %.0f}\n", bg,
               names[variant], work, per, ms, gbs);
        fflush(stdout);
      }
  return 0;
}
