// Grid-barrier micro-benchmark for the one-kernel decode step (tools/ only, not part of the library).
// 132 CTAs (one per H100 SM) x 256 threads, cooperative launch, N barriers back to back; between two barriers each CTA writes one word and
// reads its neighbour's (so a broken barrier shows as a wrong value).  Variants:
//   0  flat counter: fence + red.release + ld.acquire spin   (what decode_mega_kernel does)
//   1  flat counter without the __threadfence
//   2  flag all-gather: st.release flags[cta], warp 0 polls all flags (no atomics)
//   3  two-level counters (8 groups, last arriver of a group bumps the top counter)
//   4  flat counter, the spin polls with ld.relaxed and one fence.acquire at the end
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
  unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void bar256() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <int V>
__device__ __forceinline__ void gsync(unsigned* ctr, unsigned* flags, unsigned* grp, unsigned n /* barrier number, 1-based */) {
  bar256();
  if (V == 0 || V == 1 || V == 4) {
    if (threadIdx.x == 0) {
      if (V != 1) __threadfence();
      asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ctr), "r"(1u) : "memory");
      const unsigned target = n * gridDim.x;
      if (V == 4) { while (ld_relaxed(ctr) < target) {} asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
      else        { while (ld_acquire(ctr) < target) {} }
    }
  } else if (V == 2) {
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0) { __threadfence(); asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flags + blockIdx.x), "r"(n) : "memory"); }
      const int G = gridDim.x;
      bool ok;
      do {
        ok = true;
        for (int i = threadIdx.x; i < G; i += 32) ok = ok && (ld_acquire(flags + i) >= n);
      } while (!__all_sync(0xffffffffu, ok));
    }
  } else if (V == 3) {
    if (threadIdx.x == 0) {
      __threadfence();
      const int g = blockIdx.x & 7;
      const unsigned gsize = (gridDim.x - g + 7) / 8;
      unsigned old;
      asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(grp + g * 32), "r"(1u) : "memory");
      if (old + 1 == n * gsize) asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ctr), "r"(1u) : "memory");
      while (ld_acquire(ctr) < n * 8) {}
    }
  }
  bar256();
}

template <int V>
__global__ void __launch_bounds__(256, 1) bench(unsigned* ctr, unsigned* flags, unsigned* grp, unsigned* data, int iters, int* bad) {
  const int G = gridDim.x, c = blockIdx.x;
  int wrong = 0;
  for (int it = 1; it <= iters; ++it) {
    if (threadIdx.x == 5) data[c * 32] = it;                  // some thread other than the one that signals
    gsync<V>(ctr, flags, grp, it);
    if (threadIdx.x == 9) { const unsigned v = __ldcg(data + ((c + 37) % G) * 32); wrong += (v != (unsigned)it && v != (unsigned)it + 1); }
  }
  if (wrong) atomicAdd(bad, wrong);
}

template <int V>
static void run(const char* name, int iters) {
  unsigned *ctr, *flags, *grp, *data; int* bad;
  cudaMalloc(&ctr, 4096); cudaMalloc(&flags, 4096); cudaMalloc(&grp, 4096); cudaMalloc(&data, 132 * 128); cudaMalloc(&bad, 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9f;
  int hbad = 0;
  for (int rep = 0; rep < 4; ++rep) {
    cudaMemset(ctr, 0, 4096); cudaMemset(flags, 0, 4096); cudaMemset(grp, 0, 4096); cudaMemset(data, 0, 132 * 128); cudaMemset(bad, 0, 4);
    void* args[] = {&ctr, &flags, &grp, &data, &iters, &bad};
    cudaEventRecord(e0);
    cudaError_t rc = cudaLaunchCooperativeKernel((void*)bench<V>, dim3(132), dim3(256), args, 0, 0);
    cudaEventRecord(e1);
    if (rc != cudaSuccess || cudaEventSynchronize(e1) != cudaSuccess) { printf("%s: launch failed: %s\n", name, cudaGetErrorString(cudaGetLastError())); return; }
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
    cudaMemcpy(&hbad, bad, 4, cudaMemcpyDeviceToHost);
  }
  printf("%-64s %7.3f us per barrier   (wrong reads: %d)\n", name, best * 1e3f / iters, hbad);
}

int main() {
  const int iters = 4000;
  run<0>("0 flat counter, fence + red.release + ld.acquire spin", iters);
  run<1>("1 flat counter, no __threadfence", iters);
  run<4>("4 flat counter, ld.relaxed spin + fence", iters);
  run<2>("2 flag all-gather (st.release flags[cta]; warp 0 polls 132 flags)", iters);
  run<3>("3 two-level counters (8 groups)", iters);
  return 0;
}
