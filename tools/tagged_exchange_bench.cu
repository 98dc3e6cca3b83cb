// Activation-exchange micro-benchmark for the one-kernel decode step (tools/ only, not part of the library).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tagged_exchange_bench tools/tagged_exchange_bench.cu
//
// What one phase boundary of decode_mega_kernel costs when the 64 x 768 bf16 GEMM operand crosses it
//   B  as today: the producing CTAs store bf16 pairs, grid barrier (bar.sync, red.release.gpu, ld.acquire spin, bar.sync),
//      then every CTA loads the whole operand in the A-fragment pattern of mega_load_a (32 contiguous bytes per thread
//      and k-step group, two ld.global.cg.v4 each);
//   T  tag-checked ("LL") exchange: every bf16 pair travels as one 8-byte word {payload, tag} written with one relaxed
//      64-bit store and no fence; every CTA loads the same fragments, now 64 contiguous bytes per thread and group
//      (four ld.relaxed.gpu.v2.b64, each 64-bit element single-copy atomic) and re-loads every 16-byte piece whose two
//      tags do not yet carry the phase's value, until none is left.  No barrier.  T6 keeps all six k-step groups of a
//      thread in flight (192 registers of loaded words, more than the kernel has beside its 96 A registers), T3 two
//      halves of three, T1 one group at a time; the back-off forms sleep between two re-sweeps of a thread.
// One cooperative launch, one CTA per SM x 256 threads (8 warps: 4 row tiles x 2 k halves, as in the kernel), N phases
// back to back; in each phase every CTA produces 2-3 feature pairs of all 64 rows from what it loaded in the phase
// before, so every phase depends on the whole previous one, as the kernel's phases do.  The operand ping-pongs between
// two buffers: a CTA rewrites a buffer only after it has loaded the other one completely, which every CTA wrote after
// loading this one -- so no reader can still be waiting for the old contents.
// Also timed: the operand loads alone, bf16 (L = B without the stores and the barrier) and tagged (LT3 = T3 without the
// stores and the tag checks).
// Without the K/V and weight streams of the real kernel the release of B is cheaper than in place (it waits for the
// CTA's stores to be acknowledged), so B here is a lower bound on the barrier's cost.
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

constexpr int kRows = 64, kD = 768;

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void bar256() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void ldcg_v4(uint32_t (&r)[4], const void* p) {
  asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "l"(p) : "memory");
}
__device__ __forceinline__ void ld_tagged2(unsigned long long (&w)[2], const void* p) {
  asm volatile("ld.relaxed.gpu.global.v2.b64 {%0, %1}, [%2];" : "=l"(w[0]), "=l"(w[1]) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_tagged(void* p, uint32_t payload, uint32_t tag) {
  const unsigned long long w = (static_cast<unsigned long long>(tag) << 32) | payload;
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}

// V: 0 = B (barrier), 1 = T (tags, NJ k-step groups in flight at once), 2 = L (loads only), 3 = T's loads alone
template <int V, int NJ = 6, int BACKOFF = 0>
__global__ void __launch_bounds__(256, 1) bench(uint16_t* bf, unsigned long long* tg, unsigned* ctr, int iters, unsigned tag0,
                                                unsigned* sink, int* bad) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, mt = warp & 3, kh = warp >> 2;
  const int g = lane >> 2, t = lane & 3, r0 = mt * 16 + g, r1 = r0 + 8;
  const int c = blockIdx.x;
  uint32_t acc = c;
  for (int it = 1; it <= iters; ++it) {
    const unsigned tag = tag0 + it;
    const int buf = it & 1;
    // ---- produce: CTA c owns feature pairs c, c + G, c + 2G of all 64 rows (kh == 0 warps store, like the epilogue) ----
    if ((V == 0 || V == 1) && kh == 0) {
      for (int pr = c + static_cast<int>(gridDim.x) * t; pr < kD / 2; pr += 4 * static_cast<int>(gridDim.x)) {
        const int f = 2 * pr;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = hh ? r1 : r0;
          const uint32_t v = acc + static_cast<uint32_t>(r * kD + f) + it;
          if (V == 0) *reinterpret_cast<uint32_t*>(bf + (static_cast<size_t>(buf) * kRows + r) * kD + f) = v;
          else st_tagged(tg + (static_cast<size_t>(buf) * kRows + r) * (kD / 2) + f / 2, v, tag);
        }
      }
    }
    if (V == 0) {
      bar256();
      if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ctr), "r"(1u) : "memory");
        unsigned spins = 0;
        while (ld_acquire(ctr) < static_cast<unsigned>(it) * gridDim.x)
          if (++spins > (1u << 22) || ((spins & 1023u) == 0 && *reinterpret_cast<volatile int*>(bad) != 0)) { atomicAdd(bad, 1); break; }
      }
      bar256();
    }
    // ---- consume: this warp's 16 rows x 384 k of the whole operand ----
    uint32_t x = 0;
    if (V == 0 || V == 2) {
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        uint32_t a[4][4];
        const uint16_t* p0 = bf + (static_cast<size_t>(buf) * kRows + r0) * kD + kh * 384 + 64 * j + 16 * t;
        const uint16_t* p1 = p0 + 8 * kD;
        ldcg_v4(a[0], p0); ldcg_v4(a[1], p0 + 8); ldcg_v4(a[2], p1); ldcg_v4(a[3], p1 + 8);
#pragma unroll
        for (int q = 0; q < 4; ++q) x ^= a[q][0] ^ a[q][1] ^ a[q][2] ^ a[q][3];
      }
    } else {
      // NJ of the six k-step groups in flight at once (8 pieces of 16 bytes each); a sweep re-issues every piece whose
      // tags are not yet the phase's, all at once, until none is left
      const unsigned long long* base = tg + (static_cast<size_t>(buf) * kRows + r0) * (kD / 2) + (kh * 384 + 16 * t) / 2;
#pragma unroll
      for (int j0 = 0; j0 < 6; j0 += NJ) {
        unsigned long long w[NJ][8][2];
        auto piece = [&](int j, int q) { return base + (q >> 2) * 8 * (kD / 2) + 32 * (j0 + j) + 2 * (q & 3); };
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int q = 0; q < 8; ++q) ld_tagged2(w[j][q], piece(j, q));
        for (unsigned spins = 0;; ++spins) {
          bool done = true;
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int q = 0; q < 8; ++q)
              if (V == 1 && (static_cast<uint32_t>(w[j][q][0] >> 32) != tag || static_cast<uint32_t>(w[j][q][1] >> 32) != tag)) {
                done = false;
                ld_tagged2(w[j][q], piece(j, q));
              }
          if (done) break;
          // bounded; once any wait has given up, every other one gives up at once, so a broken run ends quickly
          if (spins > (1u << 20) || ((spins & 255u) == 255u && *reinterpret_cast<volatile int*>(bad) != 0)) { atomicAdd(bad, 1); break; }
          if (BACKOFF) __nanosleep(BACKOFF);
        }
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int q = 0; q < 8; ++q) x ^= static_cast<uint32_t>(w[j][q][0]) ^ static_cast<uint32_t>(w[j][q][1]);
      }
    }
    // a value the next phase's stores depend on (all four row tiles x both k halves of the CTA)
    acc += __shfl_xor_sync(0xffffffffu, x, 1) & 1u;
    bar256();                              // stands for the K-half exchange every GEMM phase has
  }
  if (threadIdx.x == 0) sink[c] = acc;
}

template <int V, int NJ = 6, int BACKOFF = 0>
static float run(int iters, unsigned& tag0) {
  static uint16_t* bf = nullptr; static unsigned long long* tg = nullptr; static unsigned *ctr = nullptr, *sink = nullptr; static int* bad = nullptr;
  if (!bf) {
    cudaMalloc(&bf, 2 * kRows * kD * 2); cudaMalloc(&tg, 2 * kRows * kD / 2 * 8); cudaMalloc(&ctr, 256); cudaMalloc(&sink, 4096);
    cudaMalloc(&bad, 4);
    cudaMemset(bf, 0, 2 * kRows * kD * 2); cudaMemset(tg, 0, 2 * kRows * kD / 2 * 8); cudaMemset(bad, 0, 4);
  }
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaMemset(ctr, 0, 256);
  cudaMemset(bad, 0, 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  void* args[] = {&bf, &tg, &ctr, &iters, &tag0, &sink, &bad};
  cudaEventRecord(e0);
  cudaError_t rc = cudaLaunchCooperativeKernel((void*)bench<V, NJ, BACKOFF>, dim3(sms), dim3(256), args, 0, 0);
  cudaEventRecord(e1);
  if (rc != cudaSuccess || cudaEventSynchronize(e1) != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(cudaGetLastError())); return -1.f; }
  tag0 += iters;                     // tags of the next launch never match words this one wrote
  int hbad = 0;
  cudaMemcpy(&hbad, bad, 4, cudaMemcpyDeviceToHost);
  if (hbad) printf("  %d bounded waits gave up\n", hbad);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return ms * 1e3f / iters;
}

int main() {
  const int iters = 4000;
  unsigned tag0 = 0;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs; one phase = every CTA produces part of 64 x 768 bf16 and loads all of it\n", prop.name, prop.multiProcessorCount);
  constexpr int kN = 8;
  const char* names[kN] = {"B  barrier + bf16 operand", "T6 tags, whole operand in flight", "T3 tags, two halves in flight",
                           "T1 tags, one k-step group in flight", "T3 + 200 ns back-off per re-sweep",
                           "T3 + 1000 ns back-off per re-sweep", "L  bf16 operand loads alone",
                           "LT3 tagged operand loads alone (halves)"};
  float best[kN];
  for (int k = 0; k < kN; ++k) best[k] = 1e9f;
  for (int rep = 0; rep < 5; ++rep) {     // alternating rounds; the best of each
    const float v[kN] = {run<0>(iters, tag0), run<1, 6>(iters, tag0), run<1, 3>(iters, tag0), run<1, 1>(iters, tag0),
                         run<1, 3, 200>(iters, tag0), run<1, 3, 1000>(iters, tag0), run<2>(iters, tag0), run<3, 3>(iters, tag0)};
    printf("  round %d:", rep);
    for (int k = 0; k < kN; ++k) {
      printf("  %.3f", v[k]);
      if (v[k] > 0 && v[k] < best[k]) best[k] = v[k];
    }
    printf(" us per phase\n");
    fflush(stdout);
  }
  for (int k = 0; k < kN; ++k) printf("%-40s %7.3f us per phase\n", names[k], best[k]);
  return 0;
}
