// One persistent kernel per greedy decode step (<= 64 sequences): the 6 decoder layers, the tied LM head with the
// arg-max / log-sum-exp folded into it, the reference's greedy bookkeeping and the next step's token embedding
// (reference layers/decoder.py:313-417, 65-78; layers/bert/modeling_bert.py:92-334) -- replacing the 45-launch chain of
// gitb200.cu::step_layers for that case.
//
// Why: at <= 64 rows every kernel of the chain is latency bound (TMA -> tensor core -> epilogue -> flag per hop, far above
// the HBM floor of the step's weight bytes).  Here the HBM stream is decoupled from the dependency chain:
//   * one CTA per SM (132 on an H100; cooperative launch), 8 compute warps + 1 producer warp each;
//   * every byte the step reads from HBM -- the weight tiles a CTA owns in each GEMM phase, the image K/V of its attention
//     items and the text K/V so far -- flows through a 12 x 16 KB shared-memory ring that the producer warp fills in
//     program order with TMA (bulk copies of pre-packed weight tiles, swizzled K | V boxes of up to 64 keys: only the key
//     rows attention reads), running as far ahead of the compute warps as the ring allows, across phase boundaries (only
//     the text K/V of the CURRENT layer waits for that layer's QKV phase);
//   * phases (QKV | attention | out-proj | LN | fc1 | fc2 | LN per layer, then LM head | selection + embedding) are
//     separated by a grid barrier (one release-add + acquire-spin on a global counter -- the cheapest of
//     the variants tools/barrier_bench.cu times); what crosses a barrier is only the <= 64-row activations, read straight
//     from L2 into mma.sync fragments;
//   * weights are stationary per CTA: a GEMM phase gives CTA c a few 8-feature tiles over a 768-long reduction; the 8 warps
//     split a tile 4 row tiles x 2 K halves.  The 288 q | k | v tiles go out two per CTA, three for the first 288 - 2G.  fc2 (K = 3072) is dealt as 4 k slices x 96 feature tiles over 128 CTAs, its
//     four partial sums meet in slice order in the LayerNorm phase: no atomics anywhere, the step is bit-reproducible.  One
//     schedule (mega_tiles) says which tiles a CTA owns, for the producer and the compute warps alike, and every GEMM phase
//     runs through one routine (mega_gemm);
//   * attention: the 64-key chunks of a CTA's (sequence, head) items are dealt round-robin to its 8 warps, online-softmax
//     states in shared memory, fixed-order merge.
// The skinny GEMMs and the 1-row attention are HBM-bound byte work (arithmetic intensity ~rows FLOP/B): they use the
// warp-level mma.sync path fed from shared memory; wgmma stays with the compute-bound encoder and prefill GEMMs:
// with the weights as the M operand a wgmma tile needs >= 64 weight rows per CTA (3/4 of the SMs, and of the HBM stream,
// would idle in the layer GEMMs); with the activations as the M operand every CTA would have to stage the 64 x 768
// activations (96 KB) in shared memory in every phase, which the 192 KB ring leaves no room for.
#pragma once
#include "ptx.cuh"
#include "rowops.cuh"

#include <type_traits>

namespace gitb200 {

constexpr int kMegaComputeWarps = 8;
constexpr int kMegaThreads = (kMegaComputeWarps + 1) * 32;
constexpr int kMegaSlots = 12;
constexpr int kMegaSlotBytes = 16384;
constexpr int kMegaTileBytes = 12288;      // 8 output features x 768 k x bf16, in mma-fragment order (pack_tiles_kernel)
constexpr int kMegaKvRows = 64;            // keys per attention chunk: one ring slot = K half (8 KB) | V half (8 KB)
constexpr int kMegaKvSubRows = 16;         // a chunk of fewer keys is fetched in 16-row sub-boxes (2 KB of K, 2 KB of V each)
constexpr int kMegaMaxRows = 64;
constexpr int kMegaD = 768, kMegaF = 3072, kMegaH = 12;
constexpr int kMegaAttItems = 6;           // (sequence, head) attention items of the busiest CTA: ceil(64 * 12 / 132)
constexpr int kMegaOutTiles = kMegaD / 8;  // 96 tiles of 8 output features: out-proj (one per CTA), fc2
constexpr int kMegaQkvTiles = 3 * kMegaD / 8;                  // 288 q | k | v tiles, 2-3 per CTA (needs G >= 96)
constexpr int kMegaFcTilesPerCta = 3;                          // fc1 / fc2 tiles per CTA
constexpr int kMegaFcCtas = kMegaF / 8 / kMegaFcTilesPerCta;   // 128 CTAs take fc1's 384 tiles and fc2's 96 x 4 k slices
constexpr int kMegaFc2Slices = kMegaF / kMegaD;                // fc2's 3072-long reduction as 4 slices of 768
constexpr int kMegaMinCtas = kMegaFcCtas;  // attention also needs ceil(64 * 12 / G) <= 6
constexpr int kMegaAttState = 72;          // floats per (item, warp) softmax state: 64 output dims, running max, 4 lane sums
constexpr unsigned int kMegaSpinLimit = 1u << 18;   // bounded waits: a protocol bug must end in an error code, not a hung device

struct MegaLayer {
  const uint8_t* wqkv;     // [288] tiles: features 8t .. 8t+7 of the fused q | k | v projection
  const uint8_t* wo;       // [96]
  const uint8_t* w1;       // [384]
  const uint8_t* w2;       // [96][4]: feature tile x 768-wide k slice (mega_w2_tile)
  const float* bqkv; const float* bo; const float* b1; const float* b2;
  const float* lnag; const float* lnab; const float* lnog; const float* lnob;
  __nv_bfloat16* txt_k;    // [R, T_alloc, 768]
  __nv_bfloat16* txt_v;
};

struct MegaParams {
  MegaLayer layer[6];
  const uint8_t* lm;       // [ceil(V / 8)] tiles of the tied word-embedding matrix
  const float* lm_bias;
  const float* words;      // fp32 [V, 768] (embedding gather)
  const float* positions;  // fp32 [max_pos, 768]
  const float* lnemb_g; const float* lnemb_b;
  int M, T_alloc, n_layers;
  // activations (global, L2 resident)
  float* x;                // [R, 768] residual stream (post-LayerNorm)
  float* y;                // [R, 768] pre-LayerNorm sum (after the attention block)
  float* ypart;            // [4][R, 768] fc2 partial sums of the four 768-wide k slices (summed in slice order by the LN)
  __nv_bfloat16* hb;       // [R, 768] bf16 copy of x (GEMM operand)
  __nv_bfloat16* qb;       // [R, 768] q (+bias) / 8
  __nv_bfloat16* ctx;      // [R, 768]
  __nv_bfloat16* ub;       // [R, 3072]
  // the search state greedy_select_kernel works on (R = sel.rows, V = sel.V); the LM-head partials are [R, gridDim.x]
  SelectParams sel;
  unsigned int* barrier;   // [2] grid-barrier counters, used alternately by successive steps
  int* error;              // set non-zero when a bounded spin gave up (the host reports it)
};

// ---- the tile schedule: what CTA `cta` of G owns in each GEMM phase ----------------------------------------------------
// The producer walks it to fill the ring and the compute warps to take the ring's chunks in the same order; fc2's weights are
// packed by mega_w2_tile to match.  (The attention chunks of a CTA are dealt in the kernel's prologue: round_keys.)
enum MegaGemm { kGemmQkv, kGemmOut, kGemmFc1, kGemmFc2, kGemmLm };
struct MegaTiles {
  int t0, n, stride;   // tiles t0 + j * stride (j < n) of the phase's packed weight buffer
  int f0;              // tile j computes output features 8 (f0 + j) .. 8 (f0 + j) + 7
  int a_col;           // first column of the A operand (fc2: the CTA's k slice)
};
__device__ __forceinline__ int mega_lm_per(int V, int G) { return ((V + 7) / 8 + G - 1) / G; }
// fc2's packed weights: the tile of features 8f .. 8f + 7 over k slice s (k = 768 s .. 768 s + 767)
__host__ __device__ constexpr int mega_w2_tile(int f, int s) { return f * kMegaFc2Slices + s; }
__device__ __forceinline__ MegaTiles mega_tiles(MegaGemm ph, int cta, int G, int V, int lm_per) {
  if (ph == kGemmQkv) {   // one pass: two each, three for the first 288 - 2G CTAs when G < 144 (contiguous ranges)
    const int extra = max(0, kMegaQkvTiles - 2 * G);
    const int t0 = (cta < extra) ? 3 * cta : 2 * cta + extra;
    return {t0, (cta < extra) ? 3 : max(0, min(2, kMegaQkvTiles - t0)), 1, t0, 0};
  }
  if (ph == kGemmOut) return {cta, cta < kMegaOutTiles ? 1 : 0, 1, cta, 0};
  if (ph == kGemmFc1) {
    const int t0 = cta * kMegaFcTilesPerCta;
    return {t0, cta < kMegaFcCtas ? kMegaFcTilesPerCta : 0, 1, t0, 0};
  }
  if (ph == kGemmFc2) {   // feature group cta / 4 (3 tiles) x k slice cta % 4
    const int f0 = (cta / kMegaFc2Slices) * kMegaFcTilesPerCta, ks = cta % kMegaFc2Slices;
    return {mega_w2_tile(f0, ks), cta < kMegaFcCtas ? kMegaFcTilesPerCta : 0, mega_w2_tile(1, 0), f0, ks * kMegaD};
  }
  const int t0 = cta * lm_per;   // LM head: ceil(V / 8) tiles in contiguous ranges of lm_per = mega_lm_per(V, G)
  return {t0, max(0, min(lm_per, (V + 7) / 8 - t0)), 1, t0, 0};
}

// ---- packing: [N, K] row-major bf16 -> tiles of 8 features x 768 k in fragment order ------------------------------------
// Tile layout: 48 k-steps x 32 lanes x 8 bytes.  Lane (g = lane / 4, t = lane % 4) of k-step s holds the four k values
// k0 + 64 * (s / 4) + 16 t + 4 (s % 4) + {0, 1, 2, 3} of feature 8 tile + g: the B fragment (b0 = first pair, b1 = second
// pair) of an m16n8k16 MMA whose k index has been permuted so that the matching A fragment is 16 CONTIGUOUS bf16 per
// thread and group of four k-steps -- 32 contiguous bytes of the row-major activation matrix, and the four lanes of a row
// together fetch one whole 128-byte line.
__global__ void __launch_bounds__(256) pack_tiles_kernel(const __nv_bfloat16* __restrict__ W, long long ldw, int n_feat, int k0,
                                                         uint8_t* __restrict__ dst, long long n_tiles, int tile_stride_tiles,
                                                         int tile_offset) {
  const long long total = n_tiles * 48 * 32;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int lane = static_cast<int>(i & 31);
    const int s = static_cast<int>((i >> 5) % 48);
    const long long tile = i / (48 * 32);
    const int g = lane >> 2, t = lane & 3;
    const long long f = tile * 8 + g;
    const int k = k0 + 64 * (s >> 2) + 16 * t + 4 * (s & 3);
    uint2 v = make_uint2(0u, 0u);
    if (f < n_feat) v = *reinterpret_cast<const uint2*>(W + f * ldw + k);
    *reinterpret_cast<uint2*>(dst + (tile * tile_stride_tiles + tile_offset) * kMegaTileBytes + (s * 32 + lane) * 8) = v;
  }
}

// ---- small device helpers ------------------------------------------------------------------------------------------------
// Fine-grained marks of the debug timeline build (tools/mega_timeline.py): thread 0 of CTA 0 stores (%clock64, id) pairs
// into a slice of the timeline buffer reserved once per launch -- no atomics or %globaltimer reads inside the phases.
#ifdef GITB200_TIMELINE
struct MegaTl {
  unsigned long long* buf;
  unsigned int n;
  __device__ __forceinline__ void begin() {
    buf = nullptr; n = 0;
    if (g_tl_buf != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
      const unsigned int i = atomicAdd(&g_tl_count, 160u);
      if (i + 160u <= kTimelineMax) {
        buf = g_tl_buf + 2 * i;
        for (int k = 0; k < 160; ++k) { buf[2 * k] = 0ull; buf[2 * k + 1] = 0ull; }
        mark(700000); buf[2 * n] = globaltimer_ns(); buf[2 * n + 1] = 700001ull; ++n;
      }
    }
  }
  __device__ __forceinline__ void mark(int kid) {
    if (buf != nullptr && n < 160u) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%clock64;" : "=l"(t));
      buf[2 * n] = t; buf[2 * n + 1] = static_cast<unsigned long long>(kid); ++n;
    }
  }
  __device__ __forceinline__ void end() {
    if (buf != nullptr) { mark(700002); if (n < 160u) { buf[2 * n] = globaltimer_ns(); buf[2 * n + 1] = 700003ull; ++n; } }
  }
};
#define MEGA_TL(kid) tlf.mark(kid)
// makes the next mark wait until the A operand's loads have landed
#define MEGA_TL_DEP(a, error) if (((a).lo[5][7] ^ (a).hi[5][7] ^ (a).lo[0][0]) == 0x9E3779B9u) *(error) = kWaitTimelineProbe;
#else
struct MegaTl {
  __device__ __forceinline__ void begin() {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void end() {}
};
#define MEGA_TL(kid)
#define MEGA_TL_DEP(a, error)
#endif

__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// false: gave up (or another wait already had: once the error word is set every further wait returns at once, so a broken
// launch drains in microseconds instead of timing out chunk by chunk)
__device__ __forceinline__ bool mbar_wait_bounded(uint64_t* bar, uint32_t parity, const int* error) {
  for (unsigned int i = 0; i < kMegaSpinLimit; ++i) {
    if (mbar_try_wait(bar, parity)) return true;
    if ((i & 1023u) == 1023u && *reinterpret_cast<const volatile int*>(error) != 0) return false;
  }
  return false;
}

struct MegaRing {
  uint8_t* base;
  uint64_t* full;
  uint64_t* empty;
  uint32_t idx;      // chunks consumed so far (identical in every compute warp)
  int* error;
  volatile uint32_t* issued;   // chunks the producer has armed so far (shared memory)
  __device__ __forceinline__ const uint8_t* acquire() {
    const uint32_t slot = idx % kMegaSlots;
    if (!mbar_wait_bounded(&full[slot], (idx / kMegaSlots) & 1, error)) *error = kWaitRingFull;
    return base + slot * kMegaSlotBytes;
  }
  // chunk idx + n (n < kMegaSlots) without consuming it: the GEMM phases take all tiles of a batch first, so that the MMAs
  // of one tile overlap the shared-memory reads, the K-half exchange and the epilogue of its neighbours
  __device__ __forceinline__ const uint8_t* acquire_ahead(uint32_t n) {
    const uint32_t i = idx + n, slot = i % kMegaSlots;
    if (!mbar_wait_bounded(&full[slot], (i / kMegaSlots) & 1, error)) *error = kWaitRingFull;
    return base + slot * kMegaSlotBytes;
  }
  __device__ __forceinline__ void release() {   // every compute warp, once per chunk
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[idx % kMegaSlots]);
    ++idx;
  }
  // a chunk that ONE warp consumes alone (attention items): that warp waits for it by index and frees it for all eight
  // (A parity wait alone would be ambiguous here: the warps of a CTA walk different items, so a warp may ask for a chunk
  //  whose slot is still two uses back.  It first waits until the producer has ARMED chunk i -- from then until this very
  //  warp releases it, the slot's barrier can only be in chunk i's phase -- and only then for the phase to complete.)
  __device__ __forceinline__ uint8_t* acquire_at(uint32_t i) {
    const uint32_t slot = i % kMegaSlots;
    unsigned int spins = 0;
    while (*issued <= i) {
      if (++spins > (kMegaSpinLimit << 4) || ((spins & 1023u) == 1023u && *reinterpret_cast<const volatile int*>(error) != 0)) { *error = kWaitRingArmed; break; }
    }
    if (!mbar_wait_bounded(&full[slot], (i / kMegaSlots) & 1, error)) *error = kWaitRingFull;
    return base + slot * kMegaSlotBytes;
  }
  __device__ __forceinline__ void release_at(uint32_t i) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0)
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&empty[i % kMegaSlots])), "r"(kMegaComputeWarps) : "memory");
  }
};

// Grid barrier between phases (compute warps only: 256 threads; the producer warp never waits for a phase).
__device__ __forceinline__ void mega_grid_sync(unsigned int* counter, unsigned int& epoch, int* error, MegaTl& tlf, int tl_id = 0) {
  if (tl_id) tlf.mark(tl_id + 5);                                   // this warp's phase work issued
  named_bar_sync(1, kMegaComputeWarps * 32);
  if (threadIdx.x == 0) {
    epoch += gridDim.x;
    if (tl_id) tlf.mark(tl_id + 6);                                 // all compute warps of the CTA are here
    else tl_mark_one(500000 + static_cast<int>(epoch / gridDim.x)); // this CTA arrived at barrier #n
    // release-RMW at gpu scope: cumulative over the CTA's writes that the bar.sync above ordered before this thread, so
    // no separate fence -- __threadfence() is a sequentially-consistent fence (MEMBAR.SC.GPU + L1 invalidate) that would
    // come on top of the release's own MEMBAR.ALL.GPU
    if (tl_id) tlf.mark(tl_id + 7);
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(counter), "r"(1u) : "memory");
    if (tl_id) tlf.mark(tl_id + 8);
    unsigned int spins = 0;
    while (ld_acquire_gpu(counter) < epoch) {
      if (++spins > kMegaSpinLimit || ((spins & 255u) == 255u && *reinterpret_cast<const volatile int*>(error) != 0)) {
        if (*reinterpret_cast<const volatile int*>(error) == 0) *error = kWaitGridBarrier;
        break;
      }
    }
    if (tl_id) tlf.mark(tl_id + 9);
    else tl_mark_one(600000 + static_cast<int>(epoch / gridDim.x)); // barrier #n released
  }
  named_bar_sync(1, kMegaComputeWarps * 32);
  if (tl_id) tlf.mark(tl_id + 10);
}

// A operand of one GEMM phase: this warp's 16 rows x 384 k of a row-major bf16 activation matrix, straight from L2.
struct MegaAFrag {
  uint32_t lo[6][8];   // row g     : 16 contiguous k per entry (four k-steps)
  uint32_t hi[6][8];   // row g + 8
};
// 32 contiguous bytes (sm_90 has no 256-bit loads: two 128-bit ones).  Cached in L1: each of the two instructions covers
// half of every 32-byte sector of the four lanes' 128-byte line, so with L2-only (.cg) loads the second one fetched the
// same sectors from L2 again -- twice the operand's bytes through the SM's L2 port per phase.  Weak loads are safe here:
// the operand was written before the grid barrier this CTA passed, whose acquire load invalidates the SM's L1
// (CCTL.IVALL), or by an earlier launch.
__device__ __forceinline__ void ld_256(uint32_t (&r)[8], const void* p) {
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "l"(p));
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
               : "l"(static_cast<const uint8_t*>(p) + 16));
}
__device__ __forceinline__ void mega_load_a(MegaAFrag& a, const __nv_bfloat16* A, long long lda, int rows, int mt, int kh, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int r0 = mt * 16 + g, r1 = r0 + 8;
  const __nv_bfloat16* p0 = A + static_cast<long long>(r0) * lda + kh * 384 + 16 * t;
  const __nv_bfloat16* p1 = A + static_cast<long long>(r1) * lda + kh * 384 + 16 * t;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    if (r0 < rows) ld_256(a.lo[j], p0 + 64 * j);
    else {
#pragma unroll
      for (int e = 0; e < 8; ++e) a.lo[j][e] = 0u;
    }
    if (r1 < rows) ld_256(a.hi[j], p1 + 64 * j);
    else {
#pragma unroll
      for (int e = 0; e < 8; ++e) a.hi[j][e] = 0u;
    }
  }
}
// c += A(16 x 384 of this warp) * tile(8 features, this warp's k half), NT tiles at once.  Per tile two independent
// accumulators (even / odd k-steps, added in a fixed order: bit-reproducible) -- a single one would serialise 24 dependent
// MMAs; across the NT tiles the 2 NT chains of a warp keep the tensor pipe busy over the MMA latency, and the NT tiles
// share one K-half exchange.  (9 warps cap the kernel at 168 registers per thread: NT <= 3.)
template <int NT>
__device__ __forceinline__ void mega_mma_tiles(float (&c)[NT][4], const MegaAFrag& a, const uint8_t* const (&tile)[NT], int kh, int lane) {
  const uint2* bp[NT];
  float c1[NT][4];
#pragma unroll
  for (int n = 0; n < NT; ++n) {
    bp[n] = reinterpret_cast<const uint2*>(tile[n]) + kh * 24 * 32 + lane;
    c1[n][0] = c1[n][1] = c1[n][2] = c1[n][3] = 0.f;
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      const uint32_t a0[4] = {a.lo[j][2 * i], a.hi[j][2 * i], a.lo[j][2 * i + 1], a.hi[j][2 * i + 1]};
      const uint32_t a1[4] = {a.lo[j][2 * i + 2], a.hi[j][2 * i + 2], a.lo[j][2 * i + 3], a.hi[j][2 * i + 3]};
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const uint2 b0 = bp[n][(4 * j + i) * 32];
        const uint2 b1 = bp[n][(4 * j + i + 1) * 32];
        mma_bf16_16816(c[n], a0, b0.x, b0.y);
        mma_bf16_16816(c1[n], a1, b1.x, b1.y);
      }
    }
  }
#pragma unroll
  for (int n = 0; n < NT; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) c[n][e] += c1[n][e];
}
// Sum of the two K halves of NT tiles behind one named barrier: the kh = 1 warp parks its accumulators in shared memory,
// its kh = 0 partner adds them.  Returns true in the warp that owns the result.  `red` = [2 buffers][3 tiles][4 row tiles][32 lanes] float4 (12 KB).
template <int NT>
__device__ __forceinline__ bool mega_combine_n(float (&c)[NT][4], float4* red, int buf, int mt, int kh, int lane) {
  float4* slot = red + (buf * 12 + mt) * 32 + lane;
  if (kh == 1) {
#pragma unroll
    for (int n = 0; n < NT; ++n) slot[n * 128] = make_float4(c[n][0], c[n][1], c[n][2], c[n][3]);
  }
  named_bar_sync(2 + mt, 64);
  if (kh == 0) {
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const float4 o = slot[n * 128];
      c[n][0] += o.x; c[n][1] += o.y; c[n][2] += o.z; c[n][3] += o.w;
    }
  }
  return kh == 0;
}
// Two-way variant for the LM head: both warps of a pair end up with the sum (kh0 + kh1, the same operand order in both),
// so that each can run the statistics of ONE of the two rows a thread owns.  `red2` = [2 buffers][2 tiles][8 warps][32 lanes] float4.
template <int NT>
__device__ __forceinline__ void mega_combine_both_n(float (&c)[NT][4], float4* red2, int buf, int warp, int mt, int kh, int lane) {
  float4* mine = red2 + (buf * 16 + warp) * 32 + lane;
  const float4* other = red2 + (buf * 16 + (warp ^ 4)) * 32 + lane;
#pragma unroll
  for (int n = 0; n < NT; ++n) mine[n * 256] = make_float4(c[n][0], c[n][1], c[n][2], c[n][3]);
  named_bar_sync(2 + mt, 64);
#pragma unroll
  for (int n = 0; n < NT; ++n) {
    const float4 o = other[n * 256];
    if (kh == 0) { c[n][0] += o.x; c[n][1] += o.y; c[n][2] += o.z; c[n][3] += o.w; }
    else { c[n][0] = o.x + c[n][0]; c[n][1] = o.y + c[n][1]; c[n][2] = o.z + c[n][2]; c[n][3] = o.w + c[n][3]; }
  }
}

// Zeroes c, takes the next NT ring chunks (timeline mark tl_landed once they landed), runs the MMAs and frees the chunks.
template <int NT>
__device__ __forceinline__ void mega_ring_mma(float (&c)[NT][4], MegaRing& rg, const MegaAFrag& a, int kh, int lane, MegaTl& tlf,
                                              int tl_landed) {
  const uint8_t* tb[NT];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
    tb[j] = rg.acquire_ahead(j);
  }
  if (tl_landed) tlf.mark(tl_landed);
  mega_mma_tiles<NT>(c, a, tb, kh, lane);
#pragma unroll
  for (int j = 0; j < NT; ++j) rg.release();
}
// One GEMM phase: the NT tiles s of this CTA (mega_tiles) against A[:rows, s.a_col ..) (leading dimension lda), plus bias
// when kBias.  The epilogue epi(c, f, b) runs in the warp that owns tile j's sum: c[0..1] = row r0, c[2..3] = row r0 + 8
// of output features f, f + 1, and b their bias (0 without one).  Timeline marks tl_id + 0 .. 4 (tl_id = 0: none).
// kBias is a template argument, not a null test: a bias chosen at run time compiles to selects that make the warp wait
// for the bias loads before its MMAs (in the timeline build the q | k | v and fc1 phases took ~2 us longer that way).
template <int NT, bool kBias, class Epi>
__device__ __forceinline__ void mega_gemm(MegaRing& rg, float4* red, int& red_buf, const __nv_bfloat16* A, long long lda, int rows,
                                          const MegaTiles& s, const float* bias, int mt, int kh, int lane, MegaTl& tlf, int tl_id,
                                          Epi&& epi) {
  const int t = lane & 3;
  MegaAFrag a;
  if (tl_id) tlf.mark(tl_id + 0);
  mega_load_a(a, A + s.a_col, lda, rows, mt, kh, lane);
  if (tl_id) { tlf.mark(tl_id + 1); MEGA_TL_DEP(a, rg.error) tlf.mark(tl_id + 2); }
  float2 bias_j[NT];
#pragma unroll
  for (int j = 0; j < NT; ++j)
    bias_j[j] = kBias ? __ldg(reinterpret_cast<const float2*>(bias + (s.f0 + j) * 8 + 2 * t)) : make_float2(0.f, 0.f);
  float c[NT][4];
  mega_ring_mma<NT>(c, rg, a, kh, lane, tlf, tl_id ? tl_id + 3 : 0);
  const bool own = mega_combine_n<NT>(c, red, red_buf, mt, kh, lane);
  if (tl_id) tlf.mark(tl_id + 4);
  if (own) {
#pragma unroll
    for (int j = 0; j < NT; ++j) epi(c[j], (s.f0 + j) * 8 + 2 * t, bias_j[j]);
  }
  red_buf ^= 1;
}

__device__ __forceinline__ float2 ldcg_f2(const float* p) { return __ldcg(reinterpret_cast<const float2*>(p)); }

// ---- the kernel ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMegaThreads, 1)
decode_mega_kernel(const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmTXT,
                   const __grid_constant__ CUtensorMap tmKV16, const __grid_constant__ CUtensorMap tmTXT16, const MegaParams p) {
  extern __shared__ __align__(1024) uint8_t mega_smem_raw[];
  uint8_t* smem = mega_smem_raw + ((1024u - (smem_u32(mega_smem_raw) & 1023u)) & 1023u);
  uint8_t* ring = smem;                                                  // 12 x 16 KB
  // 16 KB used by two phases that never overlap inside a CTA: attention -- per compute warp a 16-row x 128 B q tile
  // (swizzled); GEMM phases -- the K-half exchange buffers of mega_combine_n / mega_combine_both_n
  uint8_t* q_s = smem + kMegaSlots * kMegaSlotBytes;
  float4* redv = reinterpret_cast<float4*>(q_s);
  // attention: softmax states [item][warp][kMegaAttState floats], then the staged q rows of the CTA's items; the LM head keeps
  // this CTA's bias slice here
  float* att_part = reinterpret_cast<float*>(q_s + kMegaComputeWarps * 2048);
  uint4* q_stage = reinterpret_cast<uint4*>(att_part + kMegaAttItems * kMegaComputeWarps * kMegaAttState);     // [items][8] x 16 B
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(q_stage) + kMegaAttItems * 128);
  uint64_t* empty = full + kMegaSlots;
  volatile uint32_t* issued = reinterpret_cast<volatile uint32_t*>(empty + kMegaSlots);

  StepState* st = p.sel.state;
  if (st->finished) return;                     // stable: only the previous launch's selection phase writes it
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x, G = gridDim.x;
  const int R = p.sel.rows, M = p.M;
  const int pos = st->pos, step = st->step, cur_len = st->cur_len;
  const int n_kv = (M + kMegaKvRows - 1) / kMegaKvRows;
  const int n_txt = pos / 64 + 1;               // 64-position chunks of the text K/V cache holding positions 0 .. pos
  // valid keys of attention round r (image chunks 0 .. n_kv - 1, then text chunks): 64 except in the last image chunk and
  // the last text chunk.  Producer and consumers both derive it from M and pos, so they agree on which rows are fetched.
  auto round_keys = [&](int r) { return min(kMegaKvRows, r < n_kv ? M - r * kMegaKvRows : pos + 1 - (r - n_kv) * 64); };
  const int n_items = R * kMegaH;
  const int my_cta_rev = G - 1 - cta;           // attention items are dealt from the last CTA down (those own fewer weights)
  const int n_my_items = (n_items > my_cta_rev) ? (n_items - my_cta_rev + G - 1) / G : 0;
  const int lm_per = mega_lm_per(p.sel.V, G);   // the GEMM phases' weight tiles of this CTA: mega_tiles

  if (tid == 0) {
    tma_prefetch_desc(&tmKV);
    tma_prefetch_desc(&tmTXT);
    tma_prefetch_desc(&tmKV16);
    tma_prefetch_desc(&tmTXT16);
    for (int s = 0; s < kMegaSlots; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kMegaComputeWarps);
    }
    mbar_fence_init();
    *issued = 0;
    if (cta == 0) p.barrier[(step + 1) & 1] = 0;   // the counter the NEXT step will use
  }
  __syncthreads();

  if (warp == kMegaComputeWarps) {
    // ============================== producer: the step's HBM stream, in program order ==============================
    if (lane == 0) {
      uint32_t i = 0;
      auto slot_ready = [&]() -> uint8_t* {
        const uint32_t slot = i % kMegaSlots;
        if (i >= kMegaSlots && !mbar_wait_bounded(&empty[slot], ((i / kMegaSlots) - 1) & 1, p.error)) *p.error = kWaitRingEmpty;
        return ring + slot * kMegaSlotBytes;
      };
      auto publish = [&]() {          // the chunk's barrier is armed: consumers may now wait for its phase
        ++i;
        __threadfence_block();
        *issued = i;
      };
      auto tiles = [&](const uint8_t* w, const MegaTiles& s) {   // one GEMM phase's weight tiles
        for (int j = 0; j < s.n; ++j) {
          uint8_t* dst = slot_ready();
          mbar_arrive_expect_tx(&full[i % kMegaSlots], kMegaTileBytes);
          bulk_load_1d(dst, w + static_cast<size_t>(s.t0 + j * s.stride) * kMegaTileBytes, kMegaTileBytes, &full[i % kMegaSlots]);
          publish();
        }
      };
      // one attention chunk: up to 64 keys of one (sequence, head) with n valid, K rows at the slot's start, V rows 8 KB
      // in.  n = 64: one 64-row box each.  n < 64: ceil(n / 16) 16-row boxes each, sub-box s at byte 2048 s of its half --
      // the rows past the last sub-box are never fetched and never read (keys64 stops at the same 16-key step).  The 128B
      // swizzle (PTX ISA, tensor copy swizzling modes) XORs the 16-byte chunk index of a row with address bits 7..9, the
      // row's index within its 1024-byte block; both halves start 1024-byte aligned, so row j of a sub-box at 2048 s lands
      // at 2048 s + 128 j with chunk c at c ^ (j & 7) -- where row 16 s + j of a 64-row box would ((16 s + j) & 7 == j & 7),
      // and keys64's ldmatrix addressing serves both.  expect_tx counts the bytes requested (rows past the tensor's end
      // are zero-filled and still counted).
      auto kv_pair = [&](const CUtensorMap* tm, const CUtensorMap* tm16, int row_k, int row_v, int col, int n) {
        uint8_t* dst = slot_ready();
        uint64_t* bar = &full[i % kMegaSlots];
        if (n >= kMegaKvRows) {
          mbar_arrive_expect_tx(bar, kMegaSlotBytes);
          tma_load_2d(dst, tm, bar, col, row_k);
          tma_load_2d(dst + 8192, tm, bar, col, row_v);
        } else {
          const int ns = (n + kMegaKvSubRows - 1) / kMegaKvSubRows;
          mbar_arrive_expect_tx(bar, ns * 2 * (kMegaKvSubRows * 128));
          for (int s = 0; s < ns; ++s) {
            tma_load_2d(dst + s * (kMegaKvSubRows * 128), tm16, bar, col, row_k + s * kMegaKvSubRows);
            tma_load_2d(dst + 8192 + s * (kMegaKvSubRows * 128), tm16, bar, col, row_v + s * kMegaKvSubRows);
          }
        }
        publish();
      };
      for (int l = 0; l < p.n_layers; ++l) {
        const MegaLayer& L = p.layer[l];
        tiles(L.wqkv, mega_tiles(kGemmQkv, cta, G, p.sel.V, lm_per));
        // attention chunks ("units") of this CTA's items, round-major: unit u = r * n_my_items + k is keys 64r .. 64r + 63 of
        // item k (image keys first, then the text rounds), of which round_keys(r) are fetched; the consumer deals the
        // units to its 8 warps round-robin
        for (int r = 0; r < n_kv + n_txt; ++r) {
          const int n_keys = round_keys(r);
          if (r == n_kv) {
            // the text K/V of position `pos` exist once every CTA has passed barrier 7l + 1 (after this layer's QKV phase)
            const unsigned int target = static_cast<unsigned int>(G) * (7u * l + 1u);
            unsigned int spins = 0;
            while (ld_acquire_gpu(p.barrier + (step & 1)) < target) {
              if (++spins > kMegaSpinLimit || ((spins & 255u) == 255u && *reinterpret_cast<const volatile int*>(p.error) != 0)) {
                if (*reinterpret_cast<const volatile int*>(p.error) == 0) *p.error = kWaitTextKv;
                break;
              }
            }
            asm volatile("fence.proxy.async;" ::: "memory");   // other SMs' generic-proxy stores -> this thread's TMA reads
          }
          for (int kk = 0; kk < n_my_items; ++kk) {
            const int item = my_cta_rev + kk * G;
            const int b = item / kMegaH, h = item - b * kMegaH;
            if (r < n_kv)
              kv_pair(&tmKV, &tmKV16, (l * 2 + 0) * R * M + b * M + r * kMegaKvRows, (l * 2 + 1) * R * M + b * M + r * kMegaKvRows,
                      h * 64, n_keys);
            else
              kv_pair(&tmTXT, &tmTXT16, ((l * 2 + 0) * R + b) * p.T_alloc + (r - n_kv) * 64,
                      ((l * 2 + 1) * R + b) * p.T_alloc + (r - n_kv) * 64, h * 64, n_keys);
          }
        }
        tiles(L.wo, mega_tiles(kGemmOut, cta, G, p.sel.V, lm_per));
        tiles(L.w1, mega_tiles(kGemmFc1, cta, G, p.sel.V, lm_per));
        tiles(L.w2, mega_tiles(kGemmFc2, cta, G, p.sel.V, lm_per));
      }
      tiles(p.lm, mega_tiles(kGemmLm, cta, G, p.sel.V, lm_per));
    }
    return;
  }

  // ================================== compute warps ==================================
  MegaRing rg{ring, full, empty, 0u, p.error, issued};
  unsigned int* bar = p.barrier + (step & 1);
  unsigned int epoch = 0;
  MegaTl tlf;
  tlf.begin();
#ifdef GITB200_TIMELINE
#define MEGA_TL_ID(ph) ((l == 2) ? 710000 + (ph) * 100 : 0)
#else
#define MEGA_TL_ID(ph) 0
#endif
  const int mt = warp & 3, kh = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const int r0 = mt * 16 + g, r1 = r0 + 8;
  int red_buf = 0;

  for (int l = 0; l < p.n_layers; ++l) {
    const MegaLayer& L = p.layer[l];
    // ------------------------------------------------ P1: q | k | v ------------------------------------------------
    {
      const MegaTiles s = mega_tiles(kGemmQkv, cta, G, p.sel.V, lm_per);
      auto qkv_out = [&](const float (&c)[4], int f, float2 bias) {   // q / 8 | this position's text K | V
        const int seg = f / kMegaD, fo = f - seg * kMegaD;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = hh ? r1 : r0;
          if (r >= R) continue;
          const float v0 = c[2 * hh] + bias.x, v1 = c[2 * hh + 1] + bias.y;
          if (seg == 0) {
            *reinterpret_cast<uint32_t*>(p.qb + static_cast<long long>(r) * kMegaD + fo) = pack_bf16(v0 * 0.125f, v1 * 0.125f);
          } else {
            __nv_bfloat16* dst = (seg == 1 ? L.txt_k : L.txt_v) + (static_cast<long long>(r) * p.T_alloc + pos) * kMegaD + fo;
            *reinterpret_cast<uint32_t*>(dst) = pack_bf16(v0, v1);
          }
        }
      };
      if (s.n == 3) mega_gemm<3, true>(rg, redv, red_buf, p.hb, kMegaD, R, s, L.bqkv, mt, kh, lane, tlf, MEGA_TL_ID(1), qkv_out);
      else if (s.n == 2) mega_gemm<2, true>(rg, redv, red_buf, p.hb, kMegaD, R, s, L.bqkv, mt, kh, lane, tlf, MEGA_TL_ID(1), qkv_out);
    }
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(1));
    // ------------------------------------------------ P2: attention ------------------------------------------------
    // The CTA's 5-6 (sequence, head) items x (image + text) 64-key chunks form U units; warp w takes units w, w + 8, ...
    // (whatever item they belong to), so the tensor pipes of the four SM sub-partitions carry the same load -- one warp
    // per item left two of them with twice the MMAs of the others, and mma.sync issue rate is what bounds this phase.
    // The online-softmax state of (item, warp) lives in shared memory between the units of a warp; S = q K^T and
    // O += P V run on mma.sync with a 16-row q tile whose row 0 is the query (rows 1..15 zero).  At the end warp k merges
    // the 8 states of item k in warp order (bit-reproducible).  Two block-level barriers per phase, none per unit.
    {
      const int rounds = n_kv + n_txt;                      // ring chunks per item (up to 64 keys each)
      const uint32_t att_base = rg.idx;
      const int U = n_my_items * rounds;
      uint8_t* qw = q_s + warp * 2048;
      constexpr float kLog2e = 1.44269504088896340736f;
      // phase start: this warp's q tile zeroed (row 0 is rewritten per unit), its softmax states reset, the q rows staged
#pragma unroll
      for (int jq = 0; jq < 4; ++jq) reinterpret_cast<uint4*>(qw)[lane + 32 * jq] = make_uint4(0, 0, 0, 0);
      if (lane < 4) {
        for (int k = 0; k < n_my_items; ++k) {
          float* sl = att_part + (k * kMegaComputeWarps + warp) * kMegaAttState;
#pragma unroll
          for (int j = 0; j < 8; ++j) { sl[8 * j + 2 * lane] = 0.f; sl[8 * j + 2 * lane + 1] = 0.f; }
          sl[65 + lane] = 0.f;
          if (lane == 0) sl[64] = -INFINITY;
        }
      }
      if (warp < n_my_items && lane < 8) {
        const int item = my_cta_rev + warp * G;
        const int b = item / kMegaH, h = item - b * kMegaH;
        q_stage[warp * 8 + lane] = __ldcg(reinterpret_cast<const uint4*>(p.qb + static_cast<long long>(b) * kMegaD + h * 64) + lane);
      }
      named_bar_sync(1, kMegaComputeWarps * 32);
      for (int u = warp; u < U; u += kMegaComputeWarps) {
        const int r = u / n_my_items, k = u - r * n_my_items;
        // q tile (already scaled by 1/8), 128B-swizzled like the K/V boxes: row 0 <- the item's q (chunk c of row 0 sits at c << 4)
        if (lane < 8) *reinterpret_cast<uint4*>(qw + (lane << 4)) = q_stage[k * 8 + lane];
        __syncwarp();
        uint32_t qa[4][4];
        {
          const int row = (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int chunk = 2 * kk + (lane >> 4);
            ldmatrix_x4(qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3], smem_u32(qw) + row * 128 + ((chunk ^ (row & 7)) << 4));
          }
        }
        float* sl = att_part + (k * kMegaComputeWarps + warp) * kMegaAttState;
        float o[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
        float m_run = -INFINITY, l_run = 0.f;       // row g of the q tile (only g == 0 is a real row)
        if (g == 0) {
          m_run = sl[64];
          l_run = sl[65 + t];
#pragma unroll
          for (int j = 0; j < 8; ++j) { o[j][0] = sl[8 * j + 2 * t]; o[j][1] = sl[8 * j + 2 * t + 1]; }
        }
        // up to 64 keys: rows [0, 16 ns) of the K half at sK and the V half at sV -- the ns 16-key steps kv_pair fetched
        // (ns = 4 for a whole chunk); key index = key0 + row, valid below key_end.  Rows past 16 ns were not fetched and
        // are not read: their 8-key score groups are skipped (left at 0, then set to -inf by the key_end mask, since
        // key0 + 16 ns >= key_end) and so are their p.V steps.  Fetched or not, such a key had score -inf, so p = +0: it
        // added nothing to l and +-0 to o, and skipping it leaves m, l and o as they were (but for the sign of an o that is
        // exactly zero).  The loops stay fully unrolled with ns as a predicate, so sc / o keep static register indices;
        // a whole chunk (ns = 4) takes a copy without the predicates, so that its ldmatrix loads can still be issued ahead
        // of the MMAs.  The first 16-key step (ns >= 1) is unconditional in both copies.
        auto keys64 = [&](uint32_t sK, uint32_t sV, int key0, int key_end, int ns, auto whole) {
          constexpr bool kWhole = decltype(whole)::value;
          float sc[8][4];
#pragma unroll
          for (int jn = 0; jn < 8; ++jn) {
            sc[jn][0] = sc[jn][1] = sc[jn][2] = sc[jn][3] = 0.f;
            if (!kWhole && jn >= 2 && jn >= 2 * ns) continue;
            const int krow = 8 * jn + (lane & 7);
#pragma unroll
            for (int kk2 = 0; kk2 < 2; ++kk2) {
              const int chunk = 4 * kk2 + (lane >> 3);
              uint32_t b0, b1, b2, b3;
              ldmatrix_x4(b0, b1, b2, b3, sK + krow * 128 + ((chunk ^ (krow & 7)) << 4));
              mma_bf16_16816(sc[jn], qa[2 * kk2], b0, b1);
              mma_bf16_16816(sc[jn], qa[2 * kk2 + 1], b2, b3);
            }
          }
          float mx = -INFINITY;
#pragma unroll
          for (int jn = 0; jn < 8; ++jn) {
            const int key = key0 + 8 * jn + 2 * t;
            if (key >= key_end) sc[jn][0] = -INFINITY;
            if (key + 1 >= key_end) sc[jn][1] = -INFINITY;
            mx = fmaxf(mx, fmaxf(sc[jn][0], sc[jn][1]));
          }
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m_run, mx);
          const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
          const float corr = ex2_approx((m_run - m_use) * kLog2e);
          m_run = m_new;
          l_run *= corr;
#pragma unroll
          for (int j = 0; j < 8; ++j) { o[j][0] *= corr; o[j][1] *= corr; }
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {                  // 16 keys per k-step = score tiles 2kk, 2kk + 1
            if (!kWhole && kk > 0 && kk >= ns) continue;    // step 0 unconditional: l_run * corr + its sum still contracts
                                                            // to one FFMA, as it did before (bit-identical l)
            const float p0 = ex2_approx((sc[2 * kk][0] - m_use) * kLog2e), p1 = ex2_approx((sc[2 * kk][1] - m_use) * kLog2e);
            const float p2 = ex2_approx((sc[2 * kk + 1][0] - m_use) * kLog2e), p3 = ex2_approx((sc[2 * kk + 1][1] - m_use) * kLog2e);
            l_run += (p0 + p1) + (p2 + p3);
            const uint32_t pa[4] = {pack_bf16(p0, p1), 0u, pack_bf16(p2, p3), 0u};   // rows 8..15 of the q tile do not exist
            const int vrow = 16 * kk + ((lane >> 3) & 1) * 8 + (lane & 7);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int chunk = 2 * jj + (lane >> 4);
              uint32_t b0, b1, b2, b3;
              ldmatrix_x4_trans(b0, b1, b2, b3, sV + vrow * 128 + ((chunk ^ (vrow & 7)) << 4));
              mma_bf16_16816(o[2 * jj], pa, b0, b1);
              mma_bf16_16816(o[2 * jj + 1], pa, b2, b3);
            }
          }
        };
        const uint32_t ci = att_base + static_cast<uint32_t>(u);
        const uint32_t sK = smem_u32(rg.acquire_at(ci));
        const int ns = (round_keys(r) + kMegaKvSubRows - 1) / kMegaKvSubRows;
        const int key0 = (r < n_kv) ? r * kMegaKvRows : (r - n_kv) * 64;         // image keys 64r .. | text positions 64(r - n_kv) ..
        const int key_end = (r < n_kv) ? M : pos + 1;
        if (ns == kMegaKvRows / kMegaKvSubRows) keys64(sK, sK + 8192, key0, key_end, ns, std::true_type());
        else keys64(sK, sK + 8192, key0, key_end, ns, std::false_type());
        rg.release_at(ci);
        if (g == 0) {
          if (t == 0) sl[64] = m_run;
          sl[65 + t] = l_run;
#pragma unroll
          for (int j = 0; j < 8; ++j) { sl[8 * j + 2 * t] = o[j][0]; sl[8 * j + 2 * t + 1] = o[j][1]; }
        }
        __syncwarp();                                       // the q tile's row 0 and the state are rewritten by the next unit
      }
      named_bar_sync(1, kMegaComputeWarps * 32);
      if (warp < n_my_items) {
        // merge the 8 softmax states of item `warp` (fixed order: bit-reproducible); lane -> output dims 2 lane, 2 lane + 1
        const int item = my_cta_rev + warp * G;
        const int b = item / kMegaH, h = item - b * kMegaH;
        const float* p0 = att_part + (warp * kMegaComputeWarps) * kMegaAttState;
        float mm = -INFINITY;
        for (int i = 0; i < kMegaComputeWarps; ++i) mm = fmaxf(mm, p0[i * kMegaAttState + 64]);
        float lsum = 0.f, a0 = 0.f, a1 = 0.f;
        for (int i = 0; i < kMegaComputeWarps; ++i) {
          const float* pi = p0 + i * kMegaAttState;
          const float mi = pi[64];
          const float wgt = (mi == -INFINITY) ? 0.f : exp2f((mi - mm) * kLog2e);
          lsum += ((pi[65] + pi[66]) + (pi[67] + pi[68])) * wgt;
          a0 += pi[2 * lane] * wgt;
          a1 += pi[2 * lane + 1] * wgt;
        }
        *reinterpret_cast<uint32_t*>(p.ctx + static_cast<long long>(b) * kMegaD + h * 64 + 2 * lane) = pack_bf16(a0 / lsum, a1 / lsum);
      }
      rg.idx = att_base + static_cast<uint32_t>(U);
    }
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(2));
    // ------------------------------------------------ P3: attention output projection (+bias +residual) ------------------
    {
      const MegaTiles s = mega_tiles(kGemmOut, cta, G, p.sel.V, lm_per);
      if (s.n > 0) {
        const int f = s.f0 * 8 + 2 * t;
        float2 xr[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};      // residual: requested before the MMA needs the tile
        if (kh == 0 && r0 < R) xr[0] = ldcg_f2(p.x + static_cast<long long>(r0) * kMegaD + f);
        if (kh == 0 && r1 < R) xr[1] = ldcg_f2(p.x + static_cast<long long>(r1) * kMegaD + f);
        auto out_proj = [&](const float (&c)[4], int f, float2 bias) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int r = hh ? r1 : r0;
            if (r >= R) continue;
            *reinterpret_cast<float2*>(p.y + static_cast<long long>(r) * kMegaD + f) =
                make_float2(xr[hh].x + (c[2 * hh] + bias.x), xr[hh].y + (c[2 * hh + 1] + bias.y));
          }
        };
        mega_gemm<1, true>(rg, redv, red_buf, p.ctx, kMegaD, R, s, L.bo, mt, kh, lane, tlf, MEGA_TL_ID(3), out_proj);
      }
    }
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(3));
    // ------------------------------------------------ P4 / P7: LayerNorm(y) -> x, hb (warp 0 of CTA r: row r) ----------------
    // from_parts: the input row is x + ((p0 + p1) + p2) + p3 + bias (fc2's four k-slice partials, fixed order)
    auto layer_norm_rows = [&](const float* gamma, const float* beta, bool from_parts, const float* bias) {
      const int row = cta;           // one row per CTA (R <= 64 of them): 8 rows per CTA made 8 SMs pull all the rows through their L2 ports
      if (row < R && warp == 0) {
        float4 v[6];
        if (!from_parts) {
          const float4* yp = reinterpret_cast<const float4*>(p.y + static_cast<long long>(row) * kMegaD);
#pragma unroll
          for (int i = 0; i < 6; ++i) v[i] = __ldcg(yp + i * 32 + lane);
        } else {
          const long long ps = static_cast<long long>(R) * kMegaD / 4;     // float4s per partial buffer
          const float4* pp = reinterpret_cast<const float4*>(p.ypart + static_cast<long long>(row) * kMegaD);
          const float4* xp = reinterpret_cast<const float4*>(p.x + static_cast<long long>(row) * kMegaD);
          float4 q0[6], q1[6], q2[6], q3[6], xx[6];
#pragma unroll
          for (int i = 0; i < 6; ++i) {
            q0[i] = __ldcg(pp + i * 32 + lane); q1[i] = __ldcg(pp + ps + i * 32 + lane);
            q2[i] = __ldcg(pp + 2 * ps + i * 32 + lane); q3[i] = __ldcg(pp + 3 * ps + i * 32 + lane);
            xx[i] = __ldcg(xp + i * 32 + lane);
          }
#pragma unroll
          for (int i = 0; i < 6; ++i) {
            const float4 bb = __ldg(reinterpret_cast<const float4*>(bias) + i * 32 + lane);
            v[i].x = xx[i].x + ((((q0[i].x + q1[i].x) + q2[i].x) + q3[i].x) + bb.x);
            v[i].y = xx[i].y + ((((q0[i].y + q1[i].y) + q2[i].y) + q3[i].y) + bb.y);
            v[i].z = xx[i].z + ((((q0[i].z + q1[i].z) + q2[i].z) + q3[i].z) + bb.z);
            v[i].w = xx[i].w + ((((q0[i].w + q1[i].w) + q2[i].w) + q3[i].w) + bb.w);
          }
        }
        float mean, rstd;
        ln_row_stats<kMegaD>(v, 1e-12f, mean, rstd);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
          const float4 bt = __ldg(reinterpret_cast<const float4*>(beta) + i * 32 + lane);
          ln_store<kMegaD>(p.x, p.hb, 0, row, i * 32 + lane, ln_norm(v[i], mean, rstd, gm, bt));
        }
      }
    };
    layer_norm_rows(L.lnag, L.lnab, false, nullptr);
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(4));
    // ------------------------------------------------ P5: fc1 + erf-GELU ------------------------------------------------
    {
      const MegaTiles s = mega_tiles(kGemmFc1, cta, G, p.sel.V, lm_per);
      auto fc1_out = [&](const float (&c)[4], int f, float2 bias) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = hh ? r1 : r0;
          if (r >= R) continue;
          *reinterpret_cast<uint32_t*>(p.ub + static_cast<long long>(r) * kMegaF + f) =
              pack_bf16(apply_act(c[2 * hh] + bias.x, ACT_GELU_ERF), apply_act(c[2 * hh + 1] + bias.y, ACT_GELU_ERF));
        }
      };
      if (s.n > 0) mega_gemm<kMegaFcTilesPerCta, true>(rg, redv, red_buf, p.hb, kMegaD, R, s, L.b1, mt, kh, lane, tlf, MEGA_TL_ID(5), fc1_out);
    }
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(5));
    // ------------------------------------------------ P6: fc2, split over CTAs: 32 groups of 24 features x 4 k slices ------
    // (each CTA reads ONE 768-wide slice of the activations; the four partial sums of a feature meet, in slice order, in
    //  the LayerNorm phase below -- bit-reproducible, no atomics)
    {
      const MegaTiles s = mega_tiles(kGemmFc2, cta, G, p.sel.V, lm_per);
      float* yp = p.ypart + static_cast<long long>(s.a_col) * R;     // the partial buffer of k slice a_col / 768
      auto fc2_out = [&](const float (&c)[4], int f, float2) {
        if (r0 < R) *reinterpret_cast<float2*>(yp + static_cast<long long>(r0) * kMegaD + f) = make_float2(c[0], c[1]);
        if (r1 < R) *reinterpret_cast<float2*>(yp + static_cast<long long>(r1) * kMegaD + f) = make_float2(c[2], c[3]);
      };
      if (s.n > 0) mega_gemm<kMegaFcTilesPerCta, false>(rg, redv, red_buf, p.ub, kMegaF, R, s, nullptr, mt, kh, lane, tlf, MEGA_TL_ID(6), fc2_out);
    }
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(6));
    layer_norm_rows(L.lnog, L.lnob, true, L.b2);
    mega_grid_sync(bar, epoch, p.error, tlf, MEGA_TL_ID(7));
  }

  // ------------------------------------------------ LM head with the greedy statistics folded in ---------------------------
  // After the two K halves of a tile are summed, the kh = 0 warp of a pair keeps the statistics of row g, the kh = 1 warp
  // those of row g + 8: for its row and its 2 columns per tile a thread maintains the running (max, arg max, sum exp) over
  // this CTA's features -- the logits themselves never leave the SM (unless the parity hook asks for them).
  {
    const MegaTiles lm = mega_tiles(kGemmLm, cta, G, p.sel.V, lm_per);
    const int my_row = kh ? r1 : r0;
    long long last = -1;
    // no no-repeat mask at a row's first real decision, nor inside its prefix, whose token is given: row_step's first ||
    // in_prefix, spelled out here because the row_step call spills registers in this kernel
    bool unmasked = (step == 0);
    if (my_row < R) {
      last = p.sel.next_token[my_row];
      if (p.sel.row_prefix != nullptr) unmasked = cur_len <= p.sel.row_prefix_lens[my_row];
    }
    float smax = -INFINITY, ssum = 0.f;
    int sarg = 0x7fffffff;
    float* bias_s = att_part;                       // this CTA's slice of the output bias (<= 8 * lm_per floats)
    for (int i = tid; i < lm.n * 8; i += kMegaComputeWarps * 32) {
      const int col = lm.t0 * 8 + i;
      bias_s[i] = (col < p.sel.V) ? __ldg(p.lm_bias + col) : 0.f;
    }
    named_bar_sync(1, kMegaComputeWarps * 32);
    if (lm.n > 0) {
      MegaAFrag a;
      mega_load_a(a, p.hb, kMegaD, R, mt, kh, lane);
      // statistics of one tile's two columns of this thread's row (columns arrive in increasing order)
      auto lm_stats = [&](const float (&cc)[4], int j) {
        if (my_row >= R) return;
        const int f = (lm.t0 + j) * 8 + 2 * t;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = f + e;
          if (col >= p.sel.V) continue;
          float v = (kh ? cc[2 + e] : cc[e]) + bias_s[j * 8 + 2 * t + e];
          if (p.sel.step_logits != nullptr) p.sel.step_logits[(static_cast<long long>(step) * R + my_row) * p.sel.V + col] = v;
          if (!unmasked && col == static_cast<int>(last)) v = -10000.0f;     // no-repeat (reference :330)
          if (v > smax) {            // the lowest index wins exact ties
            ssum = ssum * __expf(smax - v) + 1.0f;
            smax = v;
            sarg = col;
          } else {
            ssum += __expf(v - smax);
          }
        }
      };
      int j = 0;
      MEGA_TL(720000);                                // LM head: A loads issued
      for (; j + 2 <= lm.n; j += 2) {                 // two tiles in flight per warp (see mega_mma_tiles)
        float c[2][4];
        mega_ring_mma<2>(c, rg, a, kh, lane, tlf, 720100 + j);   // mark: the pair's tiles landed
        mega_combine_both_n<2>(c, redv, red_buf, warp, mt, kh, lane);
        MEGA_TL(720200 + j);                          // MMAs + exchange done
        red_buf ^= 1;
        lm_stats(c[0], j);
        lm_stats(c[1], j + 1);
        MEGA_TL(720300 + j);                          // statistics done
      }
      if (j < lm.n) {
        float c[1][4];
        mega_ring_mma<1>(c, rg, a, kh, lane, tlf, 0);
        mega_combine_both_n<1>(c, redv, red_buf, warp, mt, kh, lane);
        red_buf ^= 1;
        lm_stats(c[0], j);
      }
    }
    // combine the 4 lanes of a quad (they hold the same row, interleaved column pairs)
#pragma unroll
    for (int o2 = 1; o2 <= 2; o2 <<= 1)
      merge_stats(smax, ssum, sarg, __shfl_xor_sync(0xffffffffu, smax, o2), __shfl_xor_sync(0xffffffffu, ssum, o2),
                  __shfl_xor_sync(0xffffffffu, sarg, o2));
    if (t == 0 && my_row < R) {
      p.sel.part_max[static_cast<long long>(my_row) * G + cta] = smax;
      p.sel.part_sum[static_cast<long long>(my_row) * G + cta] = ssum;
      p.sel.part_arg[static_cast<long long>(my_row) * G + cta] = sarg;
    }
  }
  mega_grid_sync(bar, epoch, p.error, tlf, 0);

  tlf.end();
  // ------------------------------------------------ selection (greedy bookkeeping) + next token's embedding ----------------
  if (cta < R && warp == 0) {
    const int row = cta;
    float gm = -INFINITY, gs = 0.f;
    int ga = 0x7fffffff;
    for (int k = lane; k < G; k += 32)             // increasing CTA order = increasing column order
      merge_stats(gm, gs, ga, __ldcg(p.sel.part_max + static_cast<long long>(row) * G + k),
                  __ldcg(p.sel.part_sum + static_cast<long long>(row) * G + k), __ldcg(p.sel.part_arg + static_cast<long long>(row) * G + k));
#pragma unroll
    for (int o2 = 16; o2 > 0; o2 >>= 1)
      merge_stats(gm, gs, ga, __shfl_xor_sync(0xffffffffu, gm, o2), __shfl_xor_sync(0xffffffffu, gs, o2),
                  __shfl_xor_sync(0xffffffffu, ga, o2));
    const RowStep rs = row_step(p.sel, row, step, cur_len, p.sel.next_token[row]);
    const RowChoice c = resolve_row(p.sel, row, cur_len, rs, ga, -logf(gs));
    embed_ln_row<kMegaD>(c.nxt, pos + 1, p.words, p.positions, p.lnemb_g, p.lnemb_b, p.sel.V, p.x, p.hb, 0, row, lane);
    if (lane == 0) commit_row(p.sel, row, step, cur_len, c, nullptr);
  }
}

constexpr size_t kMegaSmemBytes = 1024 + kMegaSlots * kMegaSlotBytes + kMegaComputeWarps * 2048 +
                                  kMegaAttItems * kMegaComputeWarps * kMegaAttState * 4 + kMegaAttItems * 128 + 2 * kMegaSlots * 8 + 64 + 64;

}  // namespace gitb200
