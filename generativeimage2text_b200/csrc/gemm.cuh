// C[M,N] = A[M,K] * B[N,K]^T with bf16 operands (both K-major: exactly the layout of an activation
// matrix and of an nn.Linear weight), fp32 accumulation in registers (wgmma), fused epilogues.
//
// One persistent, warp-specialised sm_90a kernel per tile width BN, 128 x BN output tiles:
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor, 128B-swizzled [rows x 64] bf16 tiles, STAGES-deep ring)
//   warpgroups 1-2 : MMA + epilogue, 64 tile rows each (wgmma m64nBNk16 from shared memory, one wgmma group in flight
//                    while the next k-block is issued); the epilogue stages 64 x 64 fp32 chunks in shared memory
// so the producer streams the next tile's operands while the MMA warpgroups run the epilogue of this one.
//
// Two epilogue shapes:
//   normal     : out[row_map(m)][n] (+bias[n]) (+act) (+resid[m][n]); N may be split into up to three equal
//                column segments with their own base pointers (QKV -> q scratch / K cache / V cache).
//   transposed : "swap-AB" for the skinny decode-step GEMMs: A = weight [features, K], B = activations
//                [rows<=BN, K]; out[n][m] (+bias[m]) (+act).  When the K dimension is split over CTAs (so a handful
//                of rows still spreads over many SMs) every split writes its own partial-sum buffer and the consumer
//                kernel adds them in split order: results are bit-reproducible from run to run.
#pragma once
#include "ptx.cuh"

namespace gitb200 {

struct GemmParams {
  int M, N, K;
  int k_splits;
  int transposed;             // epilogue shape / options below select the kernel instantiation on the host
  int partial;                // split-K: split s stores its partial sums at out[0] + s * split_stride (plain stores; the
                              // consumer adds the partials in split order -> bit-reproducible, no atomics, no zeroing)
  long long split_stride;     // elements between the partial buffers of consecutive splits
  int act;
  int out_bf16;
  const float* bias;
  const float* resid;         // normal mode only, fp32, identity row mapping
  long long ld_resid;
  void* out[3];               // column segments (normal mode): N split into equal seg_n-wide parts
  long long ldo;              // row pitch of every output segment (elements)
  long long batch_stride;     // in rows
  int seg_n;                  // segment width (normal mode); N for a single segment
  int rows_per_batch;         // row map: m -> (m / rpb) * batch_stride + (m % rpb) + row_offset
  int row_offset;
  const int* skip;            // device flag: non-zero -> the whole launch is a no-op (finished decode)
  unsigned long long* dbg;    // optional [8] %globaltimer stamps of CTA 0 (profiling aid; null in production)
  int split3;                 // bf16 output in the parity mode's operand format: row = [hi | lo | hi] (3 x N columns, ldo = 3N)
  int pdl;                    // launched with programmatic dependent launch: prefetch weights, then griddep_wait()
  ChainSync chain;            // flag-based ordering inside the decode step (see ptx.cuh); counters == null: off
  const int* lse_target;      // EPI_LSE: [M] target column of each row (-1: none); out[0] = float4 partials [M][ldo]
};

// Epilogue variants are compile-time (the runtime-flag version spent ~700 warp instructions per 32x32 chunk,
// which made every K=768 GEMM of the encoder epilogue-issue bound).
constexpr int EPI_TRANSPOSED = 1, EPI_BF16 = 2, EPI_RESID = 4, EPI_PARTIAL = 8, EPI_ACT_SHIFT = 4, EPI_SPLIT3 = 64;
// EPI_LSE (normal shape, fp32, caption scoring's LM head): no logits are stored.  Each MMA warp folds the columns it owns of
// a tile (BN / 2 of them: 32 of every 64-column chunk) into per-row statistics (max, sum exp(x - max), sum x, x[target])
// and stores them as one float4 per (row, half tile) to out[0] + row * ldo + 2 * n_blk + half; lse_combine_kernel
// (rowops.cuh) folds a row's partials in column order.
constexpr int EPI_LSE = 128;
constexpr int epi_code(bool transposed, bool bf16, bool resid, bool partial, int act) {
  return (transposed ? EPI_TRANSPOSED : 0) | (bf16 ? EPI_BF16 : 0) | (resid ? EPI_RESID : 0) | (partial ? EPI_PARTIAL : 0) |
         (act << EPI_ACT_SHIFT);
}

template <int ACT>
__device__ __forceinline__ float act_ct(float x) {
  return apply_act(x, ACT);  // ACT is a constant: the branches fold away
}

template <int BN>
struct GemmCfg {
  static constexpr int BM = 128;
  static constexpr int BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int MMA_WGS = 2;                          // 64 tile rows each
  static constexpr int THREADS = 128 * (1 + MMA_WGS);        // warpgroup 0: TMA producer
  static constexpr int WG_STAGING_BYTES = 4 * 32 * 128;     // per MMA warpgroup: 64 rows x 64 fp32 as four 32 x 32 blocks
  static constexpr int STAGING_BYTES = MMA_WGS * WG_STAGING_BYTES;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_LIMIT = 227 * 1024;
  static constexpr int STAGES_RAW = (SMEM_LIMIT - 1024 - BAR_BYTES - STAGING_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 1024 + BAR_BYTES;
  static constexpr int PRODUCER_REGS = 40, MMA_REGS = 232;  // 128 x 40 + 256 x 232 <= 64 K registers
  static_assert(BN % 64 == 0 && BN >= 64 && BN <= 256, "BN");
  static_assert(B_BYTES % 1024 == 0, "B tile must keep 1024B alignment for SWIZZLE_128B");
  static_assert(2 * STAGES * 8 <= BAR_BYTES, "barrier area");
  static_assert(STAGES >= 3, "pipeline depth");
};

// ---- epilogue building blocks ---------------------------------------------------------------------------------------------
// Output row offsets (elements) of the 8 rows a lane stores in the normal epilogue: rows row0 + it * 4 + (lane >> 3).
__device__ __forceinline__ uint32_t epi_row_offsets(const GemmParams& p, int row0, int rsub, bool store_ok, long long (&ooff)[8]) {
  uint32_t okmask = 0;
  int bq = (row0 + rsub) / p.rows_per_batch;
  int sq = (row0 + rsub) - bq * p.rows_per_batch;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    if (row0 + it * 4 + rsub < p.M && store_ok) okmask |= 1u << it;
    ooff[it] = (static_cast<long long>(bq) * p.batch_stride + sq + p.row_offset) * p.ldo;
    sq += 4;
    while (sq >= p.rows_per_batch) { sq -= p.rows_per_batch; ++bq; }
  }
  return okmask;
}

// Normal epilogue of one 32x32 fp32 accumulator chunk staged in the warp's swizzled buffer as [row][column] (16-byte
// chunk j of row r at r * 128 + ((j ^ (r & 7)) << 4)): each lane takes 4 consecutive output elements of one row
// (coalesced 128-bit accesses), then (+bias) (+act) (+residual) -> bf16 / fp32 stores into the chunk's column segment.
template <int EPI>
__device__ __forceinline__ void epi_store_normal(const GemmParams& p, const uint8_t* stg, int lane, int n0,
                                                 int row0, const long long (&ooff)[8], uint32_t okmask) {
  constexpr bool kBf16 = (EPI & EPI_BF16) != 0;
  constexpr bool kResid = (EPI & EPI_RESID) != 0;
  constexpr int kAct = (EPI >> EPI_ACT_SHIFT) & 3;
  constexpr bool kSplit3 = (EPI & EPI_SPLIT3) != 0;
  static_assert(!kSplit3 || kBf16, "split3 is a bf16 output format");
  const int c4 = lane & 7;
  const int rsub = lane >> 3;
  // 8 lanes per row (4 columns each), 4 rows per instruction
  float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias != nullptr) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + c4);
  int seg = 0;
  if (p.seg_n < p.N) seg = n0 / p.seg_n;
  const int nn = n0 - seg * p.seg_n + c4 * 4;
  float4 v[8];
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rsub;
    v[it] = *reinterpret_cast<const float4*>(stg + rr * 128 + ((c4 ^ (rr & 7)) << 4));
  }
  float4 res[8];
  if (kResid) {
    const float* rbase = p.resid + static_cast<long long>(row0 + rsub) * p.ld_resid + n0 + c4 * 4;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      res[it] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (okmask & (1u << it)) res[it] = *reinterpret_cast<const float4*>(rbase + static_cast<long long>(it) * 4 * p.ld_resid);
    }
  }
  uint8_t* obase = reinterpret_cast<uint8_t*>(p.out[seg]) + static_cast<long long>(nn) * (kBf16 ? 2 : 4);
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    float4 o = v[it];
    o.x += b4.x; o.y += b4.y; o.z += b4.z; o.w += b4.w;
    if (kAct != ACT_NONE) {
      o.x = act_ct<kAct>(o.x); o.y = act_ct<kAct>(o.y); o.z = act_ct<kAct>(o.z); o.w = act_ct<kAct>(o.w);
    }
    if (kResid) {   // out = resid + (acc + bias): the operand order of the reference's `x + f(x)`
      o.x = res[it].x + o.x; o.y = res[it].y + o.y; o.z = res[it].z + o.z; o.w = res[it].w + o.w;
    }
    if (okmask & (1u << it)) {
      if (kSplit3) {
        uint2 hi, lo;
        pack_split2(o.x, o.y, hi.x, lo.x);
        pack_split2(o.z, o.w, hi.y, lo.y);
        uint8_t* dst = obase + ooff[it] * 2;
        *reinterpret_cast<uint2*>(dst) = hi;
        *reinterpret_cast<uint2*>(dst + static_cast<long long>(p.N) * 2) = lo;
        *reinterpret_cast<uint2*>(dst + static_cast<long long>(p.N) * 4) = hi;
      } else if (kBf16) {
        uint2 pk;
        pk.x = pack_bf16(o.x, o.y);
        pk.y = pack_bf16(o.z, o.w);
        *reinterpret_cast<uint2*>(obase + ooff[it] * 2) = pk;
      } else {
        *reinterpret_cast<float4*>(obase + ooff[it] * 4) = o;
      }
    }
  }
}

// Transposed ("swap-AB") epilogue of one 32x32 chunk staged as [activation row][feature] (16-byte chunk j of row r at
// r * 128 + ((j ^ (r & 7)) << 4)): each lane owns 4 consecutive features of one activation row -- 128-bit stores.
// row0 = first feature (A row) of the chunk, n0 = first activation row (B row).
template <int EPI>
__device__ __forceinline__ void epi_store_transposed(const GemmParams& p, const uint8_t* stg, int lane, int n0, int row0,
                                                     int split, bool store_ok) {
  constexpr bool kBf16 = (EPI & EPI_BF16) != 0;
  constexpr bool kPartial = (EPI & EPI_PARTIAL) != 0;
  constexpr int kAct = (EPI >> EPI_ACT_SHIFT) & 3;
  constexpr bool kSplit3 = (EPI & EPI_SPLIT3) != 0;
  const int c4 = lane & 7;
  const int rsub = lane >> 3;
  const int f0 = row0 + c4 * 4;  // first of this lane's 4 features
  const bool full4 = (f0 + 3) < p.M;
  float bv[4] = {0.f, 0.f, 0.f, 0.f};
  if (p.bias != nullptr && split == 0) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (f0 + e < p.M) bv[e] = __ldg(p.bias + f0 + e);
  }
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rsub;
    const int arow = n0 + rr;
    const float4 t4 = *reinterpret_cast<const float4*>(stg + rr * 128 + ((c4 ^ (rr & 7)) << 4));
    float v[4] = {t4.x + bv[0], t4.y + bv[1], t4.z + bv[2], t4.w + bv[3]};
    if (kAct != ACT_NONE) {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = act_ct<kAct>(v[e]);
    }
    if (arow < p.N && store_ok && f0 < p.M) {
      const long long off = static_cast<long long>(arow) * p.ldo + f0;
      if (kPartial) {   // this split's own partial-sum buffer (plain stores; summed in split order by the consumer)
        float* dst = reinterpret_cast<float*>(p.out[0]) + static_cast<long long>(split) * p.split_stride + off;
        if (full4 && (p.ldo & 3) == 0) {
          *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
          for (int e = 0; e < 4; ++e)
            if (f0 + e < p.M) dst[e] = v[e];
        }
      } else if (kSplit3) {
        __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out[0]) + off;
        for (int e = 0; e < 4; ++e) {
          if (f0 + e < p.M) {
            __nv_bfloat16 hi, lo;
            split_bf16(v[e], hi, lo);
            dst[e] = hi; dst[p.M + e] = lo; dst[2 * p.M + e] = hi;
          }
        }
      } else if (kBf16) {
        __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out[0]) + off;
        if (full4 && (p.ldo & 3) == 0) {
          uint2 pk;
          pk.x = pack_bf16(v[0], v[1]);
          pk.y = pack_bf16(v[2], v[3]);
          *reinterpret_cast<uint2*>(dst) = pk;
        } else {
          for (int e = 0; e < 4; ++e)
            if (f0 + e < p.M) dst[e] = __float2bfloat16_rn(v[e]);
        }
      } else {
        float* dst = reinterpret_cast<float*>(p.out[0]) + off;
        if (full4 && (p.ldo & 3) == 0) {
          *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        } else if (full4 && (p.ldo & 1) == 0) {
          *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
          *reinterpret_cast<float2*>(dst + 2) = make_float2(v[2], v[3]);
        } else {
          for (int e = 0; e < 4; ++e)
            if (f0 + e < p.M) dst[e] = v[e];
        }
      }
    }
  }
}

// EPI_LSE: fold one 32 x 32 chunk staged as [row][column] (see epi_store_normal) into the running statistics of the lane's
// 8 rows (row0 + it * 4 + lane / 8) over its 4 columns n0 + 4 (lane % 8) ..; columns >= N do not exist.
__device__ __forceinline__ void epi_lse_accum(const GemmParams& p, const uint8_t* stg, int lane, int n0, const int (&tgt)[8],
                                              float (&m)[8], float (&se)[8], float (&sx)[8], float (&xt)[8]) {
  const int c4 = lane & 7;
  const int rsub = lane >> 3;
  const int col0 = n0 + c4 * 4;
  float b[4];
  bool ok[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    ok[e] = col0 + e < p.N;
    b[e] = ok[e] ? __ldg(p.bias + col0 + e) : 0.f;
  }
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rsub;
    const float4 v = *reinterpret_cast<const float4*>(stg + rr * 128 + ((c4 ^ (rr & 7)) << 4));
    const float x[4] = {v.x + b[0], v.y + b[1], v.z + b[2], v.w + b[3]};
    float cm = -INFINITY;
#pragma unroll
    for (int e = 0; e < 4; ++e) if (ok[e]) cm = fmaxf(cm, x[e]);
    const float nm = fmaxf(m[it], cm);
    if (nm == -INFINITY) continue;               // no column of this chunk exists
    float acc = (m[it] == -INFINITY) ? 0.f : se[it] * __expf(m[it] - nm);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (ok[e]) {
        acc += __expf(x[e] - nm);
        sx[it] += x[e];
        if (tgt[it] == col0 + e) xt[it] = x[e];
      }
    }
    se[it] = acc;
    m[it] = nm;
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GemmCfg<BN>::THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const GemmParams p) {
  using C = GemmCfg<BN>;
  constexpr bool kTransposed = (EPI & EPI_TRANSPOSED) != 0;
  constexpr bool kLse = (EPI & EPI_LSE) != 0;
  static_assert(!kLse || EPI == EPI_LSE, "the statistics epilogue takes no other option");
  if (p.pdl) griddep_launch_early();
  if (p.pdl) tl_mark(100000 + 1000 + static_cast<int>(gridDim.x));
  // `skip` (decode finished) only changes between steps, which are separated by full dependencies
  if ((!p.pdl || p.chain.counters != nullptr) && p.skip != nullptr && *p.skip != 0) return;  // uniform over the grid
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // keep the shared-memory provenance of the pointer (plain pointer arithmetic) so staging accesses compile to LDS/STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + C::STAGES * C::A_BYTES;
  uint8_t* sStage = smem + C::STAGES * C::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sStage + C::STAGING_BYTES);
  uint64_t* empty = full + C::STAGES;

  const int wg = threadIdx.x >> 7;
  const int warp = (threadIdx.x >> 5) & 3;   // warp within its warpgroup
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], C::MMA_WGS);   // one arrive per MMA warpgroup once its wgmmas have read the slot
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int m_tiles = (p.M + C::BM - 1) / C::BM;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int kb_total = (p.K + C::BK - 1) / C::BK;
  const int kb_per = (kb_total + p.k_splits - 1) / p.k_splits;
  const int mn_tiles = m_tiles * n_tiles;
  const int num_tiles = mn_tiles * p.k_splits;

  // PDL / chain: everything above overlapped the predecessor kernel. In the swap-AB shape the A operand is a
  // weight matrix that no kernel writes: its first tiles are requested before waiting for the predecessor.
  const bool chained = p.chain.counters != nullptr;
  int npre = 0;
  if (kTransposed && p.pdl && static_cast<int>(blockIdx.x) < num_tiles) {
    const int split = static_cast<int>(blockIdx.x) / mn_tiles;
    const int kb0 = split * kb_per;
    npre = min(C::STAGES, min(kb_total, kb0 + kb_per) - kb0);
    if (threadIdx.x == 0) {
      const int m_blk = (static_cast<int>(blockIdx.x) - split * mn_tiles) / n_tiles;
      for (int i = 0; i < npre; ++i) {
        mbar_arrive_expect_tx(&full[i], C::STAGE_BYTES);
        tma_load_2d(sA + i * C::A_BYTES, &tmA, &full[i], (kb0 + i) * C::BK, m_blk * C::BM);
      }
    }
  }
  if (chained) chain_wait(p.chain);
  else if (p.pdl) griddep_wait();
  if (p.pdl) tl_mark(1000 + static_cast<int>(gridDim.x));

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<C::PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int split = tile / mn_tiles;
        const int rem = tile - split * mn_tiles;
        const int m_blk = rem / n_tiles;
        const int n_blk = rem - m_blk * n_tiles;
        const int kb0 = split * kb_per;
        const int kb1 = min(kb_total, kb0 + kb_per);
        for (int kb = kb0; kb < kb1; ++kb) {
          if (npre > 0) {  // weight tile already in flight: add the (dependent) activation tile
            --npre;
            tma_load_2d(sB + stage * C::B_BYTES, &tmB, &full[stage], kb * C::BK, n_blk * BN);
          } else {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], C::STAGE_BYTES);
            tma_load_2d(sA + stage * C::A_BYTES, &tmA, &full[stage], kb * C::BK, m_blk * C::BM);
            tma_load_2d(sB + stage * C::B_BYTES, &tmB, &full[stage], kb * C::BK, n_blk * BN);
          }
          if (++stage == C::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------ MMA + epilogue ----------------------------
    setmaxnreg_inc<C::MMA_REGS>();
    const int mw = wg - 1;                                   // rows 64 mw .. 64 mw + 63 of the tile
    const bool store_ok = !(p.pdl && !chained && p.skip != nullptr && *p.skip != 0);  // finished decode: no stores
    uint8_t* stg_wg = sStage + mw * C::WG_STAGING_BYTES;
    uint8_t* stg = stg_wg + warp * (32 * 128);              // the 32 x 32 block this warp stores
    const int rsub = lane >> 3;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int split = tile / mn_tiles;
      const int rem = tile - split * mn_tiles;
      const int m_blk = rem / n_tiles;
      const int n_blk = rem - m_blk * n_tiles;
      const int kb0 = split * kb_per;
      const int kb1 = min(kb_total, kb0 + kb_per);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        if (p.pdl && tile == static_cast<int>(blockIdx.x) && kb == kb0 && threadIdx.x == 128) tl_mark_one(300000 + 1000 + static_cast<int>(gridDim.x));
        const uint32_t a_base = smem_u32(sA + stage * C::A_BYTES + mw * (64 * 128));
        const uint32_t b_base = smem_u32(sB + stage * C::B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < C::BK / 16; ++k)
          Wgmma<BN>::mma(acc, wgmma_desc_sw128(a_base + k * 32), wgmma_desc_sw128(b_base + k * 32), (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        if (prev >= 0) {   // the previous k-block's wgmmas have read their slot: free it
          wgmma_wait<1>();
          if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == C::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      if (p.pdl && tile == static_cast<int>(blockIdx.x) && threadIdx.x == 128) tl_mark_one(400000 + 1000 + static_cast<int>(gridDim.x));

      // ---- epilogue: 64-column chunks through the warpgroup's staging buffer (block b = 2 * column half + row half,
      //      [row][column] in the normal shape, [column][row] in the transposed one); warp w then stores block w ----
      const int row0 = m_blk * C::BM + mw * 64 + (warp & 1) * 32;   // first tile row of this warp's block
      long long ooff[8];
      uint32_t okmask = 0;
      if (!kTransposed && !kLse) okmask = epi_row_offsets(p, row0, rsub, store_ok, ooff);
      float lm[8], lse_s[8], lsx[8], lxt[8];
      int ltg[8];
      if constexpr (kLse) {
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int row = row0 + it * 4 + rsub;
          ltg[it] = row < p.M ? p.lse_target[row] : -1;
          lm[it] = -INFINITY; lse_s[it] = 0.f; lsx[it] = 0.f; lxt[it] = 0.f;
        }
      }
#pragma unroll
      for (int cc = 0; cc < BN / 64; ++cc) {
        if (n_blk * BN + cc * 64 >= p.N) break;   // uniform over the warpgroup
#pragma unroll
        for (int j8 = 0; j8 < 8; ++j8) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int r64 = warp * 16 + (lane >> 2) + 8 * hh;     // row within the warpgroup's 64
            const int c64 = j8 * 8 + 2 * (lane & 3);              // column within the chunk (even)
            const int r = r64 & 31, c = c64 & 31;
            uint8_t* blk = stg_wg + ((c64 >> 5) * 2 + (r64 >> 5)) * (32 * 128);
            const float v0 = acc[4 * (cc * 8 + j8) + 2 * hh], v1 = acc[4 * (cc * 8 + j8) + 2 * hh + 1];
            if (!kTransposed) {
              *reinterpret_cast<float2*>(blk + r * 128 + (((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4) = make_float2(v0, v1);
            } else {
              *reinterpret_cast<float*>(blk + c * 128 + (((r >> 2) ^ (c & 7)) << 4) + (r & 3) * 4) = v0;
              *reinterpret_cast<float*>(blk + (c + 1) * 128 + (((r >> 2) ^ ((c + 1) & 7)) << 4) + (r & 3) * 4) = v1;
            }
          }
        }
        named_bar_sync(1 + mw, 128);
        const int n0 = n_blk * BN + cc * 64 + (warp >> 1) * 32;
        if constexpr (kLse) {
          epi_lse_accum(p, stg, lane, n0, ltg, lm, lse_s, lsx, lxt);
        } else if (!kTransposed) {
          if (n0 < p.N) epi_store_normal<EPI>(p, stg, lane, n0, row0, ooff, okmask);
        } else {
          epi_store_transposed<EPI>(p, stg, lane, n0, row0, split, store_ok);
        }
        named_bar_sync(1 + mw, 128);   // the staging buffer is rewritten by the next chunk
      }
      if constexpr (kLse) {
        // the 8 lanes of a row merge their statistics (butterfly: every lane ends with the same values), lane 0 stores
#pragma unroll
        for (int it = 0; it < 8; ++it) {
#pragma unroll
          for (int o = 1; o < 8; o <<= 1) {
            const float m_o = __shfl_xor_sync(0xffffffffu, lm[it], o);
            const float s_o = __shfl_xor_sync(0xffffffffu, lse_s[it], o);
            const float nm = fmaxf(lm[it], m_o);
            const float sa = (lm[it] == -INFINITY) ? 0.f : lse_s[it] * __expf(lm[it] - nm);
            const float sb = (m_o == -INFINITY) ? 0.f : s_o * __expf(m_o - nm);
            lse_s[it] = sa + sb;
            lm[it] = nm;
            lsx[it] += __shfl_xor_sync(0xffffffffu, lsx[it], o);
            lxt[it] += __shfl_xor_sync(0xffffffffu, lxt[it], o);
          }
          const int row = row0 + it * 4 + rsub;
          if ((lane & 7) == 0 && row < p.M)
            reinterpret_cast<float4*>(p.out[0])[static_cast<long long>(row) * p.ldo + 2 * n_blk + (warp >> 1)] =
                make_float4(lm[it], lse_s[it], lsx[it], lxt[it]);
        }
      }
    }
  }

  __syncthreads();
  if (p.pdl) tl_mark(200000 + 1000 + static_cast<int>(gridDim.x));
  if (chained && threadIdx.x == 0) chain_signal_thread0(p.chain);
}

}  // namespace gitb200
