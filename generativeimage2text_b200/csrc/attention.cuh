// Multi-head attention kernels (head dim 64).
//
// flash_attn_wgmma_kernel : non-causal softmax(q k^T / 8) v over S keys for every (batch, head); used by the
//   ViT blocks (reference layers/CLIP/model.py:189-197 -> nn.MultiheadAttention -> SDPA, no mask) and by
//   the one-off image-row pass of the decoder (image rows attend image rows only, reference
//   layers/decoder.py:119-120; layers/bert/modeling_bert.py:41-47,138-152).  Batches are stored back to back.
// text_attn_wgmma_kernel : the text rows of a caption batch in one pass (caption scoring).  Both run attn_wg_tile:
//   TMA-fed K/V blocks on an mbarrier ring, S = Q K^T and O = P V as wgmma, online softmax in registers.
//
// decode_attn_kernel : one new text row per sequence against [image K/V || text K/V] (the KV-cached form of
//   reference layers/decoder.py:121-123 + modeling_bert.py:124-152).  Pure HBM streaming: every K/V row is
//   read once with 128-bit loads; image K/V are shared by the beams of an image; the new token's K/V are
//   appended to the text cache by the same kernel.
//
// attn_f32_kernel, text_attn_f32_kernel, decode_attn_f32_kernel : the three in plain fp32 for parity mode, one warp per
//   query row (attn_row_f32).
#pragma once
#include "ptx.cuh"
#include "rowops.cuh"

namespace gitb200 {

struct AttnParams {
  const __nv_bfloat16* q;
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  __nv_bfloat16* out;
  int B, S, H;
  long long q_rs, kv_rs, q_bs, kv_bs, o_rs, o_bs;  // row / batch strides in elements (batches back to back: q_bs = S q_rs)
  float scale_log2;                                 // (1/sqrt(64)) * log2(e)
  const int* seq_lens;                              // flash_attn_wgmma_kernel<true>: [B] valid rows of each batch (<= S)
};

// ------------------------------------------------------------------------------------------------
// attn_wg_tile: softmax(Q K^T / 8) V for one 64-row query tile of one head on Hopper's warpgroup tensor cores, the block
// loop of flash_attn_wgmma_kernel and text_attn_wgmma_kernel.
//   One CTA = one warpgroup.  Thread 0 loads the Q tile and 64-key K / V blocks by TMA (128B-swizzled 64 x 64 bf16 boxes)
//   into a two-stage ring, each stage completing on its own mbarrier, so block i + 1 is in flight while block i is
//   computed.  Per block: S = Q K^T as four wgmma m64n64k16 with both operands in shared memory; online softmax in
//   registers (thread = two query rows, a quad of lanes shares a row); O += P V as four wgmma with P straight from
//   registers (the accumulator layout of S is the A-fragment layout) and V as an MN-major B operand (V stays [key][dim] as
//   TMA delivered it).  The row sum adds the bf16-rounded weights that P V multiplies, so the output is their exact
//   weighted mean.  With the fp32 weights summed instead (measured with an mma.sync kernel on an H100), the engine's logit
//   error on the decisive-margin golden of tests/test_gpu_parity.py was 0.0625 instead of 0.0556, below that test's
//   required factor 4 under the golden's smallest decision margin (0.247).
//
// The caller chooses the keys through two callables:
//   load_kv(blk, sK, sV, bar)  thread 0: issue K / V block blk by TMA into sK / sV (8192 B each), completing on bar;
//   mask(blk, s)               set the scores of block blk that a row must not see to -inf.  Every row has to keep at
//                              least one key of every block (the running max stays finite).
// Thread 0 prefetches the tensor map descriptors before the call.  On return o holds this thread's outputs, normalised:
// register 4j + e is row warp * 16 + lane / 4 (+ 8 for e >= 2) of the tile, dims 8j + 2 (lane % 4) + (e & 1).
// ------------------------------------------------------------------------------------------------
constexpr int kAttnWgRows = 64;                 // query rows per CTA = keys per K / V block
constexpr int kAttnWgSmem = 5 * 8192 + 64 + 1024;   // Q | K x 2 | V x 2 | barriers | alignment slack

template <class LoadKV, class Mask>
__device__ __forceinline__ void attn_wg_tile(const CUtensorMap* tmQ, int q_col, int q_row, int nblk, float scale_log2,
                                             const LoadKV& load_kv, const Mask& mask, float (&o)[32]) {
  extern __shared__ __align__(1024) uint8_t attn_smem_raw[];
  uint8_t* smem = attn_smem_raw + ((1024u - (smem_u32(attn_smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + 8192;                     // [2 stages][64 keys][128 B]
  uint8_t* sV = smem + 3 * 8192;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 5 * 8192);   // [0] Q, [1 + stage] K | V
  const int tid = threadIdx.x;
  auto issue = [&](int blk, int st) {
    mbar_arrive_expect_tx(&bar[1 + st], 2 * 8192);
    load_kv(blk, sK + st * 8192, sV + st * 8192, &bar[1 + st]);
  };
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bar[0], 8192);
    tma_load_2d(sQ, tmQ, &bar[0], q_col, q_row);
    issue(0, 0);
    if (nblk > 1) issue(1, 1);
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(&bar[0], 0);
  for (int blk = 0; blk < nblk; ++blk) {
    const int st = blk & 1;
    mbar_wait(&bar[1 + st], (blk >> 1) & 1);
    // ---- S = Q K^T -----------------------------------------------------------------------------------
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      Wgmma<64>::mma(s, wgmma_desc_sw128(smem_u32(sQ) + k * 32), wgmma_desc_sw128(smem_u32(sK + st * 8192) + k * 32), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    // ---- mask, online softmax: register 4j + e is row g (e < 2) or g + 8 (e >= 2), key 8j + 2 (lane % 4) + (e & 1) of the block
    mask(blk, s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * j], s[4 * j + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
    float corr[2], m_new[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      m_new[i] = fmaxf(m_run[i], mx[i]);         // finite: mask leaves every row a key in every block
      corr[i] = exp2f((m_run[i] - m_new[i]) * scale_log2);
      m_run[i] = m_new[i];
      l_run[i] *= corr[i];
    }
    uint32_t pa[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t lo = pack_bf16(exp2f((s[4 * j] - m_new[0]) * scale_log2), exp2f((s[4 * j + 1] - m_new[0]) * scale_log2));
      const uint32_t hi = pack_bf16(exp2f((s[4 * j + 2] - m_new[1]) * scale_log2), exp2f((s[4 * j + 3] - m_new[1]) * scale_log2));
      l_run[0] += bf16_lo(lo) + bf16_hi(lo);
      l_run[1] += bf16_lo(hi) + bf16_hi(hi);
      pa[j >> 1][(j & 1) * 2 + 0] = lo;          // A fragment of k-step j / 2: (row g, keys 2t..), (row g + 8, ...), then +8 keys
      pa[j >> 1][(j & 1) * 2 + 1] = hi;
      o[4 * j] *= corr[0];
      o[4 * j + 1] *= corr[0];
      o[4 * j + 2] *= corr[1];
      o[4 * j + 3] *= corr[1];
    }
    // ---- O += P V: 16 keys per k-step = 16 rows of 128 B of the V block --------------------------------------------
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs_mn(o, pa[kk], wgmma_desc_sw128(smem_u32(sV + st * 8192) + kk * 2048));
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                             // every warp is done with stage st: refill it with block blk + 2
    if (tid == 0 && blk + 2 < nblk) issue(blk + 2, st);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 1);
    l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 2);
  }
  const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[4 * j] *= inv0;
    o[4 * j + 1] *= inv0;
    o[4 * j + 2] *= inv1;
    o[4 * j + 3] *= inv1;
  }
}

// flash_attn_wgmma_kernel: non-causal attention for any S (ViT blocks with 197 / 257 keys, the image-row prefill, 6-frame
// video with 1182 keys, 30 x 40 VQA grids with 1201); keys past S (the block may run into the next batch or past the
// tensor) are masked.  One CTA per (64 query rows, head, batch).
//   kRagged (ragged image batches): batch b occupies a slot of p.S rows of which the first p.seq_lens[b] are valid; the
//   batch is computed exactly as a uniform call with S = seq_lens[b] would compute it (the key blocks and query tiles past
//   its length are skipped, not masked) and its output rows past that length are written as zeros.
template <bool kRagged>
__global__ void __launch_bounds__(128) flash_attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                              const __grid_constant__ CUtensorMap tmK,
                                                              const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int S = kRagged ? p.seq_lens[b] : p.S;
  const int q0 = blockIdx.x * kAttnWgRows;
  const int row_base = b * p.S;                  // rows of batch b in the [B * S, H * 64] q / k / v views
  if (kRagged && q0 >= S) {                      // a query tile of the padding: zeros, no arithmetic
    __nv_bfloat16* og = p.out + b * p.o_bs + h * 64;
    for (int i = tid; i < kAttnWgRows * 8; i += 128) {
      const int r = q0 + (i >> 3);
      if (r < p.S) *reinterpret_cast<uint4*>(og + static_cast<long long>(r) * p.o_rs + (i & 7) * 8) = make_uint4(0, 0, 0, 0);
    }
    return;
  }
  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  auto load_kv = [&](int blk, uint8_t* sK, uint8_t* sV, uint64_t* bar) {
    tma_load_2d(sK, &tmK, bar, h * 64, row_base + blk * kAttnWgRows);
    tma_load_2d(sV, &tmV, bar, h * 64, row_base + blk * kAttnWgRows);
  };
  auto mask = [&](int blk, float (&s)[32]) {
    const int key0 = blk * kAttnWgRows + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = key0 + 8 * j;
      if (key >= S) { s[4 * j] = -INFINITY; s[4 * j + 2] = -INFINITY; }
      if (key + 1 >= S) { s[4 * j + 1] = -INFINITY; s[4 * j + 3] = -INFINITY; }
    }
  };
  float o[32];
  attn_wg_tile(&tmQ, h * 64, row_base + q0, (S + kAttnWgRows - 1) / kAttnWgRows, p.scale_log2, load_kv, mask, o);
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
  __nv_bfloat16* og = p.out + b * p.o_bs + h * 64 + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (r0 < S) *reinterpret_cast<uint32_t*>(og + static_cast<long long>(r0) * p.o_rs + 8 * j) = pack_bf16(o[4 * j], o[4 * j + 1]);
    else if (kRagged && r0 < p.S) *reinterpret_cast<uint32_t*>(og + static_cast<long long>(r0) * p.o_rs + 8 * j) = 0u;
    if (r1 < S) *reinterpret_cast<uint32_t*>(og + static_cast<long long>(r1) * p.o_rs + 8 * j) = pack_bf16(o[4 * j + 2], o[4 * j + 3]);
    else if (kRagged && r1 < p.S) *reinterpret_cast<uint32_t*>(og + static_cast<long long>(r1) * p.o_rs + 8 * j) = 0u;
  }
}

// ------------------------------------------------------------------------------------------------
// text_attn_wgmma_kernel: the text rows of a whole caption batch in one pass (caption scoring, the training-branch forward
// of reference layers/decoder.py:916-972 through BertEncoderAsDecoder's block mask :114-137).  Text row t of caption n
// attends to the M_b image keys of its image (image_index[n]) and to text keys 0..t of its own caption.
//   One CTA per (64 text query rows, head, caption): the image keys come first as 64-key blocks of the image K/V cache
//   (masked past M_b), then the caption's own text K/V blocks 0 .. q0 / 64, with the causal mask on the diagonal block
//   only.  Text blocks past the query tile are never loaded.
// ------------------------------------------------------------------------------------------------
struct TextAttnParams {
  __nv_bfloat16* out;          // [N * T] rows of H * 64, row stride o_rs
  int N, T, H;                 // captions, positions per caption, heads
  int M;                       // rows per image in the image K/V view (slot length)
  const int* img_lens;         // null, or [B] valid image keys of each image (ragged batches; <= M)
  const int* image_index;      // null (caption n uses image n), or [N]
  long long o_rs;
  float scale_log2;            // (1/sqrt(64)) * log2(e)
};

__global__ void __launch_bounds__(128) text_attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                             const __grid_constant__ CUtensorMap tmK,
                                                             const __grid_constant__ CUtensorMap tmV,
                                                             const __grid_constant__ CUtensorMap tmIK,
                                                             const __grid_constant__ CUtensorMap tmIV,
                                                             const TextAttnParams p) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, n = blockIdx.z;
  const int q0 = blockIdx.x * kAttnWgRows;
  const int img = p.image_index != nullptr ? p.image_index[n] : n;
  const int Mb = p.img_lens != nullptr ? p.img_lens[img] : p.M;
  const int n_img = (Mb + kAttnWgRows - 1) / kAttnWgRows;
  const int nblk = n_img + q0 / kAttnWgRows + 1;  // image blocks, then text blocks 0 .. the diagonal one
  const int trow = n * p.T;                      // rows of caption n in the [N * T, H * 64] q / k / v views
  const int g0 = warp * 16 + (lane >> 2);        // tile rows of registers e < 2 (g0) and e >= 2 (g0 + 8)
  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmIK);
    tma_prefetch_desc(&tmIV);
  }
  auto load_kv = [&](int blk, uint8_t* sK, uint8_t* sV, uint64_t* bar) {
    if (blk < n_img) {
      tma_load_2d(sK, &tmIK, bar, h * 64, img * p.M + blk * kAttnWgRows);
      tma_load_2d(sV, &tmIV, bar, h * 64, img * p.M + blk * kAttnWgRows);
    } else {
      tma_load_2d(sK, &tmK, bar, h * 64, trow + (blk - n_img) * kAttnWgRows);
      tma_load_2d(sV, &tmV, bar, h * 64, trow + (blk - n_img) * kAttnWgRows);
    }
  };
  auto mask = [&](int blk, float (&s)[32]) {
    const int kk0 = 2 * (lane & 3);              // key (of this block) of register 4j: kk0 + 8j
    if (blk < n_img) {                           // image keys: those past M_b are masked
      const int lim = Mb - blk * kAttnWgRows;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int kk = kk0 + 8 * j;
        if (kk >= lim) { s[4 * j] = -INFINITY; s[4 * j + 2] = -INFINITY; }
        if (kk + 1 >= lim) { s[4 * j + 1] = -INFINITY; s[4 * j + 3] = -INFINITY; }
      }
    } else if (blk + 1 == nblk) {                // the diagonal text block: key q0 + kk is visible to row q0 + r iff kk <= r
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int kk = kk0 + 8 * j;
        if (kk > g0) s[4 * j] = -INFINITY;
        if (kk + 1 > g0) s[4 * j + 1] = -INFINITY;
        if (kk > g0 + 8) s[4 * j + 2] = -INFINITY;
        if (kk + 1 > g0 + 8) s[4 * j + 3] = -INFINITY;
      }
    }
  };
  float o[32];
  attn_wg_tile(&tmQ, h * 64, trow + q0, nblk, p.scale_log2, load_kv, mask, o);
  const int r0 = q0 + g0, r1 = r0 + 8;
  __nv_bfloat16* og = p.out + static_cast<long long>(trow) * p.o_rs + h * 64 + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (r0 < p.T) *reinterpret_cast<uint32_t*>(og + static_cast<long long>(r0) * p.o_rs + 8 * j) = pack_bf16(o[4 * j], o[4 * j + 1]);
    if (r1 < p.T) *reinterpret_cast<uint32_t*>(og + static_cast<long long>(r1) * p.o_rs + 8 * j) = pack_bf16(o[4 * j + 2], o[4 * j + 3]);
  }
}

// one MUFU.EX2 (exp2f() adds a denormal-range fix-up the softmax does not need: those terms vanish against a row sum >= 1)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ------------------------------------------------------------------------------------------------
struct DecAttnParams {
  const float* qkv;                // [n_partials][R, 3*D] fp32 (q | k | v): the QKV GEMM's split-K partial sums, added
  int n_partials;                  //   here in split order (1..4 buffers, partial_stride elements apart)
  long long partial_stride;
  const float* bqkv;               // [3*D] bias, added here
  const __nv_bfloat16* img_k;      // [B, M, D]
  const __nv_bfloat16* img_v;
  __nv_bfloat16* txt_k;            // [R, T_alloc, D]
  __nv_bfloat16* txt_v;
  const int* src_row;              // [R, T_alloc] physical row holding text position j of logical row r (null = r)
  __nv_bfloat16* ctx;              // [R, D]
  int B, M, T_alloc, D;            // B: sequence groups of NQ rows each (R = B * NQ)
  int seqs_per_image;              // groups that share one image's K/V: group b reads image b / seqs_per_image
  const StepState* state;          // text position = state->pos (or pos_fixed when null)
  int pos_fixed;
  int chunk_rows;                  // image keys staged per TMA round (<= 512), box_rows * n_boxes
  int box_rows;                    // rows per TMA box (<= 256)
  ChainSync chain;
  const int* img_lens;             // decode_attn_kernel<., true>: [B] valid image keys of each image (M = slot length;
                                   //   chunk_rows = the staging buffer's rows, box_rows = kDecAttnRaggedBox)
};

// Image keys of one (image, head) item are staged in chunks of at most kDecAttnChunk rows, all of one length: at least two
// CTAs per SM fit (M = 257 in one piece would be 131 KB per CTA).  The chunking fixes which key group of the kernel sees
// which key, so a ragged batch derives it from each image's own key count, as a uniform call of that image would.
constexpr int kDecAttnChunk = 224;
constexpr int kDecAttnRaggedBox = 32;   // ragged batches: rows per TMA box (the chunk length varies per image)
__host__ __device__ __forceinline__ int dec_attn_chunk_rows(int M) {
  const int n_chunks = (M + kDecAttnChunk - 1) / kDecAttnChunk;
  return (M + n_chunks - 1) / n_chunks;
}

__device__ __forceinline__ void bf16x8_to_f32(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x);
  f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z);
  f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}

// One q / k / v element of this step: the split-K partial sums in split order (fixed order: bit-reproducible).
__device__ __forceinline__ float ld_partials(const float* ptr, int n, long long stride) {
  const float a = __ldcg(ptr);
  const float b = n > 1 ? __ldcg(ptr + stride) : 0.f;
  const float c = n > 2 ? __ldcg(ptr + 2 * stride) : 0.f;
  const float d = n > 3 ? __ldcg(ptr + 3 * stride) : 0.f;
  return ((a + b) + c) + d;
}

// Online-softmax state of one 8-lane key group for one query: running max m, running sum l, 8 output dims.
__device__ __forceinline__ void dec_attn_update(float (&sc)[4], const uint4 (&w)[4], float& m, float& l, float (&acc)[8]) {
  float m_new = fmaxf(fmaxf(fmaxf(sc[0], sc[1]), fmaxf(sc[2], sc[3])), m);
  if (m_new == -INFINITY) return;  // nothing valid seen yet
  const float scale = __expf(m - m_new);
  float p[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __expf(sc[i] - m_new);
  l = l * scale + (p[0] + p[1]) + (p[2] + p[3]);
#pragma unroll
  for (int d = 0; d < 8; ++d) acc[d] *= scale;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float f[8];
    bf16x8_to_f32(w[i], f);
#pragma unroll
    for (int d = 0; d < 8; ++d) acc[d] = fmaf(p[i], f[d], acc[d]);
  }
  m = m_new;
}

// Persistent, double-buffered streaming kernel: CTA c handles the (image, head) items c, c+G, c+2G, ...  Each item's
// image K/V slice (M rows of 128 B, constant during decoding) is fetched by TMA into one of two shared-memory
// buffers; the first two fetches are issued BEFORE the dependency wait, so under programmatic dependent launch most
// of this kernel's HBM stream overlaps the QKV GEMM that precedes it, and later fetches overlap the arithmetic of
// the previous item.  128 threads = 16 key groups x 8 lanes (8 head dims each, 128-bit accesses); scores are folded
// into per-group online-softmax states merged at the end (flash-decoding style), single pass over K and V.
//
// NQ == 1 (greedy decoding): software pipelining of the two global-memory round trips an item used to expose -- the step's
// own q/k/v of item k+1 are requested at the top of item k, and the text K/V rows of an item are requested before its
// image-key loop (shared memory) and consumed after it.  At 256 rows a CTA walks ~10 items, so the exposed latencies
// (not the HBM stream) bounded the kernel.
//
// kRagged: every image has its own key count img_lens[b] (<= M, the slot length) and chunk length, so each item is
// computed exactly as in a uniform call of its image; the CTA's chunk sequence is no longer one fixed count per item.
template <int NQ, bool kRagged = false>
__global__ void __launch_bounds__(128)
decode_attn_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, const DecAttnParams p) {
  extern __shared__ uint8_t attn_dyn[];
  uint8_t* sbase = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(attn_dyn) + 127) & ~uintptr_t(127));
  const size_t kv_bytes = static_cast<size_t>(p.chunk_rows) * 128;  // one of K / V of one unit
  __shared__ uint64_t bars[2];
  __shared__ float q_s[NQ][64];
  __shared__ float red_m[4][NQ];
  __shared__ float red_l[4][NQ];
  __shared__ float red_acc[4][NQ][64];

  const int tid = threadIdx.x;
  const int D = p.D;
  const int H = D / 64;
  const int n_items = p.B * H;
  const int G = gridDim.x;
  const int n_chunks = (p.M + p.chunk_rows - 1) / p.chunk_rows;
  const int n_my = (n_items - static_cast<int>(blockIdx.x) + G - 1) / G;
  int n_units = n_my * n_chunks;
  if constexpr (kRagged) {
    n_units = 0;
    for (int k = 0; k < n_my; ++k) {
      const int Mb = p.img_lens[(static_cast<int>(blockIdx.x) + k * G) / H / p.seqs_per_image];
      n_units += (Mb + dec_attn_chunk_rows(Mb) - 1) / dec_attn_chunk_rows(Mb);
    }
  }

  griddep_launch_early();
  tl_mark(100003);
  if (tid == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  int iss_k = 0, iss_c = 0;       // kRagged: item / chunk of the next unit to fetch (thread 0 issues the units in order)
  auto issue_unit = [&](int u) {  // one thread
    const int k = kRagged ? iss_k : u / n_chunks;
    const int c = kRagged ? iss_c : u - k * n_chunks;
    const int item = blockIdx.x + k * G;
    const int b = item / H, h = item - b * H;
    const int img = b / p.seqs_per_image;
    uint8_t* sK = sbase + static_cast<size_t>(u & 1) * 2 * kv_bytes;
    uint8_t* sV = sK + kv_bytes;
    const int Mb = kRagged ? p.img_lens[img] : p.M;
    const int crows = kRagged ? dec_attn_chunk_rows(Mb) : p.chunk_rows;
    const int box = kRagged ? kDecAttnRaggedBox : p.box_rows;
    const int rows_c = min(crows, Mb - c * crows);
    const int nb = (rows_c + box - 1) / box;
    mbar_arrive_expect_tx(&bars[u & 1], static_cast<uint32_t>(2 * nb * box * 128));
    for (int i = 0; i < nb; ++i) {
      const int grow = img * p.M + c * crows + i * box;
      const int gcol = h * 64;
      tma_load_2d(sK + static_cast<size_t>(i) * box * 128, &tmK, &bars[u & 1], gcol, grow);
      tma_load_2d(sV + static_cast<size_t>(i) * box * 128, &tmV, &bars[u & 1], gcol, grow);
    }
    if (kRagged && ++iss_c * crows >= Mb) { iss_c = 0; ++iss_k; }
  };
  if (tid == 0) {
    issue_unit(0);
    if (n_units > 1) issue_unit(1);
  }
  if (step_wait(p.state != nullptr ? &p.state->finished : nullptr, p.chain)) {
    // never leave with a bulk copy in flight into this CTA's shared memory
    mbar_wait(&bars[0], 0);
    if (n_units > 1) mbar_wait(&bars[1], 0);
    return;
  }
  tl_mark(3);
  const int pos = (p.state != nullptr) ? p.state->pos : p.pos_fixed;
  const int n_txt = pos + 1;
  const int grp = tid >> 3;
  const int gl = tid & 7;
  const int warp = tid >> 5;
  const int lane = tid & 31;

  // This step's q/k/v of every item of this CTA are requested together (one L2 round trip instead of one per item):
  // threads 0-63 hold (q, k) of dim tid, threads 64-127 hold v of dim tid-64.
  constexpr int kPre = (NQ == 1) ? 4 : 1;
  float pre_a[kPre], pre_b[kPre];
#pragma unroll
  for (int k = 0; k < kPre; ++k) {
    pre_a[k] = 0.f;
    pre_b[k] = 0.f;
    if (NQ == 1 && k < n_my) {
      const int item = blockIdx.x + k * G;
      const int b = item / H, h = item - b * H;
      const float* row = p.qkv + static_cast<long long>(b) * 3 * D + h * 64;
      if (tid < 64) {
        pre_a[k] = ld_partials(row + tid, p.n_partials, p.partial_stride);
        pre_b[k] = ld_partials(row + D + tid, p.n_partials, p.partial_stride);
      } else {
        pre_a[k] = ld_partials(row + 2 * D + tid - 64, p.n_partials, p.partial_stride);
      }
    }
  }

  // NQ == 1: (q, k | v) of the NEXT item, requested one item ahead
  float nxt_a = 0.f, nxt_b = 0.f;
  auto request_qkv = [&](int k, float& a, float& b2) {
    if (k < n_my) {
      const int item = blockIdx.x + k * G;
      const int b = item / H, h = item - b * H;
      const float* row = p.qkv + static_cast<long long>(b) * 3 * D + h * 64;
      if (tid < 64) {
        a = ld_partials(row + tid, p.n_partials, p.partial_stride);
        b2 = ld_partials(row + D + tid, p.n_partials, p.partial_stride);
      } else {
        a = ld_partials(row + 2 * D + tid - 64, p.n_partials, p.partial_stride);
      }
    }
  };
  if (NQ == 1) request_qkv(kPre, nxt_a, nxt_b);   // items 0..kPre-1 were requested above

  int u_base = 0;                 // units of the items before this one
  for (int k = 0; k < n_my; ++k) {
    const int item = blockIdx.x + k * G;
    const int b = item / H, h = item - b * H;
    const int Mb = kRagged ? p.img_lens[b / p.seqs_per_image] : p.M;
    const int crows = kRagged ? dec_attn_chunk_rows(Mb) : p.chunk_rows;
    const int nch = kRagged ? (Mb + crows - 1) / crows : n_chunks;
    float cur_a = 0.f, cur_b = 0.f;
    if (NQ == 1 && k >= kPre) {
      cur_a = nxt_a;
      cur_b = nxt_b;
      request_qkv(k + 1, nxt_a, nxt_b);
    }
    // ---- q (scaled by 1/8 in fp32 like the reference scales Q), append this step's K/V (bf16) ----
    for (int qi = 0; qi < NQ; ++qi) {
      const int r = b * NQ + qi;
      const float* row = p.qkv + static_cast<long long>(r) * 3 * D + h * 64;
      const float* bias = p.bqkv + h * 64;
      const bool have = (NQ == 1) && (k < kPre);
      if (tid < 64) {
        const float qv = have ? pre_a[k < kPre ? k : 0] : (NQ == 1 ? cur_a : ld_partials(row + tid, p.n_partials, p.partial_stride));
        const float kv = have ? pre_b[k < kPre ? k : 0] : (NQ == 1 ? cur_b : ld_partials(row + D + tid, p.n_partials, p.partial_stride));
        q_s[qi][tid] = (qv + bias[tid]) * 0.125f;
        p.txt_k[(static_cast<long long>(r) * p.T_alloc + pos) * D + h * 64 + tid] = __float2bfloat16_rn(kv + bias[D + tid]);
      } else {
        const int d = tid - 64;
        const float vv = have ? pre_a[k < kPre ? k : 0] : (NQ == 1 ? cur_a : ld_partials(row + 2 * D + d, p.n_partials, p.partial_stride));
        p.txt_v[(static_cast<long long>(r) * p.T_alloc + pos) * D + h * 64 + d] = __float2bfloat16_rn(vv + bias[2 * D + d]);
      }
    }
    __syncthreads();

    float qreg[NQ][8];
    float m_run[NQ], l_run[NQ], acc[NQ][8];
#pragma unroll
    for (int qi = 0; qi < NQ; ++qi) {
      m_run[qi] = -INFINITY;
      l_run[qi] = 0.f;
#pragma unroll
      for (int d = 0; d < 8; ++d) {
        qreg[qi][d] = q_s[qi][gl * 8 + d];
        acc[qi][d] = 0.f;
      }
    }
    // ---- text keys (global loads): each beam row has its own history (through the src_row indirection) ----
    auto text_chunk_load = [&](int r, int base, uint4 (&u)[4], uint4 (&w)[4]) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = base + grp + 16 * i;
        if (j < n_txt) {
          const int pr = (p.src_row != nullptr) ? p.src_row[r * p.T_alloc + j] : r;
          const long long off = (static_cast<long long>(pr) * p.T_alloc + j) * D + h * 64 + gl * 8;
          u[i] = *reinterpret_cast<const uint4*>(p.txt_k + off);
          w[i] = *reinterpret_cast<const uint4*>(p.txt_v + off);
        } else {
          u[i] = make_uint4(0, 0, 0, 0);
          w[i] = make_uint4(0, 0, 0, 0);
        }
      }
    };
    auto text_chunk_use = [&](int qi, int base, const uint4 (&u)[4], const uint4 (&w)[4]) {
      float sc[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float kf[8];
        bf16x8_to_f32(u[i], kf);
        float a = 0.f;
#pragma unroll
        for (int d = 0; d < 8; ++d) a = fmaf(qreg[qi][d], kf[d], a);
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 2);
        a += __shfl_xor_sync(0xffffffffu, a, 4);
        sc[i] = (base + grp + 16 * i < n_txt) ? a : -INFINITY;
      }
      dec_attn_update(sc, w, m_run[qi], l_run[qi], acc[qi]);
    };
    uint4 tu[4], tw[4];                       // NQ == 1: text positions 0..63 of this item, in flight across the image loop
    if (NQ == 1) {
      text_chunk_load(b, 0, tu, tw);
    } else {
#pragma unroll
      for (int qi = 0; qi < NQ; ++qi) {
        const int r = b * NQ + qi;
        for (int base = 0; base < n_txt; base += 64) {
          uint4 u[4], w[4];
          text_chunk_load(r, base, u, w);
          text_chunk_use(qi, base, u, w);
        }
      }
    }
    // ---- image keys from shared memory: shared by the NQ beams of this image ----
    for (int c = 0; c < nch; ++c) {
      const int u_idx = (kRagged ? u_base : k * n_chunks) + c;
      const uint8_t* sK = sbase + static_cast<size_t>(u_idx & 1) * 2 * kv_bytes;
      const uint8_t* sV = sK + kv_bytes;
      mbar_wait(&bars[u_idx & 1], static_cast<uint32_t>((u_idx >> 1) & 1));
      const int rows_c = min(crows, Mb - c * crows);
      for (int base = 0; base < rows_c; base += 64) {  // uniform trip count: the shuffles below stay converged
        uint4 u[4], w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int s = base + grp + 16 * i;
          const bool ok = s < rows_c;
          u[i] = ok ? *reinterpret_cast<const uint4*>(sK + static_cast<size_t>(s) * 128 + gl * 16) : make_uint4(0, 0, 0, 0);
          w[i] = ok ? *reinterpret_cast<const uint4*>(sV + static_cast<size_t>(s) * 128 + gl * 16) : make_uint4(0, 0, 0, 0);
        }
        float kf[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i) bf16x8_to_f32(u[i], kf[i]);
#pragma unroll
        for (int qi = 0; qi < NQ; ++qi) {
          float sc[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float a = 0.f;
#pragma unroll
            for (int d = 0; d < 8; ++d) a = fmaf(qreg[qi][d], kf[i][d], a);
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            a += __shfl_xor_sync(0xffffffffu, a, 2);
            a += __shfl_xor_sync(0xffffffffu, a, 4);
            sc[i] = (base + grp + 16 * i < rows_c) ? a : -INFINITY;
          }
          dec_attn_update(sc, w, m_run[qi], l_run[qi], acc[qi]);
        }
      }
      __syncthreads();  // everyone is done with this buffer: refill it with the unit after next
      if (tid == 0 && u_idx + 2 < n_units) issue_unit(u_idx + 2);
    }
    u_base += nch;
    if (NQ == 1) {
      text_chunk_use(0, 0, tu, tw);
      for (int base = 64; base < n_txt; base += 64) {   // captions longer than 64 tokens: the rest the plain way
        uint4 u[4], w[4];
        text_chunk_load(b, base, u, w);
        text_chunk_use(0, base, u, w);
      }
    }
    // ---- merge the 16 group states: 4 groups of a warp by shuffles, the 4 warps through smem ----
#pragma unroll
    for (int qi = 0; qi < NQ; ++qi) {
#pragma unroll
      for (int o = 8; o <= 16; o <<= 1) {
        const float m_o = __shfl_xor_sync(0xffffffffu, m_run[qi], o);
        const float l_o = __shfl_xor_sync(0xffffffffu, l_run[qi], o);
        const float m_n = fmaxf(m_run[qi], m_o);
        const float sa = (m_run[qi] == -INFINITY) ? 0.f : __expf(m_run[qi] - m_n);
        const float sb = (m_o == -INFINITY) ? 0.f : __expf(m_o - m_n);
        l_run[qi] = l_run[qi] * sa + l_o * sb;
#pragma unroll
        for (int d = 0; d < 8; ++d) {
          const float a_o = __shfl_xor_sync(0xffffffffu, acc[qi][d], o);
          acc[qi][d] = acc[qi][d] * sa + a_o * sb;
        }
        m_run[qi] = m_n;
      }
      if (lane < 8) {
        if (lane == 0) { red_m[warp][qi] = m_run[qi]; red_l[warp][qi] = l_run[qi]; }
#pragma unroll
        for (int d = 0; d < 8; ++d) red_acc[warp][qi][lane * 8 + d] = acc[qi][d];
      }
    }
    __syncthreads();
    for (int i = tid; i < NQ * 64; i += 128) {
      const int qi = i >> 6;
      const int d = i & 63;
      const float mm = fmaxf(fmaxf(red_m[0][qi], red_m[1][qi]), fmaxf(red_m[2][qi], red_m[3][qi]));
      float l = 0.f, a = 0.f;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float sw = (red_m[w][qi] == -INFINITY) ? 0.f : __expf(red_m[w][qi] - mm);
        l += red_l[w][qi] * sw;
        a += red_acc[w][qi][d] * sw;
      }
      p.ctx[static_cast<long long>(b * NQ + qi) * D + h * 64 + d] = __float2bfloat16_rn(a / l);
    }
    __syncthreads();  // q_s / red_* are reused by the next item
  }
  tl_mark(200003);
  chain_signal(p.chain);
}

// ------------------------------------------------------------------------------------------------
// fp32-grade parity mode (engine option "parity"): attention in plain fp32 -- q, k, v and both K/V caches stay fp32 and the
// context rows leave in the GEMMs' split operand format [hi | lo | hi].  One warp per (sequence, head, query row); scores
// live in shared memory.  Not a fast path: it exists so that the whole engine can be compared with the fp32 reference at
// the 1e-3 logit tolerance of BASELINE.json's north star.
// ------------------------------------------------------------------------------------------------
struct AttnF32Params {
  const float* q;
  const float* k;
  const float* v;
  __nv_bfloat16* out;            // split3 rows: [S, 3 * d_model] per batch element
  int B, S, H, d_model;
  long long q_rs, kv_rs, q_bs, kv_bs, o_bs;   // row / batch strides in elements (output row stride = 3 * d_model)
  const int* seq_lens;           // null, or [B] valid rows of each batch (ragged image batches): rows past it leave as zeros
};

__device__ __forceinline__ void store_split3_pair(__nv_bfloat16* row, int d_model, int col, float a, float b) {
  uint32_t hi, lo;
  pack_split2(a, b, hi, lo);
  *reinterpret_cast<uint32_t*>(row + col) = hi;
  *reinterpret_cast<uint32_t*>(row + d_model + col) = lo;
  *reinterpret_cast<uint32_t*>(row + 2 * d_model + col) = hi;
}

// One query row on one warp: softmax(q k^T) v over n_keys keys in plain fp32.  q_s: the row's q, already scaled by 1/8
// (64 floats in shared memory, visible to the warp); sc: n_keys floats of score scratch; key_row(j, want_v): the 64 fp32
// of key j's K (false) or V (true), 16-byte aligned.  Returns output dims 2 * lane and 2 * lane + 1.
template <class KeyRow>
__device__ __forceinline__ float2 attn_row_f32(const float* q_s, float* sc, int n_keys, const KeyRow& key_row) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int j0 = 0; j0 < n_keys; j0 += 32) {
    const int j = j0 + lane;
    if (j < n_keys) {
      const float4* kr = reinterpret_cast<const float4*>(key_row(j, false));
      float a = 0.f;
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        const float4 kk = kr[d];
        a = fmaf(q_s[4 * d], kk.x, a); a = fmaf(q_s[4 * d + 1], kk.y, a);
        a = fmaf(q_s[4 * d + 2], kk.z, a); a = fmaf(q_s[4 * d + 3], kk.w, a);
      }
      sc[j] = a;
      mx = fmaxf(mx, a);
    }
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < n_keys; j += 32) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float a0 = 0.f, a1 = 0.f;
  for (int j = 0; j < n_keys; ++j) {
    const float2 vv = *reinterpret_cast<const float2*>(key_row(j, true) + 2 * lane);
    a0 = fmaf(sc[j], vv.x, a0);
    a1 = fmaf(sc[j], vv.y, a1);
  }
  return make_float2(a0 / sum, a1 / sum);
}

__global__ void __launch_bounds__(128) attn_f32_kernel(const AttnF32Params p) {
  extern __shared__ __align__(16) float attn_f32_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* q_s = attn_f32_smem + warp * (64 + p.S);
  const long long item = static_cast<long long>(blockIdx.x) * 4 + warp;
  const long long total = static_cast<long long>(p.B) * p.H * p.S;
  if (item >= total) return;
  const int row = static_cast<int>(item % p.S);
  const int h = static_cast<int>((item / p.S) % p.H);
  const int b = static_cast<int>(item / (static_cast<long long>(p.S) * p.H));
  const int S = p.seq_lens != nullptr ? p.seq_lens[b] : p.S;
  __nv_bfloat16* orow = p.out + b * p.o_bs + static_cast<long long>(row) * 3 * p.d_model;
  if (row >= S) {
    store_split3_pair(orow, p.d_model, h * 64 + 2 * lane, 0.f, 0.f);
    return;
  }
  const float* qg = p.q + b * p.q_bs + static_cast<long long>(row) * p.q_rs + h * 64;
  q_s[lane] = qg[lane] * 0.125f;             // Q / sqrt(64) before the product (reference layers/bert/modeling_bert.py:42-43)
  q_s[lane + 32] = qg[lane + 32] * 0.125f;
  __syncwarp();
  const float2 r = attn_row_f32(q_s, q_s + 64, S, [&](int j, bool want_v) {
    return (want_v ? p.v : p.k) + b * p.kv_bs + static_cast<long long>(j) * p.kv_rs + h * 64;
  });
  store_split3_pair(orow, p.d_model, h * 64 + 2 * lane, r.x, r.y);
}

// Parity-mode sibling of text_attn_wgmma_kernel: plain fp32, one warp per (caption, head, text row); q / k / v fp32 rows of
// d_model elements ([N * T] text rows, [B * M] image rows), output rows in the split format [hi | lo | hi] (3 * d_model).
struct TextAttnF32Params {
  const float* q;
  const float* k;                // text K / V [N * T, d_model]
  const float* v;
  const float* img_k;            // image K / V [B * M, d_model]
  const float* img_v;
  __nv_bfloat16* out;            // [N * T, 3 * d_model]
  int N, T, H, d_model, M;
  const int* img_lens;           // null or [B]
  const int* image_index;        // null or [N]
};

__global__ void __launch_bounds__(128) text_attn_f32_kernel(const TextAttnF32Params p) {
  extern __shared__ __align__(16) float attn_f32_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* q_s = attn_f32_smem + warp * (64 + p.M + p.T);
  const long long item = static_cast<long long>(blockIdx.x) * 4 + warp;
  const long long total = static_cast<long long>(p.N) * p.H * p.T;
  if (item >= total) return;
  const int t = static_cast<int>(item % p.T);
  const int h = static_cast<int>((item / p.T) % p.H);
  const int n = static_cast<int>(item / (static_cast<long long>(p.T) * p.H));
  const int img = p.image_index != nullptr ? p.image_index[n] : n;
  const int Mb = p.img_lens != nullptr ? p.img_lens[img] : p.M;
  const long long trow = static_cast<long long>(n) * p.T;
  const float* qg = p.q + (trow + t) * p.d_model + h * 64;
  q_s[lane] = qg[lane] * 0.125f;             // Q / sqrt(64) before the product (reference layers/bert/modeling_bert.py:42-43)
  q_s[lane + 32] = qg[lane + 32] * 0.125f;
  __syncwarp();
  const float2 r = attn_row_f32(q_s, q_s + 64, Mb + t + 1, [&](int j, bool want_v) {   // image keys, then text keys 0..t
    if (j < Mb) return (want_v ? p.img_v : p.img_k) + (static_cast<long long>(img) * p.M + j) * p.d_model + h * 64;
    return (want_v ? p.v : p.k) + (trow + j - Mb) * p.d_model + h * 64;
  });
  store_split3_pair(p.out + (trow + t) * 3 * p.d_model, p.d_model, h * 64 + 2 * lane, r.x, r.y);
}

struct DecAttnF32Params {
  const float* qkv;               // split-K partial sums of this step's q | k | v, as in DecAttnParams
  int n_partials;
  long long partial_stride;
  const float* bqkv;
  const float* img_k;             // fp32 [B, M, D]
  const float* img_v;
  float* txt_k;                   // fp32 [R, T_alloc, D]
  float* txt_v;
  const int* src_row;
  __nv_bfloat16* ctx;             // split3 rows [R, 3 * D]
  int R, rows_per_image, M, T_alloc, D;   // row r reads image r / rows_per_image (sequences per image x beam)
  const StepState* state;
  int pos_fixed;
  ChainSync chain;
  const int* img_lens;            // null, or [B] valid image keys of each image (ragged batches; M is the slot length)
};

// Shared memory of one warp of decode_attn_f32_kernel in floats: q | k | v of the new token, then the scores; a multiple
// of 4 so that every warp's k / v rows are 16-byte aligned.
__host__ __device__ __forceinline__ int dec_attn_f32_warp_floats(int M, int T_alloc) { return (192 + M + T_alloc + 3) & ~3; }

// one warp per (sequence r, head h); 4 warps per CTA
__global__ void __launch_bounds__(128) decode_attn_f32_kernel(const DecAttnF32Params p) {
  extern __shared__ __align__(16) float attn_f32_smem[];
  griddep_launch_early();
  if (step_wait(p.state != nullptr ? &p.state->finished : nullptr, p.chain)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int D = p.D, H = D / 64;
  const int pos = (p.state != nullptr) ? p.state->pos : p.pos_fixed;
  float* q_s = attn_f32_smem + warp * dec_attn_f32_warp_floats(p.M, p.T_alloc);
  float* k_s = q_s + 64;
  float* v_s = q_s + 128;
  const int item = blockIdx.x * 4 + warp;
  if (item < p.R * H) {
    const int r = item / H, h = item - r * H;
    const int b = r / p.rows_per_image;
    const int Mb = p.img_lens != nullptr ? p.img_lens[b] : p.M;
    const int n_keys = Mb + pos + 1;
    const float* row = p.qkv + static_cast<long long>(r) * 3 * D + h * 64;
    const float* bias = p.bqkv + h * 64;
    for (int d = lane; d < 64; d += 32) {
      q_s[d] = (ld_partials(row + d, p.n_partials, p.partial_stride) + bias[d]) * 0.125f;
      const float kn = ld_partials(row + D + d, p.n_partials, p.partial_stride) + bias[D + d];
      const float vn = ld_partials(row + 2 * D + d, p.n_partials, p.partial_stride) + bias[2 * D + d];
      k_s[d] = kn;
      v_s[d] = vn;
      p.txt_k[(static_cast<long long>(r) * p.T_alloc + pos) * D + h * 64 + d] = kn;
      p.txt_v[(static_cast<long long>(r) * p.T_alloc + pos) * D + h * 64 + d] = vn;
    }
    __syncwarp();
    // image keys, then text positions 0..pos-1 through src_row, then the new token from shared memory
    const float2 o = attn_row_f32(q_s, q_s + 192, n_keys, [&](int j, bool want_v) -> const float* {
      if (j == n_keys - 1) return want_v ? v_s : k_s;
      if (j < Mb) return (want_v ? p.img_v : p.img_k) + (static_cast<long long>(b) * p.M + j) * D + h * 64;
      const int t = j - Mb;
      const int pr = (p.src_row != nullptr) ? p.src_row[r * p.T_alloc + t] : r;
      return (want_v ? p.txt_v : p.txt_k) + (static_cast<long long>(pr) * p.T_alloc + t) * D + h * 64;
    });
    store_split3_pair(p.ctx + static_cast<long long>(r) * 3 * D, D, h * 64 + 2 * lane, o.x, o.y);
  }
  chain_signal(p.chain);
}

}  // namespace gitb200
