// Row-wise HBM-bound kernels of the GIT hot path: LayerNorm (+bias/+residual/+temporal embedding),
// patch im2col, CLS/pos-embed/ln_pre, token embedding + LN, and the greedy selection kernels; also the CTA reductions
// and scans, the step-logits row and the step close that every selection kernel of the decode step shares.
// One warp per row, 128-bit loads/stores, fp32 statistics (two-pass: mean, then biased variance,
// like torch.nn.functional.layer_norm).
#pragma once
#include "ptx.cuh"

namespace gitb200 {

// Decode-loop state shared by the kernels of one generate() call (device memory, one per engine).
struct StepState {
  int pos;            // text position of the token fed at the current step (0-based, prefix included)
  int cur_len;        // tokens currently in tokens_out (start tokens + generated)
  int finished;       // greedy: every row ended with EOS -> remaining steps are no-ops
  int final_len;      // number of valid columns of tokens_out
  int step;           // number of decode steps executed so far
  int empty_caption;  // greedy step-0 special case (reference layers/decoder.py:279-291)
  unsigned int ticket;
  int live;           // units still live at this step, counted by close_step and reset by the last ticket: greedy rows
                      // whose next token is not EOS, beam-search images not yet done
  int error;          // decode_mega_kernel: the MegaWaitError of the first bounded wait that gave up (0: none)
  int bad_draw;       // beam_sample_kernel: 0x7fffffff - (step * rows + row) of the first row with fewer than two tokens
                      // to draw from (0: none)
};

// Why a bounded wait of decode_mega_kernel gave up: a protocol bug ends in one of these codes, not in a hung device.
enum MegaWaitError : int {
  kWaitGridBarrier = 1,   // a compute thread at a grid barrier between phases
  kWaitRingFull = 2,      // a compute warp waiting for a ring chunk to land
  kWaitRingEmpty = 3,     // the producer waiting for the compute warps to free a ring slot
  kWaitTextKv = 4,        // the producer waiting for the layer's QKV phase before it fetches the text K/V
  kWaitRingArmed = 5,     // a compute warp waiting for the producer to arm an attention chunk
  kWaitTimelineProbe = 99 // timeline build only: the probe that makes a mark wait for the A operand's loads
};
inline const char* mega_wait_error_name(int code) {
  switch (code) {
    case kWaitGridBarrier: return "grid barrier";
    case kWaitRingFull: return "ring consumer: chunk never landed";
    case kWaitRingEmpty: return "ring producer: slot never freed";
    case kWaitTextKv: return "ring producer: text K/V never written";
    case kWaitRingArmed: return "ring consumer: attention chunk never armed";
    case kWaitTimelineProbe: return "timeline probe";
    default: return "unknown code";
  }
}

struct LnParams {
  const float* x;        // [rows, D] fp32 (ldx == D)
  const float* bias;     // [D] or null: added to x first
  const float* resid;    // [rows, D] or null: added to x first
  const float* gamma;
  const float* beta;
  float eps;
  float* out_f32;        // may alias x (in place) or be null
  __nv_bfloat16* out_bf16;  // or null
  int rows;
  int n_partials;        // > 1: x is the first of n split-K partial-sum buffers, partial_stride elements apart; they are
  long long partial_stride;  // added in split order (fixed order -> bit-reproducible; nothing to re-zero)
  // optional frame remap (video path, reference layers/decoder.py:846-851): input row (f*B + b)*L + l ->
  // output row b*(F*L) + f*L + l, plus `+ temb[f]` AFTER the normalisation.
  const float* temb;     // [F, D] or null
  int remap_B, remap_F, remap_L;  // remap_F == 0 -> identity
  const int* skip_flag;  // device int: non-zero -> kernel is a no-op (finished decode)
  int split3;            // parity mode: out_bf16 rows are [hi | lo | hi] (3 x D columns, see split_bf16 in ptx.cuh)
  ChainSync chain;       // decode-step flag ordering (counters == null: plain / PDL ordering)
};

// The LayerNorm row routine of every LN kernel below: one warp holds a row of D floats as NV = D / 128 float4 per lane.
// Two-pass statistics: the mean, then rsqrtf(biased variance + eps).
template <int D>
__device__ __forceinline__ void ln_row_stats(const float4 (&v)[D / 128], float eps, float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < D / 128; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  mean = warp_sum(s) * (1.0f / D);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < D / 128; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    ss += (a * a + b * b) + (c * c + d * d);
  }
  rstd = rsqrtf(warp_sum(ss) * (1.0f / D) + eps);
}
// One float4 of the normalised row.
__device__ __forceinline__ float4 ln_norm(const float4 v, float mean, float rstd, const float4 g, const float4 b) {
  return make_float4((v.x - mean) * rstd * g.x + b.x, (v.y - mean) * rstd * g.y + b.y, (v.z - mean) * rstd * g.z + b.z,
                     (v.w - mean) * rstd * g.w + b.w);
}
// Stores float4 k (= i * 32 + lane) of output row `row`: fp32 to out_f32, and bf16 to out_bf16, or [hi | lo | hi] rows of
// 3 D there when split3 (parity mode's GEMM operand format, see split_bf16 in ptx.cuh).  A null output is skipped.
template <int D>
__device__ __forceinline__ void ln_store(float* out_f32, __nv_bfloat16* out_bf16, int split3, long long row, int k,
                                         const float4 o) {
  if (out_f32 != nullptr) reinterpret_cast<float4*>(out_f32 + row * D)[k] = o;
  if (out_bf16 != nullptr && split3) {
    uint2 hi, lo;
    pack_split2(o.x, o.y, hi.x, lo.x);
    pack_split2(o.z, o.w, hi.y, lo.y);
    uint2* dst = reinterpret_cast<uint2*>(out_bf16 + row * 3 * D) + k;
    dst[0] = hi; dst[D / 4] = lo; dst[D / 2] = hi;
  } else if (out_bf16 != nullptr) {
    uint2 pk;
    pk.x = pack_bf16(o.x, o.y);
    pk.y = pack_bf16(o.z, o.w);
    reinterpret_cast<uint2*>(out_bf16 + row * D)[k] = pk;
  }
}

// PRE: fetch gamma / beta / bias before the dependency wait (decode chain: hides one L2 round trip; costs registers,
// so the big encoder LayerNorms use PRE = false).
template <int D, bool PRE>
__global__ void __launch_bounds__(256) layernorm_kernel(const LnParams p) {
  static_assert(D % 128 == 0, "D");
  constexpr int NV = D / 128;
  griddep_launch_early();
  tl_mark(100002);
  const int lane = threadIdx.x & 31;
  // parameters are constants: fetch them before the dependency wait
  float4 gam[PRE ? NV : 1], bet[PRE ? NV : 1], bia[PRE ? NV : 1];
  if (PRE) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      gam[i] = __ldg(reinterpret_cast<const float4*>(p.gamma) + i * 32 + lane);
      bet[i] = __ldg(reinterpret_cast<const float4*>(p.beta) + i * 32 + lane);
      bia[i] = (p.bias != nullptr) ? __ldg(reinterpret_cast<const float4*>(p.bias) + i * 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if (step_wait(p.skip_flag, p.chain)) return;
  tl_mark(2);
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= p.rows) {
    chain_signal(p.chain);
    return;
  }
  float4 v[NV];
  const float4* xp = reinterpret_cast<const float4*>(p.x + static_cast<long long>(row) * D);
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = __ldcg(xp + i * 32 + lane);
  for (int s0 = 1; s0 < p.n_partials; s0 += 3) {   // three partial buffers per round trip, added in split order
    float4 w[3][NV];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const bool ok = s0 + k < p.n_partials;
      const float4* sp = reinterpret_cast<const float4*>(p.x + (ok ? s0 + k : 0) * p.partial_stride + static_cast<long long>(row) * D);
#pragma unroll
      for (int i = 0; i < NV; ++i) w[k][i] = ok ? __ldcg(sp + i * 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
      for (int i = 0; i < NV; ++i) { v[i].x += w[k][i].x; v[i].y += w[k][i].y; v[i].z += w[k][i].z; v[i].w += w[k][i].w; }
    }
  }
  if (p.resid != nullptr) {
    const float4* rp = reinterpret_cast<const float4*>(p.resid + static_cast<long long>(row) * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 r = __ldcg(rp + i * 32 + lane);
      v[i].x += r.x; v[i].y += r.y; v[i].z += r.z; v[i].w += r.w;
    }
  }
  if (PRE) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i].x += bia[i].x; v[i].y += bia[i].y; v[i].z += bia[i].z; v[i].w += bia[i].w;
    }
  } else if (p.bias != nullptr) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias) + i * 32 + lane);
      v[i].x += b.x; v[i].y += b.y; v[i].z += b.z; v[i].w += b.w;
    }
  }
  float mean, rstd;
  ln_row_stats<D>(v, p.eps, mean, rstd);

  long long orow = row;
  int frame = 0;
  if (p.remap_F > 0) {
    const int img = row / p.remap_L;
    const int l = row - img * p.remap_L;
    frame = img / p.remap_B;
    const int b = img - frame * p.remap_B;
    orow = (static_cast<long long>(b) * p.remap_F + frame) * p.remap_L + l;
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = PRE ? gam[i] : __ldg(reinterpret_cast<const float4*>(p.gamma) + i * 32 + lane);
    const float4 b = PRE ? bet[i] : __ldg(reinterpret_cast<const float4*>(p.beta) + i * 32 + lane);
    float4 o = ln_norm(v[i], mean, rstd, g, b);
    if (p.temb != nullptr) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p.temb + static_cast<long long>(frame) * D) + i * 32 + lane);
      o.x += t.x; o.y += t.y; o.z += t.z; o.w += t.w;
    }
    ln_store<D>(p.out_f32, p.out_bf16, p.split3, orow, i * 32 + lane, o);
  }
  tl_mark(200002);
  chain_signal(p.chain);
}

// Positional embedding [1 + g0*g0, d] re-sampled to a gh x gw grid for inputs whose size differs from the resolution the
// embedding was built for (reference layers/CLIP/model.py:245-251): CLS row copied, grid rows =
// F.interpolate(mode='bicubic', align_corners=False), i.e. source coordinate (o + 0.5) * in / out - 0.5, Keys cubic with
// A = -0.75 over taps floor(x) - 1 .. floor(x) + 2 clamped to the grid. One thread per (token, 4 channels).
__device__ __forceinline__ void cubic_coeffs_a075(float t, float w[4]) {
  const float A = -0.75f;
  const float x0 = t + 1.0f, x1 = t, x2 = 1.0f - t, x3 = 2.0f - t;
  w[0] = ((A * x0 - 5.0f * A) * x0 + 8.0f * A) * x0 - 4.0f * A;
  w[1] = ((A + 2.0f) * x1 - (A + 3.0f)) * x1 * x1 + 1.0f;
  w[2] = ((A + 2.0f) * x2 - (A + 3.0f)) * x2 * x2 + 1.0f;
  w[3] = ((A * x3 - 5.0f * A) * x3 + 8.0f * A) * x3 - 4.0f * A;
}
__global__ void __launch_bounds__(256)
pos_embed_bicubic_kernel(const float* __restrict__ pos, float* __restrict__ out, int g0, int gh, int gw, int d) {
  const int d4 = d >> 2;
  const long long total = static_cast<long long>(1 + gh * gw) * d4;
  const float sy = static_cast<float>(g0) / static_cast<float>(gh), sx = static_cast<float>(g0) / static_cast<float>(gw);
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % d4);
    const int tok = static_cast<int>(idx / d4);
    const float4* src = reinterpret_cast<const float4*>(pos);
    float4 acc;
    if (tok == 0) {
      acc = __ldg(src + c);
    } else {
      const int oy = (tok - 1) / gw, ox = (tok - 1) - oy * gw;
      const float ry = sy * (oy + 0.5f) - 0.5f, rx = sx * (ox + 0.5f) - 0.5f;
      const float fy = floorf(ry), fx = floorf(rx);
      float wy[4], wx[4];
      cubic_coeffs_a075(ry - fy, wy);
      cubic_coeffs_a075(rx - fx, wx);
      const int iy = static_cast<int>(fy), ix = static_cast<int>(fx);
      acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int yy = min(max(iy - 1 + a, 0), g0 - 1);
        float4 row = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int xx = min(max(ix - 1 + b, 0), g0 - 1);
          const float4 v = __ldg(src + static_cast<long long>(1 + yy * g0 + xx) * d4 + c);
          row.x += wx[b] * v.x; row.y += wx[b] * v.y; row.z += wx[b] * v.z; row.w += wx[b] * v.w;
        }
        acc.x += wy[a] * row.x; acc.y += wy[a] * row.y; acc.z += wy[a] * row.z; acc.w += wy[a] * row.w;
      }
    }
    reinterpret_cast<float4*>(out)[idx] = acc;
  }
}

// One encoded image of a call (gitb200.cu ImageBatch): [3, h, w] at src_off floats into the call's pixels, a gh x gw patch
// grid and L = gh * gw + 1 valid tokens in its slot of L_max rows; its positional embedding starts at row pos_row of the
// call's positional table.
struct RaggedImg {
  long long src_off;
  int h, w, gh, gw, L, pos_row;
};

// Patch im2col for the stride==kernel conv (reference layers/CLIP/model.py:224,242):
// A[(img, py, px)][(c, ky, kx)] = img[c, py*p+ky, px*p+kx], zero-padded to Kp columns, bf16.  Every image owns
// n_slot = L_max - 1 rows of A (one row map for the patch GEMM); rows past its own gh * gw patches are zero.
__global__ void im2col_patch_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ A,
                                    const RaggedImg* __restrict__ tab, int n_img, int n_slot, int p, int Kp, int split3) {
  const long long total = static_cast<long long>(n_img) * n_slot * (Kp / 8);
  const int K = 3 * p * p;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int kc = static_cast<int>(idx % (Kp / 8));
    const long long row = idx / (Kp / 8);
    const int im = static_cast<int>(row / n_slot);
    const int t = static_cast<int>(row - static_cast<long long>(im) * n_slot);
    const RaggedImg e = tab[im];
    float v[8];
    if (t < e.gh * e.gw) {
      const int py = t / e.gw, px = t - py * e.gw;
      const float* src = img + e.src_off;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = kc * 8 + j;
        float x = 0.f;
        if (k < K) {
          const int c = k / (p * p);
          const int r = k - c * p * p;
          const int ky = r / p;
          const int kx = r - ky * p;
          x = __ldg(src + (static_cast<long long>(c) * e.h + (py * p + ky)) * e.w + (px * p + kx));
        }
        v[j] = x;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
    }
    if (split3) {   // parity mode: [hi | lo | hi], 3 x Kp columns
      uint4 hi, lo;
      pack_split2(v[0], v[1], hi.x, lo.x);
      pack_split2(v[2], v[3], hi.y, lo.y);
      pack_split2(v[4], v[5], hi.z, lo.z);
      pack_split2(v[6], v[7], hi.w, lo.w);
      uint4* dst = reinterpret_cast<uint4*>(A + row * 3 * Kp) + kc;
      dst[0] = hi; dst[Kp / 8] = lo; dst[Kp / 4] = hi;
      continue;
    }
    uint4 o;
    o.x = pack_bf16(v[0], v[1]);
    o.y = pack_bf16(v[2], v[3]);
    o.z = pack_bf16(v[4], v[5]);
    o.w = pack_bf16(v[6], v[7]);
    reinterpret_cast<uint4*>(A + row * Kp)[kc] = o;
  }
}

// x[img, l] = ln_pre((l == 0 ? class_embedding : patch_out[img, l]) + positional_embedding[l])
// in place on the fp32 residual stream (reference layers/CLIP/model.py:254-257).
// L is the slot length L_max: image b takes its positional rows from pos + tab[b].pos_row and its rows past tab[b].L are
// set to zero (finite padding: no valid row ever reads them).
template <int D>
__global__ void __launch_bounds__(256)
cls_pos_lnpre_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos,
                     const float* __restrict__ gamma, const float* __restrict__ beta, int rows, int L,
                     const RaggedImg* __restrict__ tab) {
  constexpr int NV = D / 128;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int l = row % L;
  const RaggedImg& e = tab[row / L];
  if (l >= e.L) {
    float4* op = reinterpret_cast<float4*>(x + static_cast<long long>(row) * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) op[i * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  pos += static_cast<long long>(e.pos_row) * D;
  float4 v[NV];
  const float4* src = (l == 0) ? reinterpret_cast<const float4*>(cls)
                               : reinterpret_cast<const float4*>(x + static_cast<long long>(row) * D);
  const float4* pp = reinterpret_cast<const float4*>(pos + static_cast<long long>(l) * D);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 a = src[i * 32 + lane];
    const float4 b = __ldg(pp + i * 32 + lane);
    v[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
  float mean, rstd;
  ln_row_stats<D>(v, 1e-5f, mean, rstd);
  float4* op = reinterpret_cast<float4*>(x + static_cast<long long>(row) * D);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
    const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + i * 32 + lane);
    op[i * 32 + lane] = ln_norm(v[i], mean, rstd, g, b);
  }
}

// One embedded row: e = LN(words[tok] + positions[pos], eps 1e-8) (reference layers/decoder.py:65-78), the token clamped
// to the vocabulary, stored to output row `row` by ln_store.  One warp.
template <int D>
__device__ __forceinline__ void embed_ln_row(long long tok, int pos, const float* __restrict__ words,
                                             const float* __restrict__ positions, const float* __restrict__ gamma,
                                             const float* __restrict__ beta, int vocab, float* __restrict__ out_f32,
                                             __nv_bfloat16* __restrict__ out_bf16, int split3, long long row, int lane) {
  constexpr int NV = D / 128;
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
  const float4* wp = reinterpret_cast<const float4*>(words + tok * D);
  const float4* pp = reinterpret_cast<const float4*>(positions + static_cast<long long>(pos) * D);
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 a = __ldg(wp + i * 32 + lane);
    const float4 b = __ldg(pp + i * 32 + lane);
    v[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
  float mean, rstd;
  ln_row_stats<D>(v, 1e-8f, mean, rstd);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
    const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + i * 32 + lane);
    ln_store<D>(out_f32, out_bf16, split3, row, i * 32 + lane, ln_norm(v[i], mean, rstd, g, b));
  }
}

// The step's input embedding, one warp per row: tokens come from `tokens` (int64 [rows], stride tok_stride); position =
// pos_base + (state ? state->pos : 0).
template <int D>
__global__ void __launch_bounds__(256)
embed_ln_kernel(const long long* __restrict__ tokens, long long tok_stride, const float* __restrict__ words,
                const float* __restrict__ positions, const float* __restrict__ gamma, const float* __restrict__ beta,
                float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16, int rows, int pos_base,
                const StepState* __restrict__ state, int vocab, int split3, const ChainSync chain) {
  griddep_launch();
  griddep_wait();   // chain head: ordered after the previous step by a full dependency
  tl_mark(4);
  if (state != nullptr && state->finished) return;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) {
    chain_signal(chain);
    return;
  }
  const int pos = pos_base + (state != nullptr ? state->pos : 0);
  embed_ln_row<D>(tokens[row * tok_stride], pos, words, positions, gamma, beta, vocab, out_f32, out_bf16, split3, row,
                  threadIdx.x & 31);
  chain_signal(chain);
}

// ------------------------------------------------------------------------------------------------
// Caption scoring (teacher-forced pass over whole captions, reference layers/decoder.py:916-972)
// ------------------------------------------------------------------------------------------------
// embed_ln_kernel for rows * T positions at once: row r holds token tokens[r] at position r % T.  Also writes the LM-head
// target of each row, the next token of its caption (-1 for the last position).  Tokens are checked on the host.
template <int D>
__global__ void __launch_bounds__(256)
embed_ln_rows_kernel(const long long* __restrict__ tokens, int T, const float* __restrict__ words,
                     const float* __restrict__ positions, const float* __restrict__ gamma, const float* __restrict__ beta,
                     float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16, int rows, int vocab, int split3,
                     int* __restrict__ targets) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int pos = row % T;
  if (lane == 0) targets[row] = pos + 1 < T ? static_cast<int>(tokens[row + 1]) : -1;
  embed_ln_row<D>(tokens[row], pos, words, positions, gamma, beta, vocab, out_f32, out_bf16, split3, row, lane);
}

// One warp per text row: folds the row's n_parts LM-head partials (gemm.cuh EPI_LSE) into lse, the target's log-probability
// and the label-smoothed loss of SmoothLabelCrossEntropyLoss (reference layers/decoder.py:620-671, eps 0.1): with q the
// smoothed one-hot and lp = x - lse,
//   sum_c q_c (log q_c - lp_c) = sum q log q - (1 - eps) lp_t - eps / (V - 1) (sum_c lp_c - lp_t),  sum_c lp_c = sum x - V lse.
// Lane l folds parts l, l + 32, .. in order, then the lanes merge in a fixed tree: reproducible, no atomics.
// Row n * T + t scores token t + 1 of caption n (t < T - 1): logprob_out[n * (T - 1) + t]; it counts towards the loss when
// need_predict[n, t + 1] == 1 and the token is not the padding id 0 (:940-960, :640-643).
__global__ void __launch_bounds__(256)
lse_combine_kernel(const float4* __restrict__ parts, int n_parts, int rows, int T, int V, const int* __restrict__ targets,
                   const long long* __restrict__ need_predict, float eps, float* __restrict__ logprob_out,
                   float* __restrict__ row_loss, int* __restrict__ row_valid) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float m = -INFINITY, se = 0.f, xt = 0.f;
  double sx = 0.0;
  for (int k = lane; k < n_parts; k += 32) {
    const float4 q = __ldg(parts + static_cast<long long>(row) * n_parts + k);
    if (q.x != -INFINITY) {
      const float nm = fmaxf(m, q.x);
      se = ((m == -INFINITY) ? 0.f : se * expf(m - nm)) + q.y * expf(q.x - nm);
      m = nm;
    }
    sx += static_cast<double>(q.z);
    xt += q.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m_o = __shfl_xor_sync(0xffffffffu, m, o);
    const float s_o = __shfl_xor_sync(0xffffffffu, se, o);
    const float nm = fmaxf(m, m_o);
    se = ((m == -INFINITY) ? 0.f : se * expf(m - nm)) + ((m_o == -INFINITY) ? 0.f : s_o * expf(m_o - nm));
    m = nm;
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
    xt += __shfl_xor_sync(0xffffffffu, xt, o);
  }
  if (lane != 0) return;
  const int t = row % T;
  const int n = row / T;
  const int tgt = targets[row];
  float loss = 0.f;
  int valid = 0;
  if (t + 1 < T) {
    const double lse = static_cast<double>(m) + log(static_cast<double>(se));
    const double lp = static_cast<double>(xt) - lse;
    logprob_out[static_cast<long long>(n) * (T - 1) + t] = static_cast<float>(lp);
    valid = (need_predict[row + 1] == 1 && tgt != 0) ? 1 : 0;
    if (valid) {
      const double e = eps, off = e / (V - 1);
      const double qlogq = (1.0 - e) * log(1.0 - e) + e * log(off);
      const double sum_lp = sx - static_cast<double>(V) * lse;
      loss = static_cast<float>(qlogq - (1.0 - e) * lp - off * (sum_lp - lp));
    }
  }
  row_loss[row] = loss;
  row_valid[row] = valid;
}

// Mean of the valid rows' losses (NaN when there are none): one CTA, fixed-order tree over strided partial sums.
__global__ void __launch_bounds__(1024) loss_mean_kernel(const float* __restrict__ row_loss, const int* __restrict__ row_valid,
                                                         int rows, float* __restrict__ out) {
  __shared__ double s_sum[1024];
  __shared__ int s_cnt[1024];
  double a = 0.0;
  int c = 0;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    a += row_loss[r];
    c += row_valid[r];
  }
  s_sum[threadIdx.x] = a;
  s_cnt[threadIdx.x] = c;
  __syncthreads();
  for (int w = blockDim.x / 2; w > 0; w >>= 1) {
    if (static_cast<int>(threadIdx.x) < w) {
      s_sum[threadIdx.x] += s_sum[threadIdx.x + w];
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = s_cnt[0] > 0 ? static_cast<float>(s_sum[0] / s_cnt[0]) : __int_as_float(0x7fc00000);
}

// ------------------------------------------------------------------------------------------------
// CTA primitives of the row kernels that end a kernel-chain decode step (greedy_select_kernel below,
// constrained_select_kernel, beam_row_topk_kernel, beam_sample_kernel): kRowThreads threads per CTA.
// Every block reduction and scan combines the warps in warp order: bit-reproducible.
// ------------------------------------------------------------------------------------------------
constexpr int kRowThreads = 256;
constexpr int kRowWarps = kRowThreads / 32;

// Reduction over the CTA with `op` (every thread gets the result): a shuffle tree per warp, then the warp results folded
// in warp order.  sh holds kRowWarps entries.
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, T* sh, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T r = sh[0];
#pragma unroll
  for (int w = 1; w < kRowWarps; ++w) r = op(r, sh[w]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_reduce_max(float v, float* sh) {
  return block_reduce(v, sh, [](float a, float b) { return fmaxf(a, b); });
}
// fixed-order sum (warp tree, then the warps in order): bit-reproducible
__device__ __forceinline__ float block_reduce_sum(float v, float* sh) {
  return block_reduce(v, sh, [](float a, float b) { return a + b; });
}
__device__ __forceinline__ int block_reduce_max_int(int v, int* sh) {
  return block_reduce(v, sh, [](int a, int b) { return max(a, b); });
}
__device__ __forceinline__ int block_reduce_min_int(int v, int* sh) {
  return block_reduce(v, sh, [](int a, int b) { return min(a, b); });
}

// Inclusive scan over the lanes of a warp: lane l gets v_0 + ... + v_l, added in the shuffle tree's order.
template <class T>
__device__ __forceinline__ T warp_inclusive_scan(T v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T up = __shfl_up_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) >= o) v += up;
  }
  return v;
}

// Exclusive prefix sum of v over the CTA's threads in thread order (sh: kRowWarps ints).
__device__ __forceinline__ int block_exclusive_scan_int(int v, int* sh) {
  const int warp = threadIdx.x >> 5;
  const int inc = warp_inclusive_scan(v);
  if ((threadIdx.x & 31) == 31) sh[warp] = inc;
  __syncthreads();
  int before = 0;
#pragma unroll
  for (int w = 0; w < kRowWarps; ++w) if (w < warp) before += sh[w];
  __syncthreads();
  return before + inc - v;
}

// The index-order inverse-CDF lookup of the sampling kernels (a CTA per row): thread t owns the contiguous indices
// [i0, i1) and `mass_t` is the sum of mass(i) over them in index order.  The target is u * total, total = the thread
// masses summed in thread order (warp scans, then the warp totals in order).  The owner of the interval [lo, hi) that
// holds the target walks its indices to the first one whose running mass exceeds it; a target at or beyond the total
// (u -> 1 and rounding) falls to the last thread, whose walk ends at its last index.  Rounding can make two adjacent
// threads claim the target (lo is hi - mass_t, not the previous thread's hi): the higher index wins.  Returns the index
// (every thread), or -1 when no thread claims the target; *total_out = total.
template <class Mass>
__device__ __forceinline__ int inverse_cdf_index(float mass_t, float u, int i0, int i1, Mass mass, float* sh_scan, int* sh_pick,
                                                 float* total_out) {
  const int tid = threadIdx.x;
  const float inc = warp_inclusive_scan(mass_t);
  if ((tid & 31) == 31) sh_scan[tid >> 5] = inc;
  __syncthreads();
  // (sum of the earlier warps' totals) + inc: the order the draw's interval bounds are defined in
  float before = 0.f, total = 0.f;
#pragma unroll
  for (int w = 0; w < kRowWarps; ++w) {
    if (w < (tid >> 5)) before += sh_scan[w];
    total += sh_scan[w];
  }
  const float hi = before + inc, lo = hi - mass_t;
  const float target = u * total;
  int pick = -1;
  if ((target >= lo && target < hi && mass_t > 0.f) || (tid == kRowThreads - 1 && target >= hi)) {
    float acc = lo;
    pick = i1 - 1;
    for (int i = i0; i < i1; ++i) {
      acc += mass(i);
      if (target < acc) { pick = i; break; }
    }
  }
  *total_out = total;
  return block_reduce_max_int(pick, sh_pick);
}

// Row `row` of the step-logits dump [steps, rows_total, V] at step `step`, or null when there is no dump.
__device__ __forceinline__ float* step_logits_row(float* dump, int step, int rows_total, int row, int V) {
  return dump != nullptr ? dump + (static_cast<long long>(step) * rows_total + row) * V : nullptr;
}

// Pairwise merge of two online-softmax partials (max, sum exp(x - max), arg max); an empty partial has max -inf, and the
// lowest index wins exact ties of the maximum.
__device__ __forceinline__ void merge_stats(float& m, float& s, int& a, float m_o, float s_o, int a_o) {
  const float mn = fmaxf(m, m_o);
  const float sa = (m == -INFINITY) ? 0.f : __expf(m - mn);
  const float sb = (m_o == -INFINITY) ? 0.f : __expf(m_o - mn);
  s = s * sa + s_o * sb;
  if (m_o > m || (m_o == m && a_o < a)) a = a_o;
  m = mn;
}

// The close of decode step `step`, run by the one thread that commits a unit (a row in greedy, an image in beam search)
// after the unit's writes: the unit counts in StepState::live when it is still live, then draws one of the n_units
// tickets.  The last ticket resets the counters, advances the loop state, stops the search when no unit is live or
// max_steps is reached, and calls last(live count) before its closing fence.
template <class Last>
__device__ __forceinline__ void close_step(StepState* st, bool live, int n_units, int step, int cur_len, int max_steps,
                                           Last last) {
  // count this unit BEFORE drawing the ticket: the thread that draws the last ticket then sees every add
  if (live) atomicAdd(&st->live, 1);
  __threadfence();
  const unsigned int t = atomicAdd(&st->ticket, 1u);
  if (t == static_cast<unsigned int>(n_units) - 1) {
    __threadfence();
    const int n_live = atomicAdd(&st->live, 0);
    st->ticket = 0;
    st->live = 0;
    st->cur_len = cur_len + 1;
    st->final_len = cur_len + 1;
    st->pos = st->pos + 1;
    st->step = step + 1;
    if (n_live == 0) st->finished = 1;
    last(n_live);
    if (cur_len + 1 >= max_steps) st->finished = 1;
    __threadfence();
  }
}

// ------------------------------------------------------------------------------------------------
// Greedy selection = the body of AutoRegressiveBeamSearch.search for beam 1 / per-node 1
// (reference layers/decoder.py:258-273 first step, :313-417 loop): no-repeat scatter(-10000) on the
// input token (not on the first step), EOS forcing, log_softmax, argmax (lowest index on exact ties),
// logprob accumulation, all-EOS early exit.  One CTA per row.
// ------------------------------------------------------------------------------------------------
struct SelectParams {
  const float* logits;      // [rows, V]
  int V;
  int rows;
  int eos;
  int prefix_len;           // P
  int max_steps;
  long long* tokens_out;    // [rows, max_steps]
  float* logprob_sum;       // [rows]
  long long* next_token;    // [rows] input of the next step
  const long long* forced;  // [rows, max_steps] or null
  StepState* state;
  float* step_logits;       // optional dump [steps, rows_total, V]
  int rows_total, row0;     // this launch covers rows [row0, row0 + rows) of the batch
  // per-row prefixes (question batches, an extension of the reference's single-prefix path layers/decoder.py:985-1006):
  // row r starts from row_prefix[r * stride + 0 .. lens[r]); all rows advance in lockstep from text position 0, and while a
  // row is still inside its prefix its selection is overridden by the next prefix token (log-prob 0, no bookkeeping)
  const long long* row_prefix;
  int row_prefix_stride;
  const int* row_prefix_lens;
  // per-row partial results of the vocabulary slices (grid.x = n_split CTAs per row)
  int n_split;
  float* part_max;          // [rows, n_split]
  float* part_sum;          // [rows, n_split]  sum exp(v - part_max)
  int* part_arg;            // [rows, n_split]
  unsigned int* row_ticket; // [rows]
  ChainSync chain;          // last kernel of the chain: waits, then re-zeroes all counters when the step is over
};

// Where row `row` of the launch stands at this step.  in_prefix: it is still fed its prefix.  first: its first real
// decision (no no-repeat mask).  done: it ended, its input token is EOS (reference :347-351: one-hot EOS distribution).
struct RowStep {
  bool in_prefix, first, done;
};
__device__ __forceinline__ RowStep row_step(const SelectParams& p, int row, int step, int cur_len, long long last) {
  const int own_prefix = (p.row_prefix != nullptr) ? p.row_prefix_lens[p.row0 + row] : 0;
  RowStep r;
  r.in_prefix = (p.row_prefix != nullptr) && cur_len < own_prefix;
  r.first = (p.row_prefix != nullptr) ? (cur_len == own_prefix) : (step == 0);
  r.done = !r.first && !r.in_prefix && last == p.eos;
  return r;
}

// The row's token and log-prob at this step, and the token it feeds next (teacher forcing: forced[row, cur_len]).
struct RowChoice {
  long long tok, nxt;
  float lp;
};
// Inside the prefix: the next prefix token, nothing to score (log-prob 0).  Done: EOS, log_softmax of the one-hot EOS
// distribution is exactly 0.  Otherwise the model's choice.
__device__ __forceinline__ RowChoice resolve_row(const SelectParams& p, int row, int cur_len, const RowStep& rs,
                                                 long long choice, float choice_lp) {
  RowChoice c{choice, 0, choice_lp};
  if (rs.in_prefix) {
    c.tok = p.row_prefix[static_cast<long long>(p.row0 + row) * p.row_prefix_stride + cur_len];
    c.lp = 0.f;
  } else if (rs.done) {
    c.tok = p.eos;
    c.lp = 0.f;
  }
  c.nxt = (p.forced != nullptr) ? p.forced[static_cast<long long>(row) * p.max_steps + cur_len] : c.tok;
  return c;
}

// Commits one row's choice and closes the step with it: a row is live while the token it feeds next is not EOS (the
// reference stops once every one is).  The last ticket also marks an empty caption and re-zeroes the chain counters
// (null: none).
__device__ __forceinline__ void commit_row(const SelectParams& p, int row, int step, int cur_len, const RowChoice& c,
                                           unsigned int* chain_counters) {
  p.tokens_out[static_cast<long long>(row) * p.max_steps + cur_len] = c.tok;
  p.logprob_sum[row] += c.lp;
  p.next_token[row] = c.nxt;
  close_step(p.state, c.nxt != p.eos, p.rows, step, cur_len, p.max_steps, [&](int n_live) {
    if (n_live == 0 && step == 0 && p.row_prefix == nullptr) p.state->empty_caption = 1;
    // every CTA of every kernel of this step has passed its wait: recycle the chain counters
    if (chain_counters != nullptr)
      for (int k = 0; k < 64; ++k) chain_counters[k] = 0;
  });
}

// grid (n_split, rows): each CTA folds one vocabulary slice of one row into (max, argmax, sum exp) with a
// single online pass; the last CTA of a row combines the slices and does the reference's bookkeeping.
__global__ void __launch_bounds__(kRowThreads) greedy_select_kernel(const SelectParams p) {
  griddep_launch_early();
  tl_mark(100005);
  StepState* st = p.state;
  if (step_wait(&st->finished, p.chain)) return;
  tl_mark(5);
  const int row = blockIdx.y;
  const int split = blockIdx.x;
  const int tid = threadIdx.x;
  const int step = st->step;
  const int cur_len = st->cur_len;
  const float* z = p.logits + static_cast<long long>(row) * p.V;
  // The input token of this step (== our previous choice unless teacher forcing is on): the reference's
  // masks are functions of the *input* sequence (predictions_so_far[:, -1]).
  const long long last = p.next_token[row];
  const RowStep rs = row_step(p, row, step, cur_len, last);
  const int chunk = (p.V + p.n_split - 1) / p.n_split;
  const int lo = split * chunk;
  const int hi = min(p.V, lo + chunk);
  if (float* dst = step_logits_row(p.step_logits, step, p.rows_total, p.row0 + row, p.V))
    for (int i = lo + tid; i < hi; i += kRowThreads) dst[i] = z[i];
  float m = -INFINITY, ssum = 0.f;
  int arg = 0x7fffffff;
  for (int i0 = lo + tid; i0 < hi; i0 += 16 * kRowThreads) {   // one round for the usual 8-way split of 30522
    float v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int i = i0 + u * kRowThreads;
      v[u] = (i < hi) ? __ldcg(z + i) : -INFINITY;
      if (!rs.first && i == static_cast<int>(last)) v[u] = -10000.0f;   // no-repeat (reference :330)
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int i = i0 + u * kRowThreads;
      if (v[u] > m) {   // increasing i per thread: keeps the lowest index on exact ties
        ssum = ssum * __expf(m - v[u]) + 1.0f;
        m = v[u];
        arg = i;
      } else if (v[u] != -INFINITY) {
        ssum += __expf(v[u] - m);
      }
    }
  }
  // block reduce of (m, arg, ssum)
  __shared__ float s_m[kRowWarps], s_s[kRowWarps];
  __shared__ int s_a[kRowWarps];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    merge_stats(m, ssum, arg, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, ssum, o),
                __shfl_xor_sync(0xffffffffu, arg, o));
  if ((tid & 31) == 0) { s_m[tid >> 5] = m; s_s[tid >> 5] = ssum; s_a[tid >> 5] = arg; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kRowWarps; ++w) merge_stats(m, ssum, arg, s_m[w], s_s[w], s_a[w]);
    p.part_max[row * p.n_split + split] = m;
    p.part_sum[row * p.n_split + split] = ssum;
    p.part_arg[row * p.n_split + split] = arg;
    __threadfence();
    const unsigned int t = atomicAdd(&p.row_ticket[row], 1u);
    if (t == static_cast<unsigned int>(p.n_split) - 1) {
      __threadfence();
      p.row_ticket[row] = 0;
      // combine the slices in slice order (= index order); a row without a finite logit keeps arg 0
      float gm = -INFINITY, gs = 0.f;
      int ga = 0;
      for (int k = 0; k < p.n_split; ++k)
        merge_stats(gm, gs, ga, __ldcg(&p.part_max[row * p.n_split + k]), __ldcg(&p.part_sum[row * p.n_split + k]),
                    __ldcg(&p.part_arg[row * p.n_split + k]));
      // z[arg] - max - log(sum exp(z - max)) with z[arg] == max
      commit_row(p, row, step, cur_len, resolve_row(p, row, cur_len, rs, ga, -logf(gs)), p.chain.counters);
    }
  }
}

// logprobs / num_valid (reference layers/decoder.py:433-438) and EOS padding of the unused tail.
__global__ void greedy_finalize_kernel(long long* tokens_out, const float* logprob_sum, float* logprobs_out, int rows,
                                       int max_steps, int prefix_len, int eos, const StepState* state, const int* row_prefix_lens) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= rows) return;
  if (row_prefix_lens != nullptr) prefix_len = row_prefix_lens[row];
  const int n = state->final_len;
  for (int i = n; i < max_steps; ++i) tokens_out[static_cast<long long>(row) * max_steps + i] = eos;
  int not_eos = 0, has_eos = 0;
  for (int i = 0; i < n; ++i) {
    const long long t = tokens_out[static_cast<long long>(row) * max_steps + i];
    if (t == eos) has_eos = 1; else ++not_eos;
  }
  int num_valid = not_eos + has_eos - prefix_len;
  if (num_valid < 1) num_valid = 1;
  logprobs_out[row] = state->empty_caption ? logprob_sum[row] : logprob_sum[row] / static_cast<float>(num_valid);
}

}  // namespace gitb200
