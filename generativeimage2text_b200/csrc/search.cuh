// Device-side beam search = GeneratorWithBeamSearch.search + BeamHypotheses with num_keep_best = 1
// (reference layers/decoder.py:1083-1290, 1292-1341), without the reference's per-candidate host syncs.
//
// Per step, for `rows = B * beam` sequences:
//   beam_row_topk_kernel : per row, log-softmax statistics of the step logits and the row's own top
//                          `2*beam` candidates (the image-level top-2*beam over beam*V is a subset of the
//                          union of the per-row top-2*beam lists).
//   beam_update_kernel   : per image, merge the candidate lists (sorted, ties -> lower flat index), then
//                          replay the reference's bookkeeping loop: finished-check, hypothesis insertion on
//                          EOS / last step, next-beam selection, and re-ordering of the token history and of
//                          the text-KV indirection table by beam_idx (reference :1231; image K/V are shared).
//   beam_finalize_kernel : decoded[B, max_steps] (EOS padded) and the length-normalised score.
// The text KV cache is never copied: src_row[r][j] names the physical row that holds position j of
// logical row r's history.
//
// Candidate order: (score desc, beam asc, logit desc, token asc).  A row's list is ranked on the raw logit (lower token on
// exact ties); the score ((z - max) - log_sum) + beam_score is increasing in z in exact arithmetic, but fp32 can round two
// different logits of one row to the same score (e.g. z - max = -100 for a logit one ulp apart), and those keep the logit
// order -- the order of their exact scores.  The merge breaks equal scores of different beams by the lower flat index.
#pragma once
#include "ptx.cuh"
#include "rowops.cuh"

namespace gitb200 {

constexpr int kMaxBeam = 4;
constexpr int kMaxCand = 2 * kMaxBeam;  // per_node_beam_size * beam

__global__ void init_src_row_kernel(int* src, int rows, int T_alloc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows * T_alloc) src[i] = i / T_alloc;
}

// new[r][j < pos] = old[beam_idx[r]][j]; new[r][pos] = r  (raw decode_step API)
__global__ void reorder_src_row_kernel(const int* old_src, int* new_src, const int* beam_idx, int rows, int T_alloc, int pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * T_alloc) return;
  const int r = i / T_alloc, j = i - r * T_alloc;
  new_src[i] = (j < pos) ? old_src[beam_idx[r] * T_alloc + j] : r;
}

struct BeamState {
  // all arrays live in one engine-owned buffer; see beam_state_bytes()
  float* beam_scores;     // [rows]
  float* cand_val;        // [rows, kMaxCand]  row-local top candidates: logit - lse + beam_score
  int* cand_idx;          // [rows, kMaxCand]  vocabulary index
  long long* ids[2];      // [rows, max_steps] token history ping-pong (input_ids)
  int* src[2];            // [rows, T_alloc] text-KV indirection ping-pong
  int* cur;               // [1] which of ids/src is current
  int* done;              // [B]
  float* hyp_score;       // [B]   best finished hypothesis (n_hyp = 1)
  float* worst_score;     // [B]   BeamHypotheses.worst_score (1e9 when empty)
  int* hyp_len;           // [B]   0 = none
  long long* hyp_tok;     // [B, max_steps]
};

struct BeamParams {
  BeamState s;
  const float* logits;    // [rows, V]
  int V, B, beam, per_node, max_steps, T_alloc, eos;
  float length_penalty;
  long long* next_token;  // [rows]
  StepState* state;
  float* step_logits;     // optional dump [steps, rows, V]
  // per-image prefixes (see SelectParams): image b starts from row_prefix[b * stride + 0 .. lens[b])
  const long long* row_prefix;
  int row_prefix_stride;
  const int* row_prefix_lens;
};

__device__ __forceinline__ float beam_length_norm(int length, float lp) {
  // BeamHypotheses._length_norm, reference layers/decoder.py:1310-1313
  return powf(5.0f + static_cast<float>(length), lp) / powf(6.0f, lp);
}

// Sorted candidate list of kMaxCand entries in registers (descending value, ascending index on exact ties).  Every access is
// statically indexed: indexing the arrays with a runtime position puts them in local memory, which made this kernel
// several times slower.
struct TopList {
  float v[kMaxCand];
  int i[kMaxCand];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < kMaxCand; ++k) { v[k] = -INFINITY; i[k] = 0x7fffffff; }
  }
  static __device__ __forceinline__ bool before(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }
  __device__ __forceinline__ void push(float val, int idx) {          // insert if it beats the last entry, keep sorted
    if (!before(val, idx, v[kMaxCand - 1], i[kMaxCand - 1])) return;
    v[kMaxCand - 1] = val; i[kMaxCand - 1] = idx;
#pragma unroll
    for (int k = kMaxCand - 1; k > 0; --k) {
      if (before(v[k], i[k], v[k - 1], i[k - 1])) {
        const float tv = v[k]; v[k] = v[k - 1]; v[k - 1] = tv;
        const int ti = i[k]; i[k] = i[k - 1]; i[k - 1] = ti;
      }
    }
  }
};

// One CTA per row: lse = logsumexp(z), then the row's top-NC values of (z - lse + beam_score[row]).  One pass over the
// logits (online max / sum-exp and a sorted top-8 list per thread), then lists merged by shuffles and through shared memory.
__global__ void __launch_bounds__(256) beam_row_topk_kernel(const BeamParams p) {
  griddep_launch();
  griddep_wait();
  StepState* st = p.state;
  if (st->finished) return;
  const int row = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NC = p.per_node * p.beam;
  const float* z = p.logits + static_cast<long long>(row) * p.V;
  if (p.step_logits != nullptr) {
    float* dst = p.step_logits + (static_cast<long long>(st->step) * gridDim.x + row) * p.V;
    for (int i = tid; i < p.V; i += blockDim.x) dst[i] = z[i];
  }
  TopList top;
  top.init();
  float mx = -INFINITY, sum = 0.f;
  for (int i0 = tid; i0 < p.V; i0 += 8 * 256) {       // 8 independent loads in flight per thread
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = (i0 + u * 256 < p.V) ? __ldcg(z + i0 + u * 256) : -INFINITY;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (v[u] == -INFINITY) continue;
      if (v[u] > mx) { sum = sum * __expf(mx - v[u]) + 1.0f; mx = v[u]; } else { sum += __expf(v[u] - mx); }
      top.push(v[u], i0 + u * 256);
    }
  }
  // warp-level merge: each round a lane absorbs its partner's list (entries arrive in sorted order: push keeps ours sorted)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float m_o = __shfl_xor_sync(0xffffffffu, mx, o);
    const float s_o = __shfl_xor_sync(0xffffffffu, sum, o);
    const float mn = fmaxf(mx, m_o);
    sum = sum * ((mx == -INFINITY) ? 0.f : __expf(mx - mn)) + s_o * ((m_o == -INFINITY) ? 0.f : __expf(m_o - mn));
    mx = mn;
    float pv[kMaxCand];
    int pi[kMaxCand];
#pragma unroll
    for (int k = 0; k < kMaxCand; ++k) { pv[k] = __shfl_xor_sync(0xffffffffu, top.v[k], o); pi[k] = __shfl_xor_sync(0xffffffffu, top.i[k], o); }
#pragma unroll
    for (int k = 0; k < kMaxCand; ++k) top.push(pv[k], pi[k]);
  }
  __shared__ float s_m[8], s_s[8];
  __shared__ float s_cv[8][kMaxCand];
  __shared__ int s_ci[8][kMaxCand];
  if (lane == 0) {
    s_m[warp] = mx; s_s[warp] = sum;
#pragma unroll
    for (int k = 0; k < kMaxCand; ++k) { s_cv[warp][k] = top.v[k]; s_ci[warp][k] = top.i[k]; }
  }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) {
      const float mn = fmaxf(mx, s_m[w]);
      sum = sum * ((mx == -INFINITY) ? 0.f : __expf(mx - mn)) + s_s[w] * ((s_m[w] == -INFINITY) ? 0.f : __expf(s_m[w] - mn));
      mx = mn;
#pragma unroll
      for (int k = 0; k < kMaxCand; ++k) top.push(s_cv[w][k], s_ci[w][k]);
    }
    const float log_sum = logf(sum);
    const float bs = p.s.beam_scores[row];
#pragma unroll
    for (int k = 0; k < kMaxCand; ++k) {
      if (k < NC) {
        // log_softmax (x - max - log(sum exp(x - max))) + beam score (reference :1169-1172)
        p.s.cand_val[row * kMaxCand + k] = ((top.v[k] - mx) - log_sum) + bs;
        p.s.cand_idx[row * kMaxCand + k] = top.i[k];
      }
    }
  }
}

// One thread block per image (32 threads; the bookkeeping itself is sequential like the reference's loop).
__global__ void __launch_bounds__(32) beam_update_kernel(const BeamParams p) {
  griddep_launch();
  griddep_wait();
  StepState* st = p.state;
  if (st->finished) return;
  const int b = blockIdx.x;
  const int lane = threadIdx.x;
  const int beam = p.beam, NC = p.per_node * p.beam, V = p.V;
  const int cur = *p.s.cur;
  const int cur_len = st->cur_len;
  const long long* ids_old = p.s.ids[cur];
  long long* ids_new = p.s.ids[cur ^ 1];
  const int* src_old = p.s.src[cur];
  int* src_new = p.s.src[cur ^ 1];
  __shared__ float m_val[kMaxCand];
  __shared__ int m_word[kMaxCand];
  __shared__ int m_beam[kMaxCand];
  __shared__ int n_row[kMaxBeam];   // next beams: source row (global)
  __shared__ int n_word[kMaxBeam];
  __shared__ float n_score[kMaxBeam];
  const bool in_prefix = (p.row_prefix != nullptr) && cur_len < p.row_prefix_lens[b];
  if (lane == 0 && in_prefix) {
    // the image is still inside its prefix: every beam takes the next prefix token, scores and histories stay as they are
    for (int k = 0; k < beam; ++k) {
      n_row[k] = b * beam + k;
      n_word[k] = static_cast<int>(p.row_prefix[static_cast<long long>(b) * p.row_prefix_stride + cur_len]);
      n_score[k] = p.s.beam_scores[b * beam + k];
    }
  }
  if (lane == 0 && !in_prefix) {
    // merge the `beam` row lists into the image's top-NC, ordered by (value desc, flat index asc)
    int ptr[kMaxBeam];
    for (int k = 0; k < beam; ++k) ptr[k] = 0;
    for (int c = 0; c < NC; ++c) {
      int best = -1;
      float bv = 0.f;
      long long bflat = 0;
      for (int k = 0; k < beam; ++k) {
        if (ptr[k] >= NC) continue;
        const int r = b * beam + k;
        const float v = p.s.cand_val[r * kMaxCand + ptr[k]];
        const long long flat = static_cast<long long>(k) * V + p.s.cand_idx[r * kMaxCand + ptr[k]];
        if (best < 0 || v > bv || (v == bv && flat < bflat)) { best = k; bv = v; bflat = flat; }
      }
      m_val[c] = bv;
      m_word[c] = p.s.cand_idx[(b * beam + best) * kMaxCand + ptr[best]];
      m_beam[c] = best;
      ++ptr[best];
    }
    // ---- reference bookkeeping (layers/decoder.py:1184-1228) ----
    bool done = p.s.done[b] != 0;
    if (!done && p.s.hyp_len[b] > 0) {  // BeamHypotheses.is_done with early_stopping=False (:1330-1341)
      done = p.s.worst_score[b] >= m_val[0] / beam_length_norm(p.max_steps - 1, p.length_penalty);
    }
    p.s.done[b] = done ? 1 : 0;
    int n_next = 0;
    if (!done) {
      const bool last_step = (cur_len + 1 == p.max_steps);
      for (int c = 0; c < NC; ++c) {
        if (m_word[c] == p.eos || last_step) {
          // BeamHypotheses.add(input_ids[row, :cur_len], score)  (:1315-1328) with n_hyp = 1
          const float score = m_val[c] / beam_length_norm(cur_len, p.length_penalty);
          if (p.s.hyp_len[b] == 0 || score > p.s.worst_score[b]) {
            // with one kept hypothesis: a better one replaces the old and becomes the new worst_score
            const bool first = p.s.hyp_len[b] == 0;
            const float old = p.s.hyp_score[b];
            if (first || score > old) {
              p.s.hyp_score[b] = score;
              p.s.hyp_len[b] = cur_len;
              const long long* srcp = ids_old + static_cast<long long>(b * beam + m_beam[c]) * p.max_steps;
              for (int i = 0; i < cur_len; ++i) p.s.hyp_tok[static_cast<long long>(b) * p.max_steps + i] = srcp[i];
              p.s.worst_score[b] = first ? fminf(score, p.s.worst_score[b]) : score;
            } else {
              // score > worst but not better than the kept one cannot happen with n_hyp = 1 (worst == kept)
              p.s.worst_score[b] = old;
            }
          }
        } else {
          n_row[n_next] = b * beam + m_beam[c];
          n_word[n_next] = m_word[c];
          n_score[n_next] = m_val[c];
          ++n_next;
        }
        if (n_next == beam) break;
      }
    }
    if (n_next < beam) {  // finished image or last step: pad with (0, EOS, row 0) (:1189, :1220-1221)
      for (int k = 0; k < beam; ++k) { n_row[k] = 0; n_word[k] = p.eos; n_score[k] = 0.f; }
    }
  }
  __syncwarp();
  // re-order histories: input_ids = cat(input_ids[beam_idx], beam_words) (:1231-1232); KV indirection follows
  for (int k = 0; k < beam; ++k) {
    const int r = b * beam + k;
    const int srow = n_row[k];
    for (int i = lane; i < cur_len; i += 32)
      ids_new[static_cast<long long>(r) * p.max_steps + i] = ids_old[static_cast<long long>(srow) * p.max_steps + i];
    const int n_pos = st->pos + 1;  // text positions filled so far (this step wrote position st->pos)
    for (int j = lane; j < p.T_alloc; j += 32)
      src_new[r * p.T_alloc + j] = (j < n_pos) ? src_old[srow * p.T_alloc + j] : r;
    if (lane == 0) {
      ids_new[static_cast<long long>(r) * p.max_steps + cur_len] = n_word[k];
      p.next_token[r] = n_word[k];
      p.s.beam_scores[r] = n_score[k];
    }
  }
  // loop-state advance by the last image
  __threadfence();
  if (lane == 0) {
    // count this image as running BEFORE drawing the ticket: the block that draws the last ticket then sees every add
    if (p.s.done[b] == 0) atomicAdd(&st->not_eos, 1);  // re-used as "images still running"
    __threadfence();
    const unsigned int t = atomicAdd(&st->ticket, 1u);
    if (t == static_cast<unsigned int>(p.B) - 1) {
      __threadfence();
      const int running = atomicAdd(&st->not_eos, 0);
      st->ticket = 0;
      st->not_eos = 0;
      *p.s.cur = cur ^ 1;
      st->cur_len = cur_len + 1;
      st->final_len = cur_len + 1;
      st->pos = st->pos + 1;
      st->step = st->step + 1;
      if (running == 0 || cur_len + 1 >= p.max_steps) st->finished = 1;  // `if all(done): break` (:1253)
      __threadfence();
    }
  }
}

__global__ void beam_init_kernel(BeamState s, long long* next_token, const long long* prefix, int P, int sos, int B,
                                 int beam, int max_steps, int T_alloc, long long prefix_row_stride) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int rows = B * beam;
  if (r == 0) *s.cur = 0;
  if (r < rows) {
    s.beam_scores[r] = (r % beam == 0) ? 0.f : -1e9f;  // reference :1118-1120
    const long long* pr = prefix ? prefix + (r / beam) * prefix_row_stride : nullptr;   // stride 0: one prefix for all rows
    for (int i = 0; i < P; ++i) s.ids[0][static_cast<long long>(r) * max_steps + i] = pr ? pr[i] : sos;
    next_token[r] = pr ? pr[0] : sos;
    for (int j = 0; j < T_alloc; ++j) { s.src[0][r * T_alloc + j] = r; s.src[1][r * T_alloc + j] = r; }
  }
  if (r < B) { s.done[r] = 0; s.hyp_score[r] = -1e30f; s.worst_score[r] = 1e9f; s.hyp_len[r] = 0; }
}

// decoded row = best hypothesis, then EOS, EOS-padded to max_steps; logprobs = its score (reference :1264-1290)
__global__ void beam_finalize_kernel(BeamState s, long long* tokens_out, float* logprobs_out, int B, int max_steps, int eos) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int n = s.hyp_len[b];
  for (int i = 0; i < max_steps; ++i)
    tokens_out[static_cast<long long>(b) * max_steps + i] = (i < n) ? s.hyp_tok[static_cast<long long>(b) * max_steps + i] : eos;
  logprobs_out[b] = (n > 0) ? s.hyp_score[b] : -1e5f;
}

}  // namespace gitb200
