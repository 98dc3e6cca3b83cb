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
// The per-row kernels (and beam_sample_kernel below) use the CTA reductions, the inverse-CDF lookup and the step-logits
// row of rowops.cuh; beam_update_kernel closes each step with close_step there, as the greedy kernels do.
//
// Candidate order: (score desc, beam asc, logit desc, token asc).  A row's list is ranked on the raw logit (lower token on
// exact ties); the score ((z - max) - log_sum) + beam_score is increasing in z in exact arithmetic, but fp32 can round two
// different logits of one row to the same score (e.g. z - max = -100 for a logit one ulp apart), and those keep the logit
// order -- the order of their exact scores.  The merge breaks equal scores of different beams by the lower flat index.
#pragma once
#include "ptx.cuh"
#include "rowops.cuh"

namespace gitb200 {

// Candidate capacity (per_node_beam_size * beam, per_node 2): the per-row lists, the row stride of BeamState's candidate
// arrays and the merge width are compile-time.  Two instantiations: 8 for beams 2 .. 4, 16 for beams 5 .. 8.  The 16-entry
// beam_row_topk_kernel takes several times as long per launch (DESIGN.md §6), so beams 2 .. 4 keep the 8-entry one.
constexpr int kMaxBeam = 8;
__host__ __device__ constexpr int beam_cand_capacity(int beam) { return beam <= 4 ? 8 : 16; }

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
  float* cand_val;        // [rows, kCand]  row-local top candidates: logit - lse + beam_score (kCand: beam_cand_capacity)
  int* cand_idx;          // [rows, kCand]  vocabulary index
  long long* ids[2];      // [rows, max_steps] token history ping-pong (input_ids)
  int* src[2];            // [rows, T_alloc] text-KV indirection ping-pong
  int* cur;               // [1] which of ids/src is current
  int* done;              // [B]
  float* hyp_score;       // [B]   best finished hypothesis (n_hyp = 1)
  float* worst_score;     // [B]   BeamHypotheses.worst_score (1e9 when empty)
  int* hyp_len;           // [B]   0 = none
  long long* hyp_tok;     // [B, max_steps]
};

// The do_sample branch of GeneratorWithBeamSearch.search (reference layers/decoder.py:1138-1166): uniforms == null is the
// deterministic search.
struct BeamSample {
  const float* uniforms;  // [max_steps, rows, 2]: row r at caption length t draws with uniforms[(t * rows + r) * 2 + d]
  float temperature;
  int top_k;              // <= 0: no top-k filter
  float top_p;            // 0 or >= 1: no nucleus filter
  int* kept;              // optional [rows]: size of each row's kept set (test hook)
};

struct BeamParams {
  BeamState s;
  BeamSample smp;
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

// Sorted candidate list of kCand entries in registers (descending value, ascending index on exact ties).  Every access is
// statically indexed: indexing the arrays with a runtime position puts them in local memory, which made this kernel
// several times slower.
template <int kCand>
struct TopList {
  float v[kCand];
  int i[kCand];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < kCand; ++k) { v[k] = -INFINITY; i[k] = 0x7fffffff; }
  }
  static __device__ __forceinline__ bool before(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }
  __device__ __forceinline__ void push(float val, int idx) {          // insert if it beats the last entry, keep sorted
    if (!before(val, idx, v[kCand - 1], i[kCand - 1])) return;
    v[kCand - 1] = val; i[kCand - 1] = idx;
#pragma unroll
    for (int k = kCand - 1; k > 0; --k) {
      if (before(v[k], i[k], v[k - 1], i[k - 1])) {
        const float tv = v[k]; v[k] = v[k - 1]; v[k - 1] = tv;
        const int ti = i[k]; i[k] = i[k - 1]; i[k - 1] = ti;
      }
    }
  }
};

// One CTA per row: lse = logsumexp(z), then the row's top-NC values of (z - lse + beam_score[row]).  One pass over the
// logits (online max / sum-exp and a sorted top-kCand list per thread), then lists merged by shuffles and through shared memory.
template <int kCand>
__global__ void __launch_bounds__(kRowThreads) beam_row_topk_kernel(const BeamParams p) {
  griddep_launch();
  StepState* st = p.state;
  if (step_wait(&st->finished, ChainSync{})) return;
  const int row = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NC = p.per_node * p.beam;
  const float* z = p.logits + static_cast<long long>(row) * p.V;
  if (float* dst = step_logits_row(p.step_logits, st->step, gridDim.x, row, p.V))
    for (int i = tid; i < p.V; i += blockDim.x) dst[i] = z[i];   // a kRowThreads stride changes the kernel's code
  TopList<kCand> top;
  top.init();
  float mx = -INFINITY, sum = 0.f;
  for (int i0 = tid; i0 < p.V; i0 += 8 * kRowThreads) {       // 8 independent loads in flight per thread
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = (i0 + u * kRowThreads < p.V) ? __ldcg(z + i0 + u * kRowThreads) : -INFINITY;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (v[u] == -INFINITY) continue;
      if (v[u] > mx) { sum = sum * __expf(mx - v[u]) + 1.0f; mx = v[u]; } else { sum += __expf(v[u] - mx); }
      top.push(v[u], i0 + u * kRowThreads);
    }
  }
  // warp-level merge: each round a lane absorbs its partner's list (entries arrive in sorted order: push keeps ours sorted).
  // The (max, sum exp) merges here are merge_stats without the arg max, written out: a shared helper for them changed the
  // kernel's register allocation (62 -> 48 or 64 registers) and left the deterministic beam step slower.
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float m_o = __shfl_xor_sync(0xffffffffu, mx, o);
    const float s_o = __shfl_xor_sync(0xffffffffu, sum, o);
    const float mn = fmaxf(mx, m_o);
    sum = sum * ((mx == -INFINITY) ? 0.f : __expf(mx - mn)) + s_o * ((m_o == -INFINITY) ? 0.f : __expf(m_o - mn));
    mx = mn;
    float pv[kCand];
    int pi[kCand];
#pragma unroll
    for (int k = 0; k < kCand; ++k) { pv[k] = __shfl_xor_sync(0xffffffffu, top.v[k], o); pi[k] = __shfl_xor_sync(0xffffffffu, top.i[k], o); }
#pragma unroll
    for (int k = 0; k < kCand; ++k) top.push(pv[k], pi[k]);
  }
  __shared__ float s_m[kRowWarps], s_s[kRowWarps];
  __shared__ float s_cv[kRowWarps][kCand];
  __shared__ int s_ci[kRowWarps][kCand];
  if (lane == 0) {
    s_m[warp] = mx; s_s[warp] = sum;
#pragma unroll
    for (int k = 0; k < kCand; ++k) { s_cv[warp][k] = top.v[k]; s_ci[warp][k] = top.i[k]; }
  }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kRowWarps; ++w) {
      const float mn = fmaxf(mx, s_m[w]);
      sum = sum * ((mx == -INFINITY) ? 0.f : __expf(mx - mn)) + s_s[w] * ((s_m[w] == -INFINITY) ? 0.f : __expf(s_m[w] - mn));
      mx = mn;
#pragma unroll
      for (int k = 0; k < kCand; ++k) top.push(s_cv[w][k], s_ci[w][k]);
    }
    const float log_sum = logf(sum);
    const float bs = p.s.beam_scores[row];
#pragma unroll
    for (int k = 0; k < kCand; ++k) {
      if (k < NC) {
        // log_softmax (x - max - log(sum exp(x - max))) + beam score (reference :1169-1172)
        p.s.cand_val[row * kCand + k] = ((top.v[k] - mx) - log_sum) + bs;
        p.s.cand_idx[row * kCand + k] = top.i[k];
      }
    }
  }
}

// ---- sampled beam search ---------------------------------------------------------------------------------------------
// beam_sample_kernel replaces beam_row_topk_kernel when BeamParams::smp.uniforms is set.  Per row (reference
// layers/decoder.py:1140-1161, top_k_top_p_filtering :1343-1375): scores = logits / T; top-k keeps the values >= the k-th
// largest (k = min(max(top_k, 2), V); ties at it all kept); top-p sorts by (value desc, index asc -- torch.sort leaves ties
// unordered, this is the engine's order), finds the first position J whose cumulative softmax exceeds p and keeps the
// positions 0 .. max(J, 2) (the first two are forced, then the mask shifts right by one); two draws without replacement
// from softmax(kept), each an index-order inverse-CDF lookup with its own uniform; candidate d of the row =
// log_softmax(kept)[token_d] + beam_score[row].  No sort: the k-th value and the top-p boundary come from radix descents
// over the order-preserving keys of the scores.  Every sum runs in a fixed order, so results are bit-reproducible.
constexpr int kSampleMaxVocab = 48 * 1024;   // the row's scores are kept in shared memory

__device__ __forceinline__ unsigned int order_key(float v) {   // uint32 order == fp32 order
  const unsigned int b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct SampleSmem {
  int cnt[kRowWarps][256];      // per-warp digit histograms: counts ...
  float mass[kRowWarps][256];   // ... and masses
  float stage[kRowWarps][32];
  int scan_c[256];              // inclusive scans over the buckets, in descending key order
  float scan_m[256];
  float red[kRowWarps];
  int ired[kRowWarps];
};

// Where a descending walk over the keys stops: the key, how many keys lie strictly above it (and their mass), how many
// equal it.  found = false: the mass never exceeds the target.
struct RadixStop {
  unsigned int key;
  int above, equal;
  float mass_above;
  bool found;
};

// MSB-first radix descent over the keys of s[0 .. V), 8 bits per pass, buckets visited in descending key order.
//   kMass = false: stops at the key of the `want`-th largest value (1-based, duplicates counted).
//   kMass = true : stops at the key where the running mass first exceeds `want`; the mass of s_i is exp(s_i - m), over
//                  the keys >= live only (`above` / `equal` count those).
// The histograms are per warp and need no atomics: the lanes of a warp that share a digit add their count (and their
// masses, lane by lane) through the lowest of them.  Bucket totals add the warps in order and the bucket scan is a fixed
// shuffle tree, so the masses are summed in one fixed order.  When rounding leaves a later pass without a crossing (its
// buckets need not add up to the total the pass before saw), the descent takes the lowest non-empty bucket.
template <bool kMass>
__device__ RadixStop radix_descend(const float* s, int V, float want, unsigned int live, float m, SampleSmem& sm) {
  static_assert(kRowThreads == 256, "one thread per 8-bit digit bucket");
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  RadixStop r{0u, 0, 0, 0.f, true};
  unsigned int mask = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int d = lane; d < 256; d += 32) {
      sm.cnt[warp][d] = 0;
      if (kMass) sm.mass[warp][d] = 0.f;
    }
    __syncwarp();
    for (int base = 0; base < V; base += kRowThreads) {
      const int i = base + tid;
      unsigned int key = 0u;
      bool in = false;
      if (i < V) {
        key = order_key(s[i]);
        in = (key & mask) == r.key && (!kMass || key >= live);   // mass: only the top-k survivors can hold the crossing
      }
      if (!__any_sync(0xffffffffu, in)) continue;
      const unsigned int digit = (key >> shift) & 255u;
      const unsigned int grp = __match_any_sync(0xffffffffu, in ? digit : 0x100u);
      if (kMass) {
        sm.stage[warp][lane] = in ? expf(s[i] - m) : 0.f;
        __syncwarp();
      }
      if (in && lane == __ffs(grp) - 1) {
        sm.cnt[warp][digit] += __popc(grp);
        if (kMass) {
          float acc = 0.f;
          for (unsigned int g = grp; g != 0u; g &= g - 1u) acc += sm.stage[warp][__ffs(g) - 1];
          sm.mass[warp][digit] += acc;
        }
      }
      __syncwarp();
    }
    __syncthreads();
    const int d = 255 - tid;   // thread t: bucket 255 - t
    int c = 0;
    float ms = 0.f;
#pragma unroll
    for (int w = 0; w < kRowWarps; ++w) {
      c += sm.cnt[w][d];
      if (kMass) ms += sm.mass[w][d];
    }
    int ci = warp_inclusive_scan(c);
    float mi = kMass ? warp_inclusive_scan(ms) : 0.f;
    if (lane == 31) { sm.ired[warp] = ci; sm.red[warp] = mi; }
    __syncthreads();
    // ((inc + t_0) + t_1) + ...: the order the masses above a bucket are defined in
#pragma unroll
    for (int w = 0; w < kRowWarps; ++w) {
      if (w < warp) { ci += sm.ired[w]; if (kMass) mi += sm.red[w]; }
    }
    __syncthreads();
    sm.scan_c[tid] = ci;
    if (kMass) sm.scan_m[tid] = mi;
    const bool stop = kMass ? (c > 0 && r.mass_above + mi > want) : (static_cast<float>(r.above + ci) >= want);
    // the first bucket that stops (256: none); as a max of 255 - t: block_reduce_min_int here made ptxas give the kernel
    // 46 registers instead of 39
    int t = 255 - block_reduce_max_int(stop ? 255 - tid : -1, sm.ired);
    if (t > 255) {
      if (kMass && shift == 24) { r.found = false; return r; }
      t = block_reduce_max_int(c > 0 ? tid : -1, sm.ired);
    }
    const int c_before = t > 0 ? sm.scan_c[t - 1] : 0;
    r.above += c_before;
    if (kMass && t > 0) r.mass_above += sm.scan_m[t - 1];
    r.equal = sm.scan_c[t] - c_before;
    r.key |= static_cast<unsigned int>(255 - t) << shift;
    mask |= 255u << shift;
    __syncthreads();
  }
  return r;
}

template <int kCand>   // the row stride of the candidate arrays
__global__ void __launch_bounds__(kRowThreads) beam_sample_kernel(const BeamParams p) {
  griddep_launch();
  StepState* st = p.state;
  if (step_wait(&st->finished, ChainSync{})) return;
  extern __shared__ float srow[];   // the row's scores logits / T
  __shared__ SampleSmem sm;
  const int row = blockIdx.x, rows = gridDim.x, tid = threadIdx.x, V = p.V;
  const int cur_len = st->cur_len;
  const float* z = p.logits + static_cast<long long>(row) * V;
  float* dump = step_logits_row(p.step_logits, st->step, rows, row, V);
  float mx = -INFINITY;
  for (int i0 = tid; i0 < V; i0 += 8 * kRowThreads) {        // 8 independent loads in flight per thread
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (i0 + k * kRowThreads < V) ? __ldcg(z + i0 + k * kRowThreads) : 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int i = i0 + k * kRowThreads;
      if (i >= V) break;
      if (dump != nullptr) dump[i] = v[k];
      const float sv = v[k] / p.smp.temperature;   // a division, as the reference: a multiply by 1/T can split a tie it makes
      srow[i] = sv;
      mx = fmaxf(mx, sv);
    }
  }
  // an image still inside its prefix takes the prefix token (beam_update_kernel): nothing to draw
  if (p.row_prefix != nullptr && cur_len < p.row_prefix_lens[row / p.beam]) return;
  const float m = block_reduce_max(mx, sm.red);

  // ---- top-k: keys >= live survive ----
  unsigned int live = 0u;
  int n_live = V;
  if (p.smp.top_k > 0) {
    const RadixStop r = radix_descend<false>(srow, V, static_cast<float>(min(max(p.smp.top_k, 2), V)), 0u, m, sm);
    live = r.key;
    n_live = r.above + r.equal;
  }
  // ---- top-p: kept = keys > kkey, and the keys == kkey up to index i_last ----
  unsigned int kkey = live;
  int keep_ties = 0x7fffffff, n_kept = n_live;
  const float top_p = p.smp.top_p;
  if (top_p != 0.f && top_p < 1.f) {
    float w = 0.f;
    for (int i = tid; i < V; i += kRowThreads)
      if (order_key(srow[i]) >= live) w += expf(srow[i] - m);
    const float target = top_p * block_reduce_sum(w, sm.red);   // cumsum(softmax) > p  <=>  cumsum(exp(s - m)) > p * sum
    const RadixStop c = radix_descend<true>(srow, V, target, live, m, sm);
    if (c.found) {
      // the position J where the cumulative mass crosses: the first j of the c.equal ties at c.key (index order), each of
      // mass q, with mass_above + (j + 1) q > target (computed, not accumulated: thousands of equal terms would drift)
      const float q = expf(key_value(c.key) - m);
      const float n = floorf((target - c.mass_above) / q);
      const int j = !(n > 0.f) ? 0 : (n >= static_cast<float>(c.equal - 1) ? c.equal - 1 : static_cast<int>(n));
      const int J = c.above + j;
      const int K = max(J, 2) + 1;   // positions 0 .. max(J, 2): the first two forced, then the shift right by one
      if (K < n_live) {
        n_kept = K;
        if (J >= 2) {
          kkey = c.key;
          keep_ties = j + 1;
        } else {
          const RadixStop r3 = radix_descend<false>(srow, V, 3.f, 0u, m, sm);
          kkey = r3.key;
          keep_ties = 3 - r3.above;
        }
      }
    }
  }
  // thread t owns the contiguous indices [i0, i1): ties and draws go in index order (an odd stride: no bank conflicts)
  const int C = ((V + kRowThreads - 1) / kRowThreads) | 1;
  const int i0 = min(V, tid * C), i1 = min(V, i0 + C);
  int i_last = V;
  if (keep_ties != 0x7fffffff) {
    int nt = 0;
    for (int i = i0; i < i1; ++i) nt += order_key(srow[i]) == kkey;
    const int before = block_exclusive_scan_int(nt, sm.ired);
    int found = -1;
    if (keep_ties > before && keep_ties <= before + nt) {
      int k = before;
      for (int i = i0; i < i1; ++i)
        if (order_key(srow[i]) == kkey && ++k == keep_ties) { found = i; break; }
    }
    i_last = block_reduce_max_int(found, sm.ired);
  }
  auto mass = [&](int i) -> float {
    const unsigned int k = order_key(srow[i]);
    return (k > kkey || (k == kkey && i <= i_last)) ? expf(srow[i] - m) : 0.f;
  };

  // ---- two draws without replacement ----
  float w1 = 0.f;
  int nz1 = -1;
  for (int i = i0; i < i1; ++i) {
    const float w = mass(i);
    w1 += w;
    if (w > 0.f) nz1 = i;
  }
  const int last1 = block_reduce_max_int(nz1, sm.ired);
  const float* u = p.smp.uniforms + (static_cast<long long>(cur_len) * rows + row) * 2;
  float total1 = 0.f, total2 = 0.f;
  int t1 = inverse_cdf_index(w1, __ldg(u), i0, i1, mass, sm.red, sm.ired, &total1);
  if (t1 < 0 || !(mass(t1) > 0.f)) t1 = last1;   // rounding at the end of the distribution: never a zero-probability token
  auto mass2 = [&](int i) -> float { return i == t1 ? 0.f : mass(i); };
  float w2 = w1;
  int nz2 = nz1;
  if (t1 >= i0 && t1 < i1) {
    w2 = 0.f;
    nz2 = -1;
    for (int i = i0; i < i1; ++i) {
      const float w = mass2(i);
      w2 += w;
      if (w > 0.f) nz2 = i;
    }
  }
  const int last2 = block_reduce_max_int(nz2, sm.ired);
  int t2 = inverse_cdf_index(w2, __ldg(u + 1), i0, i1, mass2, sm.red, sm.ired, &total2);
  if (t2 < 0 || !(mass2(t2) > 0.f)) t2 = last2;
  if (tid != 0) return;
  if (!(m > -INFINITY) || !(total2 > 0.f)) {
    // torch.multinomial raises: fewer than two tokens of non-zero probability.  The first such (step, row) is reported
    // by gitb200_generate_finish; the search stops.
    atomicMax(&st->bad_draw, 0x7fffffff - (st->step * rows + row));
    st->finished = 1;
    return;
  }
  const float lse = logf(total1), bs = p.s.beam_scores[row];
  p.s.cand_val[row * kCand] = ((srow[t1] - m) - lse) + bs;
  p.s.cand_idx[row * kCand] = t1;
  p.s.cand_val[row * kCand + 1] = ((srow[t2] - m) - lse) + bs;
  p.s.cand_idx[row * kCand + 1] = t2;
  if (p.smp.kept != nullptr) p.smp.kept[row] = n_kept;
}

// One thread block per image (32 threads; the bookkeeping itself is sequential like the reference's loop).
template <int kCand>
__global__ void __launch_bounds__(32) beam_update_kernel(const BeamParams p) {
  griddep_launch();
  StepState* st = p.state;
  if (step_wait(&st->finished, ChainSync{})) return;
  const int b = blockIdx.x;
  const int lane = threadIdx.x;
  const int beam = p.beam, NC = p.per_node * p.beam, V = p.V;
  const int cur = *p.s.cur;
  const int cur_len = st->cur_len;
  const long long* ids_old = p.s.ids[cur];
  long long* ids_new = p.s.ids[cur ^ 1];
  const int* src_old = p.s.src[cur];
  int* src_new = p.s.src[cur ^ 1];
  __shared__ float m_val[kCand];
  __shared__ int m_word[kCand];
  __shared__ int m_beam[kCand];
  __shared__ int n_row[kCand / 2];   // next beams: source row (global)
  __shared__ int n_word[kCand / 2];
  __shared__ float n_score[kCand / 2];
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
    float top;   // the best candidate score
    if (p.smp.uniforms != nullptr) {
      // sampled candidates stay in (beam, draw) order (reference :1159-1166); is_done takes their maximum (:1187).  The
      // reference offsets candidate c by the beam index tiled as [0 .. beam) x per_node (:1155-1158), so the history that
      // candidate c (row c / per_node's draw c % per_node) extends is that of beam c % beam.
      top = -INFINITY;
      for (int c = 0; c < NC; ++c) {
        const int r = b * beam + c / p.per_node;
        m_val[c] = p.s.cand_val[r * kCand + c % p.per_node];
        m_word[c] = p.s.cand_idx[r * kCand + c % p.per_node];
        m_beam[c] = c % beam;
        top = fmaxf(top, m_val[c]);
      }
    } else {
      // merge the `beam` row lists into the image's top-NC, ordered by (value desc, flat index asc)
      int ptr[kCand / 2];
      for (int k = 0; k < beam; ++k) ptr[k] = 0;
      for (int c = 0; c < NC; ++c) {
        int best = -1;
        float bv = 0.f;
        long long bflat = 0;
        for (int k = 0; k < beam; ++k) {
          if (ptr[k] >= NC) continue;
          const int r = b * beam + k;
          const float v = p.s.cand_val[r * kCand + ptr[k]];
          const long long flat = static_cast<long long>(k) * V + p.s.cand_idx[r * kCand + ptr[k]];
          if (best < 0 || v > bv || (v == bv && flat < bflat)) { best = k; bv = v; bflat = flat; }
        }
        m_val[c] = bv;
        m_word[c] = p.s.cand_idx[(b * beam + best) * kCand + ptr[best]];
        m_beam[c] = best;
        ++ptr[best];
      }
      top = m_val[0];
    }
    // ---- reference bookkeeping (layers/decoder.py:1184-1228) ----
    bool done = p.s.done[b] != 0;
    if (!done && p.s.hyp_len[b] > 0) {  // BeamHypotheses.is_done with early_stopping=False (:1330-1341)
      done = p.s.worst_score[b] >= top / beam_length_norm(p.max_steps - 1, p.length_penalty);
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
  // loop-state advance by the last image: an image is live until it is done, and the search stops once every image is
  // (`if all(done): break`, :1253)
  __threadfence();
  if (lane == 0) close_step(st, p.s.done[b] == 0, p.B, st->step, cur_len, p.max_steps, [&](int) { *p.s.cur = cur ^ 1; });
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
