// Greedy selection under a vocabulary trie and / or with sampling -- the remaining decoders of SURVEY.md 8(f)-4:
//   * TrieAutoRegressiveBeamSearch.search (reference trie_decoder.py:27-218; beam 1): after the no-repeat scatter, the EOS
//     forcing and the log-softmax, the log-probs of the tokens the trie allows next are raised by
//     (max logit - min logit + 1) (:61-62, :141-142), the top-1 is taken (:67, :150) and the trie cursor moves (:70, :153);
//     the raised value is what accumulates into the caption's log-prob (:163).  The reference keeps ONE cursor and raises
//     row 0 only, i.e. it is a batch-1 decoder; here every row owns a cursor and is constrained exactly as a batch-1 call
//     would be (max / min taken over the row).
//   * the do_sample branches of AutoRegressiveBeamSearch.search (reference layers/decoder.py:260-272, 364-375): the next
//     token is drawn from softmax(logits / temperature); the log-prob that accumulates is log_softmax of the tempered
//     logits at a row's first decision (:260-265) and of the un-tempered ones afterwards (:358, :368-375 -- the division
//     happens after the log-softmax there).  torch.multinomial's random stream cannot be reproduced, so the draw is an
//     inverse-CDF lookup in index order with a caller-provided uniform number per (step, row): given the same uniforms
//     the oracle makes the same choice.  (top_k / top_p are accepted and ignored by that class: the filter call is
//     commented out, :372.)
// One CTA per row, 256 threads, two passes over the row's fp32 logits (L2 resident).  Used by the kernel-chain decode step
// in place of greedy_select_kernel; the bookkeeping (resolve_row / commit_row, rowops.cuh) is the same.
#pragma once
#include "ptx.cuh"
#include "rowops.cuh"

namespace gitb200 {

struct ConstrainParams {
  const int* trie_begin;   // [n_nodes + 1] CSR offsets (null: no trie)
  const int* trie_token;   // [n_edges] token of an edge
  const int* trie_child;   // [n_edges] node it leads to
  int* trie_cursor;        // [rows] current node per row (0 = root); advanced here
  int n_nodes;
  const float* uniforms;   // [max_steps, rows] (null: no sampling); row r at length cur_len reads uniforms[cur_len * rows + r]
  float inv_temperature;
};

__device__ __forceinline__ float block_reduce_max(float v, float* sh) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sh[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = fmaxf(r, sh[w]);
  __syncthreads();
  return r;
}
// fixed-order sum (warp tree, then warps 0..7 in order): bit-reproducible
__device__ __forceinline__ float block_reduce_sum(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sh[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r += sh[w];
  __syncthreads();
  return r;
}

// Block max of an int (every thread gets it).
__device__ __forceinline__ int block_reduce_max_int(int v, int* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  int r = sh[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = max(r, sh[w]);
  __syncthreads();
  return r;
}

// The index-order inverse-CDF lookup of the sampling kernels (a 256-thread CTA per row): thread t owns the contiguous
// indices [i0, i1) and `mass_t` is the sum of mass(i) over them in index order.  The target is u * total, total = the
// thread masses summed in thread order (warp scans, then the 8 warp totals in order).  The owner of the interval
// [lo, hi) that holds the target walks its indices to the first one whose running mass exceeds it; a target at or beyond
// the total (u -> 1 and rounding) falls to the last thread, whose walk ends at its last index.  Rounding can make two
// adjacent threads claim the target (lo is hi - mass_t, not the previous thread's hi): the higher index wins.  Returns
// the index (every thread), or -1 when no thread claims the target; *total_out = total.
template <class Mass>
__device__ __forceinline__ int inverse_cdf_index(float mass_t, float u, int i0, int i1, Mass mass, float* sh_scan, int* sh_pick,
                                                 float* total_out) {
  const int tid = threadIdx.x;
  float inc = mass_t;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float up = __shfl_up_sync(0xffffffffu, inc, o);
    if ((tid & 31) >= o) inc += up;
  }
  if ((tid & 31) == 31) sh_scan[tid >> 5] = inc;
  __syncthreads();
  float before = 0.f, total = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    if (w < (tid >> 5)) before += sh_scan[w];
    total += sh_scan[w];
  }
  const float hi = before + inc, lo = hi - mass_t;
  const float target = u * total;
  int pick = -1;
  if ((target >= lo && target < hi && mass_t > 0.f) || (tid == 255 && target >= hi)) {
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

__global__ void __launch_bounds__(256) constrained_select_kernel(const SelectParams p, const ConstrainParams q) {
  griddep_launch_early();
  StepState* st = p.state;
  if (p.chain.counters != nullptr) {
    if (st->finished) return;  // stable within a step
    chain_wait(p.chain);
  } else {
    griddep_wait();
    if (st->finished) return;
  }
  __shared__ float sh[8];
  __shared__ float sh_scan[8];
  __shared__ int sh_i[2];
  __shared__ float sh_f[2];
  const int row = blockIdx.x, tid = threadIdx.x;
  const int step = st->step, cur_len = st->cur_len;
  const float* z = p.logits + static_cast<long long>(row) * p.V;
  const long long last = p.next_token[row];
  const RowStep rs = row_step(p, row, step, cur_len, last);
  const bool sampling = q.uniforms != nullptr;
  const float it = sampling ? q.inv_temperature : 1.0f;
  if (p.step_logits != nullptr) {
    float* dst = p.step_logits + (static_cast<long long>(step) * p.rows_total + p.row0 + row) * p.V;
    for (int i = tid; i < p.V; i += 256) dst[i] = __ldcg(z + i);
  }
  // the row after the reference's masks: no-repeat scatter (:330 / trie :122), never at a row's first decision
  auto val = [&](int i) -> float {
    float v = __ldcg(z + i);
    if (!rs.first && i == static_cast<int>(last)) v = -10000.0f;
    return v;
  };
  // thread t owns the contiguous indices [t * C, (t + 1) * C): the inverse-CDF lookup needs index order
  const int C = (p.V + 255) / 256;
  const int i0 = tid * C, i1 = min(p.V, i0 + C);
  // ---- pass 1: max / min / arg max ----
  float m = -INFINITY, mn = INFINITY;
  int arg = 0x7fffffff;
  for (int i = i0; i < i1; ++i) {
    const float v = val(i);
    if (v > m) { m = v; arg = i; }
    mn = fminf(mn, v);
  }
  const float gmax = block_reduce_max(m, sh);
  const float gmin = -block_reduce_max(-mn, sh);
  // lowest index among the maxima (torch.topk / argmax of the reference; exact ties are measure-zero in practice)
  int cand = (m == gmax) ? arg : 0x7fffffff;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
  __shared__ int sh_arg[8];
  if ((tid & 31) == 0) sh_arg[tid >> 5] = cand;
  __syncthreads();
  int garg = sh_arg[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) garg = min(garg, sh_arg[w]);
  __syncthreads();
  // ---- pass 2: sum exp(v - max) (log-softmax) and, when sampling, this thread's mass of softmax(v / T) ----
  float s1 = 0.f, sT = 0.f;
  for (int i = i0; i < i1; ++i) {
    const float v = val(i);
    s1 += __expf(v - gmax);
    if (sampling) sT += __expf((v - gmax) * it);
  }
  const float sum1 = block_reduce_sum(s1, sh);
  // ---- the choice ----
  long long tok = garg;
  float lp = -logf(sum1);                   // z[arg] - max - log(sum exp(z - max)) with z[arg] == max
  int next_node = -1;
  if (sampling && !rs.done && !rs.in_prefix) {
    const float u = __ldg(q.uniforms + static_cast<long long>(cur_len) * p.rows_total + p.row0 + row);
    float total;
    int pick = inverse_cdf_index(sT, u, i0, i1, [&](int i) { return __expf((val(i) - gmax) * it); }, sh_scan, sh_arg, &total);
    if (pick < 0) pick = garg;
    tok = pick;
    const float vz = val(pick);
    // log-prob of the draw: tempered log-softmax at the row's first decision, un-tempered afterwards (see the header)
    lp = rs.first ? ((vz - gmax) * it - logf(total)) : ((vz - gmax) - logf(sum1));
  }
  if (q.trie_begin != nullptr && !rs.done && !rs.in_prefix) {
    const int node = q.trie_cursor[p.row0 + row];
    const int e0 = q.trie_begin[node], e1 = q.trie_begin[node + 1];
    if (e1 > e0) {
      // best allowed token: highest logit, lowest token id on exact ties
      float bv = -INFINITY;
      int bt = 0x7fffffff, be = -1;
      for (int e = e0 + tid; e < e1; e += 256) {
        const int t = q.trie_token[e];
        const float v = val(t);
        if (v > bv || (v == bv && t < bt)) { bv = v; bt = t; be = e; }
      }
      const float gb = block_reduce_max(bv, sh);
      int c2 = (bv == gb && be >= 0) ? bt : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c2 = min(c2, __shfl_xor_sync(0xffffffffu, c2, o));
      if ((tid & 31) == 0) sh_arg[tid >> 5] = c2;
      __syncthreads();
      int gt = sh_arg[0];
#pragma unroll
      for (int w = 1; w < 8; ++w) gt = min(gt, sh_arg[w]);
      if (bt == gt && be >= 0 && bv == gb) { sh_i[1] = q.trie_child[be]; sh_f[0] = bv; }
      __syncthreads();
      tok = gt;
      next_node = sh_i[1];
      // log_softmax value raised by (max - min + 1), in the reference's operation order: lsm + ((max - min) + 1)
      lp = ((sh_f[0] - gmax) - logf(sum1)) + ((gmax - gmin) + 1.0f);
    }
  }
  if (tid != 0) return;
  if (next_node >= 0) q.trie_cursor[p.row0 + row] = next_node;
  const RowChoice c = resolve_row(p, row, cur_len, rs, tok, lp);
  commit_row(p, row, step, cur_len, c, p.chain.counters);
}

__global__ void trie_reset_kernel(int* cursor, int rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows) cursor[i] = 0;
}

}  // namespace gitb200
