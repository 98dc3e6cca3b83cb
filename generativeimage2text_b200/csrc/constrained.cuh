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
// One CTA per row, kRowThreads threads, two passes over the row's fp32 logits (L2 resident).  Used by the kernel-chain
// decode step in place of greedy_select_kernel; the bookkeeping (resolve_row / commit_row, rowops.cuh) is the same, and
// so are the CTA reductions and the inverse-CDF lookup (rowops.cuh, shared with beam_sample_kernel).
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

__global__ void __launch_bounds__(kRowThreads) constrained_select_kernel(const SelectParams p, const ConstrainParams q) {
  griddep_launch_early();
  StepState* st = p.state;
  if (step_wait(&st->finished, p.chain)) return;
  __shared__ float sh[kRowWarps];
  __shared__ float sh_scan[kRowWarps];
  __shared__ int sh_arg[kRowWarps];
  __shared__ int sh_i[2];
  __shared__ float sh_f[2];
  const int row = blockIdx.x, tid = threadIdx.x;
  const int step = st->step, cur_len = st->cur_len;
  const float* z = p.logits + static_cast<long long>(row) * p.V;
  const long long last = p.next_token[row];
  const RowStep rs = row_step(p, row, step, cur_len, last);
  const bool sampling = q.uniforms != nullptr;
  const float it = sampling ? q.inv_temperature : 1.0f;
  if (float* dst = step_logits_row(p.step_logits, step, p.rows_total, p.row0 + row, p.V))
    for (int i = tid; i < p.V; i += kRowThreads) dst[i] = __ldcg(z + i);
  // the row after the reference's masks: no-repeat scatter (:330 / trie :122), never at a row's first decision
  auto val = [&](int i) -> float {
    float v = __ldcg(z + i);
    if (!rs.first && i == static_cast<int>(last)) v = -10000.0f;
    return v;
  };
  // thread t owns the contiguous indices [t * C, (t + 1) * C): the inverse-CDF lookup needs index order
  const int C = (p.V + kRowThreads - 1) / kRowThreads;
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
  const int garg = block_reduce_min_int((m == gmax) ? arg : 0x7fffffff, sh_arg);
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
      for (int e = e0 + tid; e < e1; e += kRowThreads) {
        const int t = q.trie_token[e];
        const float v = val(t);
        if (v > bv || (v == bv && t < bt)) { bv = v; bt = t; be = e; }
      }
      const float gb = block_reduce_max(bv, sh);
      const int gt = block_reduce_min_int((bv == gb && be >= 0) ? bt : 0x7fffffff, sh_arg);
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
