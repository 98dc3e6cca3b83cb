"""TEST INFRASTRUCTURE ONLY -- CPU restatement (fp32, plain torch ops) of the do_sample branch of the reference's
GeneratorWithBeamSearch.search (layers/decoder.py:1083-1290, 1138-1166) with top_k_top_p_filtering (:1343-1375) and
BeamHypotheses (:1292-1341), num_keep_best = 1.  The checker of the engine's sampled beam search
(tests/test_gpu_beam_sample.py); pinned against the unmodified reference by oracle/make_beam_sample_golden.py
(tests/golden/beam_sample_checks.json, tests/test_beam_sample_host.py).  The product package never imports it.

torch.multinomial's random stream cannot be reproduced, so the two draws without replacement are two sequential
index-order inverse-CDF lookups (git_oracle.inverse_cdf_draw) with caller-supplied uniforms -- the draws the engine makes.
"""
import torch
import torch.nn.functional as F

from git_oracle import EOS, inverse_cdf_draw, _length_norm


def top_k_top_p_filter(scores, top_k, top_p, min_tokens_to_keep=2):
    """top_k_top_p_filtering (layers/decoder.py:1343-1375) on a copy: top-k removes the values below the k-th largest
    (k = min(max(top_k, 2), V); ties at it stay); top-p sorts by (value desc, index asc) -- torch.sort leaves ties in no
    particular order, this is the engine's -- removes the positions whose cumulative softmax exceeds top_p, keeps the first
    two, shifts the mask right by one.  Removed entries become -inf."""
    scores = scores.clone()
    if top_k > 0:
        k = min(max(top_k, min_tokens_to_keep), scores.shape[-1])
        scores[scores < torch.topk(scores, k)[0][..., -1, None]] = float('-inf')
    if top_p and top_p < 1.0:
        V = scores.shape[-1]
        # stable sort of the negated values: descending, lower index first among equal values
        sorted_scores, sorted_idx = torch.sort(-scores, dim=-1, stable=True)
        cum = torch.cumsum(F.softmax(-sorted_scores, dim=-1), dim=-1)
        remove = cum > top_p
        remove[..., :min_tokens_to_keep] = False
        remove[..., 1:] = remove[..., :-1].clone()
        remove[..., 0] = False
        scores[remove.scatter(1, sorted_idx, remove)] = float('-inf')
        assert scores.shape[-1] == V
    return scores


def two_draws(probs, u):
    """torch.multinomial(probs, 2) without replacement as the engine draws: two sequential inverse_cdf_draws, the second
    with the first token's probability removed, u [rows, 2].  Raises, as torch.multinomial does, when a row has fewer than
    two tokens of non-zero probability."""
    if bool(((probs > 0).sum(dim=1) < 2).any()):
        raise RuntimeError('invalid multinomial distribution (fewer than two non-zero probabilities)')
    first = inverse_cdf_draw(probs, u[:, 0])
    rest = probs.scatter(1, first[:, None], 0.0)
    return torch.stack([first, inverse_cdf_draw(rest, u[:, 1])], dim=1)


def beam_sample_search(start, step, uniforms, reorder=None, max_steps=40, beam=4, per_node=2, length_penalty=0.6,
                       temperature=1.0, top_k=0, top_p=None, eos=EOS, draw=two_draws):
    """GeneratorWithBeamSearch.search, do_sample branch, num_keep_best=1 (layers/decoder.py:1083-1290, 1138-1166) with
    BeamHypotheses (:1292-1341): per row, scores = logits / T, top_k_top_p_filtering(min_tokens_to_keep=2), two draws
    without replacement from softmax(filtered), candidate = log_softmax(filtered)[token] + beam score; an image's
    candidates stay in (beam, draw) order, candidate j extends the history of beam j % beam (see below), and is_done takes
    their maximum.  `uniforms[t, r, d]` drives draw d of row r at
    caption length t.  Returns (decoded [B, max_steps] EOS-padded, logprobs [B, 1])."""
    assert per_node == 2
    B, cur_len = start.shape
    ids = start.unsqueeze(1).expand(B, beam, cur_len).reshape(B * beam, cur_len)
    hyps = [dict(hyp=[], worst=1e9) for _ in range(B)]
    beam_scores = torch.zeros(B, beam)
    beam_scores[:, 1:] = -1e9                                                   # :1118-1120
    beam_scores = beam_scores.view(-1)
    done = [False] * B
    while cur_len < max_steps:
        logits = step(ids)
        V = logits.shape[-1]
        scores = logits / temperature if temperature != 1.0 else logits        # :1140-1142
        scores = top_k_top_p_filter(scores, top_k, top_p)                      # :1144-1146
        words = draw(F.softmax(scores, dim=-1), uniforms[cur_len])              # :1148-1149
        lp = F.log_softmax(scores, dim=-1).gather(1, words)                     # :1151-1152
        nscore = (lp + beam_scores[:, None]).view(B, beam * per_node)           # :1153, :1160
        # :1155-1159: the word of candidate j (row j // per_node's draw j % per_node) is offset by beam (j % beam) -- the
        # tiled beam indices do not follow the (beam, draw) layout, so the history it extends is that of beam j % beam
        nword = words.view(B, beam * per_node) + (torch.arange(beam) * V).repeat(B, per_node)
        nxt = []
        for b in range(B):
            done[b] = done[b] or _hyp_done(hyps[b], nscore[b].max().item(), max_steps, length_penalty)   # :1187
            if done[b]:
                nxt.extend([(0.0, eos, 0)] * beam)
                continue
            sent = []
            for idx, sc in zip(nword[b].tolist(), nscore[b].tolist()):
                bid, wid = idx // V, idx % V
                if wid == eos or cur_len + 1 == max_steps:
                    _hyp_add(hyps[b], ids[b * beam + bid, :cur_len].clone(), sc, length_penalty)
                else:
                    sent.append((sc, wid, b * beam + bid))
                if len(sent) == beam:
                    break
            if len(sent) == 0:
                sent = [(0.0, eos, 0)] * beam
            assert len(sent) == beam
            nxt.extend(sent)
        beam_scores = torch.tensor([x[0] for x in nxt], dtype=torch.float32)
        bidx = torch.tensor([x[2] for x in nxt], dtype=torch.long)
        ids = torch.cat([ids[bidx], torch.tensor([x[1] for x in nxt], dtype=torch.long)[:, None]], dim=-1)
        if reorder is not None:
            reorder(bidx)
        cur_len += 1
        if all(done):
            break
    decoded = torch.full((B, max_steps), eos, dtype=torch.long)
    logprobs = torch.full((B, 1), -1e5)
    for b in range(B):
        if hyps[b]['hyp']:
            sc, seq = max(hyps[b]['hyp'], key=lambda x: x[0])
            logprobs[b, 0] = sc
            decoded[b, :len(seq)] = seq
            decoded[b, len(seq)] = eos
    return decoded, logprobs


def _hyp_add(h, seq, sum_lp, length_penalty):
    """BeamHypotheses.add with n_hyp = 1 (layers/decoder.py:1315-1328)."""
    score = sum_lp / _length_norm(len(seq), length_penalty)
    if len(h['hyp']) < 1 or score > h['worst']:
        h['hyp'].append((score, seq))
        if len(h['hyp']) > 1:
            srt = sorted([(s, i) for i, (s, _) in enumerate(h['hyp'])])
            del h['hyp'][srt[0][1]]
            h['worst'] = srt[1][0]
        else:
            h['worst'] = min(score, h['worst'])


def _hyp_done(h, best_sum_lp, max_length, length_penalty):
    """BeamHypotheses.is_done with n_hyp = 1, early_stopping=False (layers/decoder.py:1330-1341)."""
    if len(h['hyp']) < 1:
        return False
    return h['worst'] >= best_sum_lp / _length_norm(max_length - 1, length_penalty)
