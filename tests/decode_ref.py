"""fp64 statements of one decode step and of the beam-search bookkeeping, shared by the decode-step test modules.

`ref_step` computes one step of R rows from given image and text K/V (the engine's own caches, read back), rounding to
bf16 exactly where the engine stores bf16 and computing everything else in fp64.  `beam_replay` replays the reference's
beam search over dumped step logits and records the re-orderings; `ancestry` turns them into the physical text-cache row
every logical row reads at every position, which is what the engine's src_row indirection table must hold.
"""
import math

import torch

import git_oracle

V = 30522
D = 768
H = 12
EOS = 102
CLS = 101


def bf16(t):
    """Round to bfloat16 (to nearest, ties to even, from the fp32 value) and return it as fp64."""
    x = t.to(torch.float32).contiguous()
    b = x.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b)
    return b.to(torch.int32).view(torch.float32).to(torch.float64)


def _ln(x, g, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * g + b


def _gelu_erf(x):
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


class RefWeights(object):
    """The decoder's weights in fp64; GEMM weights and the tied LM-head matrix rounded to bf16 when `rounding`."""

    def __init__(self, sd, rounding=True):
        w = (lambda k: bf16(sd[k])) if rounding else (lambda k: sd[k].double())
        f = lambda k: sd[k].double()
        t = 'textual.'
        self.rounding = rounding
        self.words = f(t + 'embedding.words.weight')
        self.lm = bf16(self.words) if rounding else self.words
        self.positions = f(t + 'embedding.positions.weight')
        self.lne = (f(t + 'embedding.layer_norm.weight'), f(t + 'embedding.layer_norm.bias'))
        self.out_bias = f(t + 'output.bias')
        self.layers = []
        for j in range(6):
            b = t + 'transformer.encoder.layer.%d.' % j
            a = b + 'attention.'
            self.layers.append(dict(
                wq=w(a + 'self.query.weight'), bq=f(a + 'self.query.bias'),
                wk=w(a + 'self.key.weight'), bk=f(a + 'self.key.bias'),
                wv=w(a + 'self.value.weight'), bv=f(a + 'self.value.bias'),
                wo=w(a + 'output.dense.weight'), bo=f(a + 'output.dense.bias'),
                ln1=(f(a + 'output.LayerNorm.weight'), f(a + 'output.LayerNorm.bias')),
                w1=w(b + 'intermediate.dense.weight'), b1=f(b + 'intermediate.dense.bias'),
                w2=w(b + 'output.dense.weight'), b2=f(b + 'output.dense.bias'),
                ln2=(f(b + 'output.LayerNorm.weight'), f(b + 'output.LayerNorm.bias'))))

    def to(self, device):
        """The same weights on `device` (fp64 throughout; the GPU tests run the reference there)."""
        for name, val in list(vars(self).items()):
            if torch.is_tensor(val):
                setattr(self, name, val.to(device))
            elif isinstance(val, tuple):
                setattr(self, name, tuple(x.to(device) for x in val))
        self.layers = [{k: (tuple(x.to(device) for x in v) if isinstance(v, tuple) else v.to(device)) for k, v in L.items()}
                       for L in self.layers]
        return self

    def embed(self, tokens, pos):
        """LN(words[token] + positions[pos], eps 1e-8) in fp64 (reference layers/decoder.py:65-78)."""
        return _ln(self.words[tokens] + self.positions[pos], self.lne[0], self.lne[1], 1e-8)


def ref_step(W, img_k, img_v, txt_k, txt_v, tokens, pos, n_layers=6, q_bf16=True, defect=None):
    """One greedy decode step of R rows at text position `pos`.

    img_k / img_v: per layer [R, M, 768] (the image K/V cache); txt_k / txt_v: per layer [R, pos, 768] (text positions
    0 .. pos - 1); tokens: int64 [R], the token fed at `pos`.  q_bf16: the path stores q / 8 as bf16 (the persistent kernel;
    the chain keeps it in fp32).  defect: None or (kind, index[, layer]) -- one planted error in that layer (default: the
    last layer run)
    ('wo' | 'w1' | 'fc2' tile, 'fc2' as (tile, k slice)), in the LM head ('lm' tile), or in its attention ('chunk': a 64-key
    image chunk, 'img_last': key M - 1, 'newest': the text key at pos, all masked out).
    Returns {'layers': [per layer: qb, k, v, ctx, y, xa, ub, x], 'logits': [R, V]}."""
    bf = bf16 if W.rounding else (lambda t: t.double())
    kind, idx = defect[:2] if defect is not None else (None, None)
    at = (defect[2] if defect is not None and len(defect) > 2 else n_layers - 1)
    R = tokens.shape[0]
    x = W.embed(tokens, pos)
    out = {'layers': []}
    for j in range(n_layers):
        L = W.layers[j]
        last = j == at
        hb = bf(x)
        q = hb @ L['wq'].T + L['bq']
        qb = bf(q / 8.0) if (q_bf16 and W.rounding) else q / 8.0
        k = bf(hb @ L['wk'].T + L['bk'])
        v = bf(hb @ L['wv'].T + L['bv'])
        ik, iv = img_k[j].double(), img_v[j].double()
        M = ik.shape[1]
        K = torch.cat([ik, txt_k[j].double(), k[:, None]], dim=1)
        Vv = torch.cat([iv, txt_v[j].double(), v[:, None]], dim=1)
        S = K.shape[1]
        s = torch.einsum('rhd,rshd->rhs', qb.reshape(R, H, 64), K.reshape(R, S, H, 64))
        if last and kind in ('chunk', 'img_last', 'newest'):
            drop = {'chunk': slice(64 * idx, min(64 * idx + 64, M)), 'img_last': slice(M - 1, M),
                    'newest': slice(S - 1, S)}[kind]
            s[:, :, drop] = float('-inf')
        p = torch.softmax(s, dim=-1)
        ctx = bf(torch.einsum('rhs,rshd->rhd', p, Vv.reshape(R, S, H, 64)).reshape(R, D))
        wo, w1, w2 = L['wo'], L['w1'], L['w2']
        if last and kind == 'wo':
            wo = wo.clone()
            wo[8 * idx:8 * idx + 8] = 0
        if last and kind == 'w1':
            w1 = w1.clone()
            w1[8 * idx:8 * idx + 8] = 0
        if last and kind == 'fc2':
            w2 = w2.clone()
            w2[8 * idx[0]:8 * idx[0] + 8, 768 * idx[1]:768 * idx[1] + 768] = 0
        y = x + (ctx @ wo.T + L['bo'])
        xa = _ln(y, L['ln1'][0], L['ln1'][1], 1e-12)
        ub = bf(_gelu_erf(bf(xa) @ w1.T + L['b1']))
        x = _ln(xa + (ub @ w2.T + L['b2']), L['ln2'][0], L['ln2'][1], 1e-12)
        out['layers'].append(dict(qb=qb, k=k, v=v, ctx=ctx, y=y, xa=xa, ub=ub, x=x))
    logits = bf(x) @ W.lm.T + W.out_bias
    if kind == 'lm':
        logits[:, 8 * idx:8 * idx + 8] = W.out_bias[8 * idx:8 * idx + 8]
    out['logits'] = logits
    return out


def expected_selection(z, tokens_in, first):
    """Greedy choice and its log-prob from raw step logits z [R, V] (fp32 as dumped): the no-repeat mask (-10000 at the
    token fed, reference layers/decoder.py:330) where first[r] is False, arg-max with the lowest index on ties, fp64
    log-softmax."""
    z = z.double().clone()
    for r in range(z.shape[0]):
        if not first[r]:
            z[r, int(tokens_in[r])] = -10000.0
    tok = torch.argmax(z, dim=1)           # the first maximal index
    lp = torch.log_softmax(z, dim=1).gather(1, tok[:, None])[:, 0]
    return tok, lp


# ---------------------------------------------------------------------------------------------------------------------
# Beam search: the bookkeeping replayed over dumped step logits, and the text-K/V ancestry it implies
# ---------------------------------------------------------------------------------------------------------------------
def length_norm64(length, lp):
    return git_oracle._length_norm(length, lp)


def beam_replay(z, B, beam, max_steps, length_penalty, eos=EOS, start=CLS, prefix=None, prefix_lens=None, ties='low'):
    """git_oracle.beam_search (num_keep_best = 1, per-node width 2) replayed over step logits z [steps, B * beam, V] (fp32,
    as the engine dumped them), recording what the engine keeps on the device.

    The image-level top 2 * beam is ranked by (score desc, beam asc, raw logit desc, token asc), the engine's order
    (search.cuh): in exact arithmetic log_softmax(z) + beam score is strictly increasing in the logit z, and fp32 can
    round two different logits of one row to the same score; those stay in logit order.  Exact logit ties go to the lower
    token (TopList::before), equal scores of different beams to the lower beam (beam_update_kernel's merge).  torch.topk
    does not promise an order for equal scores.  ties='high' breaks exact logit ties the other way round (used to show
    that a planted tie decides the outcome).
    prefix [B, P] / prefix_lens [B]: per-image prefixes -- while an image's caption is shorter than its prefix every beam
    takes the next prefix token and keeps its score and history (beam_update_kernel's in_prefix branch).
    Alongside the fp32 scores the decisions are made on, every beam score is also accumulated in fp64 from the fp64
    log-softmax of the same logits ('hyp_score64').

    Returns dict(pred [B, max_steps] EOS-padded, logprobs [B] fp32, bidx / words: per step [R] int64, ids [R, max_steps]
    (the final token history, EOS-padded past the steps run), done / hyp_len [B], hyp_score [B] fp32, hyp_score64 [B],
    done_step [B]: the step at which the image was first found done, or -1; cand64: per step [R] the fp64 beam score
    each row's candidates are ranked on; gap: the smallest relative difference between the two sides of a done or
    hypothesis-replace comparison whose sides differ -- the decisions the length normalisation takes part in)."""
    R = B * beam
    V = z.shape[-1]
    NC = 2 * beam
    ids = torch.full((R, 1), start, dtype=torch.long)
    if prefix is not None:
        ids = prefix[torch.arange(R) // beam, :1].clone()
    cur_len = 1
    beam_scores = torch.zeros(B, beam)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    s64 = beam_scores.double().clone()
    hyps = [dict(score=None, score64=None, seq=None, worst=1e9) for _ in range(B)]
    done = [False] * B
    done_step = [-1] * B
    bidx_all, words_all, cand64 = [], [], []
    gap = [float('inf')]

    def note_gap(a, b):
        if a != b:
            gap[0] = min(gap[0], abs(a - b) / max(abs(a), abs(b)))
    t = 0
    while cur_len < max_steps:
        zt = z[t].float()
        lsm64 = torch.log_softmax(zt.double(), dim=-1)
        scores = torch.log_softmax(zt, dim=-1) + beam_scores[:, None]
        flat = scores.view(B, beam * V)
        order = rank_candidates(flat, zt.reshape(B, beam * V), V, NC, ties)
        nscore = flat.gather(1, order)
        cand64.append(s64.clone())
        nxt = []
        for b in range(B):
            rows = range(b * beam, b * beam + beam)
            if prefix_lens is not None and cur_len < prefix_lens[b]:
                nxt.extend((float(beam_scores[r]), int(prefix[b, cur_len]), r, float(s64[r])) for r in rows)
                continue
            h = hyps[b]
            if not done[b] and h['seq'] is not None:
                best = nscore[b, 0].item() / length_norm64(max_steps - 1, length_penalty)
                note_gap(h['worst'], best)
                done[b] = h['worst'] >= best
                if done[b]:
                    done_step[b] = t
            if done[b]:
                nxt.extend([(0.0, eos, 0, 0.0)] * beam)
                continue
            sent = []
            for idx, sc in zip(order[b].tolist(), nscore[b].tolist()):
                bid, wid = idx // V, idx % V
                r = b * beam + bid
                sc64 = float(s64[r] + lsm64[r, wid])
                if wid == eos or cur_len + 1 == max_steps:
                    score = sc / length_norm64(cur_len, length_penalty)
                    if h['seq'] is not None:
                        note_gap(score, h['worst'])
                    if h['seq'] is None or score > h['worst']:
                        # one kept hypothesis: a better one replaces it and becomes the worst score
                        h['worst'] = min(score, h['worst']) if h['seq'] is None else score
                        h['score'], h['seq'] = score, ids[r, :cur_len].clone()
                        h['score64'] = sc64 / length_norm64(cur_len, length_penalty)
                else:
                    sent.append((sc, wid, r, sc64))
                if len(sent) == beam:
                    break
            if len(sent) < beam:
                sent = [(0.0, eos, 0, 0.0)] * beam
            nxt.extend(sent)
        beam_scores = torch.tensor([x[0] for x in nxt], dtype=torch.float32)
        s64 = torch.tensor([x[3] for x in nxt], dtype=torch.float64)
        words = torch.tensor([x[1] for x in nxt], dtype=torch.long)
        bidx = torch.tensor([x[2] for x in nxt], dtype=torch.long)
        ids = torch.cat([ids[bidx], words[:, None]], dim=-1)
        bidx_all.append(bidx)
        words_all.append(words)
        cur_len += 1
        t += 1
        if all(done):
            break
    pred = torch.full((B, max_steps), eos, dtype=torch.long)
    logprobs = torch.full((B,), -1e5)
    hyp_len = torch.zeros(B, dtype=torch.long)
    hyp_score = torch.full((B,), -1e30)
    hyp_score64 = torch.full((B,), float('nan'), dtype=torch.float64)
    for b, h in enumerate(hyps):
        if h['seq'] is not None:
            n = h['seq'].numel()
            pred[b, :n] = h['seq']
            logprobs[b] = h['score']
            hyp_len[b], hyp_score[b], hyp_score64[b] = n, h['score'], h['score64']
    full_ids = torch.full((R, max_steps), eos, dtype=torch.long)
    full_ids[:, :ids.shape[1]] = ids
    return dict(pred=pred, logprobs=logprobs, bidx=bidx_all, words=words_all, ids=full_ids, n_steps=t,
                done=torch.tensor(done, dtype=torch.long), done_step=done_step, hyp_len=hyp_len, hyp_score=hyp_score,
                hyp_score64=hyp_score64, worst=torch.tensor([h['worst'] for h in hyps], dtype=torch.float64),
                cand64=cand64, gap=gap[0])


def rank_candidates(scores, z, V, NC, ties='low'):
    """Flat indices (beam * V + token) of the top NC of each row of scores [B, beam * V], ranked by (score desc, beam asc,
    logit z desc, token asc; token desc with ties='high').  Stable sorts from the least significant key up."""
    B, n = scores.shape
    perm = torch.arange(n)
    if ties == 'high':
        perm = perm // V * V + (V - 1 - perm % V)
    perm = perm.expand(B, n)
    for key, desc in ((z, True), (None, False), (scores, True)):
        k = perm // V if key is None else key.gather(1, perm)
        perm = perm.gather(1, torch.sort(k, dim=1, descending=desc, stable=True).indices)
    return perm[:, :NC]


def ancestry(bidx, R):
    """Physical text-cache row of every (logical row, position): anc[t] is [R, t] for t = 0 .. len(bidx).

    anc_0 is empty; anc_{t+1}[r][j] = anc_t[bidx_t[r]][j] for j < t, and anc_{t+1}[r][t] = bidx_t[r] -- the row that
    ran step t in row r's history wrote position t (into its own physical row, anc_t[x][t] = x)."""
    anc = [torch.zeros(R, 0, dtype=torch.long)]
    for b in bidx:
        a = torch.cat([anc[-1], torch.arange(R)[:, None]], dim=1)
        anc.append(a[b])
    return anc


def src_row_table(anc, T_alloc):
    """The indirection table the engine keeps after len(anc) - 1 steps: anc extended by the identity."""
    R, t = anc.shape
    tab = torch.arange(R)[:, None].expand(R, T_alloc).clone()
    tab[:, :t] = anc
    return tab


def gather_text(txt, anc, kv, defect=None):
    """Text K or V (kv = 0 / 1) per layer [R, t, 768] of logical rows at step t = anc.shape[1], gathered from the physical
    rows of the cache txt [layers, 2, R, T_alloc, 768].  defect: None or ('own_row', r, j) -- row r reads position j from its
    own physical row instead of its ancestor."""
    R, t = anc.shape
    if defect is not None and defect[0] == 'own_row':
        anc = anc.clone()
        anc[defect[1], defect[2]] = defect[1]
    pos = torch.arange(t, device=txt.device)
    a = anc.to(txt.device)
    return [txt[j, kv][a, pos] for j in range(txt.shape[0])]


def expand_images(img, beam, kv, shift=0):
    """Image K or V per layer [R, M, 768] from the cache img [layers, 2, B, M, 768]: row r reads image r // beam (shift:
    image (r // beam + shift) mod B instead, a planted defect)."""
    B = img.shape[2]
    idx = (torch.arange(B * beam, device=img.device) // beam + shift) % B
    return [img[j, kv][idx] for j in range(img.shape[0])]
