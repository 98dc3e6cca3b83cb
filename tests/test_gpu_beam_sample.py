"""GPU: sampled beam search (GeneratorWithBeamSearch with do_sample; reference layers/decoder.py:1138-1166, 1343-1375).

  * beam_sample_kernel through gitb200_op_beam_sample against an fp64 restatement of one step: kept sets and drawn tokens
    exactly, candidate scores within SCORE_ATOL;
  * the search: beam_sample_oracle.beam_sample_search replayed over the engine's own step logits with the engine's uniforms gives
    the engine's captions and log-probs;
  * independence (a batch row == the batch-1 call), graph / PDL / fresh-engine bit-identity, and that do_sample=False
    leaves the deterministic search bit-identical.

A draw or a top-p cut decided within BOUNDARY of a CDF step (fp64) is excluded from exact comparisons: the engine sums in
fp32, in its own order.  Every test asserts the gap of what it compares.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import beam_sample_oracle as bso
from generativeimage2text_b200 import _lib
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images, VOCAB

pytestmark = pytest.mark.gpu

EOS = 102
BOUNDARY = 1e-6
SCORE_ATOL = 3e-6      # about twice the largest |kernel - fp64| candidate score measured (1.33e-6, H100 SXM)
LOGPROB_ATOL = 1e-5    # final caption log-probs, engine vs the oracle's fp32 replay


class Tok:
    cls_token_id, sep_token_id = 101, 102


# ---------------------------------------------------------------------------------------------------------------------
# the kernel against fp64
# ---------------------------------------------------------------------------------------------------------------------
def ref_step(z, T, top_k, top_p, u, bs):
    """One row in fp64 (scores = z / T in fp32, as the reference divides) -> (kept mask, tokens, scores, gap): gap is the
    distance of the top-p cut and of both draws from their decision boundaries."""
    s = (z / T).double()
    V = s.numel()
    keep = torch.ones(V, dtype=torch.bool)
    if top_k > 0:
        keep = s >= torch.topk(s, min(max(top_k, 2), V)).values[-1]
    m = s.max()
    w = torch.where(keep, torch.exp(s - m), torch.zeros_like(s))
    gap = math.inf
    if top_p and top_p < 1.0:
        order = torch.sort(-s, stable=True).indices                       # value desc, index asc
        cum = torch.cumsum(w[order] / w.sum(), 0)
        gap = float((cum - top_p).abs().min())
        over = torch.nonzero(cum > top_p)
        if len(over):
            K = max(int(over[0]), 2) + 1
            ks = torch.zeros(V, dtype=torch.bool)
            ks[order[:K]] = True
            keep &= ks
    w = torch.where(keep, torch.exp(s - m), torch.zeros_like(s))
    toks = []
    for d in range(2):
        p = w.clone()
        for t in toks:
            p[t] = 0.0
        c = torch.cumsum(p / p.sum(), 0)
        nz = p > 0
        gap = min(gap, float((c[nz] - float(u[d])).abs().min()))
        hit = torch.nonzero(c > float(u[d]))
        toks.append(int(hit[0]) if len(hit) else int(torch.nonzero(nz)[-1]))
    lse = torch.log(w.sum())
    scores = [float((s[t] - m) - lse + bs) for t in toks]
    return keep, toks, scores, gap


def op_sample(z, bs, u, T, top_k, top_p):
    lib = _lib.load()
    rows, V = z.shape
    zd, bd, ud = z.cuda().contiguous(), bs.cuda().contiguous(), u.cuda().contiguous()
    cv = torch.empty((rows, 2), dtype=torch.float32, device='cuda')
    ci = torch.empty((rows, 2), dtype=torch.int32, device='cuda')
    kept = torch.empty((rows,), dtype=torch.int32, device='cuda')
    rc = lib.gitb200_op_beam_sample(zd.data_ptr(), rows, V, bd.data_ptr(), ud.data_ptr(), T, top_k, top_p, cv.data_ptr(),
                                    ci.data_ptr(), kept.data_ptr(), None)
    torch.cuda.synchronize()
    return rc, cv.cpu(), ci.cpu().long(), kept.cpu().long()


def _logits(kind, rows, V, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(rows, V, generator=g) * 3.0
    if kind == 'ties':              # many exact ties: at the k-th value and across the top-p boundary
        z = torch.round(z * 2.0) / 2.0
    elif kind == 'flat':            # a few equal maxima and a flat rest: ties straddle the nucleus boundary
        z = torch.zeros(rows, V)
        z[:, :: 97] = 2.0
    elif kind == 'neginf':          # -inf logits (never drawn), fewer finite values than some top_k
        z[:, 40:] = float('-inf')
    elif kind == 'tempties':        # the top logits in pairs one ulp apart, which the division by T = 0.7 often ties
        z = z / 6.0
        a = 1.5 + 0.4 * torch.rand(rows, 8, generator=g)
        z[:, :8] = a
        z[:, 8:16] = torch.from_numpy(np.nextafter(a.numpy(), np.float32(np.inf)))
        assert bool((z[:, :8] / 0.7 == z[:, 8:16] / 0.7).any()) and bool((z[:, :8] != z[:, 8:16]).all())
    return z


KERNEL_CASES = [
    # (kind, V, T, top_k, top_p)
    ('randn', VOCAB, 1.0, 0, 1.0),
    ('randn', VOCAB, 0.7, 50, 1.0),
    ('randn', VOCAB, 1.0, 0, 0.9),
    ('randn', VOCAB, 0.7, 40, 0.8),
    ('randn', VOCAB, 1.3, 0, 0.5),
    ('randn', VOCAB, 1.0, 1, 1.0),              # top_k 1 -> 2
    ('randn', 500, 1.0, 505, 1.0),              # top_k >= V
    ('randn', VOCAB, 1.0, 0, 1e-4),             # tiny top_p: the keep-three rule
    ('randn', VOCAB, 0.7, 0, 1.5),              # top_p >= 1: no nucleus filter
    ('ties', VOCAB, 1.0, 10, 1.0),
    ('ties', VOCAB, 1.0, 0, 0.6),
    ('ties', 2000, 0.7, 30, 0.7),
    ('flat', VOCAB, 1.0, 0, 0.5),
    ('flat', VOCAB, 1.0, 100, 0.3),
    ('neginf', VOCAB, 1.0, 0, 1.0),
    ('neginf', VOCAB, 1.0, 100, 0.9),
    ('tempties', VOCAB, 0.7, 12, 1.0),
    ('tempties', VOCAB, 0.7, 0, 0.2),
]


@pytest.mark.parametrize('case', KERNEL_CASES, ids=['%s-V%d-T%g-k%d-p%g' % c for c in KERNEL_CASES])
def test_kernel_against_fp64(case):
    kind, V, T, top_k, top_p = case
    rows = 24
    z = _logits(kind, rows, V, seed=KERNEL_CASES.index(case))
    g = torch.Generator().manual_seed(7)
    u = torch.rand(rows, 2, generator=g)
    u[0] = 0.0                                                       # u = 0 and u just below 1
    u[1] = float(np.nextafter(np.float32(1.0), np.float32(0.0)))
    bs = torch.randn(rows, generator=g) * 3.0
    bs[2] = -1e9                                                     # the beams the first step starts at -1e9
    rc, cv, ci, kept = op_sample(z, bs, u, T, top_k, top_p)
    assert rc == 0, _lib.last_error()
    compared, worst = 0, 0.0
    for r in range(rows):
        keep, toks, scores, gap = ref_step(z[r], T, top_k, top_p, u[r], float(bs[r]))
        assert ci[r, 0] != ci[r, 1]                                   # without replacement
        assert bool(torch.isfinite(z[r, ci[r]]).all())                # never a removed (-inf) token
        if gap < BOUNDARY:
            continue
        compared += 1
        assert int(kept[r]) == int(keep.sum()), (r, int(kept[r]), int(keep.sum()))
        assert ci[r].tolist() == toks, (r, ci[r].tolist(), toks, gap)
        err = max(abs(float(cv[r, d]) - scores[d]) for d in range(2))
        if bs[r] > -1e8:
            worst = max(worst, err)
            assert err < SCORE_ATOL, (r, err)
        else:
            assert err <= 64.0                                        # one fp32 ulp at 1e9
    print('%s: %d / %d rows compared, max |score - fp64| = %.3g' % (case, compared, rows, worst))
    assert compared >= rows // 2


def test_kernel_ties_are_cut_in_index_order():
    """Ties straddling the nucleus boundary: the engine keeps them lowest index first (torch.sort leaves them unordered)."""
    V = 1000
    z = torch.full((1, V), -5.0)
    z[0, [700, 100, 400, 900]] = 1.0                                  # four equal maxima; keep-three cuts them at three
    rc, _, ci, kept = op_sample(z, torch.zeros(1), torch.tensor([[0.999, 0.999]]), 1.0, 0, 1e-3)
    assert rc == 0 and int(kept[0]) == 3                              # 100, 400, 700 kept; 900 removed
    assert ci[0].tolist() == [700, 400]                               # thirds in index order; then halves of {100, 400}


def test_kernel_reports_fewer_than_two_drawable_tokens():
    V = 1000
    z = torch.full((3, V), float('-inf'))
    z[:, 5] = 0.0
    z[0, 6] = -1.0                                                    # row 0: two tokens; rows 1, 2: one
    z[2, 7] = -300.0                                                  # exp underflows: zero probability
    rc, _, _, _ = op_sample(z, torch.zeros(3), torch.rand(3, 2), 1.0, 0, 1.0)
    assert rc != 0 and 'fewer than two' in _lib.last_error()
    rc, _, ci, _ = op_sample(z[:1], torch.zeros(1), torch.rand(1, 2), 1.0, 0, 1.0)
    assert rc == 0 and sorted(ci[0].tolist()) == [5, 6]


# ---------------------------------------------------------------------------------------------------------------------
# the search
# ---------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(name):
    from generativeimage2text_b200.model import get_git_model
    if name not in _MODELS:
        param = {} if name == 'base' else {'image_encoder_type': 'CLIPViT_L_14', 'visual_feature_size': 1024}
        m = get_git_model(Tok(), param)
        # 'decisive': a handful of live tokens, so sampled captions differ from the deterministic ones and from each other
        missing, unexpected = m.load_state_dict(synthetic_state_dict(param, 1, 'decisive'), strict=False)
        assert not missing and not unexpected
        _MODELS[name] = m.cuda().eval()
    return _MODELS[name]


def _decoder(m, beam, max_steps, T):
    from generativeimage2text_b200.model import GeneratorWithBeamSearch
    m.decoder = GeneratorWithBeamSearch(EOS, max_steps=max_steps, beam_size=beam, length_penalty=0.6)
    m.decoder.temperature = T


def replay(out, u, start, beam, max_steps, T, top_k, top_p):
    """beam_sample_search over the engine's step logits with its uniforms -> (predictions, logprobs, images whose draws and
    top-p cuts all lie >= BOUNDARY from a decision boundary)."""
    z = out['step_logits'].cpu()
    B = start.shape[0]
    clear = torch.ones(B, dtype=torch.bool)
    it = iter(range(z.shape[0]))
    real_filter = bso.top_k_top_p_filter

    def watch_filter(scores, k, p, min_tokens_to_keep=2):
        if p and p < 1.0:
            f = real_filter(scores, k, None)
            srt = torch.sort(-f, dim=-1, stable=True).values
            cum = torch.cumsum(torch.softmax(-srt.double(), dim=-1), dim=-1)
            near = ((cum - p).abs() < BOUNDARY).any(dim=1)
            clear.mul_(~near.view(B, beam).any(dim=1))
        return real_filter(scores, k, p, min_tokens_to_keep)

    def watch_draw(probs, uu):
        words = bso.two_draws(probs, uu)
        for d in range(2):
            p = probs.double()
            if d == 1:
                p = p.scatter(1, words[:, :1], 0.0)
            c = torch.cumsum(p, dim=1) / p.sum(dim=1, keepdim=True)
            gap = torch.where(p > 0, (c - uu[:, d:d + 1].double()).abs(), torch.full_like(c, math.inf)).min(dim=1).values
            clear.mul_(~(gap < BOUNDARY).view(B, beam).any(dim=1))
        return words
    bso.top_k_top_p_filter = watch_filter
    try:
        pred, lp = bso.beam_sample_search(start, lambda ids: z[next(it)], u, max_steps=max_steps, beam=beam,
                                                 temperature=T, top_k=top_k, top_p=top_p, draw=watch_draw)
    finally:
        bso.top_k_top_p_filter = real_filter
    return pred, lp, clear


def _check_replay(out, pred, lp, clear, P=0):
    own, own_lp = out['predictions'].cpu(), out['logprobs'].cpu()
    ref = pred[:, P:] if P else pred
    assert int(clear.sum()) >= max(1, (3 * clear.numel()) // 4), clear.tolist()
    assert torch.equal(own[clear], ref[clear]), (own[clear] != ref[clear]).nonzero().tolist()
    err = float((own_lp[clear] - lp[clear]).abs().max())
    assert err < LOGPROB_ATOL, err
    return err


SEARCH_CASES = [
    # (model, beam, batch, max_steps, T, top_k, top_p)
    ('base', 4, 1, 12, 1.0, 50, None),
    ('base', 4, 3, 12, 0.7, 20, 0.9),
    ('base', 3, 5, 12, 1.0, 0, 0.3),
    ('base', 2, 8, 12, 0.7, 100, 0.5),
    ('base', 2, 2, 10, 1.0, 1, None),
    ('large', 4, 32, 10, 0.7, 40, 0.9),
    ('large', 3, 4, 10, 1.0, 30, None),
]


@pytest.mark.parametrize('case', SEARCH_CASES, ids=['%s-beam%d-B%d-s%d-T%g-k%d-p%s' % c for c in SEARCH_CASES])
def test_search_replays_the_reference_semantics(case):
    name, beam, B, steps, T, top_k, top_p = case
    m = _model(name)
    _decoder(m, beam, steps, T)
    img = synthetic_images(B, 0, seed=31 + B).cuda()
    u = torch.rand((steps, B * beam, 2), generator=torch.Generator().manual_seed(beam * 100 + B))
    out = m({'image': img}, return_step_logits=True, search_param={'do_sample': True, 'top_k': top_k, 'top_p': top_p,
                                                                   'uniforms': u})
    pred, lp, clear = replay(out, u, torch.full((B, 1), 101, dtype=torch.long), beam, steps, T, top_k, top_p)
    err = _check_replay(out, pred, lp, clear)
    print('%s: %d / %d images compared, max |logprob - replay| = %.3g' % (case, int(clear.sum()), B, err))
    plain = m({'image': img})['predictions'].cpu()
    if B >= 3:
        assert not torch.equal(plain, out['predictions'].cpu())        # it does sample


def test_prefix_and_ragged_batches_replay():
    m = _model('base')
    beam, steps, T, top_k, top_p = 3, 12, 0.7, 40, 0.9
    _decoder(m, beam, steps, T)
    # one shared prefix (batch 1)
    prefix = torch.tensor([[101, 2023, 2003]])
    u = torch.rand((steps, beam, 2), generator=torch.Generator().manual_seed(5))
    img = synthetic_images(1, 0, seed=77).cuda()
    out = m({'image': img, 'prefix': prefix.cuda()}, return_step_logits=True,
            search_param={'do_sample': True, 'top_k': top_k, 'top_p': top_p, 'uniforms': u})
    pred, lp, clear = replay(out, u, prefix, beam, steps, T, top_k, top_p)
    _check_replay(out, pred, lp, clear, P=3)
    # a ragged batch: images of their own sizes
    ims = [synthetic_images(1, 0, seed=80 + b, res=hw)[0] for b, hw in enumerate([(224, 224), (160, 288), (288, 192)])]
    u = torch.rand((steps, 3 * beam, 2), generator=torch.Generator().manual_seed(6))
    out = m({'image': [x.cuda() for x in ims]}, return_step_logits=True,
            search_param={'do_sample': True, 'top_k': top_k, 'top_p': top_p, 'uniforms': u})
    pred, lp, clear = replay(out, u, torch.full((3, 1), 101, dtype=torch.long), beam, steps, T, top_k, top_p)
    _check_replay(out, pred, lp, clear)


def test_rows_are_independent_of_the_batch():
    """Row b of a batch (plain or with a prefix per image) is bit-identical to the batch-1 call with image b and its slice
    of the uniforms."""
    m = _model('base')
    beam, steps, T = 4, 12, 0.7
    _decoder(m, beam, steps, T)
    B = 4
    img = synthetic_images(B, 0, seed=41).cuda()
    u = torch.rand((steps, B * beam, 2), generator=torch.Generator().manual_seed(9))
    sp = {'do_sample': True, 'top_k': 30, 'top_p': 0.9}
    full = m({'image': img}, search_param=dict(sp, uniforms=u))
    prefixes = torch.tensor([[101, 2000, 2001], [101, 2002, 0], [101, 0, 0], [101, 2003, 2004]])
    lens = [3, 2, 1, 3]
    pre = m({'image': img, 'prefix': prefixes.cuda(), 'prefix_len': torch.tensor(lens)}, search_param=dict(sp, uniforms=u))
    for b in range(B):
        ub = u[:, b * beam:(b + 1) * beam]
        one = m({'image': img[b:b + 1]}, search_param=dict(sp, uniforms=ub))
        assert torch.equal(one['predictions'].cpu()[0], full['predictions'].cpu()[b])
        assert torch.equal(one['logprobs'].cpu()[0], full['logprobs'].cpu()[b])
        one = m({'image': img[b:b + 1], 'prefix': prefixes[b:b + 1, :lens[b]].cuda()}, search_param=dict(sp, uniforms=ub))
        n = one['predictions'].shape[1]
        assert torch.equal(one['predictions'].cpu()[0], pre['predictions'].cpu()[b, :n])
        assert torch.equal(one['logprobs'].cpu()[0], pre['logprobs'].cpu()[b])


def test_graphs_pdl_and_a_fresh_engine_are_bit_identical():
    m = _model('base')
    beam, steps, T = 4, 14, 1.0
    _decoder(m, beam, steps, T)
    B = 3
    img = synthetic_images(B, 0, seed=51).cuda()
    u = torch.rand((steps, B * beam, 2), generator=torch.Generator().manual_seed(12))
    sp = {'do_sample': True, 'top_k': 0, 'top_p': 0.8, 'uniforms': u}
    want = m({'image': img}, search_param=sp)
    try:
        for g in (0, 1):
            for p in (0, 1):
                m.set_engine_option('use_graph', g)
                m.set_engine_option('use_pdl', p)
                got = m({'image': img}, search_param=sp)
                assert torch.equal(got['predictions'], want['predictions']) and torch.equal(got['logprobs'], want['logprobs'])
    finally:
        m.set_engine_option('use_graph', 1)
        m.set_engine_option('use_pdl', 1)
    m.release()                                                      # a fresh engine
    got = m({'image': img}, search_param=sp)
    assert torch.equal(got['predictions'], want['predictions']) and torch.equal(got['logprobs'], want['logprobs'])


def test_do_sample_false_and_parity_mode():
    m = _model('base')
    beam, steps = 4, 12
    _decoder(m, beam, steps, 0.7)
    img = synthetic_images(3, 0, seed=61).cuda()
    plain = m({'image': img})
    for sp in ({'do_sample': False}, {'do_sample': False, 'top_k': 5, 'top_p': 0.2}):
        got = m({'image': img}, search_param=sp)
        assert torch.equal(got['predictions'], plain['predictions']) and torch.equal(got['logprobs'], plain['logprobs'])
    # parity mode (fp32-grade GEMMs) runs the same search over its own logits
    u = torch.rand((steps, 3 * beam, 2), generator=torch.Generator().manual_seed(14))
    m.set_engine_option('parity', 1)
    try:
        out = m({'image': img}, return_step_logits=True, search_param={'do_sample': True, 'top_k': 50, 'top_p': 0.9,
                                                                       'uniforms': u})
        pred, lp, clear = replay(out, u, torch.full((3, 1), 101, dtype=torch.long), beam, steps, 0.7, 50, 0.9)
        _check_replay(out, pred, lp, clear)
    finally:
        m.set_engine_option('parity', 0)


def test_a_row_without_two_drawable_tokens_is_an_error():
    """A temperature so low that softmax leaves one token of non-zero probability: torch.multinomial(num_samples=2)
    raises in the reference; the engine's generate reports the step and row, and the next call works."""
    m = _model('base')
    _decoder(m, 2, 8, 1e-5)
    img = synthetic_images(1, 0, seed=71).cuda()
    with pytest.raises(RuntimeError, match='step 0, row 0 has fewer than two tokens'):
        m({'image': img}, search_param={'do_sample': True, 'top_k': 0})
    _decoder(m, 2, 8, 1.0)
    out = m({'image': img}, search_param={'do_sample': True, 'top_k': 10})
    assert out['predictions'].shape == (1, 8)
