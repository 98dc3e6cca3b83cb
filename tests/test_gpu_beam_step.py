"""The beam-search decode step -- step_layers reading the text K/V through the src_row indirection table, then
beam_row_topk_kernel and beam_update_kernel -- against an fp64 statement of every step, and its device bookkeeping
checked exactly.

Every generate call dumps its step logits.  `beam_replay` (tests/decode_ref.py) replays the reference's beam search over
them and records each step's beam_idx; `ancestry` turns those into the physical text-cache row that every logical row
reads at every position.  Each step is then recomputed by `ref_step` from the engine's own caches: image K/V of image
r // beam, text K/V gathered along the ancestry (a physical row only ever writes its own position `pos`, so the final
cache holds every step's inputs).  Compared:
  * every step's logits, and the k / v each step appended at txt[layer, k|v, r, pos], all 6 layers;
  * when the run reaches max_steps, the last step's chain buffers ctx, ub (last layer) and x (its output LayerNorm);
  * exactly: src_row (the final ancestry), the token history beam_ids, done / hyp_len, the predictions, and the last
    step's per-row candidate tokens (beam_cand) against an explicit (logit desc, token asc) ranking; within a bound:
    hyp_score, the log-probs and the candidate scores -- which carry the running beam scores of that step -- against
    the fp64 replay (fp64 log-softmax of the dumped fp32 logits, accumulated).  After the run beam_scores hold the
    (0, EOS, row 0) padding of the last step.
Every case asserts that some row reads some position from a physical row other than its own.  Planted defects in the
reference (a GEMM tile, an attention chunk, a key dropped; one position read from the row's own physical row; the wrong
image's K/V; the previous step's ancestry) must move a compared quantity by >= 4x its tolerance.

Tolerances: about 2x the largest error observed over these cases on an H100 80GB HBM3 (700 W power limit), given after
each.  The bf16 quantities differ from the reference by whole bf16 steps (0.0156 = one step at magnitudes 2 .. 4).
"""
import contextlib

import pytest
import torch

from decode_ref import (V, D, EOS, CLS, RefWeights, ref_step, beam_replay, ancestry, src_row_table, gather_text,
                        expand_images, rank_candidates)

TOL = dict(logits=0.08,     # 0.0381
           k=0.032,         # 0.0156: the text cache entry each step appended, every layer
           v=0.032,         # 0.0156
           ctx=0.016,       # 0.00781: attention output of the last layer, bf16 (q stays fp32 on the kernel chain)
           ub=0.032,        # 0.0156: erf-GELU(fc1), bf16
           x=0.019)         # 0.00931: the last layer's output LayerNorm, fp32
SCORE_TOL = 6e-7            # 2.75e-7 at |hyp_score| 1.38: hyp_score, worst_score and the log-prob against the fp64 replay
CAND_TOL = 2e-5             # 8.58e-6: the last step's row candidate scores against fp64 log-softmax + the fp64 beam score
# The done and hypothesis-replace decisions divide by fp32 powf length norms in the engine, by Python doubles in the
# reference: the norm differs by <= ~6e-7 relative (two powf of <= 2 ulp and a division), the scores by the SCORE_TOL above.
# A decision can only flip when its two sides lie within ~1.5e-6 of each other; every case asserts that they do not.
DECISION_GAP = 1e-5         # smallest relative gap seen: 4.42e-3
SENSITIVITY = 4.0
LENGTH_PENALTY = 0.6

MEASURED = {}
SENS = {}


@pytest.fixture(scope='module', autouse=True)
def _report_measured_errors():
    yield
    for name, e in sorted(MEASURED.items()):
        tol = {'score': SCORE_TOL, 'cand': CAND_TOL}.get(name, TOL.get(name))
        print('BMAX %s %.3g (tolerance %.3g)' % (name, e, tol))
    for name, r in sorted(SENS.items()):
        print('BSENS %s %.1f' % (name, r))


def _track(name, err):
    MEASURED[name] = max(MEASURED.get(name, 0.0), err)


class Tok:
    cls_token_id, sep_token_id = CLS, EOS


@pytest.fixture(scope='module')
def sd_perturbed():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    return synthetic_state_dict({}, 1, 'perturbed')


# ---------------------------------------------------------------------------------------------------------------------
# CPU checks of the reference
# ---------------------------------------------------------------------------------------------------------------------
def test_gather_step_without_rounding_is_the_reordering_cached_decoder(sd_perturbed):
    """With rounding off, ref_step over text K/V gathered along the ancestry equals git_oracle.CachedDecoder(beam), which
    physically re-orders its cache, over several re-orderings (including rows of one image that all follow global row 0)."""
    import git_oracle
    sd = sd_perturbed
    W = RefWeights(sd, rounding=False)
    g = torch.Generator().manual_seed(21)
    B, beam, M, steps = 2, 3, 5, 5
    R = B * beam
    feats = torch.randn(B, M, 768, generator=g)
    dec = git_oracle.CachedDecoder(sd, feats, beam=beam)
    img = torch.stack([torch.stack([dec.img_k[j], dec.img_v[j]]) for j in range(6)])
    phys = torch.zeros(6, 2, R, steps, D, dtype=torch.float64)
    bidx_all = [torch.tensor([0, 0, 1, 5, 3, 3]), torch.tensor([2, 1, 0, 4, 4, 5]), torch.tensor([0, 0, 0, 3, 5, 4]),
                torch.tensor([1, 2, 2, 0, 0, 0])]
    anc = ancestry(bidx_all, R)
    toks = torch.randint(1000, 30000, (steps, R), generator=g)
    toks[0] = CLS
    worst = 0.0
    for t in range(steps):
        got = ref_step(W, expand_images(img, beam, 0), expand_images(img, beam, 1), gather_text(phys, anc[t], 0),
                       gather_text(phys, anc[t], 1), toks[t], t)
        want = dec.feed(toks[t][:, None]).double()
        worst = max(worst, (got['logits'] - want).abs().max().item() / want.abs().max().item())
        for j in range(6):
            phys[j, 0, :, t] = got['layers'][j]['k']
            phys[j, 1, :, t] = got['layers'][j]['v']
            assert (got['layers'][j]['k'] - dec.txt_k[j][:, t].double()).abs().max().item() < 1e-5
        if t < len(bidx_all):
            dec.reorder(bidx_all[t])
    assert worst < 1e-5, worst
    assert not torch.equal(anc[steps - 1], torch.arange(R)[:, None].expand(R, steps - 1))


def test_beam_replay_is_the_oracle_beam_search():
    """beam_replay makes the decisions of git_oracle.beam_search (predictions, log-probs, every beam_idx) on logits
    without ties, with and without a strong EOS, at beams 2 .. 4."""
    import git_oracle
    g = torch.Generator().manual_seed(4)
    Vs = 400
    for beam, B, eos_shift, max_steps in ((2, 3, 0.0, 9), (3, 2, 3.0, 12), (4, 3, 2.0, 10), (4, 1, 0.0, 7)):
        R = B * beam
        z = torch.randn(max_steps, R, Vs, generator=g) * 2
        z[:, :, EOS] += eos_shift
        it = iter(range(max_steps))
        seen = []
        pred, lp = git_oracle.beam_search(torch.full((B, 1), CLS, dtype=torch.long), lambda ids: z[next(it)],
                                          reorder=seen.append, max_steps=max_steps, beam=beam,
                                          length_penalty=LENGTH_PENALTY)
        rep = beam_replay(z, B, beam, max_steps, LENGTH_PENALTY)
        assert torch.equal(rep['pred'], pred)
        assert torch.equal(rep['logprobs'], lp[:, 0])
        assert len(rep['bidx']) == len(seen) == rep['n_steps']
        for a, b in zip(rep['bidx'], seen):
            assert torch.equal(a, b)
        assert ((rep['hyp_score64'] - rep['hyp_score'].double()).abs() < 1e-4).all()


def test_ranking_keeps_logit_order_where_fp32_scores_collapse():
    """Token 1256 one ulp above token 1000: log_softmax + a beam score rounds both to one fp32 value at large scores.
    The ranking keeps them in logit order (the order of the exact scores), exact logit ties go to the lower token."""
    Vs = 2000
    z = torch.zeros(1, Vs)
    z[0, 7] = 140.0
    z[0, 1256] = 40.0
    z[0, 1000] = torch.nextafter(torch.tensor(40.0), torch.tensor(0.0))
    for bs, collapsed in ((0.0, True), (-150.0, True)):
        sc = torch.log_softmax(z, dim=-1) + bs
        assert bool(sc[0, 1000] == sc[0, 1256]) == collapsed
        assert rank_candidates(sc, z, Vs, 3).tolist() == [[7, 1256, 1000]]
    z[0, 1000] = 40.0
    sc = torch.log_softmax(z, dim=-1)
    assert rank_candidates(sc, z, Vs, 3).tolist() == [[7, 1000, 1256]]
    assert rank_candidates(sc, z, Vs, 3, ties='high').tolist() == [[7, 1256, 1000]]


def test_ancestry_defects_change_only_what_they_name():
    g = torch.Generator().manual_seed(9)
    R, beam, t = 6, 3, 4
    txt = torch.randn(6, 2, R, 8, D, generator=g, dtype=torch.float64)
    img = torch.randn(6, 2, 2, 5, D, generator=g, dtype=torch.float64)
    anc = ancestry([torch.tensor([1, 1, 0, 4, 3, 3])] * t, R)[t]
    base = gather_text(txt, anc, 0)
    r, j = 0, 2
    assert int(anc[r, j]) != r
    own = gather_text(txt, anc, 0, defect=('own_row', r, j))
    for L in range(6):
        diff = (own[L] != base[L]).any(-1).nonzero().tolist()
        assert diff == [[r, j]]
    a, b = expand_images(img, beam, 0), expand_images(img, beam, 0, shift=1)
    assert torch.equal(a[0][:3], img[0, 0, 0].expand(3, -1, -1)) and torch.equal(b[0][:3], img[0, 0, 1].expand(3, -1, -1))
    assert torch.equal(src_row_table(anc, 8)[:, :t], anc)
    assert torch.equal(src_row_table(anc, 8)[:, t:], torch.arange(R)[:, None].expand(R, 8 - t))


# ---------------------------------------------------------------------------------------------------------------------
# GPU plumbing
# ---------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(param, sd_key, sd):
    from generativeimage2text_b200.model import get_git_model
    key = (repr(sorted(param.items())), sd_key)
    if key not in _MODELS:
        m = get_git_model(Tok(), param)
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not missing and not unexpected
        _MODELS[key] = m.cuda().eval()
    return _MODELS[key]


def _beam(m, beam, max_steps):
    from generativeimage2text_b200.model import GeneratorWithBeamSearch
    m.decoder = GeneratorWithBeamSearch(EOS, max_steps=max_steps, beam_size=beam, length_penalty=LENGTH_PENALTY)


def _read(m, name, dtype):
    """One of the engine's buffers, caches or beam bookkeeping arrays (gitb200_debug_read), as a flat tensor."""
    from generativeimage2text_b200 import _lib
    lib = _lib.load()
    buf = torch.empty(1 << 31, dtype=torch.uint8)
    n = lib.gitb200_debug_read(m._engine, name.encode(), buf.data_ptr(), buf.numel())
    assert n > 0, 'debug_read(%s) failed' % name
    return buf[:n].view(dtype).clone()


def _caches(m, B, R):
    """(image K/V [6, 2, B, M, 768], text K/V [6, 2, R, T_alloc, 768]) as fp64 on the GPU."""
    img = _read(m, 'img_kv', torch.bfloat16).cuda().double()
    txt = _read(m, 'txt_kv', torch.bfloat16).cuda().double()
    return img.reshape(6, 2, B, -1, D), txt.reshape(6, 2, R, -1, D)


@contextlib.contextmanager
def _patched(m, sd, edits):
    """Parameters of m changed in place for the duration ({key: (index, value)}); yields the edited state dict."""
    params = m.state_dict(keep_vars=True)
    sd2, saved = dict(sd), []
    with torch.no_grad():
        for key, (idx, val) in edits.items():
            p = params[key]
            saved.append((p, idx, p[idx].clone()))
            p[idx] = val.to(p.device) if torch.is_tensor(val) else val
            t = sd2[key].clone()
            t[idx] = val
            sd2[key] = t
    if 'textual.embedding.words.weight' in edits:
        sd2['textual.output.weight'] = sd2['textual.embedding.words.weight']
    try:
        yield sd2
    finally:
        with torch.no_grad():
            for p, idx, old in saved:
                p[idx] = old


def _no_eos(sd):
    """EOS far below every other logit: every image runs to max_steps."""
    return {'textual.output.bias': (EOS, float(sd['textual.output.bias'][EOS]) - 100.0)}


def _generate(m, images, batch_extra=None):
    batch = {'image': images}
    if batch_extra:
        batch.update(batch_extra)
    out = m(batch, return_step_logits=True)
    torch.cuda.synchronize()
    return out


def _merge(parts):
    """ref_step results of consecutive row groups as one."""
    out = {'logits': torch.cat([p['logits'] for p in parts])}
    out['layers'] = [{k: torch.cat([p['layers'][j][k] for p in parts]) for k in parts[0]['layers'][j]}
                     for j in range(len(parts[0]['layers']))]
    return out


def _ref(W, img, txt, beam, anc_t, tokens, t, lens=None, defect=None, shift=0, own=None):
    """ref_step for all R rows at step t: image K/V of image r // beam (+ shift), text K/V along anc_t.  lens: the image
    token count of each image (a ragged batch: each image's rows are computed over its own keys)."""
    img_k, img_v = expand_images(img, beam, 0, shift), expand_images(img, beam, 1, shift)
    txt_k, txt_v = gather_text(txt, anc_t, 0, own), gather_text(txt, anc_t, 1, own)
    tokens = tokens.to(img.device)
    if lens is None:
        return ref_step(W, img_k, img_v, txt_k, txt_v, tokens, t, q_bf16=False, defect=defect)
    parts = []
    for b, L in enumerate(lens):
        rs = slice(b * beam, b * beam + beam)
        parts.append(ref_step(W, [k[rs, :L] for k in img_k], [v[rs, :L] for v in img_v], [k[rs] for k in txt_k],
                              [v[rs] for v in txt_v], tokens[rs], t, q_bf16=False, defect=defect))
    return _merge(parts)


def _errors(ref, z_t, txt, t, last=None):
    """max |engine - ref| per compared quantity at step t (last: the chain buffers to compare, or None)."""
    e = {'logits': (z_t - ref['logits']).abs().max().item()}
    for j in range(6):
        for kv, name in ((0, 'k'), (1, 'v')):
            e[name] = max(e.get(name, 0.0), (txt[j, kv, :, t] - ref['layers'][j][name]).abs().max().item())
    if last is not None:
        L = ref['layers'][5]
        for name, got in last.items():
            e[name] = (got - L[name]).abs().max().item()
    return e


def _ratio(d, ref, quantities):
    """How far a defect moves the compared quantities, in tolerances."""
    r = (d['logits'] - ref['logits']).abs().max().item() / TOL['logits']
    for j in range(6):
        for name in ('k', 'v'):
            r = max(r, (d['layers'][j][name] - ref['layers'][j][name]).abs().max().item() / TOL[name])
    for name in quantities:
        r = max(r, (d['layers'][5][name] - ref['layers'][5][name]).abs().max().item() / TOL[name])
    return r


def _tokens_fed(rep, t, R, beam, prefix=None):
    if t > 0:
        return rep['words'][t - 1]
    if prefix is not None:
        return prefix[torch.arange(R) // beam, 0]
    return torch.full((R,), CLS, dtype=torch.long)


def _check_candidates(m, z_t, cand64_t, beam, label):
    """The last step's per-row candidate lists (debug name beam_cand): the top 2 * beam tokens of the row's dumped logits
    ranked by (logit desc, token asc), scores non-increasing and within CAND_TOL of the fp64 log-softmax + fp64 beam score
    (rows still at the initial -1e9 are checked for order only).  Returns (values, tokens) [R, 2 * beam]."""
    R = z_t.shape[0]
    NC = 2 * beam
    raw = _read(m, 'beam_cand', torch.int32).reshape(2, R, -1)
    val, idx = raw[0].view(torch.float32)[:, :NC], raw[1][:, :NC].long()
    want = rank_candidates(z_t.float(), z_t.float(), z_t.shape[1], NC)
    assert torch.equal(idx, want), (label, 'row candidate lists', idx, want)
    assert (val[:, :-1] >= val[:, 1:]).all(), label
    live = cand64_t > -1e8
    ref = torch.log_softmax(z_t.double(), dim=-1).gather(1, idx) + cand64_t[:, None]
    e = (val.double() - ref)[live].abs().max().item() if live.any() else 0.0
    _track('cand', e)
    assert e <= CAND_TOL, (label, 'candidate scores', e)
    return val, idx


def _check_beam_run(m, W, B, beam, max_steps, out, label, lens=None, prefix=None, prefix_lens=None, sensitivity=(),
                    exempt=()):
    """Replay, ancestry, per-step numerics, exact bookkeeping and (sensitivity: defect names to assert) planted defects."""
    R = B * beam
    z = out['step_logits'].cpu()
    rep = beam_replay(z, B, beam, max_steps, LENGTH_PENALTY, prefix=prefix, prefix_lens=prefix_lens)
    n = rep['n_steps']
    assert not z[n:].any(), 'the engine ran steps past the replay\'s end'
    anc = ancestry(rep['bidx'], R)
    ident = torch.arange(R)[:, None]
    read_foreign = [t for t in range(n) if (anc[t] != ident).any()]
    assert read_foreign, (label, 'no row ever read a position from another physical row')
    img, txt = _caches(m, B, R)
    full = n == max_steps - 1
    last = None
    if full:
        last = {'ctx': _read(m, 'ctx', torch.bfloat16).cuda().double().reshape(R, D),
                'ub': _read(m, 'ub', torch.bfloat16).cuda().double().reshape(R, -1),
                'x': _read(m, 'x', torch.float32).cuda().double().reshape(R, D)}
    err = {}
    zc = z[:n].cuda().double()
    ref = None
    for t in range(n):
        toks = _tokens_fed(rep, t, R, beam, prefix)
        ref = _ref(W, img, txt, beam, anc[t], toks, t, lens)
        for k, e in _errors(ref, zc[t], txt, t, last if t == n - 1 else None).items():
            err[k] = max(err.get(k, 0.0), e)
    for k, e in err.items():
        _track(k, e)
    print('BSTEP %s n=%d foreign=%d %s' % (label, n, len(read_foreign), ' '.join('%s=%.3g' % kv for kv in sorted(err.items()))))
    for k, e in err.items():
        assert e <= TOL[k], (label, k, e, TOL[k])

    # ---- exact bookkeeping
    T_alloc = _read(m, 'src_row', torch.int32).numel() // R
    src = _read(m, 'src_row', torch.int32).reshape(R, T_alloc).long()
    assert torch.equal(src, src_row_table(anc[n], T_alloc)), label
    ids = _read(m, 'beam_ids', torch.int64).reshape(R, max_steps)
    assert torch.equal(ids[:, :n + 1], rep['ids'][:, :n + 1]), label
    # the running beam scores are consumed by the last step's candidate scores (checked there); after the run they hold
    # the (0, EOS, row 0) padding of the last step
    _check_candidates(m, z[n - 1], rep['cand64'][n - 1], beam, label)
    assert not _read(m, 'beam_scores', torch.float32).any(), label
    print('BGAP %s %.3g' % (label, rep['gap']))
    assert rep['gap'] > DECISION_GAP, (label, 'a done / replace decision too close to call in fp32', rep['gap'])
    hyp = _read(m, 'beam_hyp', torch.int32).reshape(4, B)
    assert torch.equal(hyp[0].long(), rep['done']), label
    assert torch.equal(hyp[1].long(), rep['hyp_len']), label
    hyp_score = hyp[2].view(torch.float32)
    pred, lp = out['predictions'].cpu(), out['logprobs'].cpu().reshape(-1)
    if prefix_lens is None:
        assert torch.equal(pred, rep['pred']), label
    else:
        for b, pl in enumerate(prefix_lens):
            assert torch.equal(pred[b, :max_steps - pl], rep['pred'][b, pl:]), (label, b)
    assert torch.equal(lp, hyp_score), label
    e = (hyp_score.double() - rep['hyp_score64']).abs().max().item()
    e = max(e, (hyp[3].view(torch.float32).double() - rep['worst']).abs().max().item())
    _track('score', e)
    print('BSCORE %s |hyp_score| <= %.3g err %.3g' % (label, rep['hyp_score64'].abs().max().item(), e))
    assert e <= SCORE_TOL, (label, e)

    # ---- planted defects at the last step that read a foreign row
    if sensitivity:
        # the last step whose rows were re-ordered by the step before: every planted ancestry defect changes a read there
        t = max(u for u in read_foreign if u > 0 and not torch.equal(rep['bidx'][u - 1], ident[:, 0]))
        toks = _tokens_fed(rep, t, R, beam, prefix)
        ref = _ref(W, img, txt, beam, anc[t], toks, t, lens)
        r, j = [int(x) for x in (anc[t] != ident).nonzero()[-1]]
        prev = torch.cat([anc[t - 1], ident], dim=1) if t > 0 else anc[t]
        planted = {'wo': dict(defect=('wo', 37)), 'w1': dict(defect=('w1', 200)), 'fc2': dict(defect=('fc2', (17, 3), 4)),
                   'lm': dict(defect=('lm', 500)), 'chunk': dict(defect=('chunk', 0)),
                   'img_last': dict(defect=('img_last', 0)), 'newest': dict(defect=('newest', 0)),
                   'own_row': dict(own=('own_row', r, j)), 'wrong_image': dict(shift=1), 'prev_ancestry': dict(anc=prev)}
        ratios = {}
        for name, kw in planted.items():
            if name not in sensitivity:
                continue
            a = kw.pop('anc', anc[t])
            d = _ref(W, img, txt, beam, a, toks, t, lens, **kw)
            ratios[name] = _ratio(d, ref, ('ctx', 'ub', 'x'))
            SENS[name] = max(SENS.get(name, 0.0), ratios[name])
        print('BSENS %s t=%d %s' % (label, t, ' '.join('%s=%.1f' % kv for kv in sorted(ratios.items()))))
        for name, rt in ratios.items():
            if name not in exempt:
                assert rt >= SENSITIVITY, (label, name, rt)
    return rep


ALL_DEFECTS = ('wo', 'w1', 'fc2', 'lm', 'chunk', 'img_last', 'newest', 'own_row', 'wrong_image', 'prev_ancestry')
# one key carries about 1 / (M + pos) of a row's attention weight: the single-key defects (one key dropped, one position
# read from another row) are only asserted at M = 2
MANY_KEYS = ('img_last', 'newest', 'own_row', 'prev_ancestry')

# (id, B, beam, (height, width), max_steps, defects, exempt)
CASES = [
    ('b1_k2_m2', 1, 2, (16, 16), 10, tuple(d for d in ALL_DEFECTS if d != 'wrong_image'), ()),
    ('b2_k3_m2', 2, 3, (16, 16), 8, ALL_DEFECTS, ()),
    ('b2_k3_m197', 2, 3, (224, 224), 10, ALL_DEFECTS, MANY_KEYS),
    ('b5_k4_m65', 5, 4, (128, 128), 10, ALL_DEFECTS, MANY_KEYS),
    ('b16_k4_m197', 16, 4, (224, 224), 6, (), ()),
    ('b32_k4_m257', 32, 4, (256, 256), 5, (), ()),
    ('b32_k2_m65', 32, 2, (128, 128), 5, (), ()),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_beam_step_against_fp64_reference(case, sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    label, B, beam, hw, max_steps, defects, exempt = case
    m = _model({}, 'perturbed1', sd_perturbed)
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 300 + B * beam, hw).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        W = RefWeights(sd).to('cuda')
        _check_beam_run(m, W, B, beam, max_steps, out, label, sensitivity=defects, exempt=exempt)


@pytest.mark.gpu
def test_beam_step_vatex_1182_keys():
    """Six 224x224 frames per image (1182 image keys) at beam 4."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    param = {'num_image_with_embedding': 6}
    sd = synthetic_state_dict(param, 2, 'perturbed')
    m = _model(param, 'vatex2', sd)
    B, beam, max_steps = 3, 4, 5
    _beam(m, beam, max_steps)
    frames = [f.cuda() for f in synthetic_images(B, 6, 4321)]
    with _patched(m, sd, _no_eos(sd)) as sd2:
        out = _generate(m, frames)
        _check_beam_run(m, RefWeights(sd2).to('cuda'), B, beam, max_steps, out, 'vatex_b3_k4_m1182')


@pytest.mark.gpu
def test_beam_step_ragged_batch(sd_perturbed):
    """Images of their own sizes in one call: row r attends over the L_b valid keys of its image only."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 3, 3, 8
    _beam(m, beam, max_steps)
    hws = [(128, 128), (224, 224), (160, 96)]
    images = [synthetic_images(1, 0, 40 + b, hw)[0].cuda() for b, hw in enumerate(hws)]
    lens = [(h // 16) * (w // 16) + 1 for h, w in hws]
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'ragged_b3_k3', lens=lens,
                        sensitivity=('wrong_image', 'prev_ancestry'))


@pytest.mark.gpu
def test_beam_step_per_image_prefixes(sd_perturbed):
    """Per-image prefixes: an image inside its prefix feeds the next prefix token on every beam and keeps its scores
    (beam_update_kernel's in_prefix branch) while the other images search."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 3, 3, 10
    _beam(m, beam, max_steps)
    lens = [1, 4, 2]
    prefix = torch.randint(1000, 30000, (B, 4), generator=torch.Generator().manual_seed(8))
    prefix[:, 0] = CLS
    images = synthetic_images(B, 0, 31, (128, 128)).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images, {'prefix': prefix.cuda(), 'prefix_len': torch.tensor(lens)})
        _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'prefix_b3_k3', prefix=prefix,
                        prefix_lens=lens)


@pytest.mark.gpu
def test_beam_step_images_finish_at_different_steps(sd_perturbed):
    """EOS raised until hypotheses complete: images are found done at different steps, and from then on their rows are
    padded with (0, EOS, global row 0) and read row 0's history."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 8, 3, 24
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 77, (128, 128)).cuda()
    base = float(sd_perturbed['textual.output.bias'][EOS])
    # the token just fed scores about +41 before the bias (the tied embedding), so EOS competes only near that
    for shift in [30.0 + i for i in range(21)]:
        with _patched(m, sd_perturbed, {'textual.output.bias': (EOS, base + shift)}) as sd:
            out = _generate(m, images)
            rep = beam_replay(out['step_logits'].cpu(), B, beam, max_steps, LENGTH_PENALTY)
            steps = sorted(set(rep['done_step']))
            if len(steps) >= 2 and any(s >= 0 and s < rep['n_steps'] - 1 for s in steps):
                print('BEOS shift %.0f done_step %s n_steps %d' % (shift, rep['done_step'], rep['n_steps']))
                _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'eos_b8_k3')
                return
    pytest.fail('no EOS bias made the images finish at different steps')


@pytest.mark.gpu
def test_beam_step_across_the_text_cache_growth(sd_perturbed):
    """150 steps: the text cache and both indirection tables are re-laid out from 128 to 149 positions mid-run, the
    2-step graph is captured again, and every step before and after must still read its own ancestry."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 2, 2, 150
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 12, (128, 128)).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        rep = _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'grow_b2_k2_150')
    anc = ancestry(rep['bidx'], B * beam)[rep['n_steps']]
    assert (anc[:, 128:] != torch.arange(B * beam)[:, None]).any(), 'no foreign read past the growth'


# ---------------------------------------------------------------------------------------------------------------------
# The raw decode_step API: reorder_src_row_kernel driven by the replayed beam_idx
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_raw_decode_step_api_follows_beam_idx(sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 2, 3, 12
    R = B * beam
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 51, (128, 128)).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        rep = beam_replay(out['step_logits'].cpu(), B, beam, max_steps, LENGTH_PENALTY)
        n = rep['n_steps']
        m.encode_image(images)
        m.prefill(B, beam=beam)
        zs = []
        for t in range(n):
            zs.append(m.decoding_step(_tokens_fed(rep, t, R, beam), t,
                                      beam_idx=rep['bidx'][t - 1] if t > 0 else None).cpu())
        torch.cuda.synchronize()
        anc = ancestry(rep['bidx'], R)
        src = _read(m, 'src_row', torch.int32).reshape(R, -1).long()
        assert torch.equal(src, src_row_table(anc[n - 1], src.shape[1]))
        img, txt = _caches(m, B, R)
        W = RefWeights(sd).to('cuda')
        err = {}
        for t in range(n):
            ref = _ref(W, img, txt, beam, anc[t], _tokens_fed(rep, t, R, beam), t)
            for k, e in _errors(ref, zs[t].cuda().double(), txt, t).items():
                err[k] = max(err.get(k, 0.0), e)
        same = max((zs[t] - out['step_logits'][t].cpu()).abs().max().item() for t in range(n))
        print('BRAW %s |raw - generate| %.3g' % (' '.join('%s=%.3g' % kv for kv in sorted(err.items())), same))
        assert same == 0.0, 'the raw decode_step API and generate ran the same steps to different logits'
        for k, e in err.items():
            _track(k, e)
            assert e <= TOL[k], (k, e)


# ---------------------------------------------------------------------------------------------------------------------
# Bit identity
# ---------------------------------------------------------------------------------------------------------------------
def _outputs(out):
    return {k: out[k].clone() for k in ('predictions', 'logprobs', 'step_logits')}


@pytest.mark.gpu
def test_graph_and_pdl_are_bit_identical_across_growth(sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 3, 4, 140
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 19, (128, 128)).cuda()
    runs = {}
    try:
        with _patched(m, sd_perturbed, _no_eos(sd_perturbed)):
            for g in (1, 0):
                for p in (1, 0):
                    m.set_engine_option('use_graph', g)
                    m.set_engine_option('use_pdl', p)
                    runs[(g, p)] = _outputs(_generate(m, images))
    finally:
        m.set_engine_option('use_graph', 1)
        m.set_engine_option('use_pdl', 1)
    for key, o in runs.items():
        for k in o:
            assert torch.equal(o[k], runs[(1, 1)][k]), (key, k)


@pytest.mark.gpu
def test_warm_engine_matches_a_fresh_one(sd_perturbed):
    """A greedy call and a beam call of another size first: the case is bit-identical to the same case on a fresh engine."""
    from generativeimage2text_b200.model import AutoRegressiveBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    img = synthetic_images(4, 0, 70, (128, 128)).cuda()
    m.decoder = AutoRegressiveBeamSearch(EOS, max_steps=30, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    _generate(m, synthetic_images(9, 0, 71, (224, 224)).cuda())
    _beam(m, 2, 140)
    _generate(m, synthetic_images(7, 0, 72, (128, 128)).cuda())
    _beam(m, 4, 20)
    warm = _outputs(_generate(m, img))
    m.release()
    fresh = _outputs(_generate(m, img))
    for k in warm:
        assert torch.equal(warm[k], fresh[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# Planted ties in beam_row_topk_kernel
# ---------------------------------------------------------------------------------------------------------------------
# (id, a, b, lifted): tokens a < b get a zero word-embedding row and the same LM bias, so both logits are exactly 40.0;
# `lifted` further zero-row tokens with biases 41, 42, ... sit above them in every row's list.  Each row's candidate list
# (debug name beam_cand) is compared with an explicit (logit desc, token asc) ranking; where the pair also decides a beam
# (every placement but the straddle, whose pair never reaches the kept beams) the outputs must follow the lower token.
#   one_thread: b = a + 256, one thread's consecutive loads;  warps: different warps of one round;
#   rounds: b = a + 2048, one thread's two rounds;  straddle: the pair at places 2 * beam - 1 / 2 * beam of the list.
def _tie_cases(beam):
    lift = list(range(5000, 5000 + 2 * beam - 1))
    return [('one_thread', 1000, 1256, lift[:beam - 1]), ('warps', 1000, 1100, lift[:beam - 1]),
            ('rounds', 3000, 5048, lift[:beam - 1]), ('straddle', 1000, 1256, lift)]


@pytest.mark.gpu
@pytest.mark.parametrize('beam', [2, 4])
@pytest.mark.parametrize('which', ['one_thread', 'warps', 'rounds', 'straddle'])
def test_planted_ties_keep_the_lower_index(which, beam, sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    _, a, b, lifted = [c for c in _tie_cases(beam) if c[0] == which][0]
    m = _model({}, 'perturbed1', sd_perturbed)
    B, max_steps = 2, 6
    _beam(m, beam, max_steps)
    toks = [a, b] + lifted
    bias = torch.tensor([40.0, 40.0] + [41.0 + i for i in range(len(lifted))])
    edits = {'textual.embedding.words.weight': (toks, 0.0), 'textual.output.bias': (toks, bias)}
    with _patched(m, sd_perturbed, edits):
        out = _generate(m, synthetic_images(B, 0, 55, (128, 128)).cuda())
    z = out['step_logits'].cpu()
    rep = beam_replay(z, B, beam, max_steps, LENGTH_PENALTY)
    assert (z[:rep['n_steps'], :, [a, b]] == 40.0).all()
    assert torch.equal(out['predictions'].cpu(), rep['pred'])
    ids = _read(m, 'beam_ids', torch.int64).reshape(B * beam, max_steps)
    n = rep['n_steps']
    assert torch.equal(ids[:, :n + 1], rep['ids'][:, :n + 1])
    val, idx = _check_candidates(m, z[n - 1], rep['cand64'][n - 1], beam, which)
    if which == 'straddle':
        # the pair sits at the cut of every row's list: the lower token is its last entry, the higher one is left out
        assert (idx[:, -1] == a).all() and not (idx == b).any()
    else:
        assert ((idx == a).nonzero()[:, 1] < (idx == b).nonzero()[:, 1]).all()
    flipped = beam_replay(z, B, beam, max_steps, LENGTH_PENALTY, ties='high')
    decisive = any(not torch.equal(x, y) for x, y in zip(flipped['words'] + flipped['bidx'], rep['words'] + rep['bidx']))
    print('BTIE %s beam %d decisive %s' % (which, beam, decisive))
    if which != 'straddle':
        assert decisive, 'the planted tie does not decide any beam'


@pytest.mark.gpu
@pytest.mark.parametrize('beam', [2, 4])
def test_one_ulp_pair_keeps_logit_order_where_scores_collapse(beam, sd_perturbed):
    """Token 1256 at logit 40, token 1000 one ulp below, token 7 at 140 (zero word-embedding rows, so the logits are the
    biases exactly).  (z - max) rounds both of the pair to -100, so their scores are equal in fp32 on every row.  The
    rows keep them in logit order -- the order of their exact scores -- so the second beam of step 0 continues with 1256,
    and the replay ranks the same way."""
    from generativeimage2text_b200.synthetic import synthetic_images
    a, b, top = 1000, 1256, 7
    m = _model({}, 'perturbed1', sd_perturbed)
    B, max_steps = 2, 4
    _beam(m, beam, max_steps)
    low = float(torch.nextafter(torch.tensor(40.0), torch.tensor(0.0)))
    edits = {'textual.embedding.words.weight': ([a, b, top], 0.0),
             'textual.output.bias': ([a, b, top], torch.tensor([low, 40.0, 140.0]))}
    with _patched(m, sd_perturbed, edits):
        out = _generate(m, synthetic_images(B, 0, 56, (128, 128)).cuda())
    z = out['step_logits'].cpu()
    rep = beam_replay(z, B, beam, max_steps, LENGTH_PENALTY)
    n = rep['n_steps']
    assert (z[:n, :, a] == low).all() and (z[:n, :, b] == 40.0).all()
    val, idx = _check_candidates(m, z[n - 1], rep['cand64'][n - 1], beam, 'ulp')
    pa, pb = (idx == a).nonzero(), (idx == b).nonzero()
    assert torch.equal(pa[:, 0], pb[:, 0]) and (pb[:, 1] + 1 == pa[:, 1]).all()
    assert (val.gather(1, pa[:, 1:]) == val.gather(1, pb[:, 1:])).all()      # equal scores, logit order
    assert torch.equal(out['predictions'].cpu(), rep['pred'])
    ids = _read(m, 'beam_ids', torch.int64).reshape(B * beam, max_steps)
    assert torch.equal(ids[:, :n + 1], rep['ids'][:, :n + 1])
    assert (rep['words'][0].view(B, beam)[:, 1] == b).all(), 'the second beam of step 0 should continue with %d' % b
