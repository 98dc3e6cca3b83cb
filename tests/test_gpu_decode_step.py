"""The greedy decode step -- the persistent decode_mega_kernel (<= 64 rows, use_mega = 1) and the kernel chain of
step_layers + greedy_select_kernel (use_mega = 0) -- against an fp64 statement of one step, phase by phase.

`ref_step` computes one step from the engine's OWN image and text K/V caches (read back with gitb200_debug_read), so the
encoder and the earlier steps drop out of the comparison and every step is measured on its own.  It rounds to bf16 exactly
where both paths store bf16 (weights, the GEMM operand copy of the residual stream, q / 8, the new k and v, the attention
context, the GELU output) and computes everything else in fp64.

Each GPU case runs with forced tokens that are never EOS, so every step runs, and compares
  * every step's logits, and the k / v the step appended to the text cache, with ref_step;
  * at the last step, the per-phase buffers each path writes (q, context, pre-LayerNorm sum, GELU output, residual);
  * the next step's embedding that the persistent kernel leaves in x / hb;
and checks the selection EXACTLY against the dumped logits (no-repeat mask, lowest index on ties, fp64 log-softmax).
The same step with one defect planted in the reference (a GEMM tile, an attention chunk or a key dropped) must move the
compared quantity by >= 4x its tolerance, so the tolerances are shown to be able to fail.

Exact invariants: planted ties across the LM-head slice boundaries of both paths, logits far below 0 (the padded LM-head
columns must never be chosen), row isolation, a warm engine against a fresh one, the step-logits hook, and a C-ABI
parity-mode -> default-mode sequence on one engine.
"""
import contextlib
import ctypes

import pytest
import torch

import git_oracle
from decode_ref import V, D, EOS, CLS, bf16, RefWeights, ref_step, expected_selection

# Largest |engine - ref_step| per path and compared quantity: about 2x the largest error observed over these cases on an
# H100 80GB HBM3 (132 SMs, 700 W power limit), given after each.  The bf16 quantities differ from the reference by whole
# bf16 steps where the two round a value near a rounding boundary to neighbouring bf16 numbers (0.0156 = one step at
# magnitudes 2 .. 4).
TOL = {
    'mega': dict(logits=0.08,    # 0.0389
                 k=0.032,        # 0.0156: the text cache entry the step appended, every layer
                 v=0.032,        # 0.0156
                 qb=0.004,       # 0.00195: q / 8, bf16
                 ctx=0.016,      # 0.00781: attention output, bf16
                 y=0.021,        # 0.0104: residual + attention output projection, fp32
                 ub=0.032,       # 0.0156: erf-GELU(fc1), bf16
                 emb=1.5e-6),    # 7.46e-7: the next step's embedding LN(words[next] + positions[pos + 1]), fp32
    'chain': dict(logits=0.07,   # 0.0342
                  k=0.032,       # 0.0156
                  v=0.032,       # 0.0156
                  ctx=0.008,     # 0.00391 (q stays fp32 on this path)
                  ub=0.032,      # 0.0156
                  x=0.018),      # 0.00893: the last layer's output LayerNorm, fp32
}
LOGPROB_TOL = 2e-6          # engine log-prob against the fp64 log-softmax of its own dumped logits; 8.64e-7 observed
SENSITIVITY = 4.0           # a planted defect must move a compared quantity by this many tolerances
# Cases where a single key (the last image key, the newest text key) carries enough softmax weight to be seen at the
# context tolerance.  With 64 or more image keys one key holds ~1 / (M + pos) of the weight and moves the context by
# less than 4x the tolerance (0.3x - 2.5x measured at M = 64 / 65), so there it is only reported.
SINGLE_KEY_CASES = ('r1_m2',)

MEASURED = {'mega': {}, 'chain': {}}


@pytest.fixture(scope='module', autouse=True)
def _report_measured_errors():
    """After the module: the largest error seen per path and quantity, next to its tolerance (run pytest with -s)."""
    yield
    for path in ('mega', 'chain'):
        for name, e in sorted(MEASURED[path].items()):
            tol = LOGPROB_TOL if name == 'logprob' else TOL[path][name]
            print('DMAX %s %s %.3g (tolerance %.3g)' % (path, name, e, tol))


class Tok:
    cls_token_id, sep_token_id = CLS, EOS


# ---------------------------------------------------------------------------------------------------------------------
# CPU checks of the reference itself
# ---------------------------------------------------------------------------------------------------------------------
def test_bf16_helper_matches_torch():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(100000, generator=g, dtype=torch.float64) * torch.logspace(-30, 30, 100000, dtype=torch.float64)
    # values exactly halfway between two bf16 numbers (ties to even) and their neighbours
    base = torch.randn(4096, generator=g).to(torch.bfloat16).float()
    half = (base.view(torch.int32) | 0x8000).view(torch.float32).double()
    x = torch.cat([x, half, torch.nextafter(half, half * 2), torch.nextafter(half, half * 0), torch.zeros(1)])
    ref = x.to(torch.float32).to(torch.bfloat16).to(torch.float64)
    assert torch.equal(bf16(x), ref)


@pytest.fixture(scope='module')
def sd_perturbed():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    return synthetic_state_dict({}, 1, 'perturbed')


def test_ref_step_without_rounding_is_the_cached_decoder(sd_perturbed):
    """With rounding off, ref_step is the oracle's KV-cached step (git_oracle.CachedDecoder.feed) on the same fp32 inputs."""
    sd = sd_perturbed
    W = RefWeights(sd, rounding=False)
    g = torch.Generator().manual_seed(11)
    feats = torch.randn(3, 5, 768, generator=g)
    dec = git_oracle.CachedDecoder(sd, feats)
    toks = torch.randint(1000, 30000, (3, 4), generator=g)
    toks[:, 0] = CLS
    worst = 0.0
    for pos in range(toks.shape[1]):
        txt_k = [dec.txt_k[j].clone() for j in range(6)]
        txt_v = [dec.txt_v[j].clone() for j in range(6)]
        want = dec.feed(toks[:, pos:pos + 1]).double()
        got = ref_step(W, dec.img_k, dec.img_v, txt_k, txt_v, toks[:, pos], pos)
        scale = want.abs().max().item()
        worst = max(worst, (got['logits'] - want).abs().max().item() / scale)
        for j in range(6):      # the k / v the step appends are the cache entries at pos
            assert (got['layers'][j]['k'] - dec.txt_k[j][:, pos].double()).abs().max().item() < 1e-5
            assert (got['layers'][j]['v'] - dec.txt_v[j][:, pos].double()).abs().max().item() < 1e-5
    assert worst < 1e-5, worst


def test_ref_step_defects_are_planted_where_named(sd_perturbed):
    """Each defect changes exactly the quantities it names and nothing upstream of them."""
    W = RefWeights(sd_perturbed)
    g = torch.Generator().manual_seed(5)
    R, M, pos = 2, 70, 3
    img_k = [torch.randn(R, M, D, generator=g) for _ in range(6)]
    img_v = [torch.randn(R, M, D, generator=g) for _ in range(6)]
    txt_k = [torch.randn(R, pos, D, generator=g) for _ in range(6)]
    txt_v = [torch.randn(R, pos, D, generator=g) for _ in range(6)]
    toks = torch.tensor([2000, 3000])
    base = ref_step(W, img_k, img_v, txt_k, txt_v, toks, pos, n_layers=2)
    for defect, same, moved in ((('wo', 5), 'ctx', 'y'), (('w1', 7), 'y', 'ub'), (('fc2', (3, 2)), 'ub', 'x'),
                                (('chunk', 0), 'qb', 'ctx'), (('img_last', 0), 'k', 'ctx'), (('newest', 0), 'v', 'ctx')):
        d = ref_step(W, img_k, img_v, txt_k, txt_v, toks, pos, n_layers=2, defect=defect)
        assert torch.equal(d['layers'][0]['x'], base['layers'][0]['x'])           # layer 0 is untouched
        assert torch.equal(d['layers'][1][same], base['layers'][1][same])
        assert not torch.equal(d['layers'][1][moved], base['layers'][1][moved])
    d = ref_step(W, img_k, img_v, txt_k, txt_v, toks, pos, n_layers=2, defect=('lm', 3815))
    diff = (d['logits'] != base['logits']).nonzero()[:, 1].unique()
    assert diff.tolist() == list(range(30520, 30522))


# ---------------------------------------------------------------------------------------------------------------------
# GPU plumbing
# ---------------------------------------------------------------------------------------------------------------------
def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _paths():
    return [pytest.param(1, id='mega'), pytest.param(0, id='chain')]


def _need_path(use_mega):
    if use_mega and _num_sms() < 128:
        pytest.skip('decode_mega_kernel needs >= 128 SMs (this device has %d)' % _num_sms())


_MODELS = {}


def _model(param, sd_key, sd):
    """One model per (checkpoint, geometry), kept for the module."""
    from generativeimage2text_b200.model import get_git_model
    key = (repr(sorted(param.items())), sd_key)
    if key not in _MODELS:
        m = get_git_model(Tok(), param)
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not missing and not unexpected
        _MODELS[key] = m.cuda().eval()
    return _MODELS[key]


def _greedy(m, max_steps):
    from generativeimage2text_b200.model import AutoRegressiveBeamSearch
    m.decoder = AutoRegressiveBeamSearch(EOS, max_steps=max_steps, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)


def _read(m, name, rows=None):
    """A decode-step buffer or cache of the model's engine (gitb200_debug_read) as a torch tensor."""
    from generativeimage2text_b200 import _lib
    lib = _lib.load()
    eng = m._engine
    sizes = {'x': (4, D), 'y': (4, D), 'hb': (2, D), 'ctx': (2, D), 'qb': (2, D), 'ub': (2, 3072)}
    if name in sizes:
        eb, width = sizes[name]
        cap = rows * width * eb
    else:
        cap = 1 << 31
    buf = torch.empty(cap, dtype=torch.uint8)
    n = lib.gitb200_debug_read(eng, name.encode(), buf.data_ptr(), cap)
    assert n > 0, 'debug_read(%s) failed' % name
    raw = buf[:n]
    if name in ('x', 'y'):
        return raw.view(torch.float32).reshape(rows, D).clone()
    if name in sizes:
        return raw.view(torch.bfloat16).reshape(rows, -1).clone()
    return raw.view(torch.bfloat16).clone()


def _caches(m, R):
    """(image K/V [6, 2, R, M, 768], text K/V [6, 2, R, T_alloc, 768]), bf16, as the engine holds them."""
    img = _read(m, 'img_kv')
    txt = _read(m, 'txt_kv')
    return img.reshape(6, 2, R, -1, D), txt.reshape(6, 2, R, -1, D)


@contextlib.contextmanager
def _patched(m, sd, edits):
    """Parameters of model m changed in place for the duration ({state-dict key: (index, value)}); yields the state dict with
    the same edits (CPU copy) for the reference.  The engine re-uploads the weights when they change."""
    params = m.state_dict(keep_vars=True)
    sd2, saved = dict(sd), []
    with torch.no_grad():
        for key, (idx, val) in edits.items():
            p = params[key]
            saved.append((p, idx, p[idx].clone()))
            p[idx] = val
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


_REF_W = {}


def _ref_weights(sd_key, sd):
    if sd_key not in _REF_W:
        _REF_W[sd_key] = RefWeights(sd)
    return _REF_W[sd_key]


def _track(path, name, err):
    MEASURED[path][name] = max(MEASURED[path].get(name, 0.0), err)
    return err


def _forced(R, max_steps, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randint(1000, 30000, (R, max_steps), generator=g)
    f[:, 0] = CLS
    return f


# ---------------------------------------------------------------------------------------------------------------------
# The case matrix: rows R, image keys M (from the input size), positions pos = 0 .. steps - 1
# ---------------------------------------------------------------------------------------------------------------------
# (id, R, (height, width), max_steps, debug_layers, sensitivity)
#   R: row tiles of 16 and their r0 / r0 + 8 halves; 12 R around G = 132 attention items (R = 11: one item per CTA, 12:
#      one more); 64 = kMegaMaxRows, whose 768 items put kMegaAttItems = 6 on the busiest CTA.
#   M: 2 (16x16), 64 (112x144: one whole chunk), 65 (128x128), 129 (128x256), 197 (224x224), 577 (384x384).
#   positions: every case starts at 0; 'pos66' runs to 65 (the 64-position box boundary), 'pos130' to 129 (the text cache
#      grows past 128 positions).
CASES = [
    ('r1_m2', 1, (16, 16), 6, -1, True),
    ('r2_m64_pos66', 2, (112, 144), 67, -1, True),
    ('r8_m65', 8, (128, 128), 5, -1, True),
    ('r8_m65_l1', 8, (128, 128), 4, 1, False),
    ('r9_m129', 9, (128, 256), 4, -1, False),
    ('r11_m197', 11, (224, 224), 4, -1, False),
    ('r12_m577', 12, (384, 384), 3, -1, False),
    ('r16_m197_l1', 16, (224, 224), 3, 1, False),
    ('r17_m65', 17, (128, 128), 3, -1, False),
    ('r33_m64', 33, (112, 144), 3, -1, False),
    ('r63_m197', 63, (224, 224), 3, -1, False),
    ('r64_m197', 64, (224, 224), 3, -1, False),
    ('r3_m65_pos130', 3, (128, 128), 131, -1, False),
]


def _check_run(path, m, W, R, tokens_in, first, out, n_layers, q_bf16, sensitivity, label, prefix_lens=None):
    """Compare one generate call (step logits, caches, buffers, selection, log-prob) with ref_step and the exact rules."""
    z = out['step_logits'].cpu()
    n_steps = z.shape[0]
    img, txt = _caches(m, R)
    img_k = [img[j, 0] for j in range(6)]
    img_v = [img[j, 1] for j in range(6)]
    tol = TOL[path]
    err = {}
    ref = None
    for t in range(n_steps):
        txt_k = [txt[j, 0, :, :t] for j in range(6)]
        txt_v = [txt[j, 1, :, :t] for j in range(6)]
        ref = ref_step(W, img_k, img_v, txt_k, txt_v, tokens_in[:, t], t, n_layers=n_layers, q_bf16=q_bf16)
        e = (z[t].double() - ref['logits']).abs().max().item()
        err['logits'] = max(err.get('logits', 0.0), e)
        for j in range(n_layers):
            for kv, name in ((0, 'k'), (1, 'v')):
                e = (txt[j, kv, :, t].double() - ref['layers'][j][name]).abs().max().item()
                err[name] = max(err.get(name, 0.0), e)
    # the last step's phase buffers (the last layer run)
    last = ref['layers'][n_layers - 1]
    bufs = ('qb', 'ctx', 'y', 'ub') if path == 'mega' else ('ctx', 'ub', 'x')
    for name in bufs:
        got = _read(m, name, R).double()
        err[name] = (got - last[name]).abs().max().item()
    if path == 'mega':
        # the next step's input embedding: LN(words[next] + positions[pos + 1])
        nxt = tokens_in[:, n_steps] if tokens_in.shape[1] > n_steps else None
        if nxt is not None:
            emb = W.embed(nxt, n_steps)
            err['emb'] = (_read(m, 'x', R).double() - emb).abs().max().item()
            hb = _read(m, 'hb', R).double()
            assert torch.equal(hb, bf16(_read(m, 'x', R))), label
    for name, e in err.items():
        _track(path, name, e)
    print('DSTEP %s %s %s' % (path, label, ' '.join('%s=%.3g' % kv for kv in sorted(err.items()))))
    for name, e in err.items():
        assert e <= tol[name], (label, path, name, e, tol[name])
    # exact selection against the dumped logits
    tokens_out = out['tokens_full']
    lp_sum = torch.zeros(R, dtype=torch.float64)
    for t in range(n_steps):
        tok, lp = expected_selection(z[t], tokens_in[:, t], first[:, t])
        for r in range(R):
            if prefix_lens is not None and t + 1 < prefix_lens[r]:
                continue                                  # still feeding the row's prefix
            assert int(tokens_out[r, t + 1]) == int(tok[r]), (label, path, t, r)
            lp_sum[r] += lp[r]
    P = torch.ones(R, dtype=torch.long) if prefix_lens is None else torch.tensor(prefix_lens)
    nv = (tokens_out != EOS).sum(1) + (tokens_out == EOS).any(1).long() - P
    want = lp_sum / nv.clamp(min=1).double()
    e = (out['logprobs'].cpu().double() - want).abs().max().item()
    _track(path, 'logprob', e)
    assert e <= LOGPROB_TOL, (label, path, e)
    if sensitivity:
        _check_sensitivity(path, W, img_k, img_v, txt, tokens_in, n_steps - 1, n_layers, q_bf16, ref, label)


def _check_sensitivity(path, W, img_k, img_v, txt, tokens_in, t, n_layers, q_bf16, ref, label):
    """The last step again with one planted defect: at least one quantity the path compares must move by >= SENSITIVITY x
    its tolerance (logits per row; the phase buffers of the last layer per row, the context per (row, head))."""
    txt_k = [txt[j, 0, :, :t] for j in range(6)]
    txt_v = [txt[j, 1, :, :t] for j in range(6)]
    tol = TOL[path]
    phases = ('qb', 'ctx', 'y', 'ub') if path == 'mega' else ('ctx', 'ub', 'x')
    # fc2 goes into the layer before the last: the persistent kernel leaves no buffer of the last layer's fc2 output
    # (it overwrites x with the next embedding), the residual carries the defect into the last layer's buffers
    defects = [('wo', 37), ('w1', 200), ('fc2', (17, 3), max(0, n_layers - 2)), ('lm', 500), ('lm', (V + 7) // 8 - 1),
               ('chunk', 0), ('img_last', 0), ('newest', 0)]
    ratios = {}
    for defect in defects:
        d = ref_step(W, img_k, img_v, txt_k, txt_v, tokens_in[:, t], t, n_layers=n_layers, q_bf16=q_bf16, defect=defect)
        r = (d['logits'] - ref['logits']).abs().max().item() / tol['logits']
        for name in phases:
            r = max(r, (d['layers'][-1][name] - ref['layers'][-1][name]).abs().max().item() / tol[name])
        ratios['%s_%s' % defect[:2]] = r
    print('DSENS %s %s %s' % (path, label, ' '.join('%s=%.1f' % kv for kv in sorted(ratios.items()))))
    for name, r in ratios.items():
        if name.startswith(('img_last', 'newest')) and label not in SINGLE_KEY_CASES:
            continue
        assert r >= SENSITIVITY, (label, path, name, r)


def _run(m, use_mega, images, forced=None, batch_extra=None):
    m.set_engine_option('use_mega', use_mega)
    batch = {'image': images}
    if batch_extra:
        batch.update(batch_extra)
    out = m(batch, forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    _, _, one = m.last_decode_timing()
    assert one == bool(use_mega), 'the %s path did not run' % ('one-kernel' if use_mega else 'chain')
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_decode_step_against_fp64_reference(case, use_mega, sd_perturbed):
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_images
    label, R, hw, max_steps, n_dbg, sens = case
    path = 'mega' if use_mega else 'chain'
    m = _model({}, 'perturbed1', sd_perturbed)
    m.set_engine_option('debug_layers', n_dbg)
    try:
        _greedy(m, max_steps)
        images = synthetic_images(R, 0, 700 + R, hw).cuda()
        forced = _forced(R, max_steps, 900 + R)
        out = _run(m, use_mega, images, forced)
        out['tokens_full'] = out['predictions'].cpu()
        assert out['tokens_full'].shape == (R, max_steps)
        first = torch.zeros(R, max_steps - 1, dtype=torch.bool)
        first[:, 0] = True
        n_layers = 6 if n_dbg < 0 else n_dbg
        _check_run(path, m, _ref_weights('perturbed1', sd_perturbed), R, forced, first, out, n_layers,
                   q_bf16=bool(use_mega), sensitivity=sens, label=label)
    finally:
        m.set_engine_option('debug_layers', -1)


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
def test_decode_step_vatex_1182_keys(use_mega):
    """Six 224x224 frames per row (1182 image keys, 19 chunks) at 16 rows: the VATEX geometry of the benchmark."""
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    param = {'num_image_with_embedding': 6}
    sd = synthetic_state_dict(param, 2, 'perturbed')
    m = _model(param, 'vatex2', sd)
    R, max_steps = 16, 3
    _greedy(m, max_steps)
    frames = [f.cuda() for f in synthetic_images(R, 6, 4321)]
    forced = _forced(R, max_steps, 77)
    out = _run(m, use_mega, frames, forced)
    out['tokens_full'] = out['predictions'].cpu()
    first = torch.zeros(R, max_steps - 1, dtype=torch.bool)
    first[:, 0] = True
    path = 'mega' if use_mega else 'chain'
    _check_run(path, m, RefWeights(sd), R, forced, first, out, 6, q_bf16=bool(use_mega), sensitivity=False,
               label='vatex_r16_m1182')


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
def test_decode_step_per_row_prefixes(use_mega, sd_perturbed):
    """Rows with prefixes of their own lengths: the row-specific first decision (no no-repeat mask) and prefix feeding."""
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    R, max_steps = 4, 8
    _greedy(m, max_steps)
    lens = [1, 3, 2, 4]
    prefix = torch.randint(1000, 30000, (R, 4), generator=torch.Generator().manual_seed(8))
    prefix[:, 0] = CLS
    images = synthetic_images(R, 0, 31, (128, 128)).cuda()
    eos_bias = float(sd_perturbed['textual.output.bias'][EOS]) - 100.0      # free running without EOS: every step runs
    with _patched(m, sd_perturbed, {'textual.output.bias': (EOS, eos_bias)}) as sd:
        out = _run(m, use_mega, images, batch_extra={'prefix': prefix.cuda(), 'prefix_len': torch.tensor(lens)})
        pred = out['predictions'].cpu()
        full = torch.full((R, max_steps), EOS, dtype=torch.long)
        for r, pl in enumerate(lens):
            full[r, :pl] = prefix[r, :pl]
            full[r, pl:] = pred[r, :max_steps - pl]
        assert not (full == EOS).any()
        out['tokens_full'] = full
        first = torch.zeros(R, max_steps - 1, dtype=torch.bool)
        for r, pl in enumerate(lens):
            first[r, pl - 1] = True
        path = 'mega' if use_mega else 'chain'
        _check_run(path, m, RefWeights(sd), R, full, first, out, 6, q_bf16=bool(use_mega), sensitivity=False,
                   label='prefix_r4', prefix_lens=lens)


# ---------------------------------------------------------------------------------------------------------------------
# Exact checks
# ---------------------------------------------------------------------------------------------------------------------
def _tie_pairs():
    G = 132
    lm_per = ((V + 7) // 8 + G - 1) // G * 8            # columns of one CTA's LM-head slice in decode_mega_kernel
    sel = (V + 7) // 8                                   # columns of one of greedy_select_kernel's 8 slices
    return [('mega_slice', lm_per - 1, lm_per), ('select_slice', sel - 1, sel), ('quad_lanes', 800, 802),
            ('one_thread', 1000, 1001), ('last_tile', V - 2, V - 1)]


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
@pytest.mark.parametrize('pair', _tie_pairs(), ids=[p[0] for p in _tie_pairs()])
def test_planted_exact_ties(pair, use_mega, sd_perturbed):
    """Two columns with zero word embeddings and an LM bias of +40: both logits are exactly 40.0.  Free running, the lower
    index wins the first step and the no-repeat mask makes the tokens alternate -- exactly as the oracle's greedy loop
    replays them over the dumped logits."""
    _need_path(use_mega)
    if pair[0] == 'mega_slice' and _num_sms() != 132:
        pytest.skip('the slice boundary is computed for 132 CTAs')
    from generativeimage2text_b200.synthetic import synthetic_images
    _, a, b = pair
    m = _model({}, 'perturbed1', sd_perturbed)
    R, max_steps = 2, 7
    _greedy(m, max_steps)
    edits = {'textual.embedding.words.weight': ([a, b], 0.0), 'textual.output.bias': ([a, b], 40.0)}
    with _patched(m, sd_perturbed, edits):
        out = _run(m, use_mega, synthetic_images(R, 0, 55, (128, 128)).cuda())
    z = out['step_logits'].cpu()
    assert (z[:, :, [a, b]] == 40.0).all()
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.greedy_search(torch.full((R, 1), CLS, dtype=torch.long), lambda partial: z[next(it)].double(),
                                        max_steps=max_steps)
    got = out['predictions'].cpu()
    assert torch.equal(pred, got)
    want = torch.tensor([a, b] * max_steps)[:max_steps - 1]
    assert torch.equal(got[:, 1:], want.expand(R, -1))
    assert (out['logprobs'].cpu().double() - lp).abs().max().item() <= LOGPROB_TOL


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
def test_logits_far_below_zero_never_pick_padding(use_mega, sd_perturbed):
    """LM bias -100 everywhere: every real logit is far below the 0.0 a padded LM-head column (30522 .. 30527) would
    score.  Those columns must never be chosen nor enter the log-sum-exp.  (Not -30: with the tied embedding the logit of
    the token just fed reaches about +41 before the bias.)"""
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    R, max_steps = 5, 6
    _greedy(m, max_steps)
    with _patched(m, sd_perturbed, {'textual.output.bias': (slice(None), -100.0)}):
        out = _run(m, use_mega, synthetic_images(R, 0, 56, (128, 128)).cuda())
    z = out['step_logits'].cpu()
    assert z.max().item() < -20.0
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.greedy_search(torch.full((R, 1), CLS, dtype=torch.long), lambda partial: z[next(it)].double(),
                                        max_steps=max_steps)
    got = out['predictions'].cpu()
    assert int(got.max()) < V
    assert torch.equal(pred, got)
    e = (out['logprobs'].cpu().double() - lp).abs().max().item()
    _track('mega' if use_mega else 'chain', 'logprob', e)
    assert e <= LOGPROB_TOL


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
def test_rows_are_isolated(use_mega, sd_perturbed):
    """Row r's step logits do not depend on the other rows' images and tokens (same row count: the same dealing of tiles
    and attention items over the CTAs), bit for bit."""
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    R, r, max_steps = 9, 4, 5
    _greedy(m, max_steps)
    img_a = synthetic_images(R, 0, 60, (128, 128))
    img_b = synthetic_images(R, 0, 61, (128, 128))
    img_b[r] = img_a[r]
    f_a, f_b = _forced(R, max_steps, 62), _forced(R, max_steps, 63)
    f_b[r] = f_a[r]
    za = _run(m, use_mega, img_a.cuda(), f_a)['step_logits'][:, r].clone()
    zb = _run(m, use_mega, img_b.cuda(), f_b)['step_logits'][:, r].clone()
    assert torch.equal(za, zb)


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
def test_warm_engine_matches_a_fresh_one(use_mega, sd_perturbed):
    """A longer call first (the text cache grows, later positions hold its K/V), then the case: bit-identical to the same
    case on a fresh engine -- no read of a stale cache position or of an earlier call's K/V."""
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    R = 6
    img = synthetic_images(R, 0, 70, (128, 128)).cuda()
    forced = _forced(R, 10, 71)
    _greedy(m, 140)
    _run(m, use_mega, synthetic_images(R, 0, 72, (128, 128)).cuda(), _forced(R, 140, 73))
    _greedy(m, 10)
    warm = _run(m, use_mega, img, forced)
    warm = {k: v.clone() for k, v in warm.items()}
    m.release()
    fresh = _run(m, use_mega, img, forced)
    for k in ('predictions', 'logprobs', 'step_logits'):
        assert torch.equal(warm[k], fresh[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('use_mega', _paths())
def test_step_logits_hook_changes_nothing(use_mega, sd_perturbed):
    _need_path(use_mega)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    _greedy(m, 12)
    img = synthetic_images(7, 0, 80, (224, 224)).cuda()
    m.set_engine_option('use_mega', use_mega)
    a = m({'image': img}, return_step_logits=True)
    b = m({'image': img})
    torch.cuda.synchronize()
    assert torch.equal(a['predictions'], b['predictions'])
    assert torch.equal(a['logprobs'], b['logprobs'])


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: parity mode, then default mode, on one engine
# ---------------------------------------------------------------------------------------------------------------------
def _abi_engine(lib, m, sd, parity):
    from generativeimage2text_b200 import _lib
    h = ctypes.c_void_p()
    _lib.check(lib.gitb200_create(ctypes.byref(m._cfg), 0, ctypes.byref(h)), None, 'create')
    _abi_weights(lib, h, sd, parity)
    return h


def _abi_weights(lib, h, sd, parity):
    from generativeimage2text_b200 import _lib
    _lib.check(lib.gitb200_set_option(h, b'parity', parity), h, 'set_option')
    keep = []
    for key, t in sd.items():
        t = t.cuda().float().contiguous()
        keep.append(t)
        shape = (ctypes.c_int64 * t.dim())(*t.shape)
        _lib.check(lib.gitb200_set_weight(h, key.encode(), t.data_ptr(), shape, t.dim(), _lib.F32, None), h, 'set_weight')
    _lib.check(lib.gitb200_finalize_weights(h, None), h, 'finalize_weights')


def _abi_generate(lib, h, img, max_steps):
    from generativeimage2text_b200 import _lib
    B = img.shape[0]
    sp = _lib.Search(mode=_lib.SEARCH_GREEDY, max_steps=max_steps, beam_size=1, per_node_beam=1, length_penalty=1.0)
    tok = torch.empty((B, max_steps), dtype=torch.long, device='cuda')
    lp = torch.empty((B,), dtype=torch.float32, device='cuda')
    n = ctypes.c_int32(0)
    _lib.check(lib.gitb200_generate(h, img.data_ptr(), B, 0, None, 0, ctypes.byref(sp), None, tok.data_ptr(), lp.data_ptr(),
                                    ctypes.byref(n), None, None), h, 'generate')
    torch.cuda.synchronize()
    return tok[:, :n.value].cpu(), lp.cpu()


@pytest.mark.gpu
def test_parity_then_default_mode_on_one_engine(sd_perturbed):
    """A C-ABI caller switches parity on (fp32 K/V in the text cache), generates, switches it off and generates again with
    <= 64 rows.  The one-kernel step reads whole 64-position boxes of the text cache and gives the positions past the
    caption probability 0, so they must hold finite bf16 values, not the fp32 bytes of the parity call: the outputs must be
    finite and bit-identical to those of an engine that never ran in parity mode."""
    from generativeimage2text_b200 import _lib
    from generativeimage2text_b200.synthetic import synthetic_images
    lib = _lib.load()
    m = _model({}, 'perturbed1', sd_perturbed)
    img = synthetic_images(3, 0, 90).cuda()
    h = _abi_engine(lib, m, sd_perturbed, 1)
    fresh = _abi_engine(lib, m, sd_perturbed, 0)
    try:
        _abi_generate(lib, h, img, 20)
        _abi_weights(lib, h, sd_perturbed, 0)
        tok, lp = _abi_generate(lib, h, img, 20)
        tok0, lp0 = _abi_generate(lib, fresh, img, 20)
        assert torch.isfinite(lp).all(), lp
        assert torch.equal(tok, tok0)
        assert torch.equal(lp, lp0)
    finally:
        lib.gitb200_destroy(h)
        lib.gitb200_destroy(fresh)


