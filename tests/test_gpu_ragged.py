"""GPU: ragged batches -- B single images of their own sizes in one engine call (`batch['image']` = a list of [3, H_b, W_b]
tensors).  Row b must be what the same image returns alone: checked exactly against the uniform engine path and against
sub-batches, and within the usual tolerances against the reference (tests/golden/base_ragged_*.npz hold one reference call
per image, since the reference cannot batch mixed sizes)."""
import base64
import io
import json

import numpy as np
import pytest
import torch

import git_oracle
from helpers import load_golden

pytestmark = pytest.mark.gpu

LOGIT_ATOL = {'init': 0.06, 'perturbed': 0.25}
PARITY_ATOL = 1e-3
RATIO = {'test_crop_size': 160, 'test_respect_ratio_max': 224}


class Tok:
    cls_token_id, sep_token_id = 101, 102

    def __call__(self, text, **kw):
        return {'input_ids': [1000 + (sum(map(ord, w)) * 7919) % 28000 for w in text.split()]}

    def decode(self, ids, skip_special_tokens=True):
        return ' '.join(str(i) for i in ids if not (skip_special_tokens and i in (0, 101, 102)))


def _model(param, sd, search, max_steps, use_mega=None, parity=False):
    from generativeimage2text_b200.model import get_git_model, AutoRegressiveBeamSearch, GeneratorWithBeamSearch
    m = get_git_model(Tok(), param)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    m = m.cuda().eval()
    if search == 'greedy':
        m.decoder = AutoRegressiveBeamSearch(102, max_steps=max_steps, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    else:
        m.decoder = GeneratorWithBeamSearch(102, max_steps=max_steps, beam_size=4, length_penalty=0.6)
    if use_mega is not None:
        m.set_engine_option('use_mega', use_mega)
    if parity:
        m.set_engine_option('parity', 1)
    return m


def _images(hws, seed):
    from generativeimage2text_b200.synthetic import synthetic_images
    return [synthetic_images(1, 0, seed + b, hw)[0] for b, hw in enumerate(hws)]


def _same_row(a, b):
    """Two caption rows equal up to trailing EOS padding (the width of a batch's result follows its longest row)."""
    w = min(a.numel(), b.numel())
    return torch.equal(a[:w], b[:w]) and bool((a[w:] == 102).all()) and bool((b[w:] == 102).all())


# ---- 1. the ragged machinery adds no arithmetic ------------------------------------------------------------------------
@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_same_size_ragged_list_is_bit_identical_to_a_tensor(search):
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    sd = synthetic_state_dict({}, 0, 'perturbed')
    m = _model({}, sd, search, 12, use_mega=0)
    x = synthetic_images(3, 0, 4242).cuda()
    a = m({'image': x}, return_step_logits=True)
    b = m({'image': [x[i] for i in range(3)]}, return_step_logits=True)
    torch.cuda.synchronize()
    assert torch.equal(a['predictions'], b['predictions'])
    assert torch.equal(a['logprobs'], b['logprobs'])
    assert torch.equal(a['step_logits'], b['step_logits'])


# ---- 2. composition invariance -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_ragged_rows_do_not_depend_on_the_other_images(search):
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    sd = synthetic_state_dict(RATIO, 0, 'perturbed')
    m = _model(RATIO, sd, search, 12, use_mega=0)
    imgs = [im.cuda() for im in _images([[160, 208], [208, 160], [160, 160], [160, 224], [176, 192]], 900)]
    full = m({'image': imgs})
    torch.cuda.synchronize()
    assert full['predictions'].shape[0] == 5
    for rows in ([0, 1], [1, 2], [3, 4], [4, 0], [2, 3]):
        sub = m({'image': [imgs[r] for r in rows]})
        for i, r in enumerate(rows):
            assert _same_row(full['predictions'][r], sub['predictions'][i]), (search, rows, r)
            assert torch.equal(full['logprobs'].reshape(-1)[r], sub['logprobs'].reshape(-1)[i]), (search, rows, r)


# ---- 3. against the reference, default mode ----------------------------------------------------------------------------
def _golden_images(g):
    meta = g['meta']
    return _images(meta['image_hws'], meta['img_seed'])


def test_ragged_teacher_forced_logits_against_reference():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    g = load_golden('base_ragged_greedy')
    meta = g['meta']
    sd = synthetic_state_dict(meta['param'], meta['seed'], meta['variant'])
    imgs = _golden_images(g)
    m = _model(meta['param'], sd, 'greedy', meta['max_steps'])
    feats = m.encode_image([im.cuda() for im in imgs])
    for b, f in enumerate(feats):
        np.testing.assert_allclose(f.cpu()[:, ::17, ::29].numpy(), g['feats_sample_%d' % b], rtol=0, atol=0.15)
    forced = torch.full((len(imgs), meta['max_steps']), 102, dtype=torch.long)
    for b in range(len(imgs)):
        p = torch.from_numpy(g['predictions_%d' % b])[0]
        forced[b, :p.numel()] = p
    out = m({'image': [im.cuda() for im in imgs]}, forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    cols = torch.from_numpy(g['vocab_cols'])
    atol = LOGIT_ATOL[meta['variant']]
    worst = 0.0
    for b in range(len(imgs)):
        ref = g['step_logits_%d' % b]
        for i in range(ref.shape[0]):
            worst = max(worst, float(np.abs(z[i][b, cols].numpy() - ref[i][0]).max()))
    print('ragged teacher-forced: max |logit - reference| at the sampled columns %.4f (atol %.2f)' % (worst, atol))
    assert worst < atol


# ---- 4. against the reference, parity mode -----------------------------------------------------------------------------
def test_ragged_parity_mode_greedy_against_the_fp32_reference():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    g = load_golden('base_ragged_greedy')
    meta = g['meta']
    sd = synthetic_state_dict(meta['param'], meta['seed'], meta['variant'])
    imgs = _golden_images(g)
    m = _model(meta['param'], sd, 'greedy', meta['max_steps'], parity=True)
    forced = torch.full((len(imgs), meta['max_steps']), 102, dtype=torch.long)
    raws = []
    for b, im in enumerate(imgs):
        raw = []
        ref = git_oracle.generate(sd, meta['param'], {'image': im[None]}, 'greedy', meta['max_steps'], cached=True, raw_trace=raw)
        assert np.array_equal(ref['predictions'].numpy(), g['predictions_%d' % b])     # oracle == reference
        forced[b, :ref['predictions'].shape[1]] = ref['predictions'][0]
        raws.append(raw)
    out = m({'image': [im.cuda() for im in imgs]}, forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    worst = max((z[i][b] - r[0]).abs().max().item() for b, raw in enumerate(raws) for i, r in enumerate(raw))
    print('ragged [parity] greedy: max |logit - oracle| %.2e' % worst)
    assert worst < PARITY_ATOL
    free = m({'image': [im.cuda() for im in imgs]})
    torch.cuda.synchronize()
    for b in range(len(imgs)):
        assert _same_row(free['predictions'][b].cpu(), torch.from_numpy(g['predictions_%d' % b])[0]), b


def test_ragged_parity_mode_beam_against_the_fp32_reference():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    g = load_golden('base_ragged_beam')
    meta = g['meta']
    sd = synthetic_state_dict(meta['param'], meta['seed'], meta['variant'])
    imgs = _golden_images(g)
    m = _model(meta['param'], sd, 'beam', meta['max_steps'], parity=True)
    out = m({'image': [im.cuda() for im in imgs]}, return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    worst = 0.0
    for b, im in enumerate(imgs):
        raw = []
        git_oracle.generate(sd, meta['param'], {'image': im[None]}, 'greedy', 2, cached=True, raw_trace=raw)
        worst = max(worst, (z[0][4 * b:4 * b + 4] - raw[0]).abs().max().item())     # first step: every beam row = [sos]
        assert torch.equal(out['predictions'][b].cpu(), torch.from_numpy(g['predictions_%d' % b])[0]), b
        np.testing.assert_allclose(out['logprobs'].cpu().reshape(-1)[b].item(), g['logprobs_%d' % b].reshape(-1)[0], rtol=0, atol=2e-3)
    print('ragged [parity] beam: first-step max |logit - oracle| %.2e' % worst)
    assert worst < PARITY_ATOL


# ---- 5. the VQA geometry -----------------------------------------------------------------------------------------------
def test_vqa_geometry_features_and_question_batches():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    param = {'test_crop_size': 480, 'test_respect_ratio_max': 640}
    sd = synthetic_state_dict(param, 0, 'perturbed')
    imgs = _images([[480, 640], [640, 480], [480, 480]], 31)
    m = _model(param, sd, 'beam', 10)
    feats = m.encode_image([im.cuda() for im in imgs])
    assert [f.shape[1] for f in feats] == [1201, 1201, 901]
    for b, im in enumerate(imgs):
        ref = git_oracle.visual_features(sd, param, im[None])
        err = (feats[b].cpu() - ref).abs()
        print('vqa image %d: features max %.4f mean %.5f' % (b, err.max(), err.mean()))
        assert err.mean().item() < 0.01 and err.max().item() < 0.15
    questions = [[[101, 2054, 2003], [101, 2129, 2116, 2111, 2024]], [[101, 2054, 2003, 2023], [101, 3585]],
                 [[101, 2054], [101, 2129, 2003, 1996, 2154]]]

    def pad(ps):
        t = torch.zeros((len(ps), max(len(p) for p in ps)), dtype=torch.long)
        for r, p in enumerate(ps):
            t[r, :len(p)] = torch.tensor(p)
        return {'prefix': t.cuda(), 'prefix_len': torch.tensor([len(p) for p in ps])}
    rows = [p for ps in questions for p in ps]
    ragged = m(dict(image=[im.cuda() for im in imgs for _ in range(2)], **pad(rows)))
    torch.cuda.synchronize()
    for b, (im, ps) in enumerate(zip(imgs, questions)):
        one = m(dict(image=im[None].cuda().expand(2, -1, -1, -1), **pad(ps)))
        for i in range(2):
            assert _same_row(ragged['predictions'][2 * b + i], one['predictions'][i]), (b, i)
            assert torch.equal(ragged['logprobs'].reshape(-1)[2 * b + i], one['logprobs'].reshape(-1)[i]), (b, i)


# ---- 6. the TSV driver -------------------------------------------------------------------------------------------------
def _png_b64(h, w, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    buf = io.BytesIO()
    Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(buf, format='PNG')
    return base64.b64encode(buf.getvalue())


@pytest.mark.parametrize('questions', [False, True])
def test_ratio_tsv_batches_write_what_batch_one_writes(tmp_path, questions):
    from generativeimage2text_b200 import inference as inf
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    from generativeimage2text_b200.tsv_io import tsv_writer
    sd = synthetic_state_dict(RATIO, 0, 'perturbed')
    m = _model(RATIO, sd, 'beam', 10)
    shapes = [(300, 200), (200, 300), (250, 250), (180, 400), (400, 260), (220, 330), (310, 310)]
    tsv_writer([('k%d' % i, _png_b64(h, w, i)) for i, (h, w) in enumerate(shapes)], str(tmp_path / 'img.tsv'))
    qtsv = None
    if questions:
        qtsv = str(tmp_path / 'q.tsv')
        tsv_writer([('k%d' % i, json.dumps([{'question': 'what is %d' % i, 'question_id': 2 * i},
                                            {'question': 'where are the %d things' % i, 'question_id': 2 * i + 1}]))
                    for i in range(len(shapes))], qtsv)
    outs = []
    for bs in (1, 4):
        out = str(tmp_path / ('out%d.tsv' % bs))
        inf.test_git_inference_single_tsv(str(tmp_path / 'img.tsv'), 'x', qtsv, out, tokenizer=Tok(), param=RATIO,
                                          batch_size=bs, model=m)
        outs.append(open(out, 'rb').read())
    assert outs[0] == outs[1]
    assert outs[0].count(b'\n') == len(shapes) * (2 if questions else 1)
