"""CPU: caption scoring without a GPU -- the scoring oracle (oracle/score_oracle.py) against the reference goldens
tests/golden/score_*.npz (oracle/make_score_golden.py: the unmodified reference's training-branch forward with dropout
off), and the argument checks of `model.score`, which must all fail before any engine is touched."""
import numpy as np
import pytest
import torch

import score_oracle
from helpers import load_golden

CASES = ['score_base_init', 'score_base_perturbed', 'score_large', 'score_vatex', 'score_vqa_ragged', 'score_base_b64']


def _golden_batch(g):
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    meta = g['meta']
    sd = synthetic_state_dict(meta['param'], meta['seed'], meta['variant'])
    if 'image_hws' in meta:
        image = [synthetic_images(1, 0, meta['img_seed'] + b, hw)[0] for b, hw in enumerate(meta['image_hws'])]
    else:
        image = synthetic_images(meta['batch'], meta['frames'], meta['img_seed'])
    batch = {'image': image, 'caption_tokens': torch.from_numpy(g['caption_tokens']),
             'need_predict': torch.from_numpy(g['need_predict']), 'image_index': torch.from_numpy(g['image_index'])}
    return meta, sd, batch


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference_golden(case):
    g = load_golden(case)
    meta, sd, batch = _golden_batch(g)
    out = score_oracle.score_captions(sd, meta['param'], batch, cols=g['vocab_cols'])
    ref_loss = float(g['vl_l_loss'])
    assert abs(out['vl_l_loss'].item() - ref_loss) <= 1e-5 * abs(ref_loss)
    np.testing.assert_allclose(out['token_logprobs'].numpy(), g['token_logprobs'], rtol=0, atol=1e-4)
    np.testing.assert_allclose(out['logits'].numpy(), g['logits'], rtol=0, atol=1e-3)


def test_golden_cases_cover_the_loss_filters():
    """The goldens hold question prefixes (need_predict 0), a padding target inside need_predict 1, and several captions
    per image in a non-trivial image_index."""
    g = load_golden('score_base_init')
    tok, need = g['caption_tokens'], g['need_predict']
    assert ((need[:, 1:] == 1) & (tok[:, 1:] == 0)).any()
    assert any(need[n, 1] == 0 and need[n].any() for n in range(len(tok)))
    assert len(set(g['image_index'].tolist())) < len(tok)
    v = load_golden('score_vqa_ragged')
    assert len(v['meta']['image_hws']) == 3 and len(v['caption_tokens']) == 12


def test_smooth_label_loss_formula():
    """The closed form the engine's combine kernel uses equals the KL form of SmoothLabelCrossEntropyLoss."""
    torch.manual_seed(0)
    V, eps = 300, 0.1
    z = torch.randn(7, V, dtype=torch.float64) * 3
    t = torch.randint(0, V, (7,))
    ref = score_oracle.smooth_label_ce(z, t, eps)
    lse = torch.logsumexp(z, dim=1)
    lp_t = z.gather(1, t[:, None])[:, 0] - lse
    sum_lp = z.sum(dim=1) - V * lse
    off = eps / (V - 1)
    qlogq = (1 - eps) * np.log(1 - eps) + eps * np.log(off)
    closed = (qlogq - (1 - eps) * lp_t - off * (sum_lp - lp_t)).mean()
    assert abs(closed.item() - ref.item()) < 1e-10


# ---- argument checks: all of them raise before an engine is created ----------------------------------------------------
class Tok:
    cls_token_id, sep_token_id = 101, 102


def _model():
    from generativeimage2text_b200.model import get_git_model
    return get_git_model(Tok(), {}).eval()


def _batch(N=2, T=6, B=2):
    tok = torch.tensor([[101, 2000, 2001, 2002, 102, 0]] * N)[:, :T]
    need = torch.tensor([[0, 1, 1, 1, 1, 0]] * N)[:, :T]
    return {'image': torch.zeros(B, 3, 224, 224), 'caption_tokens': tok, 'need_predict': need}


BAD = {
    'token_too_large': (lambda b: b['caption_tokens'].__setitem__((0, 2), 30522), ValueError),
    'negative_token': (lambda b: b['caption_tokens'].__setitem__((1, 1), -1), ValueError),
    'T_too_small': (lambda b: b.update(caption_tokens=b['caption_tokens'][:, :1], need_predict=b['need_predict'][:, :1]), ValueError),
    'T_too_large': (lambda b: b.update(caption_tokens=torch.full((2, 1025), 101), need_predict=torch.ones(2, 1025, dtype=torch.long)), ValueError),
    'need_shape': (lambda b: b.update(need_predict=b['need_predict'][:, :5]), ValueError),
    'need_values': (lambda b: b['need_predict'].__setitem__((0, 1), 2), ValueError),
    'tokens_1d': (lambda b: b.update(caption_tokens=b['caption_tokens'][0]), ValueError),
    'float_tokens': (lambda b: b.update(caption_tokens=b['caption_tokens'].float()), ValueError),
    'N_neq_B_without_index': (lambda b: b.update(image=torch.zeros(3, 3, 224, 224)), ValueError),
    'index_out_of_range': (lambda b: b.update(image_index=torch.tensor([0, 2])), ValueError),
    'negative_index': (lambda b: b.update(image_index=torch.tensor([-1, 0])), ValueError),
    'index_shape': (lambda b: b.update(image_index=torch.tensor([0, 1, 1])), ValueError),
    'no_valid_target': (lambda b: b.update(need_predict=torch.zeros(2, 6, dtype=torch.long)), ValueError),
    'only_padding_targets': (lambda b: b.update(caption_tokens=torch.tensor([[101, 0, 0, 0, 0, 0]] * 2)), ValueError),
    'missing_need_predict': (lambda b: b.pop('need_predict'), ValueError),
    'context': (lambda b: b.update(context=[]), NotImplementedError),
    'bi_valid_mask_caption': (lambda b: b.update(bi_valid_mask_caption=torch.ones(2, 6)), NotImplementedError),
    'image_3d_tensor': (lambda b: b.update(image=torch.zeros(3, 224, 224)), ValueError),
}


@pytest.mark.parametrize('name', sorted(BAD))
def test_score_rejects_bad_arguments_before_any_engine(name):
    m = _model()
    b = _batch()
    edit, exc = BAD[name]
    edit(b)
    with pytest.raises(exc):
        m.score(b)
    assert all(sl['engine'] is None for sl in m._slots)


def test_score_accepts_the_layouts_it_documents():
    """Valid batches pass the checks (image_index, ragged lists, video frames) and then need the GPU."""
    m = _model()
    ok = [
        _batch(),
        dict(_batch(N=4, B=2), image_index=torch.tensor([1, 0, 1, 1])),
        dict(_batch(N=3, B=2), image=[torch.zeros(3, 160, 208), torch.zeros(3, 224, 224)], image_index=[0, 1, 1]),
        dict(_batch(N=2, B=2), image=[torch.zeros(2, 3, 224, 224)] * 6),
    ]
    for b in ok:
        args = m._score_args(b)
        assert args[2].dtype == torch.long and args[3].dtype == torch.long
        if not torch.cuda.is_available():
            with pytest.raises(RuntimeError):
                m.score(b)
