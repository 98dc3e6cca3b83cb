"""CPU: beam sizes 5 .. 8 for GeneratorWithBeamSearch -- oracle/git_oracle.beam_search against the unmodified reference's
GeneratorWithBeamSearch at those sizes (tests/golden/wide_beam_*.npz, oracle/make_wide_beam_golden.py), the test replay
tests/decode_ref.beam_replay against the oracle, and the host side of the model at beam 8."""
import numpy as np
import pytest
import torch

import git_oracle
from decode_ref import CLS, beam_replay
from generativeimage2text_b200 import _lib
from generativeimage2text_b200 import model as M
from helpers import load_golden, golden_inputs

EOS = 102
GOLDENS = ['wide_beam_base_k5', 'wide_beam_base_k6', 'wide_beam_base_k8', 'wide_beam_large_k8']


@pytest.mark.parametrize('name', GOLDENS)
def test_oracle_beam_search_matches_reference_golden(name):
    g = load_golden(name)
    meta = g['meta']
    beam, B = meta['beam'], meta['batch']
    sd, batch = golden_inputs(meta)
    feats = git_oracle.visual_features(sd, meta['param'], batch['image'])
    dec = git_oracle.CachedDecoder(sd, feats, beam=beam)
    raw, fed = [], []

    def step(ids):
        fed.append(ids[:, -1].clone())
        z = dec.feed(ids[:, dec.n_text:])
        raw.append(z.clone())
        return z
    with torch.no_grad():
        pred, lp = git_oracle.beam_search(torch.full((B, 1), CLS, dtype=torch.long), step, reorder=dec.reorder,
                                          max_steps=meta['max_steps'], beam=beam)
    assert np.array_equal(pred.numpy(), g['predictions'])
    np.testing.assert_allclose(lp.numpy(), g['logprobs'], rtol=0, atol=1e-3)
    # the search trajectory: the same number of steps, the same newest token of every row at every step
    assert len(raw) == g['step_logits'].shape[0]
    assert np.array_equal(torch.stack(fed).numpy(), g['step_tokens'])
    cols = torch.from_numpy(g['vocab_cols'])
    for i, z in enumerate(raw):
        np.testing.assert_allclose(z[:, cols].numpy(), g['step_logits'][i], rtol=0, atol=5e-4)


def test_goldens_search_past_the_first_step():
    """Every golden re-orders its beams and keeps a caption that is not all EOS."""
    for name in GOLDENS:
        g = load_golden(name)
        bidx = g['step_beam_idx']
        assert (bidx[1:] != np.arange(bidx.shape[1])).any(), name
        assert (g['predictions'][:, 0] != EOS).all(), name


def test_beam_replay_is_the_oracle_beam_search_at_wide_beams():
    """beam_replay makes the decisions of git_oracle.beam_search (predictions, log-probs, every beam_idx) at beams
    5 .. 8, with and without a strong EOS."""
    g = torch.Generator().manual_seed(14)
    Vs = 400
    for beam, B, eos_shift, max_steps in ((5, 3, 0.0, 9), (6, 2, 3.0, 12), (7, 2, 2.0, 10), (8, 3, 2.5, 11), (8, 1, 0.0, 7)):
        R = B * beam
        z = torch.randn(max_steps, R, Vs, generator=g) * 2
        z[:, :, EOS] += eos_shift
        it = iter(range(max_steps))
        seen = []
        pred, lp = git_oracle.beam_search(torch.full((B, 1), CLS, dtype=torch.long), lambda ids: z[next(it)],
                                          reorder=seen.append, max_steps=max_steps, beam=beam, length_penalty=0.6)
        rep = beam_replay(z, B, beam, max_steps, 0.6)
        assert torch.equal(rep['pred'], pred), beam
        assert torch.equal(rep['logprobs'], lp[:, 0]), beam
        assert len(rep['bidx']) == len(seen) == rep['n_steps']
        for a, b in zip(rep['bidx'], seen):
            assert torch.equal(a, b)


class Tok:
    cls_token_id, sep_token_id = 101, 102


def test_model_host_side_at_beam_8():
    """GeneratorWithBeamSearch(beam_size=8) reaches the engine as beam 8 / per-node 2; sampled beam search takes
    uniforms [max_steps, B * 8, 2]."""
    m = M.get_git_model(Tok(), {})
    m.decoder = M.GeneratorWithBeamSearch(EOS, max_steps=20, beam_size=8, length_penalty=0.6)
    sp = m._search_struct()
    assert (sp.mode, sp.beam_size, sp.per_node_beam, sp.max_steps) == (_lib.SEARCH_BEAM, 8, 2, 20)
    cpu = torch.device('cpu')
    u = m._beam_sampling_setup({'do_sample': True, 'top_k': 10, 'top_p': 0.9}, sp, 3, cpu)
    assert tuple(u.shape) == (20, 24, 2)
    given = torch.rand(20, 24, 2)
    assert torch.equal(m._beam_sampling_setup({'do_sample': True, 'top_k': 0, 'uniforms': given}, sp, 3, cpu), given)
    with pytest.raises(ValueError):
        m._beam_sampling_setup({'do_sample': True, 'top_k': 0, 'uniforms': torch.rand(20, 12, 2)}, sp, 3, cpu)
