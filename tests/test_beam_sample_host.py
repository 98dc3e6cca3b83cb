"""CPU: sampled beam search (GeneratorWithBeamSearch with do_sample) -- oracle/beam_sample_oracle.beam_sample_search against what the
original code's GeneratorWithBeamSearch.search returns with torch.multinomial replaced by the same draws
(tests/golden/beam_sample_checks.json, oracle/make_beam_sample_golden.py), and the host-side argument checks."""
import json
import os

import pytest
import torch

import beam_sample_oracle as bso
from generativeimage2text_b200 import _lib
from generativeimage2text_b200 import model as M

EOS = 102
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'beam_sample_checks.json')

# (beam, batch, temperature, top_k, top_p, max_steps, seed, eos_bias): top-k only, top-p only, both, neither; a top_p small
# enough that the keep-three rule decides; top_k 1 (raised to 2); EOS biased up so that captions end early
CASES = [
    (4, 3, 1.0, 0, None, 12, 0, 0.0),
    (4, 3, 0.7, 5, None, 12, 1, 0.0),
    (3, 2, 1.0, 0, 0.8, 12, 2, 0.0),
    (2, 3, 0.7, 8, 0.9, 12, 3, 0.0),
    (4, 2, 1.0, 0, 0.05, 12, 4, 0.0),
    (2, 1, 0.7, 1, None, 10, 5, 0.0),
    (3, 4, 1.0, 50, 0.5, 6, 6, 0.0),
    (4, 3, 1.0, 10, 0.95, 16, 7, 0.6),
    (2, 2, 0.7, 0, None, 16, 8, 0.8),
]


def toy_step(vocab=64, seed=3, eos=2, eos_bias=0.0):
    """Deterministic stand-in for `decoding_step`: logits depend on the row's last token and on the caption length; EOS
    gains `eos_bias` per position."""
    g = torch.Generator().manual_seed(seed)
    table = torch.randn(vocab, vocab, generator=g) * 2.0
    drift = torch.randn(64, vocab, generator=g) * 0.5

    def step(partial):
        z = table[partial[:, -1]] + drift[partial.shape[1]]
        z[:, eos] += eos_bias * partial.shape[1]
        return z
    return step


def case_uniforms(case):
    beam, B, _, _, _, steps, seed, _ = case
    return torch.rand((steps, B * beam, 2), generator=torch.Generator().manual_seed(100 + seed))


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize('i', range(len(CASES)))
def test_beam_sample_search_equals_reference_with_the_same_draws(i):
    beam, B, T, top_k, top_p, steps, seed, eos_bias = case = CASES[i]
    gold = load_golden()['cases'][i]
    assert gold['case'] == list(case)
    start = torch.tensor([[1]] * B)
    pred, lp = bso.beam_sample_search(start, toy_step(seed=seed, eos_bias=eos_bias), case_uniforms(case),
                                             max_steps=steps, beam=beam, temperature=T, top_k=top_k, top_p=top_p, eos=2)
    assert pred.tolist() == gold['predictions']
    assert torch.allclose(lp.double(), torch.tensor(gold['logprobs'], dtype=torch.float64), rtol=0, atol=1e-6)


def test_golden_covers_the_listed_situations():
    """The golden cases reach what they are there for: EOS draws, images that finish early, searches that run to
    max_steps, and steps where the keep-three rule of the nucleus filter decides the kept set."""
    seen = load_golden()['seen']
    for what in ('eos_drawn', 'ended_early', 'ran_to_max_steps', 'keep_three_decides', 'batch_gt_1', 'beam_2', 'beam_3',
                 'beam_4'):
        assert seen[what], what


def test_filter_keeps_ties_at_the_kth_value_and_cuts_nucleus_ties_by_index():
    z = torch.tensor([[3.0, 1.0, 2.0, 2.0, 2.0, 0.0]])
    kept = torch.isfinite(bso.top_k_top_p_filter(z, 2, None))
    assert kept.tolist() == [[True, False, True, True, True, False]]                # k = 2: every value tied at the 2nd
    # softmax of [3, 2, 2, 2, 1, 0] in (value desc, index asc) order: cumsum crosses 0.6 at the 2nd position (index 2);
    # the shift keeps positions 0 .. 2 -> indices 0, 2, 3
    kept = torch.isfinite(bso.top_k_top_p_filter(z, 0, 0.6))
    assert kept.tolist() == [[True, False, True, True, False, False]]
    kept = torch.isfinite(bso.top_k_top_p_filter(z, 0, 1e-4))               # keep-three: never fewer than three
    assert int(kept.sum()) == 3


class Tok:
    cls_token_id, sep_token_id = 101, 102


def test_beam_decoder_temperature_is_its_attribute():
    """The constructor keeps taking temperature 1 only; sampled beam search reads the decoder's `temperature` attribute,
    the value the reference's search reads (layers/decoder.py:1097)."""
    with pytest.raises(AssertionError):
        M.GeneratorWithBeamSearch(EOS, max_steps=8, beam_size=4, temperature=0)
    with pytest.raises(NotImplementedError):
        M.GeneratorWithBeamSearch(EOS, max_steps=8, beam_size=4, repetition_penalty=1.2)
    m = M.get_git_model(Tok(), {})
    m.decoder = M.GeneratorWithBeamSearch(EOS, max_steps=12, beam_size=3, length_penalty=0.6)
    assert m.decoder.temperature == 1
    sp = m._search_struct()
    for bad in (0, -1.0, float('inf'), None, '0.7'):
        m.decoder.temperature = bad
        with pytest.raises(ValueError):
            m._sampling_setup({'do_sample': True, 'top_k': 5}, sp, 2, torch.device('cpu'))
    m.decoder.temperature = 0.7
    assert m._sampling_setup({'do_sample': True, 'top_k': 5}, sp, 2, torch.device('cpu')) is not None


def test_beam_search_param_validation():
    """GeneratorWithBeamSearch.search takes do_sample / top_k / top_p / num_keep_best / num_return_sequences (reference
    layers/decoder.py:1083-1092); the temperature is the decoder's."""
    m = M.get_git_model(Tok(), {})
    m.decoder = M.GeneratorWithBeamSearch(EOS, max_steps=12, beam_size=3, length_penalty=0.6)
    m.decoder.temperature = 0.7
    sp = m._search_struct()
    assert sp.mode == _lib.SEARCH_BEAM
    cpu = torch.device('cpu')
    setup = lambda param: m._sampling_setup(param, sp, 2, cpu)                                   # noqa: E731
    # do_sample off: a deterministic search whatever top_k / top_p say (they are unused there)
    for param in ({}, {'do_sample': False}, {'do_sample': False, 'top_k': 5, 'top_p': 0.3}, {'num_keep_best': 1}):
        assert setup(param) is None
    u = setup({'do_sample': True, 'top_k': 0})
    assert tuple(u.shape) == (12, 6, 2) and u.dtype == torch.float32 and bool(((u >= 0) & (u < 1)).all())
    g1 = setup({'do_sample': True, 'top_k': 4, 'top_p': 0.9, 'generator': torch.Generator().manual_seed(3)})
    g2 = setup({'do_sample': True, 'top_k': 4, 'top_p': 0.9, 'generator': torch.Generator().manual_seed(3)})
    assert torch.equal(g1, g2)
    assert setup({'do_sample': True, 'top_k': 4, 'uniforms': torch.rand(13, 6, 2)}) is not None
    assert M._beam_filter({'top_k': 0, 'top_p': None}) == (0, 1.0)
    assert M._beam_filter({'top_k': 3, 'top_p': 0}) == (3, 1.0)                               # `if top_p and ...`
    assert M._beam_filter({'top_k': 3, 'top_p': 0.25}) == (3, 0.25)
    with pytest.raises(ValueError):
        setup({'do_sample': True, 'top_k': 4, 'uniforms': torch.rand(12, 6)})
    with pytest.raises(ValueError):
        setup({'do_sample': True, 'top_k': 4, 'uniforms': torch.rand(11, 6, 2)})
    for err in (TypeError, NotImplementedError):                     # top_k defaults to None: `None > 0` raises (:1355)
        with pytest.raises(err):
            setup({'do_sample': True})
    with pytest.raises(TypeError):
        setup({'do_sample': True, 'top_k': None, 'top_p': 0.9})
    with pytest.raises(TypeError):
        setup({'do_sample': True, 'top_k': 5, 'temperature': 0.7})   # search() has no temperature argument
    with pytest.raises(TypeError):
        setup({'temperature': 1.0})
    with pytest.raises(NotImplementedError):
        setup({'do_sample': True, 'top_k': 5, 'num_return_sequences': 2})
    with pytest.raises(NotImplementedError):
        setup({'do_sample': True, 'top_k': 5, 'num_keep_best': 2})
    with pytest.raises(NotImplementedError):
        setup({'do_sample': True, 'top_k': 5, 'repetition_penalty': 1.2})
