"""CPU: num_return_sequences.

  * the oracle's search loops, run over B * n rows (each image's features repeated n times, image-major), give what the
    original code's searches return with num_return_sequences = n on a random-init GIT_BASE and distinct images
    (tests/golden/return_sequences_checks.json, oracle/make_return_sequences_golden.py; torch.multinomial replaced by the
    engine's inverse-CDF draws fed the same uniforms);
  * `submit` up to the engine call, with the engine stubbed: the value of n, the shapes of uniforms / forced tokens /
    outputs, per-image prefix expansion and what reaches the engine.
"""
import ctypes
import json
import os

import pytest
import torch

import beam_sample_oracle as bso
import git_oracle
from generativeimage2text_b200 import _lib
from generativeimage2text_b200 import model as M
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'return_sequences_checks.json')
MAX_STEPS = 8
BEAM = 4

# (search, images, n, temperature, top_k, top_p, seed of the uniforms)
CASES = [
    ('sample', 3, 2, 0.7, 0, None, 1),
    ('sample', 2, 3, 1.0, 0, None, 2),
    ('greedy', 3, 2, 1.0, 0, None, 0),
    ('trie', 2, 3, 1.0, 0, None, 0),
    ('beam', 2, 2, 1.0, 0, None, 0),
    ('beam_sample', 2, 3, 1.0, 50, 0.9, 3),
    ('beam_sample', 3, 2, 0.7, 20, None, 4),
]


def case_uniforms(case):
    search, B, n, _, _, _, seed = case
    g = torch.Generator().manual_seed(100 + seed)
    if search == 'beam_sample':
        return torch.rand((MAX_STEPS, B * n * BEAM, 2), generator=g)
    return torch.rand((MAX_STEPS, B * n), generator=g)


def case_images(case):
    """Distinct images, so that the image-major row order is pinned."""
    return synthetic_images(case[1], 0, seed=500 + case[1])


def state_dict():
    return synthetic_state_dict({}, 5, 'init')


def trie_sequences():
    """Paths longer than MAX_STEPS: the original decoder's one cursor follows row 0 and asserts if row 0 ends while other
    rows run on (trie_decoder.py:159, TokenTrie.move)."""
    g = torch.Generator().manual_seed(11)
    return [torch.randint(1000, 30000, (int(torch.randint(MAX_STEPS + 1, MAX_STEPS + 4, (1,), generator=g)),),
                          generator=g).tolist() + [102] for _ in range(40)]


def oracle_run(case, sd, feats):
    """The case's search over B * n rows: image b's features serve rows b * n .. b * n + n - 1."""
    search, B, n, T, top_k, top_p, _ = case
    beam = BEAM if search.startswith('beam') else 1
    dec = git_oracle.CachedDecoder(sd, feats.repeat_interleave(n, 0), beam=beam)

    def step(partial):
        return dec.feed(partial[:, dec.n_text:])
    start = torch.full((B * n, 1), 101, dtype=torch.long)
    u = case_uniforms(case)
    if search == 'greedy':
        return git_oracle.greedy_search(start, step, max_steps=MAX_STEPS)
    if search == 'sample':
        return git_oracle.sample_search(start, step, u, temperature=T, max_steps=MAX_STEPS)
    if search == 'trie':   # the original decoder's single cursor (per_row=False): with B * n > 1 rows it binds row 0 only
        csr = M.TokenTrie.construct(trie_sequences()).to_csr()
        return git_oracle.trie_search(start, step, csr, max_steps=MAX_STEPS, per_row=False)
    if search == 'beam':
        return git_oracle.beam_search(start, step, reorder=dec.reorder, max_steps=MAX_STEPS, beam=BEAM)
    return bso.beam_sample_search(start, step, u, reorder=dec.reorder, max_steps=MAX_STEPS, beam=BEAM, temperature=T,
                                  top_k=top_k, top_p=top_p)


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


_FEATS = {}


@pytest.mark.parametrize('i', range(len(CASES)))
def test_oracle_equals_reference_num_return_sequences(i):
    case = CASES[i]
    gold = load_golden()['cases'][i]
    assert gold['case'] == list(case)
    sd = state_dict()
    if case[1] not in _FEATS:
        _FEATS[case[1]] = git_oracle.visual_features(sd, {}, case_images(case))
    pred, lp = oracle_run(case, sd, _FEATS[case[1]])
    assert pred.shape[0] == case[1] * case[2]
    assert pred.tolist() == gold['predictions']
    # 1e-6, relative where the score exceeds 1 in magnitude (beam scores reach ~16, where one fp32 ulp is 1.9e-6)
    assert torch.allclose(lp.double(), torch.tensor(gold['logprobs'], dtype=torch.float64), rtol=1e-6, atol=1e-6)


def test_golden_rows_are_image_major_and_sampled_rows_differ():
    """Without sampling an image's n rows are equal (and greedy captions differ between images); with it, some rows of
    one image differ."""
    gold = load_golden()['cases']
    for case, g in zip(CASES, gold):
        search, B, n = case[:3]
        rows = [g['predictions'][b * n:(b + 1) * n] for b in range(B)]
        if search in ('greedy', 'beam'):
            assert all(r[i] == r[0] for r in rows for i in range(n))
        if search == 'greedy':
            assert len({tuple(r[0]) for r in rows}) > 1
        elif search in ('sample', 'beam_sample'):
            assert any(r[i] != r[0] for r in rows for i in range(n))


# ---------------------------------------------------------------------------------------------------------------------
# submit up to the engine call
# ---------------------------------------------------------------------------------------------------------------------
class Tok:
    cls_token_id, sep_token_id = 101, 102


class FakeLib:
    """Records what submit hands the engine (the calls of test_ragged_host.py's stub) and returns 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return 0
        return call

    def named(self, name):
        return [a for n, a in self.calls if n == name]


class _Stream:
    cuda_stream = 0


def _stub(monkeypatch, m):
    lib = FakeLib()
    monkeypatch.setattr(m, '_ensure_engine', lambda slot=0: (lib, None))
    monkeypatch.setattr(_lib, 'load', lambda: lib)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda dev=None: _Stream())
    m._slots[0]['engine'] = ctypes.c_void_p(1)
    return lib


def _submit(m, batch, **kw):
    return m.submit(batch, slot=0, _caller_stream=True, **kw)


@pytest.fixture
def model():
    m = M.get_git_model(Tok(), {}).eval()
    m.decoder = M.AutoRegressiveBeamSearch(102, max_steps=10, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    yield m
    m._slots[0]['pending'] = None
    m._slots[0]['engine'] = None          # a stub handle: nothing for the real library to destroy


def test_n_must_be_an_integer_of_at_least_1(model, monkeypatch):
    _stub(monkeypatch, model)
    x = torch.zeros(2, 3, 224, 224)
    for bad in (0, -1, True, False, 2.0, '2', None):
        with pytest.raises(ValueError):
            _submit(model, {'image': x}, search_param={'num_return_sequences': bad})


def test_shapes_count_sequences(model, monkeypatch):
    lib = _stub(monkeypatch, model)
    x = torch.zeros(2, 3, 224, 224)
    p = _submit(model, {'image': x}, return_step_logits=True,
                search_param={'num_return_sequences': 3, 'do_sample': True, 'temperature': 0.7})
    assert p.tokens.shape == (6, 10) and p.logprobs.shape == (6,) and p.step_logits.shape[1] == 6
    assert [a[1] for a in lib.named('gitb200_set_sequences_per_image')] == [3]
    (_, _, steps, rows, _), = lib.named('gitb200_set_sampling')
    assert (steps, rows) == (10, 6)
    (gen,) = lib.named('gitb200_generate_async')
    assert gen[2] == 2                                       # the engine encodes the 2 images
    # caller uniforms and forced tokens are [.., B * n]
    assert _submit(model, {'image': x}, search_param={'num_return_sequences': 3, 'do_sample': True,
                                                        'uniforms': torch.rand(10, 6)}).tokens.shape == (6, 10)
    with pytest.raises(ValueError):
        _submit(model, {'image': x}, search_param={'num_return_sequences': 3, 'do_sample': True, 'uniforms': torch.rand(10, 2)})
    assert _submit(model, {'image': x}, forced_tokens=torch.zeros(6, 10, dtype=torch.long),
                   search_param={'num_return_sequences': 3}).tokens.shape == (6, 10)
    with pytest.raises(AssertionError):
        _submit(model, {'image': x}, forced_tokens=torch.zeros(2, 10, dtype=torch.long), search_param={'num_return_sequences': 3})
    # the beam decoder: [max_steps, B * n * beam, 2]
    model.decoder = M.GeneratorWithBeamSearch(102, max_steps=10, beam_size=4, length_penalty=0.6)
    p = _submit(model, {'image': x}, return_step_logits=True, search_param={'num_return_sequences': 2, 'do_sample': True, 'top_k': 5})
    assert p.tokens.shape == (4, 10) and p.step_logits.shape[1] == 16
    (_, _, steps, rows, *_), = lib.named('gitb200_set_beam_sampling')
    assert (steps, rows) == (10, 16)
    with pytest.raises(ValueError):
        _submit(model, {'image': x}, search_param={'num_return_sequences': 2, 'do_sample': True, 'top_k': 5,
                                                     'uniforms': torch.rand(10, 8, 2)})


def test_n_equal_1_is_the_call_without_it(model, monkeypatch):
    lib = _stub(monkeypatch, model)
    x = torch.zeros(2, 3, 224, 224)
    _submit(model, {'image': x}).result()
    plain = list(lib.calls)
    lib.calls.clear()
    _submit(model, {'image': x}, search_param={'num_return_sequences': 1}).result()
    assert [n for n, _ in lib.calls] == [n for n, _ in plain]
    assert not lib.named('gitb200_set_sequences_per_image')


def test_per_image_prefixes_are_expanded(model, monkeypatch):
    lib = _stub(monkeypatch, model)
    x = torch.zeros(3, 3, 224, 224)
    prefix = torch.tensor([[101, 5, 6], [101, 0, 0], [101, 7, 0]])
    p = _submit(model, {'image': x, 'prefix': prefix, 'prefix_len': torch.tensor([3, 1, 2])},
                search_param={'num_return_sequences': 2})
    assert p.row_lens == [3, 3, 1, 1, 2, 2]
    (eng, ptr, rows, stride, _), = lib.named('gitb200_set_row_prefixes')
    assert (rows, stride) == (6, 3)
    kept = [t for t in p._keep if t is not None and t.dtype == torch.long and t.dim() == 2]
    assert torch.equal(kept[0], prefix.repeat_interleave(2, 0))
    # one shared prefix stays the batch-1 form: fed to every sequence
    model._slots[0]['pending'] = None        # (the stub engine decodes nothing to finish)
    lib.calls.clear()
    p = _submit(model, {'image': x[:1], 'prefix': torch.tensor([[101, 5]])}, search_param={'num_return_sequences': 4})
    assert p.tokens.shape == (4, 10) and not lib.named('gitb200_set_row_prefixes')


def test_the_private_sampling_helper_still_rejects_the_key(model):
    sp = model._search_struct()
    with pytest.raises(NotImplementedError):
        model._sampling_setup({'do_sample': True, 'num_return_sequences': 2}, sp, 2, torch.device('cpu'))


def test_the_n_sequence_call_is_never_coalesced(model, monkeypatch):
    seen = []
    monkeypatch.setattr(model, '_submit_coalesced', lambda *a, **k: seen.append('coalesced'))
    monkeypatch.setattr(model, '_ensure_engine', lambda slot=0: (_ for _ in ()).throw(RuntimeError('engine')))
    x = torch.zeros(2, 3, 224, 224)
    with pytest.raises(RuntimeError, match='engine'):
        model.submit({'image': x}, coalesce=4, search_param={'num_return_sequences': 2})
    assert seen == []
    model.submit({'image': x}, coalesce=4, search_param={'num_return_sequences': 1})
    assert seen == ['coalesced']
