"""GPU: num_return_sequences -- n sequences per image in one call, each image encoded and its K/V cached once.

The contract: an n-sequence call returns, bit for bit, what the same call returns with every image repeated n times
(`repeat_interleave(n, 0)`, or each ragged image listed n times) and the same uniforms -- tokens, log-probs and step
logits -- for every decoder, prefix form, image layout and engine switch.  Deterministic greedy runs both arms with
use_mega 0: an n > 1 call runs on the kernel chain, whose rounding the persistent kernel does not share.
"""
import ctypes

import pytest
import torch

from generativeimage2text_b200 import _lib
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images

pytestmark = pytest.mark.gpu

EOS = 102
BASE = {}
LARGE = {'image_encoder_type': 'CLIPViT_L_14', 'visual_feature_size': 1024}
VIDEO = {'num_image_with_embedding': 6}
VQA = {'test_crop_size': 480, 'test_respect_ratio_max': 640}


class Tok:
    cls_token_id, sep_token_id = 101, 102


_MODELS = {}


def _model(param, use_mega=0):
    """'decisive' weights: a handful of live tokens, so sampled sequences of one image differ."""
    from generativeimage2text_b200.model import get_git_model
    key = repr(sorted(param.items()))
    if key not in _MODELS:
        m = get_git_model(Tok(), param)
        missing, unexpected = m.load_state_dict(synthetic_state_dict(param, 1, 'decisive'), strict=False)
        assert not missing and not unexpected
        _MODELS[key] = m.cuda().eval()
    m = _MODELS[key]
    m.set_engine_option('use_mega', use_mega)
    return m


def _greedy(m, max_steps):
    from generativeimage2text_b200.model import AutoRegressiveBeamSearch
    m.decoder = AutoRegressiveBeamSearch(EOS, max_steps=max_steps, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)


def _beam(m, max_steps, beam=4):
    from generativeimage2text_b200.model import GeneratorWithBeamSearch
    m.decoder = GeneratorWithBeamSearch(EOS, max_steps=max_steps, beam_size=beam, length_penalty=0.6)


def _uniforms(m, S, seed):
    """Uniforms for S sequences of the model's decoder: [max_steps, S] (greedy) or [max_steps, S * beam, 2] (beam)."""
    d = m.decoder
    g = torch.Generator().manual_seed(seed)
    if hasattr(d, 'length_penalty'):
        return torch.rand((d.max_steps, S * d.beam_size, 2), generator=g)
    return torch.rand((d.max_steps, S), generator=g)


def _repeat(image, n):
    if isinstance(image, list) and image[0].dim() == 3:          # ragged: each image listed n times
        return [im for im in image for _ in range(n)]
    if isinstance(image, list):                                   # video frames
        return [f.repeat_interleave(n, 0) for f in image]
    return image.repeat_interleave(n, 0)


def _equal(a, b, logits=True):
    assert torch.equal(a['predictions'], b['predictions']), (a['predictions'] != b['predictions']).nonzero().tolist()[:8]
    assert torch.equal(a['logprobs'], b['logprobs'])
    if logits:
        assert torch.equal(a['step_logits'], b['step_logits'])


def _check(m, image, n, sp=None, extra=None, rep_extra=None, logits=True):
    """The n-sequence call against the repeated-image call with the same search_param; returns the n-sequence result."""
    sp = dict(sp or {})
    got = m(dict(image=image, **(extra or {})), return_step_logits=logits, search_param=dict(sp, num_return_sequences=n))
    want = m(dict(image=_repeat(image, n), **(rep_extra if rep_extra is not None else extra or {})),
             return_step_logits=logits, search_param=sp or None)
    torch.cuda.synchronize()
    _equal(got, want, logits)
    return got


def _distinct_rows(out, B, n):
    """Sampled sequences of one image differ somewhere (the rows are really drawn independently)."""
    p = out['predictions'].view(B, n, -1)
    return sum(int(not all(torch.equal(p[b, 0], p[b, i]) for i in range(n))) for b in range(B))


# ---- greedy decoder ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,n', [(3, 2), (2, 3), (4, 5)])
def test_greedy_sampling_and_deterministic(B, n):
    m = _model(BASE)
    _greedy(m, 12)
    x = synthetic_images(B, 0, seed=100 + B).cuda()
    out = _check(m, x, n, {'do_sample': True, 'temperature': 0.7, 'uniforms': _uniforms(m, B * n, B)})
    assert out['predictions'].shape[0] == B * n and out['logprobs'].shape == (B * n,)
    assert _distinct_rows(out, B, n) >= 1
    out = _check(m, x, n)
    p = out['predictions'].view(B, n, -1)
    assert all(torch.equal(p[b, 0], p[b, i]) for b in range(B) for i in range(n))   # without do_sample: n equal rows


def test_generator_draws_the_sequence_shapes():
    m = _model(BASE)
    _greedy(m, 10)
    x = synthetic_images(3, 0, seed=7).cuda()
    got = m({'image': x}, search_param={'do_sample': True, 'num_return_sequences': 2, 'generator': torch.Generator('cuda').manual_seed(4)})
    want = m({'image': x.repeat_interleave(2, 0)}, search_param={'do_sample': True, 'generator': torch.Generator('cuda').manual_seed(4)})
    _equal(got, want, logits=False)
    _beam(m, 10)
    sp = {'do_sample': True, 'top_k': 20, 'top_p': 0.9}
    got = m({'image': x}, search_param=dict(sp, num_return_sequences=3, generator=torch.Generator('cuda').manual_seed(5)))
    want = m({'image': x.repeat_interleave(3, 0)}, search_param=dict(sp, generator=torch.Generator('cuda').manual_seed(5)))
    _equal(got, want, logits=False)


def test_scst_shape_64_images_by_5():
    m = _model(BASE)
    _greedy(m, 10)
    x = synthetic_images(64, 0, seed=64).cuda()
    out = _check(m, x, 5, {'do_sample': True, 'temperature': 0.7, 'uniforms': _uniforms(m, 320, 64)})
    assert out['predictions'].shape[0] == 320
    assert _distinct_rows(out, 64, 5) >= 32


def test_trie_decoder():
    from generativeimage2text_b200.model import TrieAutoRegressiveBeamSearch, TokenTrie
    m = _model(BASE)
    _greedy(m, 12)
    x = synthetic_images(3, 0, seed=21).cuda()
    free = m({'image': x})['predictions'].cpu()
    g = torch.Generator().manual_seed(3)
    seqs = []
    for row in free.tolist():                      # the free captions with their tails cut and replaced
        body = row[1:]
        cut = max(1, (body.index(EOS) if EOS in body else len(body)) // 2)
        seqs.append(body[:cut] + torch.randint(1000, 30000, (3,), generator=g).tolist() + [EOS])
    for _ in range(30):
        seqs.append(torch.randint(1000, 30000, (int(torch.randint(2, 6, (1,), generator=g)),), generator=g).tolist() + [EOS])
    m.decoder = TrieAutoRegressiveBeamSearch(EOS, max_steps=12, beam_size=1, trie=TokenTrie.construct(seqs))
    try:
        for n in (2, 3):
            _check(m, x, n)
    finally:
        _greedy(m, 12)


# ---- beam search -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('beam,B,n', [(4, 3, 2), (3, 2, 3), (2, 2, 5)])
def test_beam_search_deterministic_and_sampled(beam, B, n):
    m = _model(BASE)
    _beam(m, 12, beam)
    x = synthetic_images(B, 0, seed=200 + B).cuda()
    out = _check(m, x, n)
    assert out['predictions'].shape[0] == B * n and out['logprobs'].shape == (B * n, 1)
    out = _check(m, x, n, {'do_sample': True, 'top_k': 50, 'top_p': 0.9, 'uniforms': _uniforms(m, B * n, beam)})
    assert out['step_logits'].shape[1] == B * n * beam
    assert _distinct_rows(out, B, n) >= 1


def test_large_32_images_by_2_beam_4_sampled():
    m = _model(LARGE)
    _beam(m, 10, 4)
    x = synthetic_images(32, 0, seed=32).cuda()
    out = _check(m, x, 2, {'do_sample': True, 'top_k': 50, 'top_p': 0.9, 'uniforms': _uniforms(m, 64, 32)})
    assert out['step_logits'].shape[1] == 256


# ---- prefixes ----------------------------------------------------------------------------------------------------------
def _row_prefixes(rows):
    t = torch.zeros((len(rows), max(len(p) for p in rows)), dtype=torch.long)
    for r, p in enumerate(rows):
        t[r, :len(p)] = torch.tensor(p)
    return {'prefix': t.cuda(), 'prefix_len': torch.tensor([len(p) for p in rows])}


@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_per_image_prefixes(search):
    m = _model(BASE)
    (_greedy if search == 'greedy' else _beam)(m, 12)
    n, prefixes = 3, [[101, 2054, 2003], [101], [101, 2129, 2116, 2111]]
    x = synthetic_images(3, 0, seed=300).cuda()
    sp = {'do_sample': True, 'top_k': 30} if search == 'beam' else {'do_sample': True, 'temperature': 0.7}
    sp['uniforms'] = _uniforms(m, 3 * n, 3)
    _check(m, x, n, sp, _row_prefixes(prefixes), _row_prefixes([p for p in prefixes for _ in range(n)]))
    _check(m, x, n, None, _row_prefixes(prefixes), _row_prefixes([p for p in prefixes for _ in range(n)]))


@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_shared_prefix_at_batch_1(search):
    """One shared prefix needs batch 1, so the repeated call gives each copy of the image that prefix as its own."""
    m = _model(BASE)
    (_greedy if search == 'greedy' else _beam)(m, 12)
    n, prefix = 3, [101, 2023, 2003]
    x = synthetic_images(1, 0, seed=301).cuda()
    sp = {'do_sample': True, 'top_k': 30} if search == 'beam' else {'do_sample': True, 'temperature': 0.7}
    sp['uniforms'] = _uniforms(m, n, 4)
    out = _check(m, x, n, sp, {'prefix': torch.tensor([prefix]).cuda()}, _row_prefixes([prefix] * n), logits=False)
    assert out['predictions'].shape[0] == n


# ---- image layouts -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_ragged_vqav2_geometry(search):
    m = _model(VQA)
    (_greedy if search == 'greedy' else _beam)(m, 10)
    ims = [synthetic_images(1, 0, 400 + b, hw)[0].cuda() for b, hw in enumerate([(480, 640), (640, 480), (480, 480)])]
    sp = {'do_sample': True, 'top_k': 50, 'top_p': 0.9} if search == 'beam' else {'do_sample': True, 'temperature': 0.7}
    sp['uniforms'] = _uniforms(m, 3 * 2, 5)
    _check(m, ims, 2, sp)
    questions = [[101, 2054, 2003], [101, 2129], [101, 2054, 2003, 1996]]
    _check(m, ims, 2, None, _row_prefixes(questions), _row_prefixes([q for q in questions for _ in range(2)]))


def test_video_six_frames():
    m = _model(VIDEO)
    _greedy(m, 10)
    frames = synthetic_images(2, 6, seed=500)
    frames = [f.cuda() for f in frames]
    _check(m, frames, 3, {'do_sample': True, 'temperature': 0.7, 'uniforms': _uniforms(m, 6, 6)})
    _beam(m, 10)
    _check(m, frames, 2, {'do_sample': True, 'top_k': 40, 'uniforms': _uniforms(m, 4, 7)})


# ---- engine switches ---------------------------------------------------------------------------------------------------
def test_parity_mode():
    m = _model(BASE)
    m.set_engine_option('parity', 1)
    try:
        x = synthetic_images(2, 0, seed=600).cuda()
        _greedy(m, 10)
        _check(m, x, 3, {'do_sample': True, 'temperature': 0.7, 'uniforms': _uniforms(m, 6, 8)})
        _check(m, x, 2)
        _beam(m, 10)
        _check(m, x, 2, {'do_sample': True, 'top_k': 50, 'top_p': 0.9, 'uniforms': _uniforms(m, 4, 9)})
    finally:
        m.set_engine_option('parity', 0)


def test_teacher_forcing_past_128_steps():
    """forced_tokens [B * n, max_steps] without EOS: the loop runs to max_steps and the text caches grow past 128."""
    m = _model(BASE)
    steps, B, n = 150, 2, 3
    _greedy(m, steps)
    x = synthetic_images(B, 0, seed=700).cuda()
    g = torch.Generator().manual_seed(10)
    forced = torch.randint(1000, 30000, (B * n, steps), generator=g)
    got = m({'image': x}, forced_tokens=forced, return_step_logits=True, search_param={'num_return_sequences': n})
    want = m({'image': x.repeat_interleave(n, 0)}, forced_tokens=forced, return_step_logits=True)
    _equal(got, want)
    assert got['step_logits'].shape[0] == steps - 1
    assert m.last_decode_timing()[1] == steps - 1


@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_graphs_and_pdl(search):
    m = _model(BASE)
    (_greedy if search == 'greedy' else _beam)(m, 12)
    x = synthetic_images(3, 0, seed=800).cuda()
    sp = {'do_sample': True, 'top_k': 0, 'top_p': 0.8} if search == 'beam' else {'do_sample': True}
    sp['uniforms'] = _uniforms(m, 9, 11)
    want = m({'image': x.repeat_interleave(3, 0)}, return_step_logits=True, search_param=sp)
    try:
        for gr in (0, 1):
            for pdl in (0, 1):
                m.set_engine_option('use_graph', gr)
                m.set_engine_option('use_pdl', pdl)
                got = m({'image': x}, return_step_logits=True, search_param=dict(sp, num_return_sequences=3))
                _equal(got, want)
    finally:
        m.set_engine_option('use_graph', 1)
        m.set_engine_option('use_pdl', 1)


def test_deterministic_greedy_with_use_mega_runs_on_the_kernel_chain():
    m = _model(BASE, use_mega=1)
    _greedy(m, 12)
    x = synthetic_images(3, 0, seed=900).cuda()
    got = m({'image': x}, search_param={'num_return_sequences': 2})
    assert not m.last_decode_timing()[2]
    m.set_engine_option('use_mega', 0)
    want = m({'image': x.repeat_interleave(2, 0)})
    _equal(got, want, logits=False)


# ---- what the call shares and what n = 1 leaves alone ------------------------------------------------------------------
def test_each_image_is_encoded_and_cached_once():
    m = _model(BASE)
    _beam(m, 8)
    B, n = 3, 4
    x = synthetic_images(B, 0, seed=1000).cuda()
    m({'image': x}, search_param={'num_return_sequences': n})
    lib = _lib.load()
    want = 6 * 2 * B * 197 * 768 * 2
    buf = (ctypes.c_uint8 * (2 * want))()
    assert lib.gitb200_debug_read(m._engine, b'img_kv', buf, 2 * want) == want    # B images, not B * n


@pytest.mark.parametrize('use_mega', [0, 1])
def test_n_equal_1_is_the_call_without_it(use_mega):
    m = _model(BASE, use_mega=use_mega)
    x = synthetic_images(3, 0, seed=1100).cuda()
    for search, sp in (('greedy', {}), ('greedy', {'do_sample': True, 'uniforms': torch.rand(12, 3)}),
                       ('beam', {}), ('beam', {'do_sample': True, 'top_k': 5, 'uniforms': torch.rand(12, 12, 2)})):
        (_greedy if search == 'greedy' else _beam)(m, 12)
        m({'image': x}, search_param=sp or None)                   # warm: graphs captured, buffers sized
        c0 = m.launch_count()
        want = m({'image': x}, return_step_logits=True, search_param=sp or None)
        c1 = m.launch_count()
        got = m({'image': x}, return_step_logits=True, search_param=dict(sp, num_return_sequences=1))
        c2 = m.launch_count()
        _equal(got, want)
        assert c2 - c1 == c1 - c0, (search, sp.keys(), c1 - c0, c2 - c1)


@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_rows_of_an_image_equal_its_call_alone(search):
    m = _model(BASE)
    (_greedy if search == 'greedy' else _beam)(m, 12)
    B, n = 3, 2
    x = synthetic_images(B, 0, seed=1200).cuda()
    sp = {'do_sample': True, 'top_k': 30, 'top_p': 0.9} if search == 'beam' else {'do_sample': True, 'temperature': 0.7}
    u = _uniforms(m, B * n, 12)
    full = m({'image': x}, search_param=dict(sp, uniforms=u, num_return_sequences=n))
    w = u.shape[1] // B
    for b in range(B):
        one = m({'image': x[b:b + 1]}, search_param=dict(sp, uniforms=u[:, b * w:(b + 1) * w], num_return_sequences=n))
        k = one['predictions'].shape[1]
        assert torch.equal(one['predictions'], full['predictions'][b * n:(b + 1) * n, :k])
        assert bool((full['predictions'][b * n:(b + 1) * n, k:] == EOS).all())
        assert torch.equal(one['logprobs'], full['logprobs'][b * n:(b + 1) * n])
