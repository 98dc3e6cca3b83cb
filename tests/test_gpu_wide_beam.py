"""GPU: GeneratorWithBeamSearch at beam sizes 5 .. 8 -- decode_attn_kernel<5 .. 8> (one (image, head) item holds all
beams of an image, so its image K/V is read once per step) and the 16-entry candidate lists of beam_row_topk_kernel<16>,
beam_sample_kernel<16> and beam_update_kernel<16>.

  * every step against the fp64 statement of test_gpu_beam_step.py (its _check_beam_run and tolerances): logits, the
    appended text K/V, the last step's chain buffers, src_row / beam_ids / hypotheses / predictions exactly, the 16-wide
    beam_cand lists and scores against the fp64 replay, and the planted defects at beam 8;
  * planted exact logit ties inside the 16-entry lists;
  * parity mode against the reference goldens of oracle/make_wide_beam_golden.py;
  * sampled beam search replayed with oracle/beam_sample_oracle.py (test_gpu_beam_sample.py's replay);
  * num_return_sequences, batch independence, graph / PDL and fresh-engine bit identity.
"""
import numpy as np
import pytest
import torch

import git_oracle
import test_gpu_beam_sample as bsm
import test_gpu_beam_step as bst
import test_gpu_parity as tpar
from decode_ref import EOS, RefWeights, beam_replay, ancestry
from helpers import load_golden, golden_inputs
from test_gpu_beam_step import (ALL_DEFECTS, MANY_KEYS, _beam, _check_beam_run, _generate, _model, _no_eos, _outputs,
                                _patched)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def sd_perturbed():
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    return synthetic_state_dict({}, 1, 'perturbed')


# ---------------------------------------------------------------------------------------------------------------------
# step-level fp64 comparison
# ---------------------------------------------------------------------------------------------------------------------
# (id, B, beam, (height, width), max_steps, defects, exempt)
CASES = [
    ('b1_k8_m2', 1, 8, (16, 16), 10, tuple(d for d in ALL_DEFECTS if d != 'wrong_image'), ()),
    ('b2_k8_m2', 2, 8, (16, 16), 8, ALL_DEFECTS, ()),
    ('b2_k5_m2', 2, 5, (16, 16), 8, ALL_DEFECTS, ()),
    ('b2_k6_m197', 2, 6, (224, 224), 8, ALL_DEFECTS, MANY_KEYS),
    ('b3_k7_m257', 3, 7, (256, 256), 6, ('chunk', 'wrong_image', 'prev_ancestry'), MANY_KEYS),
    ('b40_k8_m197', 40, 8, (224, 224), 4, (), ()),       # 320 rows
    ('b34_k7_m65', 34, 7, (128, 128), 4, (), ()),        # 238 rows
]


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_wide_beam_step_against_fp64_reference(case, sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    label, B, beam, hw, max_steps, defects, exempt = case
    m = _model({}, 'perturbed1', sd_perturbed)
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 300 + B * beam, hw).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        assert out['step_logits'].shape[1] == B * beam
        _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, label, sensitivity=defects, exempt=exempt)


def test_wide_beam_vatex_1182_keys():
    """Six 224x224 frames per image (1182 image keys, six chunks per item) at beam 8."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    param = {'num_image_with_embedding': 6}
    sd = synthetic_state_dict(param, 2, 'perturbed')
    m = _model(param, 'vatex2', sd)
    B, beam, max_steps = 2, 8, 5
    _beam(m, beam, max_steps)
    frames = [f.cuda() for f in synthetic_images(B, 6, 4322)]
    with _patched(m, sd, _no_eos(sd)) as sd2:
        out = _generate(m, frames)
        _check_beam_run(m, RefWeights(sd2).to('cuda'), B, beam, max_steps, out, 'vatex_b2_k8_m1182')


def test_wide_beam_ragged_batch(sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 3, 6, 8
    _beam(m, beam, max_steps)
    hws = [(128, 128), (224, 224), (160, 96)]
    images = [synthetic_images(1, 0, 40 + b, hw)[0].cuda() for b, hw in enumerate(hws)]
    lens = [(h // 16) * (w // 16) + 1 for h, w in hws]
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'ragged_b3_k6', lens=lens,
                        sensitivity=('wrong_image', 'prev_ancestry'))


def test_wide_beam_per_image_prefixes(sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 3, 8, 10
    _beam(m, beam, max_steps)
    lens = [1, 4, 2]
    prefix = torch.randint(1000, 30000, (B, 4), generator=torch.Generator().manual_seed(18))
    prefix[:, 0] = bst.CLS
    images = synthetic_images(B, 0, 32, (128, 128)).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images, {'prefix': prefix.cuda(), 'prefix_len': torch.tensor(lens)})
        _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'prefix_b3_k8', prefix=prefix,
                        prefix_lens=lens)


def test_wide_beam_images_finish_at_different_steps(sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 6, 5, 24
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 78, (128, 128)).cuda()
    base = float(sd_perturbed['textual.output.bias'][EOS])
    for shift in [30.0 + i for i in range(21)]:
        with _patched(m, sd_perturbed, {'textual.output.bias': (EOS, base + shift)}) as sd:
            out = _generate(m, images)
            rep = beam_replay(out['step_logits'].cpu(), B, beam, max_steps, bst.LENGTH_PENALTY)
            steps = sorted(set(rep['done_step']))
            if len(steps) >= 2 and any(s >= 0 and s < rep['n_steps'] - 1 for s in steps):
                print('BEOS shift %.0f done_step %s n_steps %d' % (shift, rep['done_step'], rep['n_steps']))
                _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'eos_b6_k5')
                return
    pytest.fail('no EOS bias made the images finish at different steps')


def test_wide_beam_across_the_text_cache_growth(sd_perturbed):
    """140 steps at beam 8: the text cache and the indirection tables are re-laid out past 128 positions mid-run."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 1, 8, 140
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 13, (128, 128)).cuda()
    with _patched(m, sd_perturbed, _no_eos(sd_perturbed)) as sd:
        out = _generate(m, images)
        rep = _check_beam_run(m, RefWeights(sd).to('cuda'), B, beam, max_steps, out, 'grow_b1_k8_140')
    anc = ancestry(rep['bidx'], B * beam)[rep['n_steps']]
    assert (anc[:, 128:] != torch.arange(B * beam)[:, None]).any(), 'no foreign read past the growth'


# ---------------------------------------------------------------------------------------------------------------------
# planted ties in the 16-entry lists: test_gpu_beam_step's placements at beam 8 (one thread, across warps, across
# 2048-element rounds, and the pair at places 15 / 16 of every row's list)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('beam', [5, 8])
@pytest.mark.parametrize('which', ['one_thread', 'warps', 'rounds', 'straddle'])
def test_wide_beam_planted_ties_keep_the_lower_index(which, beam, sd_perturbed):
    bst.test_planted_ties_keep_the_lower_index(which, beam, sd_perturbed)


@pytest.mark.parametrize('beam', [6, 8])
def test_wide_beam_one_ulp_pair_keeps_logit_order(beam, sd_perturbed, monkeypatch):
    # At beam 8 the 16-entry lists of this case reach scores near -231 (log-softmax -131 on a beam score of -100), where
    # one fp32 ulp is 1.5e-5: the engine's three roundings there came to 2.57e-5 against the fp64 replay.  The bound is
    # four ulps at that magnitude.
    monkeypatch.setattr(bst, 'CAND_TOL', max(bst.CAND_TOL, 4 * 1.53e-5))
    bst.test_one_ulp_pair_keeps_logit_order_where_scores_collapse(beam, sd_perturbed)


# ---------------------------------------------------------------------------------------------------------------------
# parity mode against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['wide_beam_base_k5', 'wide_beam_base_k8', 'wide_beam_large_k8'])
def test_wide_beam_parity_mode_against_reference(name):
    """fp32-grade parity mode: every step's logits along the oracle's own beam trajectory (raw decode-step API with the
    text-KV re-ordering) within 1e-3 of the fp32 oracle, and the free-running captions token-identical to the
    reference's."""
    from generativeimage2text_b200.model import GeneratorWithBeamSearch
    g = load_golden(name)
    meta = g['meta']
    beam, B = meta['beam'], meta['batch']
    sd, batch = golden_inputs(meta)
    m = tpar._parity_model(meta, sd)
    m.decoder = GeneratorWithBeamSearch(EOS, max_steps=meta['max_steps'], beam_size=beam, length_penalty=0.6)
    m.encode_image(tpar._to_cuda(batch)['image'])
    m.prefill(B, beam=beam)
    feats = git_oracle.visual_features(sd, meta['param'], batch['image'])
    dec = git_oracle.CachedDecoder(sd, feats, beam=beam)
    pending = {'idx': None}
    worst = [0.0]

    def step(ids):
        pos = dec.n_text
        ref = dec.feed(ids[:, pos:])
        mine = m.decoding_step(ids[:, -1], pos, beam_idx=pending['idx']).cpu()
        pending['idx'] = None
        worst[0] = max(worst[0], (mine - ref).abs().max().item())
        return ref

    def reorder(bidx):
        dec.reorder(bidx)
        pending['idx'] = bidx
    pred, _ = git_oracle.beam_search(torch.full((B, 1), 101, dtype=torch.long), step, reorder=reorder,
                                     max_steps=meta['max_steps'], beam=beam)
    assert np.array_equal(pred.numpy(), g['predictions'])
    free = m(tpar._to_cuda(batch))
    torch.cuda.synchronize()
    print('%s [parity]: beam trajectory max |logit - oracle| %.2e' % (name, worst[0]))
    assert worst[0] < tpar.PARITY_ATOL
    assert np.array_equal(free['predictions'].cpu().numpy(), g['predictions'])
    np.testing.assert_allclose(free['logprobs'].cpu().numpy().reshape(-1), g['logprobs'].reshape(-1), rtol=0, atol=2e-3)


# ---------------------------------------------------------------------------------------------------------------------
# sampled beam search
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', [('base', 6, 3, 12, 0.7, 40, 0.9), ('base', 8, 4, 12, 1.0, 0, 0.5),
                                  ('large', 8, 4, 10, 0.7, 30, None)],
                         ids=['base-beam6', 'base-beam8', 'large-beam8'])
def test_wide_beam_sampled_search_replays_the_reference_semantics(case):
    from generativeimage2text_b200.synthetic import synthetic_images
    name, beam, B, steps, T, top_k, top_p = case
    m = bsm._model(name)
    bsm._decoder(m, beam, steps, T)
    img = synthetic_images(B, 0, seed=61 + B).cuda()
    u = torch.rand((steps, B * beam, 2), generator=torch.Generator().manual_seed(beam * 100 + B))
    out = m({'image': img}, return_step_logits=True, search_param={'do_sample': True, 'top_k': top_k, 'top_p': top_p,
                                                                   'uniforms': u})
    assert out['step_logits'].shape[1] == B * beam
    pred, lp, clear = bsm.replay(out, u, torch.full((B, 1), 101, dtype=torch.long), beam, steps, T, top_k, top_p)
    err = bsm._check_replay(out, pred, lp, clear)
    print('%s: %d / %d images compared, max |logprob - replay| = %.3g' % (case, int(clear.sum()), B, err))
    plain = m({'image': img})['predictions'].cpu()
    assert not torch.equal(plain, out['predictions'].cpu())        # it does sample


# ---------------------------------------------------------------------------------------------------------------------
# bit identity
# ---------------------------------------------------------------------------------------------------------------------
def test_wide_beam_num_return_sequences_is_the_repeated_call(sd_perturbed):
    """num_return_sequences = 2 at beam 8, deterministic and sampled, is bit-identical to the call with every image
    repeated."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, n, beam, steps = 3, 2, 8, 12
    _beam(m, beam, steps)
    x = synthetic_images(B, 0, 90, (128, 128)).cuda()
    u = torch.rand((steps, B * n * beam, 2), generator=torch.Generator().manual_seed(3))
    for sp in ({}, {'do_sample': True, 'top_k': 30, 'top_p': 0.9, 'uniforms': u}):
        got = m({'image': x}, return_step_logits=True, search_param=dict(sp, num_return_sequences=n))
        want = m({'image': x.repeat_interleave(n, 0)}, return_step_logits=True, search_param=sp or None)
        torch.cuda.synchronize()
        for k in ('predictions', 'logprobs', 'step_logits'):
            assert torch.equal(got[k], want[k]), (sp.keys(), k)


def test_wide_beam_rows_are_independent_of_the_batch(sd_perturbed):
    """Each image's result in a batch of 5 at beam 7 equals its batch-1 call."""
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, steps = 5, 7, 14
    _beam(m, beam, steps)
    x = synthetic_images(B, 0, 91, (224, 224)).cuda()
    full = m({'image': x})
    torch.cuda.synchronize()
    for b in range(B):
        one = m({'image': x[b:b + 1]})
        torch.cuda.synchronize()
        assert torch.equal(one['predictions'][0], full['predictions'][b]), b
        assert torch.equal(one['logprobs'].reshape(-1)[0], full['logprobs'].reshape(-1)[b]), b


def test_wide_beam_graph_pdl_and_a_fresh_engine_are_bit_identical(sd_perturbed):
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model({}, 'perturbed1', sd_perturbed)
    B, beam, max_steps = 3, 8, 140
    _beam(m, beam, max_steps)
    images = synthetic_images(B, 0, 20, (128, 128)).cuda()
    runs = {}
    try:
        with _patched(m, sd_perturbed, _no_eos(sd_perturbed)):
            for gr in (1, 0):
                for p in (1, 0):
                    m.set_engine_option('use_graph', gr)
                    m.set_engine_option('use_pdl', p)
                    runs[(gr, p)] = _outputs(_generate(m, images))
    finally:
        m.set_engine_option('use_graph', 1)
        m.set_engine_option('use_pdl', 1)
    for key, o in runs.items():
        for k in o:
            assert torch.equal(o[k], runs[(1, 1)][k]), (key, k)
    # warm (a beam-4 and a beam-6 call of other shapes first) against a fresh engine
    img = synthetic_images(4, 0, 70, (128, 128)).cuda()
    _beam(m, 4, 30)
    _generate(m, synthetic_images(9, 0, 71, (224, 224)).cuda())
    _beam(m, 6, 20)
    _generate(m, synthetic_images(7, 0, 72, (128, 128)).cuda())
    _beam(m, 8, 20)
    warm = _outputs(_generate(m, img))
    m.release()
    fresh = _outputs(_generate(m, img))
    for k in warm:
        assert torch.equal(warm[k], fresh[k]), k
