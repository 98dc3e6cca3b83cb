"""GPU parity tests: the CUDA engine (through get_git_model / the C ABI) against the CPU oracle and the
golden vectors produced by the unmodified reference.

Why teacher forcing and margins: the engine multiplies bf16 operands (fp32 accumulate) while the reference
is fp32 end to end, and with random-init weights the greedy top-1/top-2 logit margin is often far below
the bf16 GEMM noise (SURVEY.md section 0 item 5).  So
  * numerics are compared step by step with the reference's own tokens fed back (teacher forcing), with a
    written tolerance, and token equality is required wherever the oracle's decision margin exceeds it;
  * the search semantics (no-repeat, EOS forcing, logprob normalisation, beam bookkeeping, hypothesis
    selection) are checked EXACTLY by replaying the oracle's search loop over the engine's own step logits.
"""
import ctypes
import numpy as np
import pytest
import torch

import git_oracle
from helpers import load_golden, golden_inputs, greedy_margins, golden_greedy_margins

pytestmark = pytest.mark.gpu

LOGIT_ATOL = {'init': 0.06, 'perturbed': 0.25}   # absolute, on logits with std ~0.55 / ~2.2 (bf16 operands)
MARGIN_FACTOR = 2.5                              # a decision must hold when margin > factor * observed error


class Tok:
    cls_token_id, sep_token_id = 101, 102


def _model(meta, sd, search=None, max_steps=None):
    from generativeimage2text_b200.model import get_git_model, AutoRegressiveBeamSearch, GeneratorWithBeamSearch
    m = get_git_model(Tok(), meta['param'])
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    m = m.cuda().eval()
    search = search or meta['search']
    max_steps = max_steps or meta['max_steps']
    if search == 'greedy':
        m.decoder = AutoRegressiveBeamSearch(102, max_steps=max_steps, beam_size=1, per_node_beam_size=1,
                                             fix_missing_prefix=True)
    else:
        m.decoder = GeneratorWithBeamSearch(102, max_steps=max_steps, beam_size=4, length_penalty=0.6)
    return m


def _to_cuda(batch):
    out = {}
    for k, v in batch.items():
        out[k] = [x.cuda() for x in v] if isinstance(v, (list, tuple)) else v.cuda()
    return out


@pytest.mark.parametrize('name', ['base_greedy', 'vatex_greedy', 'large_greedy', 'base_ratio_greedy', 'base_crop160_greedy',
                                  'base_vqa_ratio_greedy'])
def test_image_features_and_projection(name):
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    feats = m.encode_image(_to_cuda(batch)['image'])
    vproj = m.prefill(meta['batch'])
    torch.cuda.synchronize()
    ref = git_oracle.visual_features(sd, meta['param'], batch['image'])
    refp = git_oracle.project_visual(sd, ref)
    err = (feats.cpu() - ref).abs()
    errp = (vproj.cpu() - refp).abs()
    print('%s: features max %.4f mean %.5f | vproj max %.4f mean %.5f' % (name, err.max(), err.mean(), errp.max(), errp.mean()))
    # unit-variance LayerNorm outputs after 12/24 bf16-operand blocks
    assert err.mean().item() < 0.01 and err.max().item() < 0.15
    assert errp.mean().item() < 0.01 and errp.max().item() < 0.15
    # and directly against what the unmodified reference produced
    np.testing.assert_allclose(feats.cpu()[:, ::17, ::29].numpy(), g['feats_sample'], rtol=0, atol=0.15)
    np.testing.assert_allclose(vproj.cpu()[:, ::17, ::29].numpy(), g['vproj_sample'], rtol=0, atol=0.15)


@pytest.mark.parametrize('name', ['base_greedy_init', 'base_greedy', 'base_prefix', 'vatex_greedy', 'large_greedy',
                                  'base_ratio_greedy', 'base_crop160_greedy', 'base_vqa_ratio_greedy'])
def test_greedy_teacher_forced_against_reference(name):
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    P = len(meta.get('prefix', [101]))
    raw = []
    ref = git_oracle.generate(sd, meta['param'], batch, 'greedy', meta['max_steps'], cached=True, raw_trace=raw)
    ref_pred = ref['predictions']
    full_ref = torch.cat([batch['prefix'].long(), ref_pred], dim=1) if 'prefix' in batch else ref_pred
    assert np.array_equal(ref_pred.numpy(), g['predictions'])          # oracle == reference (pinned on CPU too)
    m = _model(meta, sd)
    forced = torch.full((meta['batch'], meta['max_steps']), 102, dtype=torch.long)
    forced[:, :full_ref.shape[1]] = full_ref
    out = m(_to_cuda(batch), forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    own = out['predictions'].cpu()
    assert own.shape == ref_pred.shape
    atol = LOGIT_ATOL[meta['variant']]
    cols = torch.from_numpy(g['vocab_cols'])
    worst = 0.0
    n_dec = n_checked = 0
    for i, r in enumerate(raw):
        e = (z[i] - r).abs().max().item()
        worst = max(worst, e)
        # the reference's own numbers at the sampled columns
        np.testing.assert_allclose(z[i][:, cols].numpy(), g['step_logits'][i], rtol=0, atol=atol)
        tok_in = None if i == 0 else full_ref[:, P + i - 1]
        margin = greedy_margins(r, tok_in)
        col = (0 if 'prefix' in batch else P) + i
        for b in range(meta['batch']):
            n_dec += 1
            if margin[b].item() > MARGIN_FACTOR * atol:
                n_checked += 1
                assert own[b, col].item() == ref_pred[b, col].item(), (name, i, b, margin[b].item())
    print('%s: max |logit - oracle| %.4f (atol %.2f); %d/%d decisions above the margin all agree' % (
        name, worst, atol, n_checked, n_dec))
    assert worst < atol
    agree = (own == ref_pred).float().mean().item()
    print('%s: teacher-forced argmax agreement overall %.3f' % (name, agree))
    assert agree > 0.8


@pytest.mark.parametrize('name', ['base_greedy', 'base_prefix'])
def test_greedy_search_semantics_replay(name):
    """Exact: the oracle's AutoRegressiveBeamSearch restatement run over the ENGINE's logits must give the
    engine's tokens and logprobs (no-repeat, EOS forcing, accumulation, / num_valid, prefix stripping)."""
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    out = m(_to_cuda(batch), return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    it = iter(range(z.shape[0]))
    start = batch['prefix'].long() if 'prefix' in batch else torch.full((meta['batch'], 1), 101, dtype=torch.long)
    pred, lp = git_oracle.greedy_search(start, lambda partial: z[next(it)], max_steps=meta['max_steps'])
    if 'prefix' in batch:
        pred = pred[:, start.shape[1]:]
    assert torch.equal(pred, out['predictions'].cpu())
    assert torch.allclose(lp, out['logprobs'].cpu(), atol=2e-3)


def test_greedy_eos_forcing_and_early_exit():
    """Bias the LM head towards EOS so rows end at different steps: exercises EOS forcing (one-hot
    distribution), the all-EOS early break and the num_valid normalisation, replayed exactly."""
    g = load_golden('base_greedy')
    meta = dict(g['meta'])
    sd, batch = golden_inputs(meta)
    sd = dict(sd)
    bias = sd['textual.output.bias'].clone()
    bias[102] += 9.5
    sd['textual.output.bias'] = bias
    m = _model(meta, sd, max_steps=40)
    out = m(_to_cuda(batch), return_step_logits=True)
    torch.cuda.synchronize()
    own = out['predictions'].cpu()
    z = out['step_logits'].cpu()
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.greedy_search(torch.full((meta['batch'], 1), 101, dtype=torch.long),
                                        lambda partial: z[next(it)], max_steps=40)
    print('eos test: lengths', own.shape, 'first eos cols', [(row == 102).nonzero()[:1].flatten().tolist() for row in own])
    assert torch.equal(pred, own)
    assert torch.allclose(lp, out['logprobs'].cpu(), atol=2e-3)
    assert (own == 102).any()


@pytest.mark.parametrize('name', ['base_beam', 'large_beam'])
def test_beam_search_semantics_replay(name):
    """Exact: GeneratorWithBeamSearch restatement over the engine's own step logits reproduces the engine's
    device-side bookkeeping (top-2*beam, hypotheses, is_done, beam re-ordering, EOS padding, scores)."""
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    out = m(_to_cuda(batch), return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.beam_search(torch.full((meta['batch'], 1), 101, dtype=torch.long),
                                      lambda ids: z[next(it)], max_steps=meta['max_steps'])
    assert torch.equal(pred, out['predictions'].cpu())
    assert torch.allclose(lp, out['logprobs'].cpu(), atol=2e-3)


@pytest.mark.parametrize('name', ['base_beam', 'large_beam'])
def test_beam_decode_path_against_oracle_trajectory(name):
    """The reference's beam trajectory (oracle-decided) drives the engine's raw decode-step API including the
    text-KV re-ordering by beam_idx; logits are compared at every step, and the final result with the golden."""
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    B = meta['batch']
    m.encode_image(_to_cuda(batch)['image'])
    m.prefill(B, beam=4)
    feats = git_oracle.visual_features(sd, meta['param'], batch['image'])
    dec = git_oracle.CachedDecoder(sd, feats, beam=4)
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

    pred, lp = git_oracle.beam_search(torch.full((B, 1), 101, dtype=torch.long), step, reorder=reorder,
                                      max_steps=meta['max_steps'])
    assert np.array_equal(pred.numpy(), g['predictions'])
    print('%s: beam trajectory max |logit - oracle| %.4f' % (name, worst[0]))
    assert worst[0] < LOGIT_ATOL[meta['variant']]


def test_generate_host_and_tensor_vs_list_input():
    """C-ABI host-buffer entry point == device entry point; a bare tensor and a one-element list give the same
    captions for an image model (no temporal embeddings)."""
    import ctypes
    from generativeimage2text_b200 import _lib
    g = load_golden('base_greedy')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd, max_steps=12)
    a = m({'image': batch['image'].cuda()})
    b = m({'image': [batch['image'].cuda()]})
    _same_captions(a, b)
    lib, stream = m._ensure_engine()
    img = batch['image'].contiguous().pin_memory()
    toks = torch.empty((meta['batch'], 12), dtype=torch.long).pin_memory()
    lps = torch.empty((meta['batch'],), dtype=torch.float32).pin_memory()
    n = ctypes.c_int32(0)
    sp = m._search_struct()
    _lib.check(lib.gitb200_generate_host(m._engine, img.data_ptr(), meta['batch'], 0, None, 0, ctypes.byref(sp),
                                         toks.data_ptr(), lps.data_ptr(), ctypes.byref(n), stream), m._engine, 'generate_host')
    assert n.value == a['predictions'].shape[1]
    _same_captions(a, {'predictions': toks[:, :n.value].cuda(), 'logprobs': lps.cuda()})


def _same_captions(a, b):
    """Two runs of the same input must agree BIT FOR BIT: split-K partial sums are stored per split and added in split
    order by the consumer kernel (no floating-point atomics anywhere on the path), so neither the launch mode (one call,
    calls in flight on several engine slots, batches coalesced into one launch) nor the run changes a result."""
    pa, pb = a['predictions'], b['predictions']
    assert pa.shape == pb.shape
    assert torch.equal(pa, pb)
    assert torch.equal(a['logprobs'].reshape(-1), b['logprobs'].reshape(-1))


def test_one_kernel_decode_step_matches_the_kernel_chain():
    """Greedy batches of <= 64 run each decode step as ONE persistent kernel (decode_mega.cuh); the same call through the
    45-launch chain (use_mega = 0) must give the same step logits up to the two paths' different bf16 roundings inside the
    attention (the chain multiplies fp32 q with bf16 K on CUDA cores, the persistent kernel runs q.K and p.V on mma.sync)."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    meta = {'param': {}, 'search': 'greedy', 'max_steps': 20}
    sd = synthetic_state_dict({}, 1, 'perturbed')
    for rows in (64, 37, 3):
        img = synthetic_images(rows, 0, 555 + rows).cuda()
        m = _model(meta, sd)
        a = m({'image': img}, return_step_logits=True)
        forced = torch.full((rows, 20), 102, dtype=torch.long)
        forced[:, :a['predictions'].shape[1]] = a['predictions'].cpu()
        za = m({'image': img}, forced_tokens=forced, return_step_logits=True)['step_logits'].clone()
        m.set_engine_option('use_mega', 0)
        zb = m({'image': img}, forced_tokens=forced, return_step_logits=True)['step_logits'].clone()
        torch.cuda.synchronize()
        err = (za - zb).abs().max().item()
        print('rows %d: one-kernel step vs kernel chain, max |dlogit| %.4f' % (rows, err))
        assert err < 0.1


def test_runs_are_bit_reproducible():
    """The same batch three times (fresh launches, replayed step graphs): identical tokens, logprobs and step logits."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    meta = {'param': {}, 'search': 'greedy', 'max_steps': 24}
    sd = synthetic_state_dict({}, 0, 'init')
    img = synthetic_images(48, 0, 4242).cuda()
    m = _model(meta, sd)
    outs = [m({'image': img}, return_step_logits=True) for _ in range(3)]
    torch.cuda.synchronize()
    for o in outs[1:]:
        _same_captions(outs[0], o)
        assert torch.equal(outs[0]['step_logits'], o['step_logits'])
    mb = _model(dict(meta, search='beam', max_steps=12), sd)
    b1, b2 = mb({'image': img[:6]}), mb({'image': img[:6]})
    _same_captions(b1, b2)


def test_pipelined_submit_matches_sync_calls():
    """Two batches in flight on the two engine slots give the same captions as one-at-a-time calls."""
    g = load_golden('base_greedy')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model(meta, sd, max_steps=12)
    imgs = [synthetic_images(2, 0, 500 + i).cuda() for i in range(4)]
    sync = [m({'image': x}) for x in imgs]
    pend = [m.submit({'image': x}) for x in imgs[:2]]
    outs = [pend[0].result(), pend[1].result()]
    pend = [m.submit({'image': x}) for x in imgs[2:]]
    outs += [p.result() for p in pend]
    for a, b in zip(sync, outs):
        _same_captions(a, b)
    assert m.launch_count() > 0


def test_engine_slots_share_one_weight_copy():
    """All engine slots borrow slot 0's parameters (gitb200_share_weights); four batches in flight on four slots give the
    captions of one-at-a-time calls."""
    g = load_golden('base_greedy')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    from generativeimage2text_b200.synthetic import synthetic_images
    from generativeimage2text_b200 import _lib
    m = _model(meta, sd, max_steps=12)
    imgs = [synthetic_images(2, 0, 700 + i).cuda() for i in range(4)]
    sync = [m({'image': x}) for x in imgs]
    pend = [m.submit({'image': x}, depth=4) for x in imgs]
    for a, p in zip(sync, pend):
        _same_captions(a, p.result())
    # a borrowing engine refuses its own parameters; its owner does not
    lib = _lib.load()
    eng1 = m._slots[1]['engine']
    assert eng1 is not None
    w = torch.zeros(768, device='cuda')
    shape = (ctypes.c_int64 * 1)(768)
    rc = lib.gitb200_set_weight(eng1, b'image_encoder.class_embedding', w.data_ptr(), shape, 1, _lib.F32, None)
    assert rc != 0 and b'borrows' in lib.gitb200_last_error(eng1)


def test_coalesced_submit_matches_sync_calls():
    """Dynamic batching: batches submitted one by one with coalesce=k share one engine launch (one decode chain over
    all their rows); every handle must return its own batch's result -- shapes as the reference's per-batch loop would
    give them, captions equal to one-at-a-time calls up to run-to-run noise."""
    g = load_golden('base_greedy')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    from generativeimage2text_b200.synthetic import synthetic_images
    m = _model(meta, sd, max_steps=12)
    imgs = [synthetic_images(2 + (i % 2), 0, 900 + i).cuda() for i in range(5)]     # batches of 2 and 3 rows
    sync = [m({'image': x}) for x in imgs]
    launches0 = m.launch_count()
    pend = [m.submit({'image': x}, depth=2, coalesce=3) for x in imgs]      # groups: [0,1,2] launched, [3,4] still open
    assert m._open_group is not None and len(m._open_group.rows) == 2
    outs = [p.result() for p in pend]                                       # asking for a result launches the open group
    assert m._open_group is None
    for a, b, x in zip(sync, outs, imgs):
        assert b['predictions'].shape[0] == x.shape[0]
        _same_captions(a, b)
    assert m.launch_count() > launches0
    # a list input (video frames) coalesces frame by frame; a prefix or a parity hook is never coalesced
    vg = load_golden('vatex_greedy')
    vsd, vbatch = golden_inputs(vg['meta'])
    vm = _model(vg['meta'], vsd, max_steps=8)
    frames_a = [f.cuda() for f in vbatch['image']]
    frames_b = [f.flip(-1).contiguous() for f in frames_a]
    ra, rb = vm({'image': frames_a}), vm({'image': frames_b})
    pa, pb = vm.submit({'image': frames_a}, coalesce=2), vm.submit({'image': frames_b}, coalesce=2)
    _same_captions(ra, pa.result())
    _same_captions(rb, pb.result())
    h = m.submit({'image': imgs[0][:1], 'prefix': torch.tensor([[101, 2054]]).cuda()}, coalesce=4)
    assert h.result()['predictions'].shape[0] == 1 and m._open_group is None


# ------------------------------------------------------------------------------------------------------------------
# The benchmarked configurations themselves (BASELINE.json configs 2-4), against goldens of the unmodified reference
# ------------------------------------------------------------------------------------------------------------------
def _teacher_forced_vs_golden(name):
    """Teacher-forced run with the reference's tokens; every step's logits at the golden's sampled columns within the
    written tolerance of the reference's own numbers, and the engine's decision equal to the reference's wherever the
    reference's margin (from its stored top-4) is decisive."""
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    ref_pred = torch.from_numpy(g['predictions'])
    B = ref_pred.shape[0]
    m = _model(meta, sd)
    forced = torch.full((B, meta['max_steps']), 102, dtype=torch.long)
    forced[:, :ref_pred.shape[1]] = ref_pred
    out = m(_to_cuda(batch), forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    own = out['predictions'].cpu()
    assert own.shape == ref_pred.shape
    atol = LOGIT_ATOL[meta['variant']]
    cols = torch.from_numpy(g['vocab_cols']).cuda()
    worst, n_dec, n_checked = 0.0, 0, 0
    for i in range(g['step_logits'].shape[0]):
        z = out['step_logits'][i][:, cols].cpu().numpy()
        worst = max(worst, float(np.abs(z - g['step_logits'][i]).max()))
        margin = golden_greedy_margins(g, i, None if i == 0 else g['predictions'][:, i])
        for b in range(B):
            n_dec += 1
            if margin[b] > MARGIN_FACTOR * atol:
                n_checked += 1
                assert own[b, i + 1].item() == ref_pred[b, i + 1].item(), (name, i, b, margin[b])
    print('%s: max |logit - reference| at the sampled columns %.4f (atol %.2f); %d/%d decisions above the margin all agree' % (
        name, worst, atol, n_checked, n_dec))
    assert worst < atol


def test_config2_base_greedy_batch64_against_reference():
    """BASELINE.json config 2 as benchmarked (GIT_BASE, 64 images, greedy, max_len 40, bench.py's checkpoint and pixels):
    64-row swap-AB decode GEMM tiles, 296-CTA decode attention with several items per CTA."""
    _teacher_forced_vs_golden('base_greedy_b64')


def test_config4_vatex_batch16_against_reference():
    """BASELINE.json config 4 (GIT_BASE_VATEX, 16 x 6 frames, M = 1182 image tokens: chunked K/V staging)."""
    _teacher_forced_vs_golden('vatex_greedy_b16')


def test_config3_large_beam_batch32_against_reference_trajectory():
    """BASELINE.json config 3 (GIT_LARGE, 32 images x beam 4 = 128 rows): the engine's raw decode-step API driven along
    the trajectory of the reference's own beam search (newest tokens + re-ordering from the golden), logits compared with
    the reference's at the sampled columns at every step; then the engine's own device-side search, replayed exactly."""
    g = load_golden('large_beam_b32')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    B = meta['batch']
    m.encode_image(batch['image'].cuda())
    m.prefill(B, beam=4)
    cols = torch.from_numpy(g['vocab_cols']).cuda()
    atol = LOGIT_ATOL[meta['variant']]
    worst = 0.0
    for i in range(g['step_tokens'].shape[0]):
        bidx = None if i == 0 else torch.from_numpy(g['step_beam_idx'][i])
        z = m.decoding_step(torch.from_numpy(g['step_tokens'][i]), i, beam_idx=bidx)
        worst = max(worst, float((z[:, cols].cpu().numpy() - g['step_logits'][i]).__abs__().max()))
    print('large_beam_b32: %d steps x 128 rows, max |logit - reference| at the sampled columns %.4f' % (g['step_tokens'].shape[0], worst))
    assert worst < atol
    out = m({'image': batch['image'].cuda()}, return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.beam_search(torch.full((B, 1), 101, dtype=torch.long), lambda ids: z[next(it)], max_steps=meta['max_steps'])
    assert torch.equal(pred, out['predictions'].cpu())
    assert torch.allclose(lp, out['logprobs'].cpu(), atol=2e-3)


def test_coalesced_256_rows_against_reference():
    """bench.py's serving mode: four batches of 64 submitted one by one share ONE engine launch (256-row decode tiles, ~10
    (image, head) items per attention CTA).  Each member must return exactly what a call of its own returns, and the
    256-row launch is checked against the reference teacher-forced (rows 0-63 = the golden's batch, the other members are
    different pixels)."""
    from generativeimage2text_b200.synthetic import synthetic_images
    g = load_golden('base_greedy_b64')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    # like with like: a 256-row launch runs the kernel chain, so the one-call-at-a-time results it is compared with must
    # too (64-row calls default to the persistent one-kernel step, whose attention rounds differently;
    # test_one_kernel_decode_step_matches_the_kernel_chain bounds that difference)
    m.set_engine_option('use_mega', 0)
    imgs = [batch['image'].cuda()] + [synthetic_images(64, 0, 9000 + i).cuda() for i in range(3)]
    solo = [m({'image': x}) for x in imgs]
    pend = [m.submit({'image': x}, depth=2, coalesce=4) for x in imgs]
    for a, p in zip(solo, pend):
        _same_captions(a, p.result())
    # the 256-row launch itself against the reference: teacher forcing needs one call, so the four batches go in as one
    big = torch.cat(imgs, dim=0)
    ref_pred = torch.from_numpy(g['predictions'])
    forced = torch.full((256, meta['max_steps']), 102, dtype=torch.long)
    forced[:64, :ref_pred.shape[1]] = ref_pred
    forced[64:] = torch.cat([s['predictions'] for s in solo[1:]], dim=0).cpu()
    out = m({'image': big}, forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    cols = torch.from_numpy(g['vocab_cols']).cuda()
    worst = 0.0
    for i in range(g['step_logits'].shape[0]):
        worst = max(worst, float(np.abs(out['step_logits'][i][:64][:, cols].cpu().numpy() - g['step_logits'][i]).max()))
    print('256-row launch, rows 0-63: max |logit - reference| at the sampled columns %.4f' % worst)
    assert worst < LOGIT_ATOL[meta['variant']]


def test_decisive_checkpoint_free_running_token_identity():
    """SURVEY.md section 7 hard part 1b: on a checkpoint whose every greedy decision has a margin many times the engine's
    logit error, the FREE-RUNNING engine output must equal the unmodified reference's `predictions` token for token."""
    g = load_golden('base_decisive')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    # measured error of this checkpoint (teacher-forced, all 30522 columns, against the oracle)
    raw = []
    ref = git_oracle.generate(sd, meta['param'], batch, 'greedy', meta['max_steps'], cached=True, raw_trace=raw)
    assert np.array_equal(ref['predictions'].numpy(), g['predictions'])
    forced = torch.full((meta['batch'], meta['max_steps']), 102, dtype=torch.long)
    forced[:, :ref['predictions'].shape[1]] = ref['predictions']
    tf = m(_to_cuda(batch), forced_tokens=forced, return_step_logits=True)
    err = max((tf['step_logits'][i].cpu() - r).abs().max().item() for i, r in enumerate(raw))
    min_margin = float(g['min_margin'])
    print('decisive checkpoint: min reference margin %.3f, measured max |logit error| %.4f (ratio %.1f)' % (min_margin, err, min_margin / err))
    assert min_margin >= 4.0 * err
    out = m(_to_cuda(batch))
    torch.cuda.synchronize()
    assert np.array_equal(out['predictions'].cpu().numpy(), g['predictions'])
    np.testing.assert_allclose(out['logprobs'].cpu().numpy(), g['logprobs'], rtol=0, atol=5e-2)


def test_beam_images_finish_at_different_steps():
    """Beam search with B > 1 where images end at different steps (EOS-biased LM head): the device-side bookkeeping
    (per-image done flags, the all-done early exit) replayed exactly by the oracle's loop over the engine's step logits."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    sd = dict(synthetic_state_dict({}, 0, 'perturbed'))
    bias = sd['textual.output.bias'].clone()
    bias[102] += 7.0
    sd['textual.output.bias'] = bias
    meta = {'param': {}, 'search': 'beam', 'max_steps': 24}
    m = _model(meta, sd)
    img = synthetic_images(12, 0, 31337).cuda()
    for rep_ in range(3):
        out = m({'image': img}, return_step_logits=True)
        torch.cuda.synchronize()
        z = out['step_logits'].cpu()
        it = iter(range(z.shape[0]))
        pred, lp = git_oracle.beam_search(torch.full((12, 1), 101, dtype=torch.long), lambda ids: z[next(it)], max_steps=24)
        assert torch.equal(pred, out['predictions'].cpu())
        assert torch.allclose(lp, out['logprobs'].cpu(), atol=2e-3)
    ends = [(row == 102).nonzero()[:1].flatten().tolist() for row in out['predictions'].cpu()]
    print('beam: first EOS column per image', ends)


def test_long_max_steps_grows_the_text_cache():
    """The shipped default decoder has max_steps = 1024: the text K/V cache starts at 128 positions and is re-laid-out when
    a caption outgrows it; steps go out in chunks of 64 with the `finished` flag read back in between."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    sd = synthetic_state_dict({}, 0, 'init')
    img = synthetic_images(3, 0, 99).cuda()
    short = _model({'param': {}, 'search': 'greedy', 'max_steps': 200}, sd)
    a = short({'image': img})
    long_ = _model({'param': {}, 'search': 'greedy', 'max_steps': 320}, sd)
    b = long_({'image': img})
    torch.cuda.synchronize()
    assert a['predictions'].shape[1] == 200 and b['predictions'].shape[1] == 320      # random weights never emit EOS
    assert torch.equal(a['predictions'], b['predictions'][:, :200])
    # an EOS-biased checkpoint ends early: the loop must stop enqueueing (default beam decoder, max_steps 1024)
    sd2 = dict(sd)
    bias = sd2['textual.output.bias'].clone()
    bias[102] += 12.0
    sd2['textual.output.bias'] = bias
    from generativeimage2text_b200.model import get_git_model
    m = get_git_model(Tok(), {})
    m.load_state_dict(sd2, strict=False)
    m = m.cuda().eval()                       # decoder: GeneratorWithBeamSearch(max_steps=1024), the shipped default
    before = m.launch_count()
    out = m({'image': img})
    torch.cuda.synchronize()
    assert out['predictions'].shape == (3, 1024)
    assert m.launch_count() - before < 400 * 48, 'the beam loop enqueued (almost) all 1023 steps'


# ------------------------------------------------------------------------------------------------------------------
# fp32-grade parity mode (engine option 'parity'): the north star's "logits within 1e-3", token-identical greedy output
# ------------------------------------------------------------------------------------------------------------------
PARITY_ATOL = 1e-3


def _parity_model(meta, sd, **kw):
    m = _model(meta, sd, **kw)
    m.set_engine_option('parity', 1)
    return m


@pytest.mark.parametrize('name', ['base_greedy_init', 'base_greedy', 'base_prefix', 'vatex_greedy', 'large_greedy',
                                  'base_ratio_greedy', 'base_decisive'])
def test_parity_mode_logits_within_1e3_of_the_fp32_reference(name):
    """Every GEMM as a three-term (hi, lo) bf16 split product through the same wgmma kernels, fp32 attention and caches:
    image features, visual projection and every step's full logit row within 1e-3 of the fp32 oracle (and of the
    reference's own numbers at the golden's sampled columns), teacher-forced; decisions equal wherever the margin exceeds
    2.5x the measured error; and the FREE-RUNNING captions equal the reference's whenever every margin along the way does."""
    g = load_golden(name)
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    P = len(meta.get('prefix', [101]))
    raw = []
    ref = git_oracle.generate(sd, meta['param'], batch, 'greedy', meta['max_steps'], cached=True, raw_trace=raw)
    ref_pred = ref['predictions']
    full_ref = torch.cat([batch['prefix'].long(), ref_pred], dim=1) if 'prefix' in batch else ref_pred
    m = _parity_model(meta, sd)
    feats = m.encode_image(_to_cuda(batch)['image'])
    vproj = m.prefill(meta['batch'])
    torch.cuda.synchronize()
    rf = git_oracle.visual_features(sd, meta['param'], batch['image'])
    e_f = (feats.cpu() - rf).abs().max().item()
    e_p = (vproj.cpu() - git_oracle.project_visual(sd, rf)).abs().max().item()
    forced = torch.full((meta['batch'], meta['max_steps']), 102, dtype=torch.long)
    forced[:, :full_ref.shape[1]] = full_ref
    out = m(_to_cuda(batch), forced_tokens=forced, return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    own = out['predictions'].cpu()
    cols = torch.from_numpy(g['vocab_cols'])
    worst = max((z[i] - r).abs().max().item() for i, r in enumerate(raw))
    print('%s [parity]: features max err %.2e, vproj %.2e, logits %.2e (north star: 1e-3)' % (name, e_f, e_p, worst))
    assert e_f < PARITY_ATOL and e_p < PARITY_ATOL and worst < PARITY_ATOL
    min_margin = float('inf')
    for i, r in enumerate(raw):
        np.testing.assert_allclose(z[i][:, cols].numpy(), g['step_logits'][i], rtol=0, atol=PARITY_ATOL + 5e-4)
        tok_in = None if i == 0 else full_ref[:, P + i - 1]
        margin = greedy_margins(r, tok_in)
        col = (0 if 'prefix' in batch else P) + i
        for b in range(meta['batch']):
            if tok_in is not None and tok_in[b].item() == 102:
                continue                                     # the row has ended: EOS is forced
            min_margin = min(min_margin, margin[b].item())
            if margin[b].item() > 2.5 * worst:
                assert own[b, col].item() == ref_pred[b, col].item(), (name, i, b, margin[b].item())
    free = m(_to_cuda(batch))
    torch.cuda.synchronize()
    same = free['predictions'].shape == ref_pred.shape and bool((free['predictions'].cpu() == ref_pred).all())
    print('%s [parity]: smallest reference margin %.2e; free-running captions token-identical: %s' % (name, min_margin, same))
    if min_margin > 4 * worst:
        assert same
        np.testing.assert_allclose(free['logprobs'].cpu().numpy().reshape(-1), g['logprobs'].reshape(-1), rtol=0, atol=2e-3)


def test_parity_mode_beam_trajectory():
    """Beam search rows (4 beams per image sharing the fp32 image K/V, text K/V re-ordered by beam_idx) in parity mode."""
    g = load_golden('base_beam')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _parity_model(meta, sd)
    B = meta['batch']
    m.encode_image(_to_cuda(batch)['image'])
    m.prefill(B, beam=4)
    feats = git_oracle.visual_features(sd, meta['param'], batch['image'])
    dec = git_oracle.CachedDecoder(sd, feats, beam=4)
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

    pred, lp = git_oracle.beam_search(torch.full((B, 1), 101, dtype=torch.long), step, reorder=reorder, max_steps=meta['max_steps'])
    assert np.array_equal(pred.numpy(), g['predictions'])
    print('base_beam [parity]: beam trajectory max |logit - oracle| %.2e' % worst[0])
    assert worst[0] < PARITY_ATOL


# ------------------------------------------------------------------------------------------------------------------
# SURVEY.md section 8f-4: prefix batches with B > 1 (the reference asserts batch 1, layers/decoder.py:985-989)
# ------------------------------------------------------------------------------------------------------------------
def _prefix_batch(m, img, prefixes):
    P = max(len(p) for p in prefixes)
    pad = torch.full((len(prefixes), P), 0, dtype=torch.long)
    for r, p in enumerate(prefixes):
        pad[r, :len(p)] = torch.tensor(p)
    return m({'image': img, 'prefix': pad.cuda(), 'prefix_len': torch.tensor([len(p) for p in prefixes])})


@pytest.mark.parametrize('search', ['greedy', 'beam'])
def test_prefix_batches_one_prefix_per_image(search):
    """A batch of (image, question) pairs with ragged question lengths: every row must be what a batch-1 call with that
    row's own prefix returns.  (1) The result of a row does not depend on which other rows share its batch (exact).
    (2) Against the reference-shaped batch-1 path (shared prefix fed first, then the search): token-identical on every row
    whose reference decisions are all decisive (margins from the CPU oracle), logprobs within the bf16 noise."""
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    meta = {'param': {}, 'search': search, 'max_steps': 14}
    sd = synthetic_state_dict({}, 0, 'decisive')
    m = _model(meta, sd)
    img = synthetic_images(5, 0, 4711)
    prefixes = [[101, 2054, 2003], [101, 2129, 2116, 2111, 2024], [101], [101, 2054], [101, 3585, 2003, 1996]]
    full = _prefix_batch(m, img.cuda(), prefixes)
    torch.cuda.synchronize()
    assert full['predictions'].shape[0] == 5
    # (1) composition invariance
    for rows in ([0, 1], [1, 2], [3, 4], [4, 0]):
        sub = _prefix_batch(m, img[rows].cuda(), [prefixes[r] for r in rows])
        for i, r in enumerate(rows):
            a, b = full['predictions'][r], sub['predictions'][i]
            w = min(a.numel(), b.numel())
            assert torch.equal(a[:w], b[:w]) and bool((a[w:] == 102).all()) and bool((b[w:] == 102).all()), (search, rows, r)
            assert torch.equal(full['logprobs'].reshape(-1)[r], sub['logprobs'].reshape(-1)[i])
    # (2) against batch-1 calls through the reference-shaped path
    n_checked = 0
    for r, p in enumerate(prefixes):
        one = m({'image': img[r:r + 1].cuda(), 'prefix': torch.tensor([p]).cuda()}) if len(p) > 1 else m({'image': img[r:r + 1].cuda()})
        pred1 = one['predictions'][0]
        if len(p) == 1 and search == 'greedy':
            pred1 = pred1[1:]                     # the un-prefixed greedy result keeps its start token
        if len(p) == 1 and search == 'beam':
            pred1 = pred1[1:]
        trace = []
        git_oracle.generate(sd, {}, {'image': img[r:r + 1], **({'prefix': torch.tensor([p])} if len(p) > 1 else {})}, search, 14,
                            cached=True, trace=trace)
        if search == 'greedy':
            margins = [float((z.topk(2, dim=1).values[:, 0] - z.topk(2, dim=1).values[:, 1]).min()) for z in trace]
            decisive = min(m_ for m_ in margins if np.isfinite(m_)) > 0.3
        else:
            decisive = False                      # beam margins involve the candidate lists: reported, not asserted
        a = full['predictions'][r]
        w = min(a.numel(), pred1.numel())
        same = torch.equal(a[:w], pred1[:w]) and bool((a[w:] == 102).all()) and bool((pred1[w:] == 102).all())
        print('%s row %d (prefix %d tokens): batch row == batch-1 call: %s%s' % (search, r, len(p), same, ' [decisive]' if decisive else ''))
        if decisive:
            n_checked += 1
            assert same
            assert abs(full['logprobs'].reshape(-1)[r].item() - one['logprobs'].reshape(-1)[0].item()) < 5e-2
    print('%s: %d rows had only decisive reference decisions' % (search, n_checked))


# ---- the remaining decoders (SURVEY.md 8f-4) --------------------------------------------------------------------------------
def _trie_from_reference_captions(pred, extra_seed=0):
    """A vocabulary trie that contains the free-running greedy captions' first tokens plus decoys, so that the constraint
    both binds and leaves real choices: sequences of 3-6 tokens ending in EOS."""
    g = torch.Generator().manual_seed(extra_seed)
    seqs = []
    for row in pred.tolist():
        body = [t for t in row[1:] if t != 102][:4]
        seqs.append(body + [102])
        for _ in range(6):                                   # decoys sharing a prefix of the row's own caption
            cut = int(torch.randint(0, len(body) + 1, (1,), generator=g))
            tail = torch.randint(1000, 30000, (int(torch.randint(1, 4, (1,), generator=g)),), generator=g).tolist()
            seqs.append(body[:cut] + tail + [102])
    for _ in range(40):
        seqs.append(torch.randint(1000, 30000, (int(torch.randint(2, 6, (1,), generator=g)),), generator=g).tolist() + [102])
    return seqs


def test_trie_decoder_replays_the_reference_semantics():
    """TrieAutoRegressiveBeamSearch (reference trie_decoder.py:27-218) on the device: the oracle's restatement (pinned
    against the reference class in tests/test_oracle_vs_reference.py) run over the ENGINE's own step logits must give the
    engine's tokens and log-probs exactly; every caption is a path of the trie; rows of a batch equal their batch-1 calls."""
    from generativeimage2text_b200.model import TrieAutoRegressiveBeamSearch, TokenTrie
    g = load_golden('base_greedy')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd, max_steps=12)
    free = m(_to_cuda(batch))['predictions'].cpu()
    seqs = _trie_from_reference_captions(free)
    trie = TokenTrie.construct(seqs)
    m.decoder = TrieAutoRegressiveBeamSearch(102, max_steps=12, beam_size=1, trie=trie)
    out = m(_to_cuda(batch), return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    it = iter(range(z.shape[0]))
    B = meta['batch']
    start = torch.full((B, 1), 101, dtype=torch.long)
    pred, lp = git_oracle.trie_search(start, lambda partial: z[next(it)], trie.to_csr(), max_steps=12)
    own = out['predictions'].cpu()
    print('trie captions:', own.tolist())
    assert torch.equal(pred, own)
    assert torch.allclose(lp, out['logprobs'].cpu(), rtol=1e-4, atol=2e-3)
    for row in own.tolist():
        body = row[1:]
        cut = body.index(102) + 1 if 102 in body else len(body)
        assert body[:cut] in seqs, body                      # the constraint binds
    # a batch row == its own batch-1 call (each row owns a trie cursor), and the trie can be swapped / removed
    one = m({'image': batch['image'][1:2].cuda()})
    n = one['predictions'].shape[1]
    assert torch.equal(one['predictions'].cpu()[0], own[1, :n]) and bool((own[1, n:] == 102).all())
    from generativeimage2text_b200.model import AutoRegressiveBeamSearch
    m.decoder = AutoRegressiveBeamSearch(102, max_steps=12, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    again = m(_to_cuda(batch))['predictions'].cpu()
    assert torch.equal(again, free)


@pytest.mark.parametrize('temperature', [1.0, 0.7])
def test_sampling_replays_the_reference_semantics(temperature):
    """do_sample branches of AutoRegressiveBeamSearch.search (reference layers/decoder.py:260-276, 364-375): the oracle's
    restatement (pinned against the reference with the same draws) over the ENGINE's step logits and uniforms gives the
    engine's tokens (a draw that lands within fp32 rounding of a CDF step may differ: at most one row) and log-probs."""
    g = load_golden('base_greedy')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd, max_steps=14)
    B = meta['batch']
    u = torch.rand((14, B), generator=torch.Generator().manual_seed(21))
    out = m(_to_cuda(batch), return_step_logits=True, search_param={'do_sample': True, 'temperature': temperature, 'uniforms': u})
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    own = out['predictions'].cpu()
    # teacher-forced replay: feed the oracle the engine's own history so that one near-tie cannot derail the comparison
    start = torch.full((B, 1), 101, dtype=torch.long)
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.sample_search(start, lambda partial: z[next(it)], u, temperature=temperature, max_steps=14)
    same = (pred == own).all(dim=1)
    print('sampled captions:', own.tolist(), 'rows identical to the replay:', same.tolist())
    assert int(same.sum()) >= B - 1
    assert torch.allclose(lp[same], out['logprobs'].cpu()[same], rtol=1e-4, atol=2e-3)
    greedy = m(_to_cuda(batch))['predictions'].cpu()
    assert not torch.equal(greedy[:, :own.shape[1]], own[:, :greedy.shape[1]])          # it does sample
    # same uniforms -> same captions; a generator works too
    out2 = m(_to_cuda(batch), search_param={'do_sample': True, 'temperature': temperature, 'uniforms': u})
    assert torch.equal(out2['predictions'].cpu(), own)
    gen = torch.Generator(device='cuda').manual_seed(3)
    out3 = m(_to_cuda(batch), search_param={'do_sample': True, 'temperature': temperature, 'generator': gen})
    assert out3['predictions'].shape[0] == B


@pytest.mark.parametrize('beam', [2, 3])
def test_beam_sizes_other_than_the_default(beam):
    """GeneratorWithBeamSearch with beam_size 2 / 3 (per-node 2; the shipped default is 4): exact replay of the oracle's
    restatement over the engine's own step logits, as for the default size."""
    from generativeimage2text_b200.model import GeneratorWithBeamSearch
    g = load_golden('base_beam')
    meta = g['meta']
    sd, batch = golden_inputs(meta)
    m = _model(meta, sd)
    m.decoder = GeneratorWithBeamSearch(102, max_steps=meta['max_steps'], beam_size=beam, length_penalty=0.6)
    out = m(_to_cuda(batch), return_step_logits=True)
    torch.cuda.synchronize()
    z = out['step_logits'].cpu()
    assert z.shape[1] == meta['batch'] * beam
    it = iter(range(z.shape[0]))
    pred, lp = git_oracle.beam_search(torch.full((meta['batch'], 1), 101, dtype=torch.long),
                                      lambda ids: z[next(it)], max_steps=meta['max_steps'], beam=beam)
    assert torch.equal(pred, out['predictions'].cpu())
    assert torch.allclose(lp, out['logprobs'].cpu(), atol=2e-3)
