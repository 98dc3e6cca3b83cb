"""GPU: caption scoring (`model.score`, C ABI gitb200_score) -- one teacher-forced pass over given captions that returns the
per-token log-probabilities and the reference's smoothed captioning loss.

* text_attn_wgmma_kernel / text_attn_f32_kernel (gitb200_op_text_attention) against an fp64 statement of the masked
  attention, with planted keys at the image tail, the diagonal and the 64-key block edges, and NaN rows that must never
  be read;
* the whole call against the reference goldens tests/golden/score_*.npz (oracle/make_score_golden.py), in the default and
  in the parity mode, and against the engine's own teacher-forced generate path;
* exact invariances: a caption's results do not depend on the other captions, on extra padding, on image_index grouping,
  on the other images of a ragged batch, or on the call."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import load_golden

pytestmark = pytest.mark.gpu

# Bounds set from what was measured on an H100 80GB HBM3 (700 W power limit), largest over the cases:
#   default mode: token log-probs 0.0082 (init) / 0.0388 (perturbed) from the reference, loss 3.3e-5 relative;
#                 0.023 from the engine's own teacher-forced step logits;
#   parity mode:  token log-probs 7.2e-4, loss 4.7e-4 (the fp32 targets 2e-3 / 1e-3); 4.4e-4 from the step logits;
#   text_attn_wgmma_kernel 3.63e-3, text_attn_f32_kernel 6.1e-6 (|out - ref| / max|v|).
LP_ATOL = {'init': 0.03, 'perturbed': 0.1}
LOSS_RTOL = {'init': 2e-4, 'perturbed': 2e-4}
GEN_ATOL = 0.1
PARITY_LP_ATOL, PARITY_LOSS_ATOL, PARITY_GEN_ATOL = 2e-3, 1e-3, 1e-3
ATTN_TOL, ATTN_F32_TOL = 7e-3, 1e-5       # |out - ref| / max|v|
CASES = ['score_base_init', 'score_base_perturbed', 'score_large', 'score_vatex', 'score_vqa_ragged', 'score_base_b64']


class Tok:
    cls_token_id, sep_token_id = 101, 102


def _lib():
    from generativeimage2text_b200 import _lib
    return _lib, _lib.load()


def _model(param, sd, parity=False):
    from generativeimage2text_b200.model import get_git_model
    m = get_git_model(Tok(), param)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    m = m.cuda().eval()
    if parity:
        m.set_engine_option('parity', 1)
    return m


def _golden_batch(g):
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    meta = g['meta']
    sd = synthetic_state_dict(meta['param'], meta['seed'], meta['variant'])
    if 'image_hws' in meta:
        image = [synthetic_images(1, 0, meta['img_seed'] + b, hw)[0].cuda() for b, hw in enumerate(meta['image_hws'])]
    else:
        image = synthetic_images(meta['batch'], meta['frames'], meta['img_seed'])
        image = [f.cuda() for f in image] if isinstance(image, list) else image.cuda()
    batch = {'image': image, 'caption_tokens': torch.from_numpy(g['caption_tokens']),
             'need_predict': torch.from_numpy(g['need_predict']), 'image_index': torch.from_numpy(g['image_index'])}
    return meta, sd, batch


# ---- 1. the attention kernel ------------------------------------------------------------------------------------------
def ref_text_attention(q, k, v, ik, iv, lens, index, T, H):
    """fp64: row t of caption n attends to image index[n]'s first lens[b] keys and to its own text keys 0..t."""
    N = q.shape[0] // T
    out = torch.zeros(q.shape, dtype=torch.float64)
    M = ik.shape[0] // len(lens)
    for n in range(N):
        b = index[n]
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            qq = q[n * T:(n + 1) * T, c].double() / 8
            kk = torch.cat([ik[b * M:b * M + lens[b], c], k[n * T:(n + 1) * T, c]]).double()
            vv = torch.cat([iv[b * M:b * M + lens[b], c], v[n * T:(n + 1) * T, c]]).double()
            s = qq @ kk.T
            mask = torch.ones(T, T, dtype=torch.bool).triu(1)
            s[:, lens[b]:][mask] = float('-inf')
            out[n * T:(n + 1) * T, c] = torch.softmax(s, dim=1) @ vv
    return out


def _attn_inputs(M, T, ragged, seed, H=2, B=3, per=2):
    g = torch.Generator().manual_seed(seed)
    N = B * per
    D = 64 * H
    q = torch.randn(N * T, D, generator=g)
    k = torch.randn(N * T, D, generator=g)
    v = torch.randn(N * T, D, generator=g)
    ik = torch.randn(B * M, D, generator=g)
    iv = torch.randn(B * M, D, generator=g)
    lens = [M, max(1, M - 37), max(1, (M + 1) // 2)] if ragged else [M] * B
    index = [(n * 2 + 1) % B for n in range(N)]                      # several captions per image, not in image order
    # planted keys (each about half of its row's weight): the last image key, the diagonal, the 64-key block edges
    for n in range(N):
        b = index[n]
        for t in range(T):
            if t % 64 in (0, 63) or t == T - 1 or t % 7 == 3:
                k[n * T + t] = q[n * T + t] * 2.0                     # the diagonal key of row t
        ik[b * M + lens[b] - 1] = q[n * T:(n + 1) * T].mean(0) * 3.0
    return q, k, v, ik, iv, lens, index, N, B


def _run_text_attention(q, k, v, ik, iv, lens, index, N, T, B, M, H, fp32, ragged):
    _l, lib = _lib()
    dt = torch.float32 if fp32 else torch.bfloat16
    dq, dk, dv, dik, div = (t.to(dt).cuda().contiguous() for t in (q, k, v, ik, iv))
    out = torch.zeros((N * T, (3 if fp32 else 1) * H * 64), dtype=torch.bfloat16, device='cuda')
    lens_h = (ctypes.c_int32 * B)(*lens) if ragged else None
    idx_h = (ctypes.c_int32 * N)(*index)
    _l.check(lib.gitb200_op_text_attention(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), dik.data_ptr(), div.data_ptr(),
                                           out.data_ptr(), N, T, B, M, lens_h, idx_h, H, 1 if fp32 else 0,
                                           torch.cuda.current_stream().cuda_stream), None, 'op_text_attention')
    torch.cuda.synchronize()
    if fp32:
        D = H * 64
        return out[:, :D].float() + out[:, D:2 * D].float()
    return out.float()


@pytest.mark.parametrize('fp32', [0, 1])
@pytest.mark.parametrize('ragged', [False, True])
@pytest.mark.parametrize('M', [2, 197, 257, 1182, 1201])
def test_text_attention_against_fp64(M, ragged, fp32):
    H = 2
    worst = 0.0
    for T in (1, 2, 63, 64, 65, 129):
        q, k, v, ik, iv, lens, index, N, B = _attn_inputs(M, T, ragged, seed=M * 1000 + T)
        if fp32:
            ref = ref_text_attention(q, k, v, ik, iv, lens, index, T, H)
        else:   # the kernel's operands are bf16
            bq, bk, bv, bik, biv = (t.bfloat16().float() for t in (q, k, v, ik, iv))
            ref = ref_text_attention(bq, bk, bv, bik, biv, lens, index, T, H)
        out = _run_text_attention(q, k, v, ik, iv, lens, index, N, T, B, M, H, fp32, ragged)
        assert torch.isfinite(out).all()
        err = ((out.cpu().double() - ref).abs().max() / max(v.abs().max(), iv.abs().max())).item()
        worst = max(worst, err)
    print('text attention M=%d ragged=%s fp32=%d: max |out - ref| / max|v| = %.3g' % (M, ragged, fp32, worst))
    assert worst < (ATTN_F32_TOL if fp32 else ATTN_TOL)


@pytest.mark.parametrize('fp32', [0, 1])
def test_text_attention_never_reads_the_future(fp32):
    """K rows in every query's future may hold NaN (the score is replaced, not added to); K and V rows in the text blocks
    past a query tile are never loaded.  The rows that may not see them must come out bit-identical."""
    M, T, H = 197, 129, 2
    q, k, v, ik, iv, lens, index, N, B = _attn_inputs(M, T, False, seed=7)
    base = _run_text_attention(q, k, v, ik, iv, lens, index, N, T, B, M, H, fp32, False)
    for p0 in (1, 40, 63, 64, 100):                 # K = NaN at positions >= p0 of every caption: rows < p0 unchanged
        k2 = k.clone().view(N, T, -1)
        k2[:, p0:] = float('nan')
        out = _run_text_attention(q, k2.view(N * T, -1), v, ik, iv, lens, index, N, T, B, M, H, fp32, False)
        rows = (torch.arange(N * T) % T) < p0
        assert torch.equal(out[rows.cuda()], base[rows.cuda()]), p0
    if not fp32:
        for kb in (1, 2):                           # K and V = NaN from text block kb on: rows of the blocks before unchanged
            k2, v2 = k.clone().view(N, T, -1), v.clone().view(N, T, -1)
            k2[:, 64 * kb:] = float('nan')
            v2[:, 64 * kb:] = float('nan')
            out = _run_text_attention(q, k2.view(N * T, -1), v2.view(N * T, -1), ik, iv, lens, index, N, T, B, M, H, fp32, False)
            rows = (torch.arange(N * T) % T) < 64 * kb
            assert torch.equal(out[rows.cuda()], base[rows.cuda()]), kb


def test_text_attention_rejects_bad_arguments():
    _l, lib = _lib()
    x = torch.zeros(64, 128, dtype=torch.bfloat16, device='cuda')
    idx = (ctypes.c_int32 * 2)(0, 5)
    rc = lib.gitb200_op_text_attention(x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                                       2, 32, 2, 32, None, idx, 2, 0, None)
    assert rc != 0 and 'image_index' in _l.last_error()
    lens = (ctypes.c_int32 * 2)(32, 33)
    rc = lib.gitb200_op_text_attention(x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                                       2, 32, 2, 32, lens, None, 2, 0, None)
    assert rc != 0


# ---- 2. the whole call against the reference ---------------------------------------------------------------------------
@pytest.mark.parametrize('case', CASES)
def test_score_against_reference(case):
    g = load_golden(case)
    meta, sd, batch = _golden_batch(g)
    m = _model(meta['param'], sd)
    out = m.score(batch)
    torch.cuda.synchronize()
    lp = out['token_logprobs'].cpu().numpy()
    ref_lp = g['token_logprobs']
    err_lp = float(np.abs(lp - ref_lp).max())
    loss, ref_loss = out['vl_l_loss'].item(), float(g['vl_l_loss'])
    rel = abs(loss - ref_loss) / abs(ref_loss)
    print('%s: max |token logprob - reference| %.4f, loss %.6f vs %.6f (rel %.2e)' % (case, err_lp, loss, ref_loss, rel))
    assert err_lp < LP_ATOL[meta['variant']]
    assert rel < LOSS_RTOL[meta['variant']]


@pytest.mark.parametrize('case', CASES)
def test_score_parity_mode_against_reference(case):
    g = load_golden(case)
    meta, sd, batch = _golden_batch(g)
    m = _model(meta['param'], sd, parity=True)
    out = m.score(batch)
    torch.cuda.synchronize()
    err_lp = float(np.abs(out['token_logprobs'].cpu().numpy() - g['token_logprobs']).max())
    err_loss = abs(out['vl_l_loss'].item() - float(g['vl_l_loss']))
    print('%s [parity]: max |token logprob - reference| %.2e, |loss - reference| %.2e' % (case, err_lp, err_loss))
    assert err_lp < PARITY_LP_ATOL
    assert err_loss < PARITY_LOSS_ATOL


def _edge_captions():
    """Captions whose targets sit at the LM head's column-tile edges (0, 255, 256, 30521) and one row with no valid target."""
    tok = torch.tensor([[101, 2054, 255, 256, 30521, 102, 0, 0],
                        [101, 30521, 256, 255, 7, 3000, 102, 0],
                        [101, 500, 600, 102, 0, 0, 0, 0]])
    need = torch.tensor([[0, 1, 1, 1, 1, 1, 0, 0],
                         [0, 1, 1, 1, 1, 1, 1, 0],
                         [0, 0, 0, 0, 0, 0, 0, 0]])
    return tok, need


@pytest.mark.parametrize('parity', [False, True])
def test_score_against_teacher_forced_generate(parity):
    """score() == log-softmax / gather of the step logits the engine's generate path computes for the same captions."""
    from generativeimage2text_b200.model import AutoRegressiveBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    sd = synthetic_state_dict({}, 0, 'perturbed')
    m = _model({}, sd, parity=parity)
    tok, need = _edge_captions()
    image = synthetic_images(3, 0, 77).cuda()
    out = m.score({'image': image, 'caption_tokens': tok, 'need_predict': need})
    T = tok.shape[1]
    m.decoder = AutoRegressiveBeamSearch(102, max_steps=T, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    gen = m({'image': image}, forced_tokens=tok, return_step_logits=True)
    torch.cuda.synchronize()
    z = gen['step_logits'].cpu()                     # [T - 1, 3, V]: step s predicts position s + 1
    ref = torch.log_softmax(z, dim=-1).gather(2, tok[:, 1:].T[..., None])[..., 0].T
    # the generate path stops early once every row has emitted EOS; compare the steps it ran
    steps = int((z.abs().sum(dim=(1, 2)) > 0).sum())
    err = (out['token_logprobs'].cpu()[:, :steps] - ref[:, :steps]).abs().max().item()
    print('score vs teacher-forced generate (parity=%s): max |difference| %.2e over %d steps' % (parity, err, steps))
    assert steps >= 5
    assert err < (PARITY_GEN_ATOL if parity else GEN_ATOL)


# ---- 3. exact invariances ------------------------------------------------------------------------------------------------
def test_rows_are_independent_of_the_batch_and_the_call():
    g = load_golden('score_base_perturbed')
    meta, sd, batch = _golden_batch(g)
    m = _model(meta['param'], sd)
    a = m.score(batch)['token_logprobs']
    b = m.score(batch)['token_logprobs']
    assert torch.equal(a, b)                                            # repeated calls
    tok, need, idx = batch['caption_tokens'], batch['need_predict'], batch['image_index']
    # extra padding positions
    pad = m.score(dict(batch, caption_tokens=torch.nn.functional.pad(tok, (0, 70)),
                       need_predict=torch.nn.functional.pad(need, (0, 70))))['token_logprobs']
    assert torch.equal(pad[:, :tok.shape[1] - 1], a)
    # a subset of the captions, in another order
    rows = [5, 0, 7]
    sub = m.score(dict(batch, caption_tokens=tok[rows], need_predict=need[rows], image_index=idx[rows]))['token_logprobs']
    assert torch.equal(sub, a[rows])
    # image_index grouping == the images repeated one per caption
    rep = m.score({'image': batch['image'][idx.cuda()], 'caption_tokens': tok, 'need_predict': need})['token_logprobs']
    assert torch.equal(rep, a)


def test_ragged_rows_equal_their_image_alone():
    g = load_golden('score_vqa_ragged')
    meta, sd, batch = _golden_batch(g)
    m = _model(meta['param'], sd)
    full = m.score(batch)['token_logprobs']
    idx = batch['image_index']
    for b, im in enumerate(batch['image']):
        rows = torch.nonzero(idx == b)[:, 0]
        one = m.score({'image': im[None], 'caption_tokens': batch['caption_tokens'][rows],
                       'need_predict': batch['need_predict'][rows],
                       'image_index': torch.zeros(len(rows), dtype=torch.long)})['token_logprobs']
        assert torch.equal(one, full[rows.cuda()]), b
