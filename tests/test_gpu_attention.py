"""Every attention kernel through a C-ABI op entry point against a plain fp64 PyTorch statement of the same operation.

Kernels (csrc/attention.cuh) and their entry points:
  gitb200_op_decode_attention: decode_attn_kernel<beam, ragged> and decode_attn_f32_kernel (parity mode);
  gitb200_op_attention_ex: flash_attn_wgmma_kernel<false / true> and attn_f32_kernel (parity mode).

Random data alone lets a dropped key hide inside the tolerance, so every case plants keys: for some (row, head) pairs
one key at a boundary of the kernel (the last valid key, the first and last key of each 64-key block or decode chunk,
text positions 0, 63, 64 and the newest one) gets the log-sum-exp of that row's other scores as its score, so that it
carries about half of the softmax weight.  Building a case asserts that masking any planted key moves its output row by
at least 4x the tolerance: a kernel that drops or double-counts one of those keys fails.  The case builders and those
sensitivity checks run on the CPU; the kernels need an H100.
"""
import ctypes
import math

import pytest
import torch

# |out - ref| <= TOL * max|v| + ABS.  Each TOL is about 3.5x the largest |out - ref| / max|v| its kernel showed over
# these cases on an H100 80GB HBM3 (400 W power limit), given after it.
TOL_DECODE = 5.5e-3       # decode_attn_kernel: fp32 softmax, bf16 output; observed 1.58e-3
TOL_DECODE_F32 = 1e-5     # decode_attn_f32_kernel: fp32, output hi + lo; observed 2.84e-6
TOL_WGMMA = 3.5e-3        # flash_attn_wgmma_kernel: bf16 P, bf16 output; observed 9.11e-4
TOL_ATTN_F32 = 7e-6       # attn_f32_kernel: fp32, output hi + lo; observed 1.90e-6
ABS = 1e-5
PAD = 3e4                 # a large finite value in rows no valid row may read
SENTINEL = 1000.0          # output rows no kernel may write (exact in bf16)

DEC_CHUNK = 224           # kDecAttnChunk: image keys of one decode chunk at most


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def ref_attention(q, k, v, lens=None):
    """softmax(q k^T / 8) v per (batch, head) over the first lens[b] keys (all S when lens is None).
    q, k, v [B, S, H, 64]; returns fp64 [B, S, H, 64] whose rows past lens[b] are zero."""
    B, S, H, _ = q.shape
    out = torch.zeros(B, S, H, 64, dtype=torch.float64)
    for b in range(B):
        n = S if lens is None else int(lens[b])
        qb, kb, vb = (t[b, :n].double().transpose(0, 1) for t in (q, k, v))    # [H, n, 64]
        p = torch.softmax(qb @ kb.transpose(-1, -2) / 8.0, dim=-1)
        out[b, :n] = (p @ vb).transpose(0, 1)
    return out


def decode_new_qkv(qkv_parts, bias, bf16):
    """q (scaled by 1/8) and the k / v a decode step appends, from split-K partials [n, R, 3D] and bias [3D]: the
    partials are summed in split order in fp32, then the bias is added; k / v are stored (bf16 in bf16 mode)."""
    s = qkv_parts[0].clone()
    for p in qkv_parts[1:]:
        s = s + p
    s = s + bias
    D = bias.numel() // 3
    q, k, v = s[:, :D] * 0.125, s[:, D:2 * D], s[:, 2 * D:]
    if bf16:
        k, v = k.bfloat16(), v.bfloat16()
    return q, k, v


def _decode_keys(r, kn, vn, img_k, img_v, txt_k, txt_v, src_row, lens, pos, beam):
    """Keys and values [n, D] (fp64) that row r attends: image keys 0 .. M_b - 1 of image r // beam, then text positions
    0 .. pos gathered through src_row from the caches with this step's k / v written at pos."""
    b = r // beam
    mb = img_k.shape[1] if lens is None else int(lens[b])
    tk, tv = txt_k.clone(), txt_v.clone()
    tk[:, pos], tv[:, pos] = kn, vn
    t = torch.arange(pos + 1)
    phys = torch.full((pos + 1,), r) if src_row is None else src_row[r, :pos + 1].long()
    K = torch.cat([img_k[b, :mb].double(), tk[phys, t].double()])
    V = torch.cat([img_v[b, :mb].double(), tv[phys, t].double()])
    return K, V


def ref_decode(qkv_parts, bias, img_k, img_v, txt_k, txt_v, src_row, lens, pos, beam):
    """One decode step's attention, fp64 [R, D]: row r's q against image r // beam's first lens[b] keys (M when lens is
    None) and text positions 0 .. pos, softmax over them all, per 64-wide head."""
    q, kn, vn = decode_new_qkv(qkv_parts, bias, img_k.dtype == torch.bfloat16)
    R, D = q.shape
    H = D // 64
    out = torch.empty(R, H, 64, dtype=torch.float64)
    for r in range(R):
        K, V = _decode_keys(r, kn, vn, img_k, img_v, txt_k, txt_v, src_row, lens, pos, beam)
        Kh, Vh = K.view(-1, H, 64).transpose(0, 1), V.view(-1, H, 64).transpose(0, 1)    # [H, n, 64]
        p = torch.softmax(torch.einsum('hd,hnd->hn', q[r].double().view(H, 64), Kh), dim=-1)
        out[r] = torch.einsum('hn,hnd->hd', p, Vh)
    return out.view(R, D)


def _planted(q, K, j):
    """Key vector along q whose score q . k is the log-sum-exp of the other keys' scores (about half the weight)."""
    s = K @ q
    target = torch.logsumexp(torch.cat([s[:j], s[j + 1:]]), 0)
    return q * (target / (q @ q))


def _masked_change(q, K, V, j):
    """Largest change of softmax(K q) V when key j is left out."""
    full = torch.softmax(K @ q, 0) @ V
    keep = torch.ones(K.shape[0], dtype=torch.bool)
    keep[j] = False
    return (full - torch.softmax(K[keep] @ q, 0) @ V[keep]).abs().max().item()


def _bound(tol, vmax):
    return tol * vmax + ABS


# ---------------------------------------------------------------------------------------------------------------------
# decode cases
# ---------------------------------------------------------------------------------------------------------------------
def dec_chunk_bounds(mb):
    """First and last key of every chunk a decode CTA stages for an image of mb keys (dec_attn_chunk_rows)."""
    n = -(-mb // DEC_CHUNK)
    rows = -(-mb // n)
    out = set()
    for c in range(n):
        out |= {c * rows, min((c + 1) * rows, mb) - 1}
    return out


def make_decode_case(beam, M, pos, n_partials, B=2, D=768, lens=None, fp32=False, seed=0, pad=PAD):
    """Inputs of one decode step with planted boundary keys, and its fp64 reference.  Text positions after pos hold NaN;
    image slot rows past lens[b] hold `pad`."""
    g = torch.Generator().manual_seed(seed)
    dt = torch.float32 if fp32 else torch.bfloat16
    tol = TOL_DECODE_F32 if fp32 else TOL_DECODE
    R, H, T = B * beam, D // 64, pos + 3
    parts = torch.randn(n_partials, R, 3 * D, generator=g) / math.sqrt(n_partials)
    bias = 0.1 * torch.randn(3 * D, generator=g)
    img_k, img_v = (torch.randn(B, M, D, generator=g).to(dt) for _ in range(2))
    txt_k, txt_v = (torch.randn(R, T, D, generator=g).to(dt) for _ in range(2))
    txt_k[:, pos + 1:] = float('nan')
    txt_v[:, pos + 1:] = float('nan')
    src_row = None
    if beam > 1:     # ancestry within each image's beams; the newest position is the row's own
        src_row = (torch.arange(R) // beam * beam)[:, None] + torch.randint(0, beam, (R, T), generator=g)
        src_row[:, pos:] = torch.arange(R)[:, None]
        src_row = src_row.int()
    mbs = [M] * B if lens is None else list(lens)
    case = dict(beam=beam, M=M, pos=pos, B=B, D=D, T=T, lens=lens, fp32=fp32, parts=parts, bias=bias, img_k=img_k,
                img_v=img_v, txt_k=txt_k, txt_v=txt_v, src_row=src_row, tol=tol)

    def keys(r):
        _, kn, vn = decode_new_qkv(parts, bias, not fp32)
        return _decode_keys(r, kn, vn, img_k, img_v, txt_k, txt_v, src_row, lens, pos, beam)

    # plant: every boundary key of image b, dealt to the (row, head) pairs of its beams
    plants = []
    for b in range(B):
        mb = mbs[b]
        bounds = sorted(dec_chunk_bounds(mb)) + [mb + t for t in sorted({0, 63, 64, pos}) if t <= pos]
        slots = [(b * beam + i, h) for h in range(H) for i in range(beam)]
        for n, j in enumerate(bounds):
            r, h = slots[(n * 5) % len(slots)]
            cs = slice(h * 64, (h + 1) * 64)
            q = decode_new_qkv(parts, bias, not fp32)[0][r, cs].double()
            K, _ = keys(r)
            vec = _planted(q, K[:, cs], j)
            if j < mb:
                img_k[b, j, cs] = vec.to(dt)
            elif j - mb < pos:
                t = j - mb
                pr = r if src_row is None else int(src_row[r, t])
                txt_k[pr, t, cs] = vec.to(dt)
            else:            # this step's own key: what the partials sum to
                rest = bias[D:][cs].double() + sum(parts[i, r, D:][cs].double() for i in range(1, n_partials))
                parts[0, r, D + h * 64:D + (h + 1) * 64] = (vec - rest).float()
            plants.append((r, h, j))
    for b in range(B):
        img_k[b, mbs[b]:] = pad
        img_v[b, mbs[b]:] = pad
    case['ref'] = ref_decode(parts, bias, img_k, img_v, txt_k, txt_v, src_row, lens, pos, beam)
    q = decode_new_qkv(parts, bias, not fp32)[0].double()
    case['vmax'] = max(keys(r)[1].abs().max().item() for r in range(R))
    for r, h, j in plants:
        cs = slice(h * 64, (h + 1) * 64)
        K, V = keys(r)
        change = _masked_change(q[r, cs], K[:, cs], V[:, cs], j)
        assert _bound(tol, case['vmax']) <= change / 4, (r, h, j, change)
    case['n_plants'] = len(plants)
    return case


BEAMS = (1, 2, 3, 4)
DEC_M = (2, 50, 197, 224, 225, 257, 449, 1182, 1201)   # one chunk, the 224 edge, even / uneven splits, video, VQA
DEC_POS = (0, 62, 63, 64, 65, 129)
DEC_NP = (1, 3, 4)
# every beam size with every M; pos and n_partials cycle so that each beam size also meets every pos and n_partials
DEC_CASES = [(beam, M, DEC_POS[(mi + bi) % 6], DEC_NP[(mi + 2 * bi) % 3], 768)
             for bi, beam in enumerate(BEAMS) for mi, M in enumerate(DEC_M)] + [(2, 449, 65, 3, 128)]
DEC_F32_CASES = [(1, 2, 0, 1), (2, 225, 64, 3), (3, 449, 129, 4), (4, 1201, 63, 3), (1, 1182, 65, 1)]
RAGGED_LENS = [2, 197, 1201, 449, 50, 1201]     # mixed chunk counts, the longest image first and last


def _dec_case(beam, M, pos, n_partials, D, fp32=False):
    return make_decode_case(beam, M, pos, n_partials, B=2 if D == 768 else 4, D=D, fp32=fp32,
                            seed=1000 * beam + M + pos)


def _ragged_case(beam, fp32=False, pad=PAD):
    return make_decode_case(beam, max(RAGGED_LENS), 64, 3, B=len(RAGGED_LENS), lens=RAGGED_LENS, fp32=fp32,
                            seed=77 + beam, pad=pad)


# ---------------------------------------------------------------------------------------------------------------------
# prefill / ViT attention cases
# ---------------------------------------------------------------------------------------------------------------------
def make_attention_case(B, S, H, lens=None, fp32=False, seed=0, pad=PAD, tol=TOL_WGMMA):
    """q | k | v packed as [B, S, 3 * H * 64] (the engine's QKV GEMM output) with planted boundary keys; rows past
    lens[b] hold `pad`."""
    g = torch.Generator().manual_seed(seed)
    dt = torch.float32 if fp32 else torch.bfloat16
    qkv = torch.randn(B, S, 3, H, 64, generator=g).to(dt)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    lens_ = [S] * B if lens is None else list(lens)
    plants = []
    for b in range(B):
        n = lens_[b]
        bounds = sorted({0, n - 1} | {x for c in range(0, n, 64) for x in (c, min(c + 63, n - 1))})
        for h in range(H):
            rows = torch.randperm(n, generator=g)[:len(bounds)].tolist()
            for j, i in zip(bounds, rows):
                qi = q[b, i, h].double() / 8.0
                k[b, j, h] = _planted(qi, k[b, :n, h].double(), j).to(dt)
                plants.append((b, h, i, j))
        qkv[b, n:] = pad
    ref = ref_attention(q, k, v, lens)
    vmax = max(v[b, :lens_[b]].double().abs().max().item() for b in range(B))
    for b, h, i, j in plants:
        n = lens_[b]
        change = _masked_change(q[b, i, h].double() / 8.0, k[b, :n, h].double(), v[b, :n, h].double(), j)
        assert _bound(tol, vmax) <= change / 4, (b, h, i, j, change)
    return dict(qkv=qkv.reshape(B, S, 3 * H * 64), q=q, k=k, v=v, ref=ref.reshape(B, S, H * 64), vmax=vmax, B=B, S=S,
                H=H, lens=lens, tol=tol, n_plants=len(plants))


WGMMA_RAGGED_LENS = [2, 63, 64, 65, 128, 197, 1201]
F32_ATTN_CASES = [(2, 197, 2, None), (3, 1201, 2, [2, 65, 1201])]
UNIFORM_CASES = [(2, 197, 12), (1, 1201, 2)]


def _wgmma_ragged_case(pad=PAD):
    return make_attention_case(len(WGMMA_RAGGED_LENS), max(WGMMA_RAGGED_LENS), 2, lens=WGMMA_RAGGED_LENS, seed=11, pad=pad)


def _uniform_case(B, S, H):
    return make_attention_case(B, S, H, seed=12)


def _f32_attn_case(B, S, H, lens, pad=PAD):
    return make_attention_case(B, S, H, lens=lens, fp32=True, seed=15, pad=pad, tol=TOL_ATTN_F32)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the references against SDPA, and every case's sensitivity to its planted keys
# ---------------------------------------------------------------------------------------------------------------------
def test_ref_attention_matches_sdpa():
    g = torch.Generator().manual_seed(3)
    B, S, H, lens = 3, 9, 2, [9, 4, 1]
    q, k, v = (torch.randn(B, S, H, 64, generator=g, dtype=torch.float64) for _ in range(3))
    out = ref_attention(q, k, v, lens)
    for b, n in enumerate(lens):
        want = torch.nn.functional.scaled_dot_product_attention(
            q[b, :n].transpose(0, 1), k[b, :n].transpose(0, 1), v[b, :n].transpose(0, 1)).transpose(0, 1)
        torch.testing.assert_close(out[b, :n], want, rtol=1e-12, atol=1e-12)
        assert not out[b, n:].any()
    torch.testing.assert_close(ref_attention(q, k, v), ref_attention(q, k, v, [S] * B), rtol=0, atol=0)


@pytest.mark.parametrize('fp32', [False, True])
def test_ref_decode_matches_sdpa_and_explicit_gather(fp32):
    """Beam search: the src_row gather of ref_decode against a loop over positions, and its softmax against SDPA."""
    g = torch.Generator().manual_seed(4)
    dt = torch.float32 if fp32 else torch.bfloat16
    B, beam, M, lens, T, pos, D, npart = 2, 3, 7, [7, 3], 6, 4, 128, 3
    R, H = B * beam, D // 64
    parts = torch.randn(npart, R, 3 * D, generator=g)
    bias = torch.randn(3 * D, generator=g)
    img_k, img_v = (torch.randn(B, M, D, generator=g).to(dt) for _ in range(2))
    txt_k, txt_v = (torch.randn(R, T, D, generator=g).to(dt) for _ in range(2))
    src = ((torch.arange(R) // beam * beam)[:, None] + torch.randint(0, beam, (R, T), generator=g)).int()
    src[:, pos] = torch.arange(R).int()
    out = ref_decode(parts, bias, img_k, img_v, txt_k, txt_v, src, lens, pos, beam)
    s = ((parts[0] + parts[1]) + parts[2]) + bias
    q = s[:, :D] * 0.125
    kn, vn = s[:, D:2 * D].to(dt), s[:, 2 * D:].to(dt)
    for r in range(R):
        b = r // beam
        ks = [img_k[b, j] for j in range(lens[b])]
        vs = [img_v[b, j] for j in range(lens[b])]
        for t in range(pos + 1):
            ks.append(kn[r] if t == pos else txt_k[int(src[r, t]), t])
            vs.append(vn[r] if t == pos else txt_v[int(src[r, t]), t])
        K, V = (torch.stack(x).double().view(-1, H, 64).transpose(0, 1)[None] for x in (ks, vs))
        want = torch.nn.functional.scaled_dot_product_attention(q[r].double().view(1, H, 1, 64), K, V, scale=1.0)
        torch.testing.assert_close(out[r].view(H, 64), want.view(H, 64), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('beam,M,pos,n_partials,D', DEC_CASES)
def test_decode_case_sensitivity(beam, M, pos, n_partials, D):
    """Every GPU decode case, built: each planted key moves its row by at least 4x the tolerance."""
    assert _dec_case(beam, M, pos, n_partials, D)['n_plants'] >= 4


@pytest.mark.parametrize('beam', BEAMS)
def test_ragged_decode_case_sensitivity(beam):
    assert _ragged_case(beam)['n_plants'] >= 6 * 4


@pytest.mark.parametrize('build', ['wgmma_ragged', 'uniform', 'f32'])
def test_attention_case_sensitivity(build):
    """Every GPU attention case, built: each planted key moves its row by at least 4x the tolerance."""
    if build == 'wgmma_ragged':
        _wgmma_ragged_case()
    for args in {'uniform': UNIFORM_CASES, 'f32': F32_ATTN_CASES, 'wgmma_ragged': []}[build]:
        {'uniform': _uniform_case, 'f32': _f32_attn_case}[build](*args)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from generativeimage2text_b200 import _lib
    return _lib


def _lens_arg(lens):
    return None if lens is None else (ctypes.c_int32 * len(lens))(*lens)


def _run_decode(case, grid=0, img_k=None, img_v=None, rows=None):
    """One gitb200_op_decode_attention call on fresh copies of the caches.  Returns ctx, txt_k, txt_v (CPU)."""
    L = _lib()
    parts = case['parts'].cuda()
    img_k = (case['img_k'] if img_k is None else img_k).cuda()
    img_v = (case['img_v'] if img_v is None else img_v).cuda()
    txt_k, txt_v = case['txt_k'].cuda(), case['txt_v'].cuda()
    bias = case['bias'].cuda()
    src = case['src_row'].cuda() if case['src_row'] is not None else None
    R, D = parts.shape[1], case['D']
    ctx = torch.zeros(R, 3 * D if case['fp32'] else D, dtype=torch.bfloat16, device='cuda')
    B = img_k.shape[0]
    rc = L.load().gitb200_op_decode_attention(
        parts.data_ptr(), parts.shape[0], bias.data_ptr(), img_k.data_ptr(), img_v.data_ptr(),
        txt_k.data_ptr(), txt_v.data_ptr(), src.data_ptr() if src is not None else None, ctx.data_ptr(), B,
        case['beam'], img_k.shape[1], _lens_arg(case['lens']), case['T'], case['pos'], D, int(case['fp32']), grid,
        torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    return ctx.cpu(), txt_k.cpu(), txt_v.cpu()


def _split_value(ctx, D):
    """[hi | lo | hi] split rows -> hi + lo (fp32); the two hi copies must be equal."""
    hi, lo, hi2 = ctx.split(D, dim=-1)
    assert torch.equal(hi.view(torch.int16), hi2.view(torch.int16))
    return hi.float() + lo.float()


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _check_decode(case, ctx, txt_k, txt_v, what):
    """ctx against the reference; the cache entry at pos is this step's k / v bit for bit and nothing else changed."""
    D, pos = case['D'], case['pos']
    out = _split_value(ctx, D) if case['fp32'] else ctx.float()
    assert torch.isfinite(out).all(), what
    err = (out.double() - case['ref']).abs().max().item()
    print('%s: max err / max|v| = %.3g (tol %.3g)' % (what, err / case['vmax'], case['tol']))
    assert err <= _bound(case['tol'], case['vmax']), (what, err, case['vmax'])
    _, kn, vn = decode_new_qkv(case['parts'], case['bias'], not case['fp32'])
    for got, old, new in ((txt_k, case['txt_k'], kn), (txt_v, case['txt_v'], vn)):
        want = old.clone()
        want[:, pos] = new
        assert torch.equal(_bits(got), _bits(want)), what


@pytest.mark.gpu
@pytest.mark.parametrize('beam,M,pos,n_partials,D', DEC_CASES)
def test_decode_attention(beam, M, pos, n_partials, D):
    case = _dec_case(beam, M, pos, n_partials, D)
    ctx, tk, tv = _run_decode(case)
    _check_decode(case, ctx, tk, tv, 'decode beam=%d M=%d pos=%d np=%d D=%d' % (beam, M, pos, n_partials, D))
    for grid in (1, 7):      # one CTA walking every item (the beam-1 look-ahead past kPre), several items per CTA
        assert torch.equal(_run_decode(case, grid)[0].view(torch.int16), ctx.view(torch.int16)), grid


@pytest.mark.gpu
@pytest.mark.parametrize('beam', BEAMS)
def test_ragged_decode_attention(beam):
    case = _ragged_case(beam)
    ctx, tk, tv = _run_decode(case)
    _check_decode(case, ctx, tk, tv, 'ragged decode beam=%d' % beam)
    for grid in (1, 7):      # one CTA walking items of different chunk counts, in the order thread 0 issues them
        assert torch.equal(_run_decode(case, grid)[0].view(torch.int16), ctx.view(torch.int16)), grid
    zero = _ragged_case(beam, pad=0.0)          # padding rows are never read
    assert torch.equal(_run_decode(zero)[0].view(torch.int16), ctx.view(torch.int16))
    for b, mb in enumerate(RAGGED_LENS):        # row b gets exactly the arithmetic of a call of its own size
        rows = slice(b * beam, (b + 1) * beam)
        one = dict(case, lens=None, parts=case['parts'][:, rows].contiguous(), txt_k=case['txt_k'][rows].contiguous(),
                   txt_v=case['txt_v'][rows].contiguous(),
                   src_row=None if case['src_row'] is None else (case['src_row'][rows] - b * beam).contiguous())
        got = _run_decode(one, img_k=case['img_k'][b:b + 1, :mb].contiguous(), img_v=case['img_v'][b:b + 1, :mb].contiguous())
        assert torch.equal(got[0].view(torch.int16), ctx[rows].view(torch.int16)), b


@pytest.mark.gpu
@pytest.mark.parametrize('beam,M,pos,n_partials', DEC_F32_CASES)
def test_decode_attention_f32(beam, M, pos, n_partials):
    case = _dec_case(beam, M, pos, n_partials, 768, fp32=True)
    ctx, tk, tv = _run_decode(case)
    _check_decode(case, ctx, tk, tv, 'decode f32 beam=%d M=%d pos=%d np=%d' % (beam, M, pos, n_partials))


@pytest.mark.gpu
@pytest.mark.parametrize('beam', [1, 3])
def test_ragged_decode_attention_f32(beam):
    case = _ragged_case(beam, fp32=True)
    ctx, tk, tv = _run_decode(case)
    _check_decode(case, ctx, tk, tv, 'ragged decode f32 beam=%d' % beam)
    assert torch.equal(_run_decode(_ragged_case(beam, fp32=True, pad=0.0))[0].view(torch.int16), ctx.view(torch.int16))


def _run_attention(qkv, B, S, H, lens=None, fp32=False, out=None, legacy=False):
    """gitb200_op_attention(_ex) on q | k | v rows of 3 * H * 64 elements; out defaults to [B, S, d] (bf16; split rows
    [B, S, 3d] in parity mode)."""
    L = _lib()
    d = H * 64
    qkv = qkv.cuda()
    if out is None:
        out = torch.zeros(B, S, 3 * d if fp32 else d, dtype=torch.bfloat16)
    out = out.cuda()
    q_bs, o_bs = S * 3 * d, S * out.shape[-1]
    es = qkv.element_size()
    base = qkv.data_ptr()
    args = (base, base + d * es, base + 2 * d * es, out.data_ptr(), B, S, H, 3 * d, 3 * d, q_bs, q_bs, d, o_bs)
    if legacy:
        rc = L.load().gitb200_op_attention(*args, torch.cuda.current_stream().cuda_stream)
    else:
        rc = L.load().gitb200_op_attention_ex(*args, _lens_arg(lens), int(fp32), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    return out.cpu()


def _check_attention(case, out, what):
    err = (out.double() - case['ref']).abs().max().item()
    print('%s: max err / max|v| = %.3g (tol %.3g)' % (what, err / case['vmax'], case['tol']))
    assert err <= _bound(case['tol'], case['vmax']), (what, err, case['vmax'])


@pytest.mark.gpu
def test_flash_wgmma_ragged():
    lens = WGMMA_RAGGED_LENS
    B, S, H = len(lens), max(lens), 2
    case = _wgmma_ragged_case()
    out = _run_attention(case['qkv'], B, S, H, lens)
    _check_attention(case, out.float(), 'wgmma ragged')
    for b, n in enumerate(lens):
        assert not out[b, n:].view(torch.int16).any(), b          # padding rows: exact (+0) zeros
        one = _run_attention(case['qkv'][b:b + 1, :n].contiguous(), 1, n, H, legacy=True)
        assert torch.equal(one[0].view(torch.int16), out[b, :n].view(torch.int16)), b
    zero = _wgmma_ragged_case(pad=0.0)
    assert torch.equal(_run_attention(zero['qkv'], B, S, H, lens).view(torch.int16), out.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize('B,S,H', UNIFORM_CASES)
def test_flash_wgmma_uniform_stays_in_bounds(B, S, H):
    """Output rows past B * S of an over-allocated buffer stay untouched."""
    case = _uniform_case(B, S, H)
    d = H * 64
    out = torch.full((B * S + 70, d), SENTINEL, dtype=torch.bfloat16)
    out = _run_attention(case['qkv'], B, S, H, out=out)
    assert (out[B * S:] == SENTINEL).all()
    _check_attention(case, out[:B * S].view(B, S, d).float(), 'wgmma B=%d S=%d H=%d' % (B, S, H))


@pytest.mark.gpu
@pytest.mark.parametrize('B,S,H,lens', F32_ATTN_CASES)
def test_attn_f32(B, S, H, lens):
    case = _f32_attn_case(B, S, H, lens)
    out = _run_attention(case['qkv'], B, S, H, lens, fp32=True)
    _check_attention(case, _split_value(out, H * 64), 'attn f32 S=%d ragged=%s' % (S, lens is not None))
    if lens is not None:
        for b, n in enumerate(lens):
            assert not out[b, n:].view(torch.int16).any(), b
        zero = _f32_attn_case(B, S, H, lens, pad=0.0)
        assert torch.equal(_run_attention(zero['qkv'], B, S, H, lens, fp32=True).view(torch.int16), out.view(torch.int16))


@pytest.mark.gpu
def test_op_argument_checks():
    """Bad arguments are refused on the host with a message, before anything is launched."""
    L = _lib()
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    x = torch.zeros(16, device='cuda')
    p = x.data_ptr()

    def dec(beam=2, n_partials=3, lens=None, pos=5, T=8, grid=0, fp32=0, M=50):
        return lib.gitb200_op_decode_attention(p, n_partials, p, p, p, p, p, None, p, 2, beam, M, _lens_arg(lens), T, pos,
                                               768, fp32, grid, st)
    for kw, msg in ((dict(beam=5), 'beam'), (dict(beam=0), 'beam'), (dict(n_partials=5), 'n_partials'),
                    (dict(lens=[50, 51]), 'outside 1 .. 50'), (dict(lens=[0, 3]), 'outside 1 .. 50'),
                    (dict(pos=8), 'position'), (dict(grid=25), 'grid'),
                    (dict(fp32=1, M=16000, T=8), 'shared memory')):
        assert dec(**kw) != 0, kw
        assert msg in L.last_error(None), (kw, L.last_error(None))
    rc = lib.gitb200_op_attention_ex(p, p, p, p, 2, 10, 1, 192, 192, 1920, 1920, 64, 640, _lens_arg([3, 11]), 0, st)
    assert rc != 0 and 'outside 1 .. 10' in L.last_error(None)
    rc = lib.gitb200_op_attention_ex(p, p, p, p, 1, 20000, 1, 192, 192, 192 * 20000, 192 * 20000, 64, 0, None, 1, st)
    assert rc != 0 and 'shared memory' in L.last_error(None)
    rc = lib.gitb200_op_attention_ex(p, p, p, p, 2, 10, 1, 192, 192, 1920 + 192, 1920 + 192, 64, 640, None, 0, st)
    assert rc != 0 and 'back to back' in L.last_error(None)          # gap rows between the batches
