"""fp64 statement of hot path A: the image encoder and the image rows of the prefill, stage by stage.

The stages are the ones the engine runs (encode_impl, image_rows):
  * `resample_pos`: the positional embedding re-sampled to a gh x gw patch grid, F.interpolate(mode='bicubic',
    align_corners=False) as the reference does (layers/CLIP/model.py:245-251);
  * `stem`: patch conv, class row, positional add, ln_pre (eps 1e-5);
  * `block`: one ViT block -- LN1, QKV, softmax attention, out-proj + residual, LN2, fc1, QuickGELU, fc2 + residual;
  * `ln_post`: ln_post on every token, input row (f*B + b)*L + l to output [b, f*L + l], `+ temb[f]` after the norm
    for list inputs only (frames truncated to the number of temporal embeddings by the caller);
  * `feats_operand`: the GEMM-operand copy of the features the prefill reads;
  * `vproj`: the visual projection, Linear + LN (eps 1e-5);
  * `image_layers`: the decoder layers over the image rows (post-LN, eps 1e-12, erf-GELU, no mask among image rows),
    their per-layer K and V; the last layer stops after its QKV.

With `rounding` (the engine's default mode) every stage rounds to bf16 exactly where the engine stores bf16: pixels and
conv weights, every GEMM weight, the LN outputs that feed GEMMs, q / k / v, the attention context, the fc1 output and the
features' operand copy.  Everything else is fp64 with the exact sigmoid.  Two differences to the kernels are left to
the tolerances: the fc1 epilogue's QuickGELU uses tanh.approx, and the flash-attention kernel rounds P to bf16 before
the P.V product.  Without `rounding` (the engine's parity mode, fp32-grade) everything is fp64.

Every stage takes `defect=`: None or (kind, ...) -- one planted error, used to show that a tolerance can fail:
  resample_pos: ('bicubic_a05',) Keys cubic with A = -0.5; ('align_corners',) align_corners=True;
  stem:         ('patch_kxky',) (ky, kx) transposed in the patch; ('cls_nopos',) the class row without pos[0];
                ('operand', ) the pixels rounded to bf16 (in parity mode: what a dropped lo half of that operand does);
  block:        ('attn_keys', head, j) keys 64j .. 64j + 63 masked out of one head; ('fc1_tile', j) fc1 output columns
                64j .. 64j + 63 zeroed; ('operand',) the LN2 output (fc1's input operand) rounded to bf16;
  ln_post:      ('frames_swapped',) frames 0 and 1 exchanged in the output layout; ('temb0',) temb[0] on every frame;
  vproj:        ('vproj_nobias',);
  image_layers: ('k_from_prev', j) layer j's K computed from layer j - 1's input.
"""
import math

import torch
import torch.nn.functional as F

from decode_ref import bf16, _ln, _gelu_erf

ENCODERS = {'CLIPViT_B_16': dict(patch=16, width=768, layers=12, heads=12),
            'CLIPViT_L_14': dict(patch=14, width=1024, layers=24, heads=16)}


def _dev(x, device):
    if torch.is_tensor(x):
        return x.to(device)
    if isinstance(x, tuple):
        return tuple(_dev(v, device) for v in x)
    if isinstance(x, dict):
        return {k: _dev(v, device) for k, v in x.items()}
    if isinstance(x, list):
        return [_dev(v, device) for v in x]
    return x


class EncWeights(object):
    """The encoder's weights and the visual projection in fp64; GEMM weights rounded to bf16 when `rounding`."""

    def __init__(self, sd, param=None, rounding=True, n_blocks=None):
        param = param or {}
        cfg = ENCODERS[param.get('image_encoder_type', 'CLIPViT_B_16')]
        self.patch, self.d, self.heads = cfg['patch'], cfg['width'], cfg['heads']
        self.n_layers = cfg['layers'] if n_blocks is None else n_blocks
        self.rounding = rounding
        w = (lambda k: bf16(sd[k])) if rounding else (lambda k: sd[k].double())
        f = lambda k: sd[k].double()
        e = 'image_encoder.'
        self.conv = w(e + 'conv1.weight')                           # [d, 3, p, p]
        self.cls = f(e + 'class_embedding')
        self.pos = f(e + 'positional_embedding')
        self.g0 = int(round(math.sqrt(self.pos.shape[0] - 1)))
        self.ln_pre = (f(e + 'ln_pre.weight'), f(e + 'ln_pre.bias'))
        self.ln_post_w = (f(e + 'ln_post.weight'), f(e + 'ln_post.bias'))
        self.blocks = []
        for i in range(self.n_layers):
            b = e + 'transformer.resblocks.%d.' % i
            self.blocks.append(dict(
                ln1=(f(b + 'ln_1.weight'), f(b + 'ln_1.bias')),
                wqkv=w(b + 'attn.in_proj_weight'), bqkv=f(b + 'attn.in_proj_bias'),
                wo=w(b + 'attn.out_proj.weight'), bo=f(b + 'attn.out_proj.bias'),
                ln2=(f(b + 'ln_2.weight'), f(b + 'ln_2.bias')),
                w1=w(b + 'mlp.c_fc.weight'), b1=f(b + 'mlp.c_fc.bias'),
                w2=w(b + 'mlp.c_proj.weight'), b2=f(b + 'mlp.c_proj.bias')))
        n_emb = param.get('num_image_with_embedding') or 0
        self.temb = torch.stack([f('img_temperal_embedding.%d' % i).reshape(-1) for i in range(n_emb)]) if n_emb else None
        t = 'textual.visual_projection.'
        self.wvp, self.bvp = w(t + '0.weight'), f(t + '0.bias')
        self.lnvp = (f(t + '1.weight'), f(t + '1.bias'))

    def bf(self, t):
        return bf16(t) if self.rounding else t.double()

    def to(self, device):
        for name, val in list(vars(self).items()):
            setattr(self, name, _dev(val, device))
        return self


def _cubic_matrix(n_in, n_out, A, align_corners, dtype, device):
    """[n_out, n_in] 1-D bicubic interpolation matrix: Keys cubic with parameter A over taps floor(x) - 1 .. floor(x) + 2
    clamped to the input, source coordinate (o + 0.5) * n_in / n_out - 0.5 (align_corners: o * (n_in - 1) / (n_out - 1))."""
    o = torch.arange(n_out, dtype=dtype, device=device)
    if align_corners:
        x = o * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
    else:
        x = (o + 0.5) * (n_in / n_out) - 0.5
    fl = torch.floor(x)
    t = x - fl
    taps = [t + 1, t, 1 - t, 2 - t]
    m = torch.zeros(n_out, n_in, dtype=dtype, device=device)
    for a, s in enumerate(taps):
        near = ((A + 2) * s - (A + 3)) * s * s + 1
        far = ((A * s - 5 * A) * s + 8 * A) * s - 4 * A
        wgt = near if a in (1, 2) else far
        idx = (fl.long() - 1 + a).clamp(0, n_in - 1)
        m.index_put_((torch.arange(n_out, device=device), idx), wgt, accumulate=True)
    return m


def resample_pos(pos, gh, gw, defect=None):
    """The positional table [1 + gh*gw, d] for a gh x gw patch grid from the stored [1 + g0*g0, d] (fp64)."""
    pos = pos.double()
    d = pos.shape[1]
    g0 = int(round(math.sqrt(pos.shape[0] - 1)))
    if (gh, gw) == (g0, g0) and defect is None:
        return pos
    grid = pos[1:].reshape(g0, g0, d).permute(2, 0, 1)[None]
    kind = defect[0] if defect is not None else None
    if kind == 'bicubic_a05':
        my = _cubic_matrix(g0, gh, -0.5, False, pos.dtype, pos.device)
        mx = _cubic_matrix(g0, gw, -0.5, False, pos.dtype, pos.device)
        out = torch.einsum('yi,dij,xj->dyx', my, grid[0], mx)[None]
    else:
        out = F.interpolate(grid, size=(gh, gw), mode='bicubic', align_corners=(kind == 'align_corners'))
    return torch.cat([pos[:1], out[0].permute(1, 2, 0).reshape(-1, d)], dim=0)


def stem(W, pixels, pos, defect=None):
    """ln_pre(cls | patch + pos) of pixels [N, 3, H, W] (a trailing partial patch is dropped) with the positional table
    pos [1 + gh*gw, d] of their grid -> [N, 1 + gh*gw, d]."""
    kind = defect[0] if defect is not None else None
    p, d = W.patch, W.d
    N, _, H, Wd = pixels.shape
    gh, gw = H // p, Wd // p
    x = pixels[:, :, :gh * p, :gw * p].double()
    x = bf16(x) if (W.rounding or kind == 'operand') else x
    # [N, 3, gh, p, gw, p] -> [N, gh, gw, 3, p(ky), p(kx)]
    x = x.reshape(N, 3, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5)
    if kind == 'patch_kxky':
        x = x.transpose(-1, -2)
    a = x.reshape(N, gh * gw, 3 * p * p)
    patches = a @ W.conv.reshape(d, -1).T
    cls = W.cls if kind == 'cls_nopos' else W.cls + pos[0]
    tok = torch.cat([cls.expand(N, 1, d), patches + pos[1:]], dim=1)
    return _ln(tok, W.ln_pre[0], W.ln_pre[1], 1e-5)


def block(W, i, x, lens=None, defect=None):
    """ViT block i on x [N, L, d]; lens: None or the valid tokens of each image (keys past them are masked; the rows past
    them are computed but meaningless)."""
    kind = defect[0] if defect is not None else None
    Bk = W.blocks[i]
    N, L, d = x.shape
    H = W.heads
    hd = d // H
    h = W.bf(_ln(x, Bk['ln1'][0], Bk['ln1'][1], 1e-5))
    qkv = W.bf(h @ Bk['wqkv'].T + Bk['bqkv'])
    q, k, v = (t.reshape(N, L, H, hd).transpose(1, 2) for t in qkv.split(d, dim=-1))
    s = (q @ k.transpose(-1, -2)) / math.sqrt(hd)
    if lens is not None:
        keys = torch.arange(L, device=x.device)
        s = s.masked_fill((keys[None, :] >= torch.as_tensor(lens, device=x.device)[:, None])[:, None, None, :], float('-inf'))
    if kind == 'attn_keys':
        s[:, defect[1], :, 64 * defect[2]:64 * defect[2] + 64] = float('-inf')
    ctx = W.bf((torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(N, L, d))
    x = x + (ctx @ Bk['wo'].T + Bk['bo'])
    h = _ln(x, Bk['ln2'][0], Bk['ln2'][1], 1e-5)
    h = bf16(h) if kind == 'operand' else W.bf(h)
    u = h @ Bk['w1'].T + Bk['b1']
    u = W.bf(u * torch.sigmoid(1.702 * u))
    if kind == 'fc1_tile':
        u[..., 64 * defect[1]:64 * defect[1] + 64] = 0
    return x + (u @ Bk['w2'].T + Bk['b2'])


def ln_post(W, x, B, frames, list_input, defect=None):
    """x [frames*B, L, d] in the encoder's image order (f*B + b) -> features [B, frames*L, d]: ln_post (eps 1e-5), frame f
    of image b at tokens f*L .. f*L + L - 1, + temb[f] after the norm for list inputs of a model with temporal embeddings."""
    kind = defect[0] if defect is not None else None
    L, d = x.shape[1], x.shape[2]
    y = _ln(x.double(), W.ln_post_w[0], W.ln_post_w[1], 1e-5).reshape(frames, B, L, d)
    if list_input and W.temb is not None:
        idx = [0] * frames if kind == 'temb0' else list(range(frames))
        y = y + W.temb[idx][:, None, None, :]
    order = list(range(frames))
    if kind == 'frames_swapped':
        order[0], order[1] = 1, 0
    return y[order].permute(1, 0, 2, 3).reshape(B, frames * L, d)


def feats_operand(f, parity):
    """What the engine keeps of features f [rows, d] (fp32) as the prefill's GEMM operand, as fp64: bf16(f) [rows, d], or in
    parity mode [hi | lo | hi] rows of 3d with hi = bf16(f), lo = bf16(f - hi)."""
    f = f.float()
    hi = bf16(f)
    if not parity:
        return hi
    lo = bf16(f.double() - hi)
    return torch.cat([hi, lo, hi], dim=-1)


def vproj(W, feats, defect=None):
    """Linear(d -> 768) + LN (eps 1e-5) of the features as the GEMM reads them ([..., d] fp64)."""
    kind = defect[0] if defect is not None else None
    y = feats.double() @ W.wvp.T
    if kind != 'vproj_nobias':
        y = y + W.bvp
    return _ln(y, W.lnvp[0], W.lnvp[1], 1e-5)


def image_layers(RW, x, lens=None, defect=None):
    """The decoder layers over image rows x [B, M, 768] (the visual projection's output) with decode_ref.RefWeights RW;
    lens: None or the valid tokens of each image (keys past them masked).  Returns per layer dict(k, v) [B, M, 768];
    the last layer stops after its QKV."""
    kind = defect[0] if defect is not None else None
    bf = bf16 if RW.rounding else (lambda t: t.double())
    B, M, D = x.shape
    H = 12
    out = []
    prev_h = None
    for j, Lj in enumerate(RW.layers):
        h = bf(x)
        hk = prev_h if (kind == 'k_from_prev' and defect[1] == j) else h
        q = bf(h @ Lj['wq'].T + Lj['bq'])
        k = bf(hk @ Lj['wk'].T + Lj['bk'])
        v = bf(h @ Lj['wv'].T + Lj['bv'])
        out.append(dict(k=k, v=v))
        prev_h = h
        if j + 1 == len(RW.layers):
            break
        qh, kh, vh = (t.reshape(B, M, H, 64).transpose(1, 2) for t in (q, k, v))
        s = (qh / 8.0) @ kh.transpose(-1, -2)
        if lens is not None:
            keys = torch.arange(M, device=x.device)
            s = s.masked_fill((keys[None, :] >= torch.as_tensor(lens, device=x.device)[:, None])[:, None, None, :],
                              float('-inf'))
        ctx = bf((torch.softmax(s, dim=-1) @ vh).transpose(1, 2).reshape(B, M, D))
        xa = _ln(x + (ctx @ Lj['wo'].T + Lj['bo']), Lj['ln1'][0], Lj['ln1'][1], 1e-12)
        u = bf(_gelu_erf(bf(xa) @ Lj['w1'].T + Lj['b1']))
        x = _ln(xa + (u @ Lj['w2'].T + Lj['b2']), Lj['ln2'][0], Lj['ln2'][1], 1e-12)
    return out
