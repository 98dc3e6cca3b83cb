"""GPU: every hand-written kernel through its C-ABI entry point against a plain PyTorch fp32 statement of
the same op on the same (bf16-rounded) inputs.  The GEMM and LayerNorm tests here are a smoke layer: every GEMM
instantiation, epilogue form and split-K / LM-head consumer is compared with fp64 in tests/test_gpu_gemm.py."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from generativeimage2text_b200 import _lib
    return _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gemm(a, w, bias=None, resid=None, act=0, out_bf16=False, transposed=False, k_splits=1, bn=0):
    L = _lib()
    M, K = a.shape
    N = w.shape[0]
    out = torch.zeros((M, N), dtype=torch.bfloat16 if out_bf16 else torch.float32, device='cuda')
    rc = L.load().gitb200_op_gemm(a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                  resid.data_ptr() if resid is not None else None, out.data_ptr(), M, N, K, act,
                                  int(out_bf16), int(transposed), k_splits, bn, _stream())
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    return out


def _ref_gemm(a, w, bias=None, resid=None, act=0):
    y = a.double() @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    if act == 1:
        y = y * torch.sigmoid(1.702 * y)
    elif act == 2:
        y = y * 0.5 * (1.0 + torch.erf(y / 2 ** 0.5))
    if resid is not None:
        y = y + resid.double()
    return y.float()


def _rand(shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


@pytest.mark.parametrize('M,N,K,bn', [
    (128, 128, 64, 128),      # one tile, one k-block
    (128, 128, 256, 128),     # accumulate over k-blocks inside one swizzle ring
    (256, 256, 1024, 128),    # pipeline wrap-around (16 k-blocks > stages)
    (1000, 768, 768, 128), (1000, 768, 768, 192), (1000, 768, 768, 256),
    (12608, 768, 768, 0),     # persistent: several tiles per CTA, tail rows
    (300, 3072, 776, 256),    # K tail (776 = 12*64 + 8) relies on TMA zero fill
])
def test_gemm_plain(M, N, K, bn):
    a, w = _rand((M, K), 1.0, 1), _rand((N, K), 0.05, 2)
    out = _gemm(a, w, bn=bn)
    ref = _ref_gemm(a, w)
    err = (out - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize('M,N,K,bn,act,out_bf16,use_resid', [
    (256, 256, 64, 256, 0, False, False),      # one tile, one k-block
    (512, 512, 512, 256, 0, True, False),      # several tiles, ring wrap-around
    (1000, 768, 768, 192, 0, False, True),     # M tail, 192-wide tiles, residual epilogue
    (12608, 3072, 768, 256, 1, True, False),   # ViT c_fc: persistent CTAs, several tiles each
    (12608, 768, 3072, 192, 0, False, True),   # ViT c_proj
])
def test_gemm_wide_tiles(M, N, K, bn, act, out_bf16, use_resid):
    """128 x 256 / 128 x 192 tiles at the encoder's GEMM shapes, with the epilogues those GEMMs use."""
    a, w = _rand((M, K), 1.0, 41), _rand((N, K), 0.05, 42)
    bias = _rand((N,), 0.5, 43, torch.float32)
    resid = _rand((M, N), 1.0, 44, torch.float32) if use_resid else None
    out = _gemm(a, w, bias, resid, act, out_bf16, False, 1, bn)
    ref = _ref_gemm(a, w, bias, resid, act)
    tol = 3e-2 if out_bf16 else 2e-3
    assert (out.float() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('act,out_bf16,use_resid', [(0, False, True), (1, True, False), (2, True, False), (0, True, False)])
def test_gemm_epilogues(act, out_bf16, use_resid):
    M, N, K = 777, 1536, 768
    a, w = _rand((M, K), 1.0, 3), _rand((N, K), 0.05, 4)
    bias = _rand((N,), 0.5, 5, torch.float32)
    resid = _rand((M, N), 1.0, 6, torch.float32) if use_resid else None
    out = _gemm(a, w, bias, resid, act, out_bf16)
    ref = _ref_gemm(a, w, bias, resid, act)
    tol = 3e-2 if out_bf16 else 2e-3
    assert (out.float() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('rows,feats,K,splits', [
    (64, 2304, 768, 1), (64, 2304, 768, 3), (64, 768, 768, 6), (64, 768, 3072, 8), (5, 768, 768, 1), (1, 3072, 768, 1),
    (128, 768, 3072, 4), (256, 768, 3072, 8), (64, 30522, 768, 1), (200, 1024, 768, 1),
])
def test_gemm_skinny_transposed(rows, feats, K, splits):
    x, w = _rand((rows, K), 1.0, 7), _rand((feats, K), 0.05, 8)
    bias = _rand((feats,), 0.5, 9, torch.float32) if splits == 1 else None
    out = _gemm(x, w, bias, None, 0, False, True, splits)
    ref = _ref_gemm(x, w, bias)
    assert (out - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    if splits > 1:     # split-K partial buffers are summed in split order: bit-identical from run to run
        assert torch.equal(out, _gemm(x, w, bias, None, 0, False, True, splits))


def test_gemm_skinny_gelu_bf16():
    x, w = _rand((64, 768), 1.0, 10), _rand((3072, 768), 0.05, 11)
    bias = _rand((3072,), 0.5, 12, torch.float32)
    out = _gemm(x, w, bias, None, 2, True, True, 1)
    ref = _ref_gemm(x, w, bias, None, 2)
    assert (out.float() - ref).abs().max().item() < 3e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('D,rows', [(768, 1000), (1024, 257), (768, 3)])
def test_layernorm(D, rows):
    L = _lib()
    x = _rand((rows, D), 2.0, 20, torch.float32)
    bias = _rand((D,), 0.5, 21, torch.float32)
    resid = _rand((rows, D), 1.0, 22, torch.float32)
    g = 1 + _rand((D,), 0.1, 23, torch.float32)
    b = _rand((D,), 0.1, 24, torch.float32)
    of = torch.empty_like(x)
    ob = torch.empty((rows, D), dtype=torch.bfloat16, device='cuda')
    rc = L.load().gitb200_op_layernorm(x.data_ptr(), bias.data_ptr(), resid.data_ptr(), g.data_ptr(), b.data_ptr(),
                                       ctypes.c_float(1e-12), of.data_ptr(), ob.data_ptr(), rows, D, _stream())
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x + bias + resid, (D,), g, b, 1e-12)
    assert (of - ref).abs().max().item() < 2e-5
    assert (ob.float() - ref).abs().max().item() < 3e-2


@pytest.mark.parametrize('B,S,H', [(2, 197, 12), (1, 257, 16), (1, 64, 1), (1, 1182, 12), (3, 5, 2), (2, 513, 3), (1, 640, 2),
                                   (2, 1201, 12), (3, 600, 1)])
def test_flash_attention(B, S, H):
    L = _lib()
    d = H * 64
    qkv = _rand((B, S, 3 * d), 1.0, 30)
    out = torch.zeros((B, S, d), dtype=torch.bfloat16, device='cuda')
    base = qkv.data_ptr()
    rc = L.load().gitb200_op_attention(base, base + d * 2, base + 2 * d * 2, out.data_ptr(), B, S, H, 3 * d, 3 * d,
                                       S * 3 * d, S * 3 * d, d, S * d, _stream())
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    q, k, v = qkv.float().split(d, dim=-1)
    q = q.view(B, S, H, 64).transpose(1, 2)
    k = k.view(B, S, H, 64).transpose(1, 2)
    v = v.view(B, S, H, 64).transpose(1, 2)
    ref = (torch.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1) @ v).transpose(1, 2).reshape(B, S, d)
    # the flash_attn_wgmma_kernel bound of tests/test_gpu_attention.py
    assert (out.float() - ref).abs().max().item() <= 3.5e-3 * v.abs().max().item() + 1e-5
