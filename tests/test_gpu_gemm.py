"""Every instantiation of gemm_bf16_wgmma<BN, EPI> (csrc/gemm.cuh), in every epilogue form the engine launches, and the
consumers of its split-K partials and LM-head statistics, against plain fp64 PyTorch statements of the same operations.

Kernels and their entry points:
  gitb200_op_gemm_ex:      gemm_bf16_wgmma<BN, EPI> through launch_gemm, with the row map, column segments, split3, the
                           statistics epilogue (EPI_LSE), raw split-K partial buffers, in-place residual and the skip flag;
  gitb200_op_layernorm_ex: layernorm_kernel<768 / 1024, PRE> with n_partials, split3, the frame remap and the skip flag;
  gitb200_op_lse_combine:  lse_combine_kernel + loss_mean_kernel on caller-supplied partials.

How cases are built.  INSTANTIATIONS mirrors launch_gemm_bn: every (BN, EPI) pair in it is run.  ENGINE_CALLS lists every
launch_gemm( call site of gitb200.cu / engine_api.inc with the form it launches.  Output buffers carry guard rows and
columns filled with SENTINEL: rows a row map skips, rows past M, columns past a segment, splits that were dropped and the
whole output under skip != 0 must still hold it.

Exact layer (no tolerance).  Operands are small integers stored as bf16; the builder asserts that |A| @ |W|^T (+ |bias|
+ |resid|) stays below 2^24, so every product and every fp32 partial sum is exact in any order.  fp32 output must equal the
fp64 reference, bf16 output its round-to-nearest-even, split3 (bf16(x), bf16(x - hi), bf16(x)), and each split-K partial
the fp64 sum over exactly its k range.  Epilogues with an activation run in this layer with a bias that lifts every
pre-activation to >= 40, where all three activations return x itself (tanh.approx(0.851 x) == 1, exp(-x^2 / 2) == 0,
1 + expf(-1.702 x) == 1); their curves are checked in the real-valued layer.  A mismatch is reported as (tile row, tile
column, 64-column chunk, segment, split) of the first wrong element.

Real-valued layer.  Gaussian operands at the engine's scales.  Per element
  |out - ref| <= LIP * C_ACC * (|A| @ |W|^T) + C_ACT[act] * |pre-activation| + C_OUT * |ref| + ABS
with C_OUT = 2^-8 for bf16 output (8 significant bits: half an ulp is up to 2^-8 relative) and 2^-23 for fp32 output (the bias and residual adds
round twice), LIP = 1.13 (the largest slope of either GELU) when an activation follows.  The constants below are about
2x the largest ratio seen over these cases on an H100 80GB HBM3 (700 W power limit), given after each.

The suite must be able to fail: the unmarked tests at the end corrupt the reference the way a kernel bug would (a dropped
k-step, a k-block taken twice, a 32-column block stored one block to the right, a row map off by one image, swapped
segments, moved split boundaries, partials added in reverse, a statistics half tile merged without rescaling, the last two
vocabulary columns ignored) and assert that the comparison used by the GPU tests rejects it, by >= 4x the bound in the
real-valued layer.  Case builders, references and those checks run on the CPU; kernel runs need an H100.

Setting GITB200_GEMM_OBSERVED=<file> writes the largest ratio each bound saw as JSON (how the constants were measured).
"""
import ctypes
import json
import math
import os

import pytest
import torch

gpu = pytest.mark.gpu

SENTINEL = 1000.0            # exact in bf16; no reference value equals it where it matters (guards only)
BM, BK = 128, 64

C_ACC = 3.2e-6               # fp32 accumulation of exact bf16 products, relative to |A| @ |W|^T; observed 1.6e-6 on a
                             # logit whose 768 products share one sign (test_lse_statistics plants it as the row maximum)
                             # and 6.84e-7 on Gaussian operands at K = 4096: wgmma does not round its fp32 sums to nearest
C_ACC_PARITY = 5.4e-6        # (hi, lo) operands at 3K against the fp64 product of the fp32 values; observed 2.67e-6 = 2^-18.5
C_OUT = {True: 2.0 ** -8, False: 2.0 ** -23}
LIP = 1.13
# Activation error beyond the output rounding, relative to |pre-activation|, seen at the planted pre-activations:
C_ACT = {0: 0.0,
         1: 1.3e-8,          # tanh.approx QuickGELU (looser: one MUFU op); observed 6.36e-9
         2: 2.0e-9,          # A&S 7.1.26 erf with ex2 / rcp; observed 9.83e-10
         3: 0.0}             # expf sigmoid, full-precision division; observed 0 beyond the 2^-16 of hi + lo
ABS = 1e-7
C_LSE = 2.8e-6               # statistics: log(sum exp) and the fp32 sums, relative to max(1, |max|); observed 1.38e-6
C_LN = {True: 2.0 ** -8, False: 1.2e-6}     # LayerNorm output, relative to max(1, |ref|); fp32 observed 5.73e-7
C_LOGPROB = 3.0e-7           # lse_combine_kernel log-probability, relative to max(1, |log-probability|); observed 1.35e-7
C_LOSS = 1.6e-5              # smoothed loss, relative to max(1, |loss|); observed 7.73e-6

OBSERVED = {}


def _observe(name, value):
    """Keeps the largest value a bound saw on the device (the CPU tests plant defects: they are not observations)."""
    if isinstance(value, torch.Tensor) and not value.is_cuda:
        return
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), float(value))


@pytest.fixture(scope='module', autouse=True)
def _dump_observed():
    yield
    path = os.environ.get('GITB200_GEMM_OBSERVED')
    if path and OBSERVED:
        with open(path, 'w') as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)


# ---------------------------------------------------------------------------------------------------------------------
# models of the kernel's geometry (mirrors of csrc/gemm.cuh and launch_gemm in csrc/gitb200.cu)
# ---------------------------------------------------------------------------------------------------------------------
def stages(bn):
    """GemmCfg<BN>::STAGES."""
    stage = BM * BK * 2 + bn * BK * 2
    return min(8, (227 * 1024 - 1024 - 256 - 2 * 4 * 32 * 128) // stage)


def pick_bn(N, transposed):
    """pick_bn of gitb200.cu; N is the kernel's N (activation rows in the transposed shape)."""
    if transposed:
        return 64 if N <= 64 else (128 if N <= 128 else 256)
    if N % 256 == 0 and N >= 1024:
        return 256
    if N % 192 == 0:
        return 192
    if N % 256 == 0:
        return 256
    if N % 128 == 0:
        return 128
    return 256 if N > 192 else (192 if N > 128 else 128)


def split_ranges(K, requested):
    """k ranges [k0, k1) of the splits launch_gemm runs for `requested`: ceil(k-blocks / requested) 64-wide k-blocks
    each, empty splits dropped."""
    kb_total = -(-K // BK)
    splits = max(1, min(requested, kb_total))
    kb_per = -(-kb_total // splits)
    eff = -(-kb_total // kb_per)
    return [(s * kb_per * BK, min(K, (s + 1) * kb_per * BK)) for s in range(eff)]


def row_map(m, rpb, bstride, roff):
    """Output row of GEMM row m: (m / rpb) * bstride + m % rpb + roff (rpb <= 0: identity)."""
    if rpb <= 0:
        return m
    return (m // rpb) * bstride + m % rpb + roff


def lse_owned_columns(N, part):
    """Columns whose statistics land in float4 `part` = 2 * tile + half of a row: 32 of every 64-column chunk of the
    256-column tile (n_blk * 256 + cc * 64 + half * 32 + 0..31, cc 0..3), clipped to N."""
    tile, half = divmod(part, 2)
    cols = [tile * 256 + cc * 64 + half * 32 + j for cc in range(4) for j in range(32)]
    return [c for c in cols if c < N]


def bf16_rne(x):
    """fp32 -> nearest bf16 (ties to even), returned as fp32; by integer arithmetic on the bit pattern."""
    b = x.float().contiguous().view(torch.int32)
    r = b + 0x7fff + ((b >> 16) & 1)
    return (r & -65536).view(torch.float32)


def split3_rows(x):
    """[hi | lo | hi] rows of the parity mode: hi = bf16(x), lo = bf16(x - hi), as fp32."""
    x = x.float()
    hi = bf16_rne(x)
    lo = bf16_rne(x - hi)
    return torch.cat([hi, lo, hi], dim=1)


def act_ref(x, act):
    """The activations in fp64: 1 and 3 QuickGELU x sigmoid(1.702 x), 2 erf-GELU."""
    if act in (1, 3):
        return x * torch.sigmoid(1.702 * x)
    if act == 2:
        return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))
    return x


class Layout:
    """Where the normal epilogue puts logical element (m, n): segment n // seg_n, physical row row_map(m), column
    n % seg_n, in buffers of pitch ldo with guard rows and columns.  split3 rows are 3 * N wide (one segment)."""

    def __init__(self, M, N, segs=1, rpb=0, bstride=0, roff=0, split3=False, guard_cols=8, guard_rows=2):
        assert N % segs == 0 and not (split3 and segs > 1)
        self.M, self.N, self.segs, self.seg_n = M, N, segs, N // segs
        self.rpb, self.bstride, self.roff, self.split3 = rpb, bstride, roff, split3
        self.width = self.seg_n * (3 if split3 else 1)
        self.ldo = self.width + guard_cols
        self.rows = row_map(torch.arange(M), rpb, bstride, roff)
        self.phys_rows = (-(-M // rpb) * bstride if rpb > 0 else M) + guard_rows

    def scatter(self, logical, dtype=torch.float32, fill=SENTINEL):
        """Buffers as a correct kernel leaves them: `logical` [M, N] ([M, 3N] for split3) in place, `fill` elsewhere."""
        rows = self.rows.to(logical.device)
        bufs = []
        for s in range(self.segs):
            buf = torch.full((self.phys_rows, self.ldo), fill, dtype=dtype, device=logical.device)
            buf[rows, :self.width] = logical[:, s * self.width:(s + 1) * self.width].to(dtype)
            bufs.append(buf)
        return bufs

    def gather(self, bufs):
        rows = self.rows.to(bufs[0].device)
        return torch.cat([b[rows, :self.width] for b in bufs], dim=1)

    def guards_ok(self, bufs, fill=SENTINEL):
        """None, or a message naming the first guard element that no longer holds `fill`."""
        for s, b in enumerate(bufs):
            keep = torch.ones_like(b, dtype=torch.bool)
            keep[self.rows.to(b.device), :self.width] = False
            bad = keep & (b.float() != fill)
            if bad.any():
                r, c = (int(v) for v in bad.nonzero()[0])
                return 'guard element overwritten: segment %d physical row %d column %d holds %r' % (s, r, c, b[r, c].item())
        return None


def where(m, n, N, bn, seg_n=None, split=None, transposed=False):
    """Names the tile that owns logical element (m, n) (n modulo N in split3 rows)."""
    n = n % N
    if transposed:      # kernel M = features (columns of the logical matrix), kernel N = activation rows
        return 'feature tile %d, row tile %d, 64-row chunk %d%s (row %d, feature %d)' % (
            n // BM, m // bn, (m % bn) // 64, '' if split is None else ', split %d' % split, m, n)
    return 'tile row %d, tile column %d, 64-column chunk %d, segment %d%s (row %d, column %d)' % (
        m // BM, n // bn, (n % bn) // 64, n // (seg_n or N), '' if split is None else ', split %d' % split, m, n)


def check_exact(got, exp, N, bn, seg_n=None, split=None, transposed=False):
    """None when the logical matrices are equal, else a message naming the first wrong element's tile."""
    bad = got.float() != exp.float()
    if not bad.any():
        return None
    m, n = (int(v) for v in bad.nonzero()[0])
    return '%d wrong elements, first at %s: got %r, expected %r' % (
        int(bad.sum()), where(m, n, N, bn, seg_n, split, transposed), got[m, n].item(), exp[m, n].item())


def check_bound(got, ref, bound, N, bn, seg_n=None, transposed=False):
    """(largest |got - ref| / bound, message naming the worst element's tile)."""
    ratio = (got.double() - ref).abs() / bound
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float('inf')), ratio)
    worst = ratio.max().item()
    m, n = (int(v) for v in (ratio == ratio.max()).nonzero()[0])
    return worst, '|got - ref| = %.3g is %.2f x its bound at %s' % (
        abs(got[m, n].item() - ref[m, n].item()), worst, where(m, n, N, bn, seg_n, None, transposed))


# ---------------------------------------------------------------------------------------------------------------------
# operands and fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def int_operands(M, N, K, seed, amax=3, wmax=2, density=1.0):
    """Integer A [M, K] in -amax..amax and W [N, K] in -wmax..wmax as bf16; asserts every partial sum < 2^24."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randint(-amax, amax + 1, (M, K), generator=g).float()
    W = torch.randint(-wmax, wmax + 1, (N, K), generator=g).float()
    if density < 1.0:
        A = A * (torch.rand((M, K), generator=g) < density)
        W = W * (torch.rand((N, K), generator=g) < density)
    assert K * amax * wmax < 2 ** 24
    return A.bfloat16(), W.bfloat16()


def int_vector(shape, seed, lim=8):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-lim, lim + 1, shape, generator=g).float()


def real_operands(M, N, K, seed, wscale=0.04):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((M, K), generator=g).bfloat16(), (torch.randn((N, K), generator=g) * wscale).bfloat16()


def ref_product(A, W, k0=0, k1=None):
    """fp64 A[:, k0:k1] @ W[:, k0:k1]^T."""
    return A[:, k0:k1].double() @ W[:, k0:k1].double().t()


def abs_product(A, W):
    return A.double().abs() @ W.double().abs().t()


def saturating_bias(A, W, N):
    """Integer bias that lifts every pre-activation of integer operands to >= 40, where each activation returns x."""
    lift = float(abs_product(A, W).max().item()) + 40.0
    assert 2 * lift < 256, 'keep the lifted values exactly representable in bf16'
    return torch.full((N,), lift, dtype=torch.float32, device=A.device)


def expected_output(x, out_bf16, split3):
    """What an exact fp64 result x is stored as: fp32, bf16 (RNE) or split3 rows; as fp32 values."""
    assert x.abs().max().item() < 2 ** 24
    if split3:
        return split3_rows(x)
    return bf16_rne(x) if out_bf16 else x.float()


def lse_stats_ref(x, targets):
    """fp64 [M, n_parts, 4] = (max, sum exp(x - max), sum x, x[target]) over the columns each float4 owns (see
    lse_owned_columns); parts that own no column hold (-inf, 0, 0, 0).  x fp64 [M, N]; targets [M] (-1: none)."""
    M, N = x.shape
    nt = -(-N // 256)
    xp = torch.full((M, nt * 256), float('-inf'), dtype=torch.float64, device=x.device)
    xp[:, :N] = x
    col = torch.arange(nt * 256, device=x.device)

    def parts(t):      # [.., nt * 256] -> [.., 2 * nt, 128]: part 2 * tile + half owns 32 of every 64 columns
        lead = t.shape[:-1]
        return t.reshape(*lead, nt, 4, 2, 32).transpose(-3, -2).reshape(*lead, 2 * nt, 128)

    xs, cs = parts(xp), parts(col)
    valid = cs < N
    m = xs.max(dim=-1).values
    e = torch.where(valid, torch.exp(xs - torch.where(torch.isinf(m), torch.zeros_like(m), m)[..., None]), torch.zeros_like(xs))
    xz = torch.where(valid, xs, torch.zeros_like(xs))
    hit = valid & (cs[None] == targets.to(x.device).long()[:, None, None])
    return torch.stack([m, e.sum(-1), xz.sum(-1), (xz * hit).sum(-1)], dim=-1)


def lse_fold_ref(stats, rescale=True):
    """log(sum exp) of a row from its parts [.., n_parts, 4] in fp64 (rescale=False: the planted defect of adding the
    parts' sums without bringing them to a common max)."""
    m, se = stats[..., 0], stats[..., 1]
    top = m.max(dim=-1).values
    w = torch.exp(m - top[..., None]) if rescale else torch.ones_like(m)
    w = torch.where(torch.isinf(m), torch.zeros_like(w), w)
    return top + torch.log((se * w).sum(-1))


def smoothed_loss_ref(x, targets, eps=0.1):
    """Per-row SmoothLabelCrossEntropyLoss in fp64 (the formula of oracle/score_oracle.py smooth_label_ce)."""
    V = x.shape[1]
    one_hot = torch.zeros_like(x).scatter(1, targets.view(-1, 1).long(), 1.0)
    q = one_hot * (1 - eps) + (1 - one_hot) * eps / (V - 1)
    lp = torch.log_softmax(x, dim=1)
    return (q * (q.log() - lp)).sum(dim=1)


def ln_ref(parts, bias, resid, gamma, beta, eps):
    """LayerNorm of split-K partials [n, rows, D]: added in split order in fp32 (as the kernel must), the rest in fp64."""
    s = parts[0].clone()
    for p in parts[1:]:
        s = s + p
    v = s.double()
    if resid is not None:
        v = v + resid.double()
    if bias is not None:
        v = v + bias.double()
    mean = v.mean(-1, keepdim=True)
    var = ((v - mean) ** 2).mean(-1, keepdim=True)
    return (v - mean) / torch.sqrt(var + eps) * gamma.double() + beta.double()


def remap_rows(rows, B, F, L):
    """Frame remap of the video path: input row (f * B + b) * L + l -> output row (b * F + f) * L + l; (out row, frame)."""
    r = torch.arange(rows)
    img, l = r // L, r % L
    f, b = img // B, img % B
    return (b * F + f) * L + l, f


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations of launch_gemm_bn and the engine's call sites
# ---------------------------------------------------------------------------------------------------------------------
# (bn, transposed, out_bf16, resid, partial, act, split3) -- one line per case label of launch_gemm_bn
_NORMAL_EPIS = [(True, False, 0), (False, True, 0), (False, False, 0), (True, False, 1), (True, False, 2)]   # bf16, resid, act
INSTANTIATIONS = (
    [(bn, False, bf, rs, False, act, False) for bn in (128, 192, 256) for bf, rs, act in _NORMAL_EPIS] +
    [(256, False, True, False, False, act, True) for act in (3, 2)] +
    [(bn, True, True, False, False, 2, True) for bn in (64, 128, 256)] +
    [(bn, True, False, False, True, 0, False) for bn in (64, 128, 256)] +
    [(bn, True, False, False, False, 0, False) for bn in (64, 128, 256)] +
    [(bn, True, True, False, False, 2, False) for bn in (64, 128, 256)])
N_INSTANTIATIONS = len(INSTANTIATIONS) + 1     # + <256, EPI_LSE>, run by the statistics tests


def _inst_id(p):
    bn, tr, bf, rs, pa, act, s3 = p
    return 'bn%d-%s-%s%s%s-act%d%s' % (bn, 'T' if tr else 'N', 'bf16' if bf else 'f32', '+resid' if rs else '',
                                        '+partial' if pa else '', act, '+split3' if s3 else '')


# Normal-shape calls: name -> (site, M, N, K, dict(bias, act, out_bf16, resid: None / 'inplace' / 'other', segs, map)).
# map = (rows_per_batch, batch_stride, row_offset).  Sites are the launch_gemm( lines of csrc/gitb200.cu (g:) and
# csrc/engine_api.inc (e:).  The parity mode launches the same calls at 3 K with split3 / fp32 outputs: those
# instantiations are in INSTANTIATIONS and the (hi, lo) arithmetic in test_parity_operands.
ENGINE_CALLS = {
    # encode_impl: patch embedding, rows land at token 1 + patch of each image
    'patch_b16_1img': ('g:1214', 196, 768, 768, dict(map=(196, 197, 1))),
    'patch_b16_2img': ('g:1214', 2 * 196, 768, 768, dict(map=(196, 197, 1))),
    'patch_b16_64img': ('g:1214', 64 * 196, 768, 768, dict(map=(196, 197, 1))),
    'patch_l14_1img': ('g:1214', 256, 1024, 640, dict(map=(256, 257, 1))),          # K = 588 padded to 640
    'patch_l14_2img': ('g:1214', 2 * 256, 1024, 640, dict(map=(256, 257, 1))),
    'patch_l14_64img': ('g:1214', 64 * 256, 1024, 640, dict(map=(256, 257, 1))),
    'patch_video_2x6': ('g:1214', 12 * 196, 768, 768, dict(map=(196, 197, 1))),      # 2 clips x 6 frames
    'patch_ragged_lmax141': ('g:1214', 3 * 140, 768, 768, dict(map=(140, 141, 1))),  # every image owns L_max - 1 rows
    'patch_ragged_tiny': ('g:1214', 40 * 3, 768, 768, dict(map=(3, 4, 1))),          # a 32-row block spans 11 images
    # encode_impl: the encoder layers
    'enc_qkv_768': ('g:1238', 2 * 197, 2304, 768, dict(bias=True, out_bf16=True)),
    'enc_qkv_1024': ('g:1238', 2 * 257, 3072, 1024, dict(bias=True, out_bf16=True)),
    'enc_outproj_768': ('g:1240', 2 * 197, 768, 768, dict(bias=True, resid='inplace')),
    'enc_outproj_1024': ('g:1240', 2 * 257, 1024, 1024, dict(bias=True, resid='inplace')),
    'enc_cfc_768': ('g:1242', 2 * 197, 3072, 768, dict(bias=True, act=1, out_bf16=True)),
    'enc_cfc_1024': ('g:1242', 2 * 257, 4096, 1024, dict(bias=True, act=1, out_bf16=True)),
    'enc_cproj_768': ('g:1243', 2 * 197, 768, 3072, dict(bias=True, resid='inplace')),
    'enc_cproj_1024': ('g:1243', 2 * 257, 1024, 4096, dict(bias=True, resid='inplace')),
    'enc_cproj_768_64img': ('g:1243', 64 * 197 + 5, 768, 3072, dict(bias=True, resid='inplace')),
    # image_rows: the visual projection, then decoder_layers over the image rows
    'visual_projection_768': ('g:1342', 2 * 197, 768, 768, dict(bias=True)),
    'visual_projection_1024': ('g:1342', 2 * 257, 768, 1024, dict(bias=True)),
    'prefill_qkv': ('g:1321', 2 * 197, 2304, 768, dict(bias=True, out_bf16=True, segs=3)),   # q scratch | K cache | V cache
    'prefill_qkv_row_map': ('g:1321', 2 * 197, 2304, 768, dict(bias=True, out_bf16=True, segs=3, map=(197, 200, 2))),
    'prefill_outproj': ('g:1324', 2 * 197, 768, 768, dict(bias=True, resid='other')),
    'prefill_fc1': ('g:1326', 2 * 197, 3072, 768, dict(bias=True, act=2, out_bf16=True)),
    'prefill_fc2': ('g:1327', 2 * 197, 768, 3072, dict(bias=True, resid='other')),
    # score_impl: decoder_layers over the caption text rows (the LM head at e:696 is the statistics epilogue: test_lse_*)
    'score_qkv': ('g:1321', 5 * 13, 2304, 768, dict(bias=True, out_bf16=True, segs=3)),       # q | text K | text V
    'score_qkv_parity': ('g:1321', 5 * 13, 2304, 768, dict(bias=True, segs=3)),               # fp32 segments
    'score_outproj': ('g:1324', 5 * 13, 768, 768, dict(bias=True, resid='other')),
    'score_fc1': ('g:1326', 5 * 13, 3072, 768, dict(bias=True, act=2, out_bf16=True)),
    'score_fc2': ('g:1327', 5 * 13, 768, 3072, dict(bias=True, resid='other')),
}
# Sites not in the table: step_layers' skinny calls (g:1434, DECODE_CALLS), the LM-head statistics (e:696, test_lse_*) and the
# two hooks themselves (gitb200_op_gemm e:757, which tests/test_gpu_kernels.py runs, and gitb200_op_gemm_ex e:813).
OTHER_SITES = ('g:1434', 'e:696', 'e:757', 'e:813')
# step_layers' skinny calls (g:1434 through the `skinny` lambda): name -> (features, K, requested splits, bias, act, bf16)
DECODE_CALLS = {
    'decode_qkv': (2304, 768, 3, False, 0, False),        # kQkvSplits
    'decode_outproj': (768, 768, 6, False, 0, False),     # kOutProjSplits
    'decode_fc1': (3072, 768, 1, True, 2, True),
    'decode_fc2': (768, 3072, 8, False, 0, False),        # kFc2Splits
    'decode_lm_head': (30522, 768, 1, True, 0, False),    # ldo = 30522: float2 stores, feature tail of 2
}
DECODE_ROWS = (1, 5, 64, 65, 128, 200, 256)


# ---------------------------------------------------------------------------------------------------------------------
# GPU plumbing
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from generativeimage2text_b200 import _lib
    return _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _padded(t, ld, junk=7.0):
    """t [rows, K] stored with row pitch ld > K; the padding holds a value no k range may pick up."""
    buf = torch.full((t.shape[0], ld), junk, dtype=t.dtype, device=t.device)
    buf[:, :t.shape[1]] = t
    return buf


def launch(expect_error=False, **kw):
    """gitb200_op_gemm_ex with the descriptor fields in kw (tensors for pointers).  Returns the effective split count."""
    L = _lib()
    d = L.GemmDesc()
    outs = kw.pop('out')
    for i, o in enumerate(outs):
        d.out[i] = o.data_ptr()
    for k, v in kw.items():
        setattr(d, k, _ptr(v) if isinstance(v, torch.Tensor) or v is None else v)
    eff = ctypes.c_int(0)
    rc = L.load().gitb200_op_gemm_ex(ctypes.byref(d), ctypes.byref(eff), _stream())
    if expect_error:
        assert rc != 0 and L.last_error(None), 'the call should have been refused'
        return L.last_error(None)
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    return eff.value


def run_normal(A, W, lay, bias=None, resid=None, act=0, out_bf16=False, bn=0, inplace=False, skip=0, lda=None, ldb=None):
    """The normal epilogue on device tensors; returns the output buffers.  inplace: the residual lives in out[0]."""
    M, K = A.shape
    N = W.shape[0]
    dtype = torch.bfloat16 if out_bf16 else torch.float32
    if inplace:
        outs = lay.scatter(resid, dtype)
        resid_t, ld_resid = outs[0], lay.ldo
    else:
        outs = [torch.full((lay.phys_rows, lay.ldo), SENTINEL, dtype=dtype, device='cuda') for _ in range(lay.segs)]
        resid_t, ld_resid = resid, N
    a_t = A if lda is None else _padded(A, lda)
    w_t = W if ldb is None else _padded(W, ldb)
    flag = torch.tensor([skip], dtype=torch.int32, device='cuda')
    launch(a=a_t, b=w_t, lda=lda or K, ldb=ldb or K, M=M, N=N, K=K, bias=bias, resid=resid_t, ld_resid=ld_resid, act=act,
           out_bf16=int(out_bf16), split3=int(lay.split3), transposed=0, k_splits=1, bn=bn, out=outs,
           seg_n=lay.seg_n if lay.segs > 1 else 0, ldo=lay.ldo, rows_per_batch=lay.rpb, batch_stride=lay.bstride,
           row_offset=lay.roff, skip=flag)
    return outs


def run_skinny(X, W, bias=None, act=0, out_bf16=False, split3=False, k_splits=1, bn=0, pad=8, skip=0):
    """The transposed (swap-AB) epilogue: X [rows, K] activations, W [features, K].  Returns (buffers
    [requested splits, rows + 2, ldo], effective split count)."""
    rows, K = X.shape
    feats = W.shape[0]
    ldo = feats * (3 if split3 else 1) + pad
    out = torch.full((k_splits, rows + 2, ldo), SENTINEL, dtype=torch.bfloat16 if out_bf16 else torch.float32, device='cuda')
    flag = torch.tensor([skip], dtype=torch.int32, device='cuda')
    eff = launch(a=W, b=X, lda=K, ldb=K, M=feats, N=rows, K=K, bias=bias, act=act, out_bf16=int(out_bf16),
                 split3=int(split3), transposed=1, k_splits=k_splits, bn=bn, out=[out], ldo=ldo,
                 split_stride=(rows + 2) * ldo, skip=flag)
    return out, eff


def skinny_guards_ok(out, rows, width, eff):
    keep = torch.ones_like(out, dtype=torch.bool)
    keep[:eff, :rows, :width] = False
    bad = keep & (out.float() != SENTINEL)
    if bad.any():
        return 'guard element overwritten at (split, row, column) = %s' % (tuple(int(v) for v in bad.nonzero()[0]),)
    return None


def run_lse(A, W, bias, targets):
    """EPI_LSE; returns the float4 partials [M + 2, n_parts + 1, 4] (one guard row pair, one guard float4 per row)."""
    M, K = A.shape
    N = W.shape[0]
    n_parts = 2 * -(-N // 256)
    out = torch.full((M + 2, n_parts + 1, 4), SENTINEL, dtype=torch.float32, device='cuda')
    launch(a=A, b=W, lda=K, ldb=K, M=M, N=N, K=K, bias=bias, act=0, out_bf16=0, split3=0, transposed=0, k_splits=1, bn=0,
           out=[out], ldo=n_parts + 1, lse_target=targets)
    return out


def run_ln(parts, bias, resid, gamma, beta, eps, want_f32=True, want_bf16=True, split3=False, inplace=False, temb=None,
           remap=(0, 0, 0), skip=0, pre=False, expect_error=False):
    """layernorm_kernel on partials [n, rows + guard.., D]-like storage: parts is [n, rows, D] fp32 on the device."""
    L = _lib()
    n, rows, D = parts.shape
    of = parts[0] if inplace else torch.full((rows + 1, D), SENTINEL, device='cuda')
    ob = torch.full((rows + 1, D * (3 if split3 else 1)), SENTINEL, dtype=torch.bfloat16, device='cuda')
    flag = torch.tensor([skip], dtype=torch.int32, device='cuda')
    rc = L.load().gitb200_op_layernorm_ex(parts.data_ptr(), n, rows * D, _ptr(bias), _ptr(resid), gamma.data_ptr(),
                                          beta.data_ptr(), ctypes.c_float(eps), of.data_ptr() if want_f32 else None,
                                          ob.data_ptr() if want_bf16 else None, rows, D, int(split3), _ptr(temb), remap[0],
                                          remap[1], remap[2], flag.data_ptr(), int(pre), _stream())
    if expect_error:
        assert rc != 0 and L.last_error(None)
        return None, None
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    return of, ob


def run_lse_combine(parts, rows, T, V, targets, need_predict, eps=0.1):
    L = _lib()
    n_parts = parts.shape[1]
    lp = torch.full((rows // T * max(T - 1, 1) + 1,), SENTINEL, device='cuda')
    row_loss = torch.full((rows + 1,), SENTINEL, device='cuda')
    row_valid = torch.full((rows + 1,), 77, dtype=torch.int32, device='cuda')
    loss = torch.full((2,), SENTINEL, device='cuda')
    rc = L.load().gitb200_op_lse_combine(parts.data_ptr(), n_parts, rows, T, V, targets.data_ptr(), need_predict.data_ptr(),
                                         ctypes.c_float(eps), lp.data_ptr(), row_loss.data_ptr(), row_valid.data_ptr(),
                                         loss.data_ptr(), _stream())
    assert rc == 0, L.last_error(None)
    torch.cuda.synchronize()
    assert lp[-1].item() == SENTINEL and row_loss[-1].item() == SENTINEL and row_valid[-1].item() == 77
    assert loss[1].item() == SENTINEL
    return lp[:-1], row_loss[:-1], row_valid[:-1], loss[0]


# ---------------------------------------------------------------------------------------------------------------------
# exact layer
# ---------------------------------------------------------------------------------------------------------------------
def exact_normal_case(M, N, K, seed, bias=False, act=0, out_bf16=False, resid=None, segs=1, map=(0, 0, 0), split3=False,
                      bn=0, lda=None, ldb=None):
    """Runs one normal-shape call on integer operands and fails with the first wrong tile."""
    dense = act == 0
    A, W = int_operands(M, N, K, seed, 3 if dense else 1, 2 if dense else 1, 1.0 if dense else 0.25)
    A, W = A.cuda(), W.cuda()
    bias_t = None
    if act:
        bias_t = saturating_bias(A, W, N)
    elif bias:
        bias_t = int_vector((N,), seed + 1).cuda()
    resid_t = int_vector((M, N), seed + 2).cuda() if resid else None
    x = ref_product(A, W)
    if bias_t is not None:
        x = x + bias_t.double()
    if resid_t is not None:
        x = x + resid_t.double()      # act(x) == x here: see saturating_bias
    lay = Layout(M, N, segs, *map, split3=split3)
    exp = expected_output(x, out_bf16, split3)
    outs = run_normal(A, W, lay, bias_t, resid_t, act, out_bf16, bn, inplace=(resid == 'inplace'), lda=lda, ldb=ldb)
    eff_bn = 256 if split3 else (bn or pick_bn(N, False))
    msg = check_exact(lay.gather(outs), exp, N, eff_bn, lay.seg_n) or lay.guards_ok(outs)
    assert msg is None, msg
    return A, W, lay, bias_t, resid_t


def exact_skinny_case(rows, feats, K, seed, splits=1, bias=False, act=0, out_bf16=False, split3=False, bn=0, pad=8):
    dense = act == 0
    X, W = int_operands(rows, feats, K, seed, 3 if dense else 1, 2 if dense else 1, 1.0 if dense else 0.25)
    X, W = X.cuda(), W.cuda()
    bias_t = None
    if act:
        bias_t = saturating_bias(X, W, feats)
    elif bias:
        bias_t = int_vector((feats,), seed + 1).cuda()
    out, eff = run_skinny(X, W, bias_t, act, out_bf16, split3, splits, bn, pad)
    ranges = split_ranges(K, splits)
    assert eff == len(ranges), 'effective split count %d, expected %d' % (eff, len(ranges))
    eff_bn = bn or pick_bn(rows, True)
    width = feats * (3 if split3 else 1)
    for s, (k0, k1) in enumerate(ranges):
        x = ref_product(X, W, k0, k1)
        if bias_t is not None and s == 0:
            x = x + bias_t.double()
        msg = check_exact(out[s, :rows, :width], expected_output(x, out_bf16, split3), feats, eff_bn,
                          split=s if splits > 1 else None, transposed=True)
        assert msg is None, msg
    msg = skinny_guards_ok(out, rows, width, eff)
    assert msg is None, msg
    return X, W, out, eff


@gpu
@pytest.mark.parametrize('inst', INSTANTIATIONS, ids=_inst_id)
def test_exact_every_instantiation(inst):
    """Every launch_gemm_inst<BN, EPI> of launch_gemm_bn: two tile rows with a row tail, three tile columns with the
    last one partial, K = 64 * (STAGES + 1) + 8 (the ring wraps, the last k-block leans on TMA zero fill)."""
    bn, transposed, out_bf16, resid, partial, act, split3 = inst
    K = BK * (stages(bn) + 1) + 8
    if not transposed:
        exact_normal_case(197, 2 * bn + 32, K, 100 + bn, bias=True, act=act, out_bf16=out_bf16,
                          resid='other' if resid else None, split3=split3, bn=bn)
    else:
        rows = {64: 37, 128: 101, 256: 200}[bn]
        exact_skinny_case(rows, 300, K, 200 + bn, splits=3 if partial else 1, bias=not partial, act=act,
                          out_bf16=out_bf16, split3=split3, bn=bn)


def test_instantiation_table_matches_the_launcher():
    """INSTANTIATIONS is compared with the case labels of launch_gemm_bn in the source."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, 'generativeimage2text_b200', 'csrc', 'gitb200.cu')).read()
    body = src[src.index('static int launch_gemm_bn('):src.index('static int pick_bn(')]
    acts = {'ACT_NONE': 0, 'ACT_QUICKGELU': 1, 'ACT_GELU_ERF': 2, 'ACT_QUICKGELU_EXACT': 3}
    found = set()
    bns = None
    for line in body.splitlines():
        g = re.search(r'if constexpr \((BN == \d+(?: \|\| BN == \d+)*)\)', line)
        if g:
            bns = [int(v) for v in re.findall(r'\d+', g.group(1))]
        for call in re.finditer(r'launch_gemm_inst<BN, (EPI_LSE|epi_code\((\w+), (\w+), (\w+), (\w+), (\w+)\)( \| EPI_SPLIT3)?)>', line):
            if call.group(1) == 'EPI_LSE':
                found.add('lse')
                continue
            tr, bf, rs, pa = (v == 'true' for v in call.group(2, 3, 4, 5))
            for bn in bns:
                found.add((bn, tr, bf, rs, pa, acts[call.group(6)], call.group(7) is not None))
    assert 'lse' in found
    found.discard('lse')
    assert found == set(INSTANTIATIONS) and len(INSTANTIATIONS) == len(set(INSTANTIATIONS))
    assert N_INSTANTIATIONS == 30


@gpu
def test_refused_calls():
    """Argument errors come back as return codes with a message; nothing is launched."""
    A, W = (t.cuda() for t in int_operands(64, 128, 64, 1))
    out = torch.full((64, 128), SENTINEL, dtype=torch.bfloat16, device='cuda')
    resid = torch.zeros((64, 128), device='cuda')
    base = dict(a=A, b=W, lda=64, ldb=64, M=64, N=128, K=64, act=0, out_bf16=1, split3=0, transposed=0, k_splits=1, bn=128,
                out=[out], ldo=128)
    assert 'not instantiated' in launch(expect_error=True, **dict(base, resid=resid, ld_resid=128))    # bf16 + residual
    launch(expect_error=True, **dict(base, act=4))
    launch(expect_error=True, **dict(base, k_splits=2))               # split-K needs the transposed shape
    launch(expect_error=True, **dict(base, N=120))                    # N % 32
    launch(expect_error=True, **dict(base, bn=96))
    launch(expect_error=True, **dict(base, ldo=64))
    launch(expect_error=True, **dict(base, seg_n=32))                 # four segments
    launch(expect_error=True, **dict(base, lse_target=torch.zeros(64, dtype=torch.int32, device='cuda')))   # no bias
    launch(expect_error=True, **dict(base, transposed=1, resid=resid, ld_resid=128))
    launch(expect_error=True, **dict(base, lda=60))                   # TMA pitch
    torch.cuda.synchronize()
    assert (out.float() == SENTINEL).all()


def _edge_cases():
    """Shapes at the kernel's edges: every M with N / K / epilogue cycling, every K at M = 197, per tile width."""
    cases = []
    epis = [dict(), dict(bias=True, out_bf16=True), dict(bias=True, resid='inplace'), dict(bias=True, resid='other')]
    for bn, ns in ((128, (32, 96, 768, 1056)), (192, (1024, 768, 96, 2304)), (256, (768, 2304, 3072, 32))):
        ks = (64, 8, 72, 640, 776, 768, 3072, BK * (stages(bn) + 1))
        ms = (1, 63, 64, 65, 127, 128, 129, 197, 12608 + 5)
        for i, M in enumerate(ms):
            N, K = ns[i % 4], ks[(i + 2) % 8]
            if M > 12608:
                N, K = 768, 768                     # 297 / 396 / 297 tiles: more than the 132 CTAs
            cases.append((bn, M, N, K, epis[i % 4], None, None))
        for i, K in enumerate(ks):
            cases.append((bn, 197, ns[(i + 1) % 4], K, epis[(i + 1) % 4], None, None))
        cases.append((bn, 129, 96, 72, dict(bias=True), 136, 200))         # lda > K, ldb > K with junk in the padding
        cases.append((bn, 65, 2304, 776, dict(out_bf16=True), 1024, 784))
    return cases


def _edge_id(c):
    bn, M, N, K, epi, lda, ldb = c
    return 'bn%d-M%d-N%d-K%d-%s%s' % (bn, M, N, K, '+'.join(sorted('%s' % k for k in epi)) or 'plain',
                                      '-lda%d-ldb%d' % (lda, ldb) if lda else '')


@gpu
@pytest.mark.parametrize('case', _edge_cases(), ids=_edge_id)
def test_exact_edges(case):
    bn, M, N, K, epi, lda, ldb = case
    exact_normal_case(M, N, K, 7 * M + N + K, bn=bn, lda=lda, ldb=ldb, **epi)


@gpu
@pytest.mark.parametrize('name', sorted(ENGINE_CALLS))
def test_exact_engine_calls(name):
    _, M, N, K, form = ENGINE_CALLS[name]
    exact_normal_case(M, N, K, sum(name.encode()), **form)


@gpu
@pytest.mark.parametrize('rows', DECODE_ROWS)
@pytest.mark.parametrize('name', sorted(DECODE_CALLS))
def test_exact_decode_calls(name, rows):
    feats, K, splits, bias, act, out_bf16 = DECODE_CALLS[name]
    exact_skinny_case(rows, feats, K, rows + feats, splits, bias, act, out_bf16, pad=0 if feats == 30522 else 8)


@gpu
@pytest.mark.parametrize('rows,feats,K,splits,bn,bias,out_bf16,pad', [
    (64, 768, 768, 3, 64, False, False, 8),      # 64-row tiles with split-K
    (37, 766, 776, 4, 64, True, False, 1),       # odd pitch: scalar stores; bias goes to split 0 only; K tail
    (65, 770, 640, 1, 64, True, False, 0),       # two row tiles of 64; pitch % 4 == 2: float2 stores, feature tail of 2
    (128, 770, 72, 1, 128, True, True, 1),       # bf16 scalar stores
    (200, 64, 8, 1, 256, True, False, 8),        # one k-block of 8 columns: the rest is TMA zero fill
    (256, 3072, 3072, 8, 256, False, False, 8),
    (5, 2304, 768, 16, 0, False, False, 8),      # 16 requested over 12 k-blocks -> 12
    (5, 768, 768, 8, 0, False, False, 8),        # 8 requested over 12 k-blocks -> 6, two buffers stay untouched
])
def test_exact_skinny_edges(rows, feats, K, splits, bn, bias, out_bf16, pad):
    # bf16 leaves the transposed shape only behind the erf-GELU (saturated here: see the header)
    exact_skinny_case(rows, feats, K, rows * 3 + feats + K, splits, bias, 2 if out_bf16 else 0, out_bf16, bn=bn, pad=pad)


@gpu
def test_skip_flag_stores_nothing():
    """A finished decode: with *skip != 0 neither epilogue shape may store anything."""
    A, W = (t.cuda() for t in int_operands(197, 768, 768, 5))
    lay = Layout(197, 768, 3, 197, 200, 2)
    for o in run_normal(A, W, lay, skip=1):
        assert (o == SENTINEL).all()
    out, _ = run_skinny(A[:64], W, k_splits=6, skip=1)
    assert (out == SENTINEL).all()
    out, _ = run_skinny(A[:64], W, skip=1)
    assert (out == SENTINEL).all()
    g = torch.ones(768, device='cuda')
    of, ob = run_ln(torch.randn(1, 9, 768, device='cuda'), None, None, g, g, 1e-5, skip=1)
    assert (of == SENTINEL).all() and (ob.float() == SENTINEL).all()


# ---------------------------------------------------------------------------------------------------------------------
# real-valued layer
# ---------------------------------------------------------------------------------------------------------------------
PLANTED_X = (0.0, 1e-4, -1e-4, 6.0, -6.0, 12.0, -12.0, 40.0, -40.0)


def real_bound(absdot, pre, ref, act, out_bf16, c_acc=None):
    c_acc = C_ACC if c_acc is None else c_acc
    return (LIP if act else 1.0) * c_acc * absdot + C_ACT[act] * pre.abs() + C_OUT[out_bf16] * ref.abs() + ABS


@gpu
@pytest.mark.parametrize('M,N,K,bn,act,out_bf16,resid,transposed', [
    (394, 2304, 768, 256, 0, False, False, False), (394, 768, 3072, 192, 0, False, True, False),
    (514, 1024, 4096, 128, 0, False, True, False), (394, 768, 776, 128, 0, True, False, False),
    (394, 3072, 768, 256, 1, True, False, False), (394, 3072, 768, 192, 1, True, False, False),
    (394, 3072, 768, 128, 2, True, False, False), (394, 3072, 768, 256, 2, True, False, False),
    (394, 3072, 768, 256, 3, True, False, False),                  # split3 (the only exact-QuickGELU form)
    (64, 3072, 768, 64, 2, True, False, True), (200, 3072, 768, 256, 2, True, False, True),
    (128, 30522, 768, 128, 0, False, False, True), (64, 768, 3072, 64, 0, False, False, True),
])
def test_real_valued(M, N, K, bn, act, out_bf16, resid, transposed):
    """Gaussian operands; activations against fp64 sigmoid / erf, with pre-activations of PLANTED_X planted through the
    bias in the first columns (their rows of W are zero, so the pre-activation is the bias itself)."""
    A, W = real_operands(M, N, K, M + N + K + act)
    g = torch.Generator().manual_seed(9)
    bias = torch.randn((N,), generator=g) * 0.5
    if act:
        W[:len(PLANTED_X)] = 0
        bias[:len(PLANTED_X)] = torch.tensor(PLANTED_X)
    A, W, bias = A.cuda(), W.cuda(), bias.cuda()
    resid_t = torch.randn((M, N), generator=g).cuda() if resid else None
    split3 = act == 3
    pre = ref_product(A, W) + bias.double()
    ref = act_ref(pre, act) + (resid_t.double() if resid else 0.0)
    absdot = abs_product(A, W)
    if transposed:
        out, _ = run_skinny(A, W, bias, act, out_bf16, split3, 1, bn)
        got = out[0, :M, :N].float()
        assert skinny_guards_ok(out, M, N, 1) is None
    else:
        lay = Layout(M, N, split3=split3)
        outs = run_normal(A, W, lay, bias, resid_t, act, out_bf16, bn)
        got = lay.gather(outs).float()
        assert lay.guards_ok(outs) is None
        if split3:
            assert torch.equal(got[:, :N], got[:, 2 * N:])
            got = got[:, :N].double() + got[:, N:2 * N].double()      # hi + lo carries the value to ~2^-17
    bound = real_bound(absdot, pre, ref, act, out_bf16 and not split3)
    if split3:
        bound = bound + 2.0 ** -16 * ref.abs()
    err = (got.double() - ref).abs()
    if act == 0 and not out_bf16:
        _observe('c_acc', (err / absdot).max())
    if act and not split3:
        far = absdot == 0          # planted columns: the pre-activation is exact, what is left is the activation + output
        _observe('c_act%d' % act, ((err - C_OUT[out_bf16] * ref.abs()).clamp(min=0)[far] / pre.abs()[far].clamp(min=1e-30)).max())
    if split3:
        far = absdot == 0
        _observe('c_act3', ((err - 2.0 ** -16 * ref.abs()).clamp(min=0)[far] / pre.abs()[far].clamp(min=1e-30)).max())
    worst, msg = check_bound(got, ref, bound, N, bn, transposed=transposed)
    _observe('real_worst_over_bound', worst)
    assert worst <= 1.0, msg


@gpu
@pytest.mark.parametrize('M,N,K', [(394, 768, 768), (65, 2304, 768), (200, 768, 3072)])
def test_parity_operands(M, N, K):
    """The parity mode's arithmetic: fp32 A and W split into [hi | lo | hi] / [hi | hi | lo] and run at 3 K give
    sum a_hi w_hi + a_lo w_hi + a_hi w_lo, compared with the fp64 product of the fp32 values."""
    g = torch.Generator().manual_seed(M + N)
    A32, W32 = torch.randn((M, K), generator=g), torch.randn((N, K), generator=g) * 0.04
    a_hi, w_hi = bf16_rne(A32), bf16_rne(W32)
    a_lo, w_lo = bf16_rne(A32 - a_hi), bf16_rne(W32 - w_hi)
    A3 = torch.cat([a_hi, a_lo, a_hi], 1).bfloat16().cuda()
    W3 = torch.cat([w_hi, w_hi, w_lo], 1).bfloat16().cuda()
    lay = Layout(M, N)
    got = lay.gather(run_normal(A3, W3, lay))
    ref = A32.double().cuda() @ W32.double().cuda().t()
    absdot = A32.double().abs().cuda() @ W32.double().abs().cuda().t()
    _observe('c_acc_parity', ((got.double() - ref).abs() / absdot).max())
    worst, msg = check_bound(got, ref, C_ACC_PARITY * absdot + ABS, N, pick_bn(N, False))
    assert worst <= 1.0, msg


# ---------------------------------------------------------------------------------------------------------------------
# LM-head statistics
# ---------------------------------------------------------------------------------------------------------------------
def check_lse_stats(got, ref, delta, exact):
    """got / ref [M, n_parts, 4].  exact: max, sum x and x[target] must be equal.  Otherwise each is within the logit
    error delta [M, 1] (sum x: 128 of them).  log(sum exp) + max is compared within delta + C_LSE.  Returns the worst
    ratio over its bound, or a message."""
    empty = torch.isinf(ref[..., 0])
    if empty.any():
        e = got[empty]
        if not ((e[:, 0] == float('-inf')).all() and (e[:, 1:] == 0).all()):
            return 'a half tile that owns no column does not hold (-inf, 0, 0, 0)'
    g, r = got[~empty].double(), ref[~empty]
    d = delta.expand(-1, ref.shape[1])[~empty]
    if exact:
        for i, nm in ((0, 'max'), (2, 'sum x'), (3, 'x[target]')):
            if not torch.equal(g[:, i], r[:, i]):
                return '%s differs in %d (row, half tile) statistics' % (nm, int((g[:, i] != r[:, i]).sum()))
    lse_g, lse_r = g[:, 0] + torch.log(g[:, 1]), r[:, 0] + torch.log(r[:, 1])
    scale = r[:, 0].abs().clamp(min=1.0)
    ratios = [(lse_g - lse_r).abs() / (d + C_LSE * scale), (g[:, 0] - r[:, 0]).abs() / (d + 1e-30),
              (g[:, 2] - r[:, 2]).abs() / (128 * (d + C_LSE * scale)), (g[:, 3] - r[:, 3]).abs() / (d + 1e-30)]
    _observe('c_lse', ((lse_g - lse_r).abs() - d).clamp(min=0).div(scale).max())
    return max(float(x.max()) for x in ratios)


def lse_case(M, N, K, seed, exact, shift=0.0):
    """A, W, bias, targets (CPU) of one LM-head call.  exact: sparse integer operands (logits within about +-25),
    otherwise Gaussian.  shift moves every logit through the bias: +80 overflows and -1e4 underflows the exponentials
    unless the maximum is subtracted first."""
    g = torch.Generator().manual_seed(seed)
    if exact:
        A, W = int_operands(M, N, K, seed, 1, 1, 0.2)
        bias = int_vector((N,), seed + 1, 4) + shift
    else:
        A, W = real_operands(M, N, K, seed, 0.05)
        bias = torch.randn((N,), generator=g) * 0.5 + shift
    targets = torch.randint(0, N, (M,), generator=g, dtype=torch.int32)
    targets[0] = N - 1
    if M > 1:
        targets[M - 1] = -1
    if M > 2:
        targets[1] = 0
    return A, W, bias, targets


@gpu
@pytest.mark.parametrize('exact', [True, False], ids=['int', 'real'])
@pytest.mark.parametrize('M,N,shift', [(1, 58, 0.0), (64, 256, 0.0), (129, 257, 0.0), (64, 30522, 0.0), (2560, 30522, 0.0),
                                       (129, 58, 0.0), (1, 30522, 0.0), (129, 257, 80.0), (129, 257, -1e4),
                                       (64, 30522, 80.0), (64, 30522, -1e4)])
def test_lse_statistics(M, N, shift, exact):
    """EPI_LSE: every stored float4 against fp64 over exactly the columns it owns; N = 58 / 257 / 30522 end in a partial
    tile (30522: 58 valid columns in the last of 120 tiles, N % 4 == 2), 257 leaves a half tile without a column."""
    K = 768 if N == 30522 else 136
    A, W, bias, targets = lse_case(M, N, K, M + N, exact, shift)
    if M > 3:                                   # the row maximum in the last valid column
        W[N - 1] = A[3] if exact else (A[3].float() * (30.0 / K)).bfloat16()
    A, W, bias, targets = A.cuda(), W.cuda(), bias.cuda(), targets.cuda()
    x = ref_product(A, W) + bias.double()
    if M > 3:
        assert int(x[3].argmax()) == N - 1
    out = run_lse(A, W, bias, targets)
    n_parts = 2 * -(-N // 256)
    assert (out[M:] == SENTINEL).all() and (out[:, n_parts] == SENTINEL).all(), 'guard statistics overwritten'
    ref = lse_stats_ref(x, targets)
    delta = torch.zeros((M, 1), dtype=torch.float64, device='cuda') if exact else \
        (C_ACC * abs_product(A, W) + 2.0 ** -23 * x.abs()).max(dim=1, keepdim=True).values
    res = check_lse_stats(out[:M, :n_parts], ref, delta, exact)
    assert not isinstance(res, str), res
    assert res <= 1.0, 'statistics are %.2f x their bound' % res
    # and through the consumer: log-probabilities of the targets against fp64 log_softmax
    T = 1 if M == 1 else (2 if M % 2 == 0 else 3 if M % 3 == 0 else 1)
    if T > 1:
        need = torch.ones(M, dtype=torch.int64, device='cuda')
        lp, _, _, _ = run_lse_combine(out[:M, :n_parts].contiguous(), M, T, N, targets, need)
        rows = torch.arange(M, device='cuda').view(-1, T)[:, :T - 1].reshape(-1)
        rows = rows[targets[rows] >= 0]
        want = torch.log_softmax(x, dim=1)[rows, targets[rows].long()]
        lp_rows = (rows // T) * (T - 1) + rows % T
        err = (lp[lp_rows].double() - want).abs()
        tol = 2 * delta[rows, 0] + C_LOGPROB * want.abs().clamp(min=1.0)
        _observe('c_logprob', ((err - 2 * delta[rows, 0]).clamp(min=0) / want.abs().clamp(min=1.0)).max())
        assert (err <= tol).all(), 'log-probability off by %.3g (bound %.3g)' % (err.max().item(), tol[err.argmax()].item())


def combine_case(N_cap, T, V, seed, shift=True):
    """Logits [N_cap * T, V] fp64 (values exactly representable in fp32), targets and need_predict of a scoring call:
    the last position of a caption has no target (-1); targets include 0 (padding: never counted) and V - 1; one row is
    shifted by +80 and one by -1e4 (overflow / underflow unless the maximum is subtracted)."""
    g = torch.Generator().manual_seed(seed)
    rows = N_cap * T
    x = (torch.randn((rows, V), generator=g) * 2.0).float()
    if shift:
        x[0] += 80.0
        x[min(2, rows - 1)] -= 1e4
    x = x.double()
    targets = torch.randint(1, V, (rows,), generator=g, dtype=torch.int32)
    targets[T - 1::T] = -1
    targets[0] = V - 1
    if rows > T:
        targets[T] = 0
    need = torch.randint(0, 2, (rows,), generator=g, dtype=torch.int64)
    need[:2] = 1
    return x, targets, need


def combine_ref(x, targets, need, T, eps=0.1):
    """(log-probabilities [N_cap, T - 1], row losses, row validity, mean loss) in fp64."""
    rows, V = x.shape
    t = torch.arange(rows, device=x.device) % T
    scored = t + 1 < T
    tg = targets.long().clamp(min=0)
    lp = torch.log_softmax(x, dim=1).gather(1, tg[:, None])[:, 0]
    nxt = torch.cat([need[1:], need[:1]])
    valid = scored & (nxt == 1) & (targets != 0)
    loss = torch.where(valid, smoothed_loss_ref(x, tg, eps), torch.zeros(rows, dtype=torch.float64, device=x.device))
    mean = loss.sum() / valid.sum() if valid.any() else torch.tensor(float('nan'))
    return lp[scored].view(-1, T - 1), loss, valid, mean


@gpu
@pytest.mark.parametrize('N_cap,T,V', [(5, 13, 30522), (64, 2, 30522), (3, 40, 257), (700, 4, 58)])
def test_lse_combine(N_cap, T, V):
    """lse_combine_kernel + loss_mean_kernel on fp64-made partials: n_parts = 240 leaves lane tails (240 = 7 * 32 + 16)."""
    x, targets, need = (t.cuda() for t in combine_case(N_cap, T, V, N_cap + T))
    parts = lse_stats_ref(x, targets).float().contiguous()
    lp, row_loss, row_valid, loss = run_lse_combine(parts, N_cap * T, T, V, targets, need)
    lp_ref, loss_ref, valid_ref, mean_ref = combine_ref(x, targets, need, T)
    err = (lp.view(-1, T - 1).double() - lp_ref).abs() / lp_ref.abs().clamp(min=1.0)
    _observe('c_logprob', err.max())
    assert err.max().item() <= C_LOGPROB
    assert torch.equal(row_valid.bool(), valid_ref)
    lerr = (row_loss.double() - loss_ref).abs() / loss_ref.abs().clamp(min=1.0)
    _observe('c_loss', lerr.max())
    assert lerr.max().item() <= C_LOSS
    assert abs(loss.item() - mean_ref.item()) <= C_LOSS * max(1.0, abs(mean_ref.item()))
    # need_predict all zero: no valid row, the loss is NaN by contract
    _, row_loss, row_valid, loss = run_lse_combine(parts, N_cap * T, T, V, targets, torch.zeros_like(need))
    assert not row_valid.any() and (row_loss == 0).all() and math.isnan(loss.item())


# ---------------------------------------------------------------------------------------------------------------------
# split-K consumers
# ---------------------------------------------------------------------------------------------------------------------
def ln_case(n, rows, D, seed, cancel=False):
    g = torch.Generator().manual_seed(seed)
    parts = torch.randn((n, rows, D), generator=g) * 2.0
    if cancel and n >= 3:          # (1e8 + -1e8) + x == x, but x + -1e8 + 1e8 loses x: the order is visible
        parts[0] = 1e8 * torch.sign(torch.randn((rows, D), generator=g))
        parts[1] = -parts[0]
    return (parts, torch.randn((D,), generator=g) * 0.5, torch.randn((rows, D), generator=g),
            1 + 0.1 * torch.randn((D,), generator=g), 0.1 * torch.randn((D,), generator=g))


def check_ln(of, ob, ref, split3, orow=None):
    """Worst |out - ref| over its bound across the outputs present; ref fp64 [rows, D]; orow: output row of each row."""
    rows, D = ref.shape
    idx = torch.arange(rows, device=ref.device) if orow is None else orow.to(ref.device)
    scale = ref.abs().clamp(min=1.0)
    worst = 0.0
    if of is not None:
        worst = max(worst, ((of[idx].double() - ref).abs() / (C_LN[False] * scale)).max().item())
        _observe('c_ln', ((of[idx].double() - ref).abs() / scale).max())
    if ob is not None:
        o = ob[idx].float()
        if split3:
            if not torch.equal(o[:, :D], o[:, 2 * D:]):
                return float('inf')
            worst = max(worst, ((o[:, :D].double() + o[:, D:2 * D].double() - ref).abs() /
                                (C_LN[False] * scale + 2.0 ** -16 * ref.abs())).max().item())
        else:
            worst = max(worst, ((o.double() - ref).abs() / ((C_LN[True] + C_LN[False]) * scale)).max().item())
    return worst


@gpu
@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize('rows,eps,form', [(1, 1e-12, 'plain'), (7, 1e-5, 'bias_resid'), (8, 1e-12, 'split3'),
                                           (9, 1e-12, 'inplace'), (64, 1e-12, 'pre'), (256, 1e-5, 'pre_split3')])
def test_layernorm_partials(n, rows, eps, form):
    """layernorm_kernel<768> over n partial buffers (three per trip: 2, 4, 5, 7, 8 end in a tail), with cancelling
    partials so that any other summation order is far outside the bound."""
    parts, bias, resid, gamma, beta = (t.cuda() for t in ln_case(n, rows, 768, n * 1000 + rows, cancel=True))
    plain = form in ('plain', 'split3')
    b, r = (None, None) if plain else (bias, resid)
    ref = ln_ref(parts, b, r, gamma, beta, eps)
    split3 = 'split3' in form
    of, ob = run_ln(parts.clone(), b, r, gamma, beta, eps, split3=split3, inplace=(form == 'inplace'), pre='pre' in form)
    assert (ob[rows:].float() == SENTINEL).all() and (form == 'inplace' or (of[rows:] == SENTINEL).all())
    worst = check_ln(of, ob, ref, split3)
    assert worst <= 1.0, 'LayerNorm output is %.2f x its bound' % worst


@gpu
@pytest.mark.parametrize('rows', [1, 9, 257])
def test_layernorm_1024(rows):
    parts, bias, resid, gamma, beta = (t.cuda() for t in ln_case(1, rows, 1024, rows))
    of, ob = run_ln(parts, bias, resid, gamma, beta, 1e-5)
    assert check_ln(of, ob, ln_ref(parts, bias, resid, gamma, beta, 1e-5), False) <= 1.0
    run_ln(parts, bias, resid, gamma, beta, 1e-5, pre=True, expect_error=True)      # no <1024, PRE> instantiation


@gpu
def test_layernorm_frame_remap():
    """ln_post of a video batch: rows (f * B + b) * L + l land at (b * F + f) * L + l, temb[f] added after the norm."""
    B, F, L, D = 2, 6, 197, 768
    rows = B * F * L
    parts, _, _, gamma, beta = (t.cuda() for t in ln_case(1, rows, D, 3))
    temb = torch.randn((F, D), generator=torch.Generator().manual_seed(4)).cuda()
    orow, frame = remap_rows(rows, B, F, L)
    ref = ln_ref(parts, None, None, gamma, beta, 1e-5) + temb.double()[frame.cuda()]
    of, ob = run_ln(parts, None, None, gamma, beta, 1e-5, temb=temb, remap=(B, F, L))
    assert sorted(orow.tolist()) == list(range(rows))
    assert check_ln(of, ob, ref, False, orow) <= 1.0
    assert (of[rows:] == SENTINEL).all()


@gpu
def test_gemm_partials_into_layernorm():
    """The decode chain's round trip: a skinny GEMM with 8 requested splits leaves 6 raw partial buffers, LayerNorm adds
    them in split order with the bias and the residual; bit-equal on two runs."""
    rows, D, K = 64, 768, 768
    X, W = (t.cuda() for t in real_operands(rows, D, K, 11))
    _, bias, resid, gamma, beta = (t.cuda() for t in ln_case(1, rows, D, 12))
    results = []
    for _ in range(2):
        out, eff = run_skinny(X, W, k_splits=8, pad=0)
        assert eff == 6
        parts = out[:eff, :rows].contiguous()
        results.append(run_ln(parts, bias, resid, gamma, beta, 1e-12, pre=True))
    assert torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1])
    worst, msg = check_bound(parts.double().sum(0), ref_product(X, W), C_ACC * abs_product(X, W) + ABS, D, 64, transposed=True)
    assert worst <= 1.0, msg
    assert check_ln(results[0][0], results[0][1], ln_ref(parts, bias, resid, gamma, beta, 1e-12), False) <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the references themselves
# ---------------------------------------------------------------------------------------------------------------------
def test_bf16_helper_matches_torch():
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(100000, generator=g) * 100, torch.randn(100000, generator=g) * 1e-3,
                   torch.tensor([0.0, -0.0, 1.0, 1.00390625, 1.01171875, -1.00390625, 255.5, 256.5, 3.0e38, 1e-40])])
    assert torch.equal(bf16_rne(x), x.bfloat16().float())
    s = split3_rows(x[None])
    n = x.numel()
    assert torch.equal(s[:, :n], s[:, 2 * n:]) and torch.equal(s[0, n:2 * n], (x - x.bfloat16().float()).bfloat16().float())


def test_row_map_matches_a_naive_walk():
    """The closed form against walking the rows the way epi_row_offsets does (four rows per step, any number of images)."""
    for rpb, bstride, roff, M in ((196, 197, 1, 700), (3, 4, 1, 120), (1, 2, 1, 70), (256, 257, 1, 1000), (20, 25, 3, 333)):
        for start in range(4):
            bq, sq = divmod(start, rpb)
            for m in range(start, M, 4):
                assert row_map(m, rpb, bstride, roff) == bq * bstride + sq + roff
                sq += 4
                while sq >= rpb:
                    sq -= rpb
                    bq += 1
    lay = Layout(392, 64, 1, 196, 197, 1)
    assert lay.phys_rows == 2 * 197 + 2 and 0 not in lay.rows and 197 not in lay.rows and int(lay.rows[196]) == 198


@pytest.mark.parametrize('N', [58, 256, 257, 30522])
def test_lse_ownership_covers_every_column_once(N):
    n_parts = 2 * -(-N // 256)
    owned = [c for p in range(n_parts) for c in lse_owned_columns(N, p)]
    assert sorted(owned) == list(range(N))
    if N == 257:
        assert lse_owned_columns(N, 2) == [256] and lse_owned_columns(N, 3) == []
    if N == 30522:
        assert n_parts == 240 and len(lse_owned_columns(N, 238)) == 32 and len(lse_owned_columns(N, 239)) == 26
    g = torch.Generator().manual_seed(N)
    x = torch.randn((3, N), generator=g).double()
    t = torch.tensor([0, N - 1, -1], dtype=torch.int32)
    ref = lse_stats_ref(x, t)
    for p in range(n_parts):
        cols = lse_owned_columns(N, p)
        if not cols:
            assert ref[:, p].tolist() == [[float('-inf'), 0.0, 0.0, 0.0]] * 3
            continue
        sub = x[:, cols]
        assert torch.equal(ref[:, p, 0], sub.max(1).values)
        assert torch.allclose(ref[:, p, 1], torch.exp(sub - sub.max(1, keepdim=True).values).sum(1), rtol=1e-12)
        assert torch.allclose(ref[:, p, 2], sub.sum(1), rtol=1e-12, atol=1e-12)
        for r in range(3):
            assert ref[r, p, 3].item() == (x[r, int(t[r])].item() if int(t[r]) in cols else 0.0)
    assert torch.allclose(lse_fold_ref(ref), torch.logsumexp(x, 1), rtol=1e-12)


def test_every_engine_gemm_call_site_is_named():
    """A new launch_gemm( call in the engine needs a case here: the sites named above are as many as the source has."""
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'generativeimage2text_b200', 'csrc')
    calls = sum(open(os.path.join(root, f)).read().count('launch_gemm(h, ') for f in ('gitb200.cu', 'engine_api.inc'))
    named = {v[0] for v in ENGINE_CALLS.values()} | set(OTHER_SITES)
    assert calls == len(named) == 14


def test_split_ranges_and_stages():
    assert [stages(bn) for bn in (64, 128, 192, 256)] == [8, 6, 4, 4]
    assert len(split_ranges(768, 8)) == 6 and len(split_ranges(768, 16)) == 12 and len(split_ranges(3072, 8)) == 8
    assert split_ranges(776, 4) == [(0, 256), (256, 512), (512, 768), (768, 776)]
    assert split_ranges(8, 3) == [(0, 8)]
    for K, req in ((768, 3), (768, 6), (3072, 8), (776, 5), (640, 7)):
        r = split_ranges(K, req)
        assert r[0][0] == 0 and r[-1][1] == K and all(a[1] == b[0] for a, b in zip(r, r[1:])) and all(b > a for a, b in r)


def test_combine_reference_matches_the_oracle_formula():
    """smoothed_loss_ref / combine_ref against the closed form lse_combine_kernel evaluates."""
    x, targets, need = combine_case(3, 5, 300, 1)
    lp, loss, valid, mean = combine_ref(x, targets, need, 5)
    V, e = 300, 0.1
    lse = torch.logsumexp(x, 1)
    tg = targets.long().clamp(min=0)
    lpt = x.gather(1, tg[:, None])[:, 0] - lse
    closed = (1 - e) * math.log(1 - e) + e * math.log(e / (V - 1)) - (1 - e) * lpt - e / (V - 1) * (x.sum(1) - V * lse - lpt)
    assert torch.allclose(loss[valid], closed[valid], rtol=1e-10)
    assert valid.sum() > 0 and not valid[4::5].any() and not valid[5]
    assert abs(mean.item() - loss[valid].mean().item()) < 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the suite must be able to fail (defects planted in the reference)
# ---------------------------------------------------------------------------------------------------------------------
def _exact_pair(M=197, N=544, K=328, bn=256):
    A, W = int_operands(M, N, K, 1)
    return A, W, ref_product(A, W), bn


def _tile_cols(N, bn, tile):
    return slice(tile * bn, min(N, (tile + 1) * bn))


def test_planted_dropped_k_step_is_named():
    A, W, x, bn = _exact_pair()
    cols = _tile_cols(544, bn, 1)
    bad = x.clone()
    bad[:, cols] -= ref_product(A, W[cols], 48, 64)            # the last k-step of 16 of the first k-block, tile column 1
    msg = check_exact(bad.float(), x.float(), 544, bn)
    assert msg is not None and 'tile row 0, tile column 1, 64-column chunk 0' in msg
    msg = check_exact(bf16_rne(bad.float()), bf16_rne(x.float()), 544, bn)
    assert msg is not None and 'tile column 1' in msg
    # real-valued layer: the same defect is >= 4x the bound
    Ar, Wr = real_operands(197, 544, 768, 2)
    ref, absdot = ref_product(Ar, Wr), abs_product(Ar, Wr)
    bad = ref.clone()
    bad[:, cols] -= ref_product(Ar, Wr[cols], 48, 64)
    for out_bf16 in (False, True):
        bound = real_bound(absdot, ref, ref, 0, out_bf16)
        worst, msg = check_bound(bad, ref, bound, 544, bn)
        assert worst >= 4.0 and 'tile column 1' in msg, (out_bf16, worst)


def test_planted_k_block_taken_twice():
    A, W, x, bn = _exact_pair()
    cols = _tile_cols(544, bn, 2)
    bad = x.clone()
    bad[128:, cols] += ref_product(A[128:], W[cols], 256, 320)        # k-block 4 again (a phase slip on ring wrap-around)
    msg = check_exact(bad.float(), x.float(), 544, bn)
    assert msg is not None and 'tile row 1, tile column 2' in msg
    Ar, Wr = real_operands(197, 544, 768, 3)
    ref, absdot = ref_product(Ar, Wr), abs_product(Ar, Wr)
    bad = ref.clone()
    bad[128:, cols] += ref_product(Ar[128:], Wr[cols], 256, 320)
    for out_bf16 in (False, True):
        assert check_bound(bad, ref, real_bound(absdot, ref, ref, 0, out_bf16), 544, bn)[0] >= 4.0


def test_planted_block_stored_one_block_to_the_right():
    A, W, x, bn = _exact_pair()
    bad = x.clone()
    bad[:, 352:384] = x[:, 320:352]            # tile column 1, chunk 1: its first 32 columns land on its second 32
    msg = check_exact(bad.float(), x.float(), 544, bn)
    assert msg is not None and 'tile column 1, 64-column chunk 1' in msg
    Ar, Wr = real_operands(197, 544, 768, 4)
    ref, absdot = ref_product(Ar, Wr), abs_product(Ar, Wr)
    bad = ref.clone()
    bad[:, 352:384] = ref[:, 320:352]
    assert check_bound(bad, ref, real_bound(absdot, ref, ref, 0, True), 544, bn)[0] >= 4.0


def test_planted_row_map_off_by_one_image():
    A, W = int_operands(3 * 20, 64, 64, 5)
    x = ref_product(A, W).float()
    lay = Layout(60, 64, 1, 20, 21, 1)
    wrong = Layout(60, 64, 1, 20, 21, 1)
    wrong.rows = row_map(torch.arange(60), 20, 21, 1) - 21 * (torch.arange(60) >= 40)      # image 2 lands on image 1
    bufs = wrong.scatter(x)
    assert check_exact(lay.gather(bufs), x, 64, 128) is not None
    no_offset = Layout(60, 64, 1, 20, 21, 1)
    no_offset.rows = row_map(torch.arange(60), 20, 21, 0)                                   # `ooff` without row_offset
    bufs = no_offset.scatter(x)
    assert check_exact(lay.gather(bufs), x, 64, 128) is not None and 'physical row 0' in lay.guards_ok(bufs)
    assert lay.guards_ok(lay.scatter(x)) is None and check_exact(lay.gather(lay.scatter(x)), x, 64, 128) is None


def test_planted_segments_swapped():
    A, W = int_operands(65, 96, 64, 6)
    x = ref_product(A, W).float()
    lay = Layout(65, 96, 3)
    bufs = lay.scatter(x)
    msg = check_exact(lay.gather([bufs[0], bufs[2], bufs[1]]), x, 96, 128, lay.seg_n)
    assert msg is not None and 'segment 1' in msg
    beyond = lay.scatter(x)
    beyond[0][:, lay.width] = 0.0              # a column past the segment
    assert 'column 32' in lay.guards_ok(beyond)


def test_planted_split_boundaries_moved():
    X, W = int_operands(5, 96, 768, 7)
    ranges = split_ranges(768, 8)
    assert len(ranges) == 6
    (k0, k1) = ranges[2]
    good = ref_product(X, W, k0, k1).float()
    moved = ref_product(X, W, k0 + 64, k1 + 64).float()
    msg = check_exact(moved, good, 96, 64, split=2, transposed=True)
    assert msg is not None and 'split 2' in msg
    assert torch.equal(sum(ref_product(X, W, a, b) for a, b in ranges), ref_product(X, W))


def test_planted_partials_added_in_reverse():
    parts, bias, resid, gamma, beta = ln_case(5, 8, 768, 8, cancel=True)
    ref = ln_ref(parts, bias, resid, gamma, beta, 1e-12)
    rev = ln_ref(parts.flip(0), bias, resid, gamma, beta, 1e-12)
    assert check_ln(rev.float(), None, ref, False) >= 4.0 and check_ln(None, rev.bfloat16(), ref, False) >= 4.0
    assert check_ln(ref.float(), ref.bfloat16(), ref, False) <= 1.0
    orow, _ = remap_rows(2 * 3 * 4, 2, 3, 4)
    assert orow.tolist()[:8] == [0, 1, 2, 3, 12, 13, 14, 15] and sorted(orow.tolist()) == list(range(24))


def test_planted_lse_defects():
    x, targets, need = combine_case(2, 3, 30522, 9, shift=False)
    x[1, 30521] = x[1].max() + 3.0             # the row maximum in the last valid column
    x[2, 30520] = x[2].max() + 3.0
    stats = lse_stats_ref(x, targets)
    good = torch.logsumexp(x, 1)
    assert torch.allclose(lse_fold_ref(stats), good, rtol=1e-12)
    scale = 25.0                              # no log-probability of this case is larger in magnitude
    assert (good - x.min(1).values).max().item() < scale
    # a half tile merged without rescaling by its maximum
    assert ((lse_fold_ref(stats, rescale=False) - good).abs() / (C_LOGPROB * scale)).min().item() >= 4.0
    # the last two vocabulary columns ignored: the statistics of the last float4 change, and so do the rows' lse
    short = lse_stats_ref(x[:, :30520], targets)
    delta = torch.zeros((6, 1), dtype=torch.float64)
    res = check_lse_stats(short.float(), stats, delta, exact=False)
    assert isinstance(res, str) or res >= 4.0
    assert ((lse_fold_ref(short) - good).abs() / (C_LOGPROB * scale))[1:3].min().item() >= 4.0
    assert check_lse_stats(stats.float(), stats, delta + 1e-6, exact=False) <= 1.0


def test_saturated_activations_are_the_identity_in_fp64_too():
    """The exact layer's activation trick: at x >= 40 both GELUs differ from x by less than half an fp32 ulp."""
    x = torch.tensor([40.0, 64.0, 200.0], dtype=torch.float64)
    for act in (1, 2, 3):
        assert ((act_ref(x, act) - x).abs() < 2.0 ** -25 * x).all()
