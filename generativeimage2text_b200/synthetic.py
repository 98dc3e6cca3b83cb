"""Reference state-dict layout and seeded synthetic checkpoints.

There are no reachable pretrained checkpoints (SURVEY.md section 8c: `output/{model}/snapshot/model.pt`
lives on Azure blob storage), so benches and parity tests use *random-init weights of the named
size* (BASELINE.json).  The key names / shapes below are the reference's own
(`CaptioningModel.state_dict()`, SURVEY.md section 8b "State-dict key families"; verified against the
reference in tests/test_oracle_vs_reference.py) so that `torch_common.load_state_dict`
(reference generativeimage2text/torch_common.py:93-145) can drive this engine unchanged.

Weights are generated with numpy's PCG64 keyed by (seed, crc32(key)) so that every machine and
every torch version produces bit-identical tensors -- the golden fixtures under tests/golden were
produced by loading exactly these tensors into the unmodified reference.
"""
import zlib
from collections import OrderedDict

import numpy as np
import torch

ENCODER_CFG = {
    # reference model.py:64-67 name map -> layers/CLIP/model.py:405-410 (`build_model` derivation)
    'CLIPViT_B_16': dict(patch=16, width=768, layers=12, heads=12, output_dim=512),
    'CLIPViT_L_14': dict(patch=14, width=1024, layers=24, heads=16, output_dim=768),
}

# decoder hyper-parameters hard-coded by reference model.py:14-26
VOCAB = 30522
HIDDEN = 768
DEC_LAYERS = 6
DEC_HEADS = 12
FFN = 3072
MAX_POS = 1024


def state_spec(param=None):
    """Ordered list of (key, shape, (kind, scale)) for the model `get_git_model(tok, param)` builds.

    kind: 'normal' (std=scale), 'ones', 'zeros'.  Scales follow the reference's initialisers
    (layers/CLIP/model.py:226-228, torch defaults for Linear/Conv2d/MultiheadAttention,
    layers/decoder.py:507-517 N(0,0.02); uniform(+-b) initialisers are represented by a normal of
    the same std b/sqrt(3)).
    """
    param = param or {}
    enc = ENCODER_CFG[param.get('image_encoder_type', 'CLIPViT_B_16')]
    res = param.get('test_crop_size', 224)
    p, d, nl = enc['patch'], enc['width'], enc['layers']
    L = (res // p) ** 2 + 1
    dv = param.get('visual_feature_size', 768)
    spec = []

    def add(k, shape, kind, scale=0.0):
        spec.append((k, tuple(shape), (kind, float(scale))))

    s3 = 3 ** -0.5
    ie = 'image_encoder.'
    add(ie + 'class_embedding', (d,), 'normal', d ** -0.5)
    add(ie + 'positional_embedding', (L, d), 'normal', d ** -0.5)
    add(ie + 'proj', (d, enc['output_dim']), 'normal', d ** -0.5)  # unused by GIT (output_grid=True)
    add(ie + 'conv1.weight', (d, 3, p, p), 'normal', s3 * (3 * p * p) ** -0.5)
    add(ie + 'ln_pre.weight', (d,), 'ones')
    add(ie + 'ln_pre.bias', (d,), 'zeros')
    for i in range(nl):
        b = ie + 'transformer.resblocks.%d.' % i
        add(b + 'attn.in_proj_weight', (3 * d, d), 'normal', s3 * (6.0 / (4 * d)) ** 0.5)
        add(b + 'attn.in_proj_bias', (3 * d,), 'zeros')
        add(b + 'attn.out_proj.weight', (d, d), 'normal', s3 * d ** -0.5)
        add(b + 'attn.out_proj.bias', (d,), 'zeros')
        add(b + 'ln_1.weight', (d,), 'ones')
        add(b + 'ln_1.bias', (d,), 'zeros')
        add(b + 'mlp.c_fc.weight', (4 * d, d), 'normal', s3 * d ** -0.5)
        add(b + 'mlp.c_fc.bias', (4 * d,), 'normal', s3 * d ** -0.5)
        add(b + 'mlp.c_proj.weight', (d, 4 * d), 'normal', s3 * (4 * d) ** -0.5)
        add(b + 'mlp.c_proj.bias', (d,), 'normal', s3 * (4 * d) ** -0.5)
        add(b + 'ln_2.weight', (d,), 'ones')
        add(b + 'ln_2.bias', (d,), 'zeros')
    add(ie + 'ln_post.weight', (d,), 'ones')
    add(ie + 'ln_post.bias', (d,), 'zeros')

    t = 'textual.'
    D = HIDDEN
    add(t + 'visual_projection.0.weight', (D, dv), 'normal', 0.02)
    add(t + 'visual_projection.0.bias', (D,), 'normal', s3 * dv ** -0.5)
    add(t + 'visual_projection.1.weight', (D,), 'ones')
    add(t + 'visual_projection.1.bias', (D,), 'zeros')
    add(t + 'embedding.words.weight', (VOCAB, D), 'normal', 0.02)
    add(t + 'embedding.positions.weight', (MAX_POS, D), 'normal', 0.02)
    add(t + 'embedding.layer_norm.weight', (D,), 'ones')
    add(t + 'embedding.layer_norm.bias', (D,), 'zeros')
    for j in range(DEC_LAYERS):
        b = t + 'transformer.encoder.layer.%d.' % j
        for n in ('query', 'key', 'value'):
            add(b + 'attention.self.%s.weight' % n, (D, D), 'normal', 0.02)
            add(b + 'attention.self.%s.bias' % n, (D,), 'normal', s3 * D ** -0.5)
        add(b + 'attention.output.dense.weight', (D, D), 'normal', 0.02)
        add(b + 'attention.output.dense.bias', (D,), 'normal', s3 * D ** -0.5)
        add(b + 'attention.output.LayerNorm.weight', (D,), 'ones')
        add(b + 'attention.output.LayerNorm.bias', (D,), 'zeros')
        add(b + 'intermediate.dense.weight', (FFN, D), 'normal', 0.02)
        add(b + 'intermediate.dense.bias', (FFN,), 'normal', s3 * D ** -0.5)
        add(b + 'output.dense.weight', (D, FFN), 'normal', 0.02)
        add(b + 'output.dense.bias', (D,), 'normal', s3 * FFN ** -0.5)
        add(b + 'output.LayerNorm.weight', (D,), 'ones')
        add(b + 'output.LayerNorm.bias', (D,), 'zeros')
    # textual.output.weight is tied to textual.embedding.words.weight (layers/decoder.py:503-505)
    add(t + 'output.weight', (VOCAB, D), 'tied', 0.0)
    add(t + 'output.bias', (VOCAB,), 'normal', s3 * D ** -0.5)
    n_frames = param.get('num_image_with_embedding') or 0
    for i in range(n_frames):
        add('img_temperal_embedding.%d' % i, (1, 1, dv), 'zeros')
    return spec


def _rng(seed, key):
    return np.random.Generator(np.random.PCG64([int(seed), zlib.crc32(key.encode())]))


def synthetic_state_dict(param=None, seed=0, variant='init'):
    """Seeded checkpoint with the reference's keys.

    variant 'init'     : the reference initialisers' distributions (LayerNorm = (1, 0), temporal
                         embeddings = 0) -- "random-init weights of the named size".
    variant 'decisive' : 'perturbed' with the LM-head bias of decisive_output_bias() (free-running token identity).
    variant 'perturbed': same, but (a) the tied word embedding / LM-head matrix is 4x larger (logit std
                         ~2 instead of ~0.5, so the softmax is not near-uniform), and (b) LayerNorm
                         scales/shifts, the zero biases and the temporal embeddings get small random
                         values so every fused epilogue term is exercised.  Note that top-1/top-2
                         margins stay small relative to bf16 GEMM noise for ANY random checkpoint
                         (the ratio is scale-invariant; SURVEY.md section 0 item 5) -- parity tests are
                         therefore teacher-forced and margin-aware.
    """
    assert variant in ('init', 'perturbed', 'decisive')
    decisive = variant == 'decisive'
    if decisive:
        variant = 'perturbed'
    sd = OrderedDict()
    for key, shape, (kind, scale) in state_spec(param):
        if kind == 'tied':
            sd[key] = sd['textual.embedding.words.weight']
            continue
        g = _rng(seed, key)
        if kind == 'normal':
            a = g.standard_normal(shape, dtype=np.float32) * np.float32(scale)
            if variant == 'perturbed' and key == 'textual.embedding.words.weight':
                a = a * np.float32(4.0)
        elif kind == 'ones':
            a = np.ones(shape, dtype=np.float32)
            if variant == 'perturbed':
                a = a + g.standard_normal(shape, dtype=np.float32) * np.float32(0.05)
        else:
            a = np.zeros(shape, dtype=np.float32)
            if variant == 'perturbed':
                a = a + g.standard_normal(shape, dtype=np.float32) * np.float32(0.02)
        if decisive and key == 'textual.output.bias':
            a = decisive_output_bias(a, seed)
        if decisive and key.startswith('textual.transformer.encoder.layer.'):
            # sharper decoder attention (q, k x8) whose output weighs more in the residual stream (x4): the ranking of
            # the live tokens then depends on WHICH image tokens a row attends to, i.e. on the image and the history
            if key.endswith('attention.self.query.weight') or key.endswith('attention.self.key.weight'):
                a = a * np.float32(DECISIVE_QK_SCALE)
            elif key.endswith('attention.output.dense.weight'):
                a = a * np.float32(DECISIVE_AO_SCALE)
        sd[key] = torch.from_numpy(np.ascontiguousarray(a))
    return sd


DECISIVE_LIVE = 8      # tokens that stay in play in the 'decisive' variant (EOS is one of them)
# decoder attention sharpening of the 'decisive' variant (q, k weights / attention output weights).  Chosen with
# tools/decisive_pick.py: the sharper the softmax the more the captions depend on the image -- and the more bf16 rounding is
# amplified; x8 / x4 made the decoder chaotic (12.5 max logit error), these values keep the error at the random-init level
DECISIVE_QK_SCALE = 2.0
DECISIVE_AO_SCALE = 2.0


def decisive_output_bias(bias, seed):
    """'decisive' variant = 'perturbed' with an LM-head bias that takes all but DECISIVE_LIVE seeded tokens out of play
    (-30) and handicaps EOS (-3, so captions end at different steps).  The ranking among the live tokens still comes
    from the whole network (image, history), but the top-1/top-2 gap is no longer the gap of the two largest of 30522
    near-iid values: tests/golden/*decisive* pick (seed, image seed) pairs whose smallest free-running greedy margin is
    many times the engine's measured logit error, and assert token identity with the unmodified reference on them."""
    g = _rng(seed, 'decisive.live_tokens')
    live = g.choice(np.arange(1000, VOCAB), size=DECISIVE_LIVE - 1, replace=False)
    out = bias - np.float32(30.0)
    out[live] = bias[live]
    out[102] = bias[102] - np.float32(3.0)
    return out.astype(np.float32)


def synthetic_images(batch, frames=0, seed=1234, res=224):
    """Synthetic CLIP-normalised pixels: one fp32 [B,3,res,res] tensor (frames=0) or a list of
    `frames` such tensors (video path, reference inference.py:89 passes a list).  `res` may be (height, width)."""
    rh, rw = (res, res) if isinstance(res, int) else (int(res[0]), int(res[1]))

    def one(i):
        g = np.random.Generator(np.random.PCG64([int(seed), int(i)]))
        return torch.from_numpy(g.standard_normal((batch, 3, rh, rw), dtype=np.float32))
    if not frames:
        return one(0)
    return [one(i) for i in range(frames)]
