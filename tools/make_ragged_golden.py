"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/base_ragged_{greedy,beam}.npz, the reference goldens of ragged batches
(a list of images of their own sizes in one engine call), by running the UNMODIFIED reference through oracle/ref_shim.py.

The reference cannot batch images of different sizes, so every image is its own batch-1 reference call; image b uses
pixels synthetic_images(1, 0, img_seed + b, image_hws[b]).  Per image the file keeps what oracle/make_golden.py keeps per
batch, with a `_<b>` suffix: predictions, logprobs, the raw last-position logits of every decoding_step at the 256 fixed
vocabulary columns of oracle/make_golden.py plus the top-4 values / indices, and strided samples of the image features
and of their visual projection.

Run where the reference is importable:  python tools/make_ragged_golden.py [case ...]
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, ROOT)

import ref_shim  # noqa: E402
from make_golden import GOLDEN_DIR, vocab_sample  # noqa: E402
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images  # noqa: E402

# four MinMaxResizeForTest sizes of a 160 / 224 model: four different patch grids (10x13, 13x10, 10x10, 10x14 =
# 131 / 131 / 101 / 141 image tokens)
RATIO = {'test_crop_size': 160, 'test_respect_ratio_max': 224}
HWS = [[160, 208], [208, 160], [160, 160], [160, 224]]
CASES = {
    'base_ragged_greedy': dict(param=RATIO, variant='perturbed', batch=4, frames=0, search='greedy', max_steps=12,
                               image_hws=HWS, ragged=True),
    'base_ragged_beam': dict(param=RATIO, variant='init', batch=4, frames=0, search='beam', max_steps=12,
                             image_hws=HWS, ragged=True),
}


def run_ragged_case(name, cfg, seed=0, img_seed=1234):
    sd = synthetic_state_dict(cfg['param'], seed, cfg['variant'])
    model = ref_shim.load_reference_model(cfg['param'], cfg['search'], cfg['max_steps'], state_dict=sd)
    cols = torch.from_numpy(vocab_sample(cfg.get('n_cols', 256)))
    arrays = {}
    t0 = time.time()
    orig = model.decoding_step
    for b, hw in enumerate(cfg['image_hws']):
        image = synthetic_images(1, 0, img_seed + b, hw)
        steps = []

        def spy(*a, **kw):
            z = orig(*a, **kw)
            top = z.topk(4, dim=1)
            steps.append((z[:, cols].clone(), top.values.clone(), top.indices.clone()))
            return z
        model.decoding_step = spy
        with torch.no_grad():
            out = model({'image': image})
            vf = model.image_encoder(image)
            vproj = model.textual.visual_projection(vf)
        arrays.update({
            'predictions_%d' % b: out['predictions'].numpy(),
            'logprobs_%d' % b: out['logprobs'].numpy(),
            'step_logits_%d' % b: torch.stack([s[0] for s in steps]).numpy(),
            'step_top4_val_%d' % b: torch.stack([s[1] for s in steps]).numpy(),
            'step_top4_idx_%d' % b: torch.stack([s[2] for s in steps]).numpy(),
            'feats_sample_%d' % b: vf[:, ::17, ::29].numpy(),
            'vproj_sample_%d' % b: vproj[:, ::17, ::29].numpy(),
        })
        print('%-18s image %d %s: steps=%d pred=%s lp=%s' % (name, b, hw, len(steps), out['predictions'].tolist(),
                                                             np.round(out['logprobs'].flatten().numpy(), 4).tolist()))
    meta = dict(cfg)
    meta.update(seed=seed, img_seed=img_seed, reference_commit='faae4fb9', torch=torch.__version__,
                generator='tools/make_ragged_golden.py', seconds=round(time.time() - t0, 2))
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + '.npz'), meta=np.array(json.dumps(meta)), vocab_cols=cols.numpy(),
                        **arrays)


if __name__ == '__main__':
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for n in sys.argv[1:] or list(CASES):
        run_ragged_case(n, CASES[n])
