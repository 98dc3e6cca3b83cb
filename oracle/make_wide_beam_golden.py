"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/wide_beam_*.npz: the unmodified reference's GeneratorWithBeamSearch
(layers/decoder.py:1056-1290) at beam sizes above the shipped 4 (per-node 2, length_penalty 0.6), imported through
oracle/ref_shim.py, on random-init synthetic checkpoints.

Run where the reference is importable (GIT_REFERENCE_ROOT):  python oracle/make_wide_beam_golden.py [case ...]

Per case, as oracle/make_golden.py stores its beam cases: the config, `predictions`, `logprobs`, every `decoding_step`
call's raw logits at 64 fixed vocabulary columns plus the top-4 values / indices per row, and the search trajectory (the
newest token of every row at every step and the source row of its history).  The reference's source is not modified:
its decoder is built here with the case's beam size and `decoding_step` is observed by wrapping the bound method.
"""
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import ref_shim  # noqa: E402
from make_golden import GOLDEN_DIR, LARGE, vocab_sample, beam_idx_from_histories  # noqa: E402
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images  # noqa: E402

CASES = {
    # name: param, batch, beam, max_steps (every case: variant 'init', weight seed 0, image seed 1234, 224x224)
    'wide_beam_base_k5': dict(param={}, batch=2, beam=5, max_steps=40),
    'wide_beam_base_k6': dict(param={}, batch=2, beam=6, max_steps=40),
    'wide_beam_base_k8': dict(param={}, batch=2, beam=8, max_steps=40),
    'wide_beam_large_k8': dict(param=LARGE, batch=4, beam=8, max_steps=16),
}


def run_case(name, cfg, seed=0, img_seed=1234):
    _, ref_decoder = ref_shim._import_reference()
    sd = synthetic_state_dict(cfg['param'], seed, 'init')
    model = ref_shim.load_reference_model(cfg['param'], 'stock', state_dict=sd)
    model.decoder = ref_decoder.GeneratorWithBeamSearch(eos_index=ref_shim.Tok.sep_token_id, max_steps=cfg['max_steps'],
                                                        beam_size=cfg['beam'], length_penalty=0.6)
    image = synthetic_images(cfg['batch'], 0, img_seed, 224)
    cols = torch.from_numpy(vocab_sample(64))
    steps, inputs = [], []
    orig = model.decoding_step

    def spy(*a, **kw):
        z = orig(*a, **kw)
        top = z.topk(4, dim=1)
        steps.append((z[:, cols].clone(), top.values.clone(), top.indices.clone()))
        inputs.append(a[3].clone())          # partial_captions of this call [rows, cur_len]
        return z
    model.decoding_step = spy
    t0 = time.time()
    with torch.no_grad():
        out = model({'image': image})
    dt = time.time() - t0
    ids = [x.numpy() for x in inputs]
    bidx = [np.arange(ids[0].shape[0], dtype=np.int32)]
    for prev, cur in zip(ids[:-1], ids[1:]):
        bidx.append(beam_idx_from_histories(prev, cur, cfg['beam']))
    meta = dict(cfg, search='beam', variant='init', frames=0, seed=seed, img_seed=img_seed, torch=torch.__version__,
                generator='oracle/make_wide_beam_golden.py', seconds=round(dt, 2))
    np.savez_compressed(
        os.path.join(GOLDEN_DIR, name + '.npz'),
        meta=np.array(json.dumps(meta)),
        predictions=out['predictions'].numpy(),
        logprobs=out['logprobs'].numpy(),
        vocab_cols=cols.numpy(),
        step_logits=torch.stack([s[0] for s in steps]).numpy(),
        step_top4_val=torch.stack([s[1] for s in steps]).numpy(),
        step_top4_idx=torch.stack([s[2] for s in steps]).numpy(),
        step_tokens=np.stack([x[:, -1] for x in ids]),
        step_beam_idx=np.stack(bidx),
    )
    print('%-20s %6.1fs steps=%d pred=%s lp=%s' % (name, dt, len(steps), tuple(out['predictions'].shape),
                                                  np.round(out['logprobs'].flatten().numpy(), 4).tolist()))


if __name__ == '__main__':
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for n in sys.argv[1:] or list(CASES):
        run_case(n, CASES[n])
