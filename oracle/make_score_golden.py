"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/score_*.npz, the reference goldens of caption scoring, by running the
UNMODIFIED reference's training-branch forward (CaptioningModel.forward_one_ce, layers/decoder.py:916-972) through
oracle/ref_shim.py.

The model is put in training mode (the branch that takes `caption_tokens` / `need_predict` and returns `vl_l_loss`) and every
nn.Dropout module is then switched back to eval: dropout (0.1 in the BERT layers and the embedding) is the only randomness
of that branch, so the forward becomes deterministic; every case is run twice and must give the same loss.  Images are
repeated by `image_index` (the reference has no such argument).  The reference cannot batch images of different sizes, so
the ragged case makes one call per image and combines the per-call losses weighted by their token counts.

Per case: tokens, need_predict, image_index, vl_l_loss, the target log-probabilities [N, T-1], the logits at the fixed
vocabulary columns of oracle/make_golden.py [N, T, cols] (captured by wrapping `model.textual.forward` on the instance),
and a strided sample of the image features.

Run where the reference is importable:  python oracle/make_score_golden.py [case ...]
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
from make_golden import GOLDEN_DIR, LARGE, vocab_sample  # noqa: E402
from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images  # noqa: E402

VQA = {'test_crop_size': 480, 'test_respect_ratio_max': 640}


def captions(n_img, per_img, T, seed, min_len=5, max_len=20, question=True, zero_inside=True):
    """[N, T] token rows CLS .. SEP padded with 0 (the reference's collate_fn) and their need_predict (train.py:38-61):
    every second caption starts with a question prefix (need_predict 0); the first caption holds a 0 token inside its
    predicted part (a target the loss ignores)."""
    g = np.random.Generator(np.random.PCG64(seed))
    N = n_img * per_img
    tok = np.zeros((N, T), dtype=np.int64)
    need = np.zeros((N, T), dtype=np.int64)
    for n in range(N):
        L = int(g.integers(min_len, max_len + 1))            # CLS + payload + SEP
        payload = g.integers(1000, 29000, size=L - 2)
        n_q = int(g.integers(1, L - 3)) if (question and n % 2 == 1) else 0
        tok[n, :L] = np.concatenate([[101], payload, [102]])
        need[n, :L] = [0] + [0] * n_q + [1] * (L - 2 - n_q) + [1]
    if zero_inside:
        k = int(np.nonzero(need[0])[0][1])
        tok[0, k] = 0
    return tok, need, np.repeat(np.arange(n_img), per_img).astype(np.int64)


def vqa_captions(n_img, n_ans, seed):
    """One question per image followed by each of n_ans candidate answers: need_predict 0 on CLS + question, 1 on answer + SEP."""
    g = np.random.Generator(np.random.PCG64(seed))
    rows = []
    for b in range(n_img):
        q = list(g.integers(1000, 29000, size=int(g.integers(3, 7))))
        for a in range(n_ans):
            ans = list(g.integers(1000, 29000, size=int(g.integers(1, 4))))
            rows.append(([101] + q + ans + [102], [0] * (1 + len(q)) + [1] * (len(ans) + 1), b))
    T = max(len(r[0]) for r in rows)
    tok = np.zeros((len(rows), T), dtype=np.int64)
    need = np.zeros((len(rows), T), dtype=np.int64)
    for n, (t, m, _) in enumerate(rows):
        tok[n, :len(t)] = t
        need[n, :len(m)] = m
    return tok, need, np.array([r[2] for r in rows], dtype=np.int64)


CASES = {
    'score_base_init': dict(param={}, variant='init', batch=4, frames=0, caps=dict(per_img=3, T=22)),
    'score_base_perturbed': dict(param={}, variant='perturbed', batch=4, frames=0, caps=dict(per_img=3, T=22)),
    'score_large': dict(param=LARGE, variant='perturbed', batch=2, frames=0, caps=dict(per_img=2, T=16, max_len=16)),
    'score_vatex': dict(param={'num_image_with_embedding': 6}, variant='perturbed', batch=2, frames=6,
                        caps=dict(per_img=2, T=18, max_len=18)),
    'score_vqa_ragged': dict(param=VQA, variant='perturbed', image_hws=[[480, 640], [640, 480], [480, 480]], vqa=4),
    'score_base_b64': dict(param={}, variant='init', batch=64, frames=0, n_cols=64,
                           caps=dict(per_img=1, T=40, min_len=40, max_len=40, question=False, zero_inside=False)),
}


def _reference(param, sd):
    model = ref_shim.load_reference_model(param, 'greedy', 12, state_dict=sd)
    model.train()                                         # the branch that scores given captions
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.eval()                                      # ... without its only source of randomness
    return model


def _run(model, image, tok, need):
    """One reference forward -> (vl_l_loss, output logits [N, T, V])."""
    seen = []
    orig = model.textual.forward

    def spy(*a, **kw):
        out = orig(*a, **kw)
        seen.append(out)
        return out
    model.textual.forward = spy
    try:
        with torch.no_grad():
            out = model({'image': image, 'caption_tokens': torch.from_numpy(tok), 'need_predict': torch.from_numpy(need)})
    finally:
        del model.textual.forward
    assert len(seen) == 1
    return out['vl_l_loss'], seen[0]


def run_case(name, cfg, seed=0, img_seed=1234, cap_seed=99):
    sd = synthetic_state_dict(cfg['param'], seed, cfg['variant'])
    model = _reference(cfg['param'], sd)
    cols = torch.from_numpy(vocab_sample(cfg.get('n_cols', 256)))
    t0 = time.time()
    arrays = {}
    if 'image_hws' in cfg:
        tok, need, index = vqa_captions(len(cfg['image_hws']), cfg['vqa'], cap_seed)
        N, T = tok.shape
        logits = torch.zeros(N, T, len(cols))
        loss_sum, count, zs = 0.0, 0, []
        for b, hw in enumerate(cfg['image_hws']):
            rows = np.nonzero(index == b)[0]
            image = synthetic_images(1, 0, img_seed + b, hw)
            loss, z = _run(model, image.expand(len(rows), -1, -1, -1), tok[rows], need[rows])
            loss2, _ = _run(model, image.expand(len(rows), -1, -1, -1), tok[rows], need[rows])
            assert loss.item() == loss2.item(), 'the reference forward is not deterministic'
            n_valid = int(((need[rows, 1:] == 1) & (tok[rows, 1:] != 0)).sum())
            loss_sum += loss.item() * n_valid
            count += n_valid
            logits[rows] = z[:, :, cols]
            zs.append(z)                                 # the rows of image b follow those of image b - 1
            with torch.no_grad():
                arrays['feats_sample_%d' % b] = model.image_encoder(image)[:, ::17, ::29].numpy()
        loss = torch.tensor(loss_sum / count)
        z_all = torch.cat(zs)
    else:
        tok, need, index = captions(cfg['batch'], seed=cap_seed, **cfg['caps'])
        image = synthetic_images(cfg['batch'], cfg['frames'], img_seed)
        idx = torch.from_numpy(index)
        rep = [f[idx] for f in image] if isinstance(image, list) else image[idx]
        loss, z_all = _run(model, rep, tok, need)
        loss2, _ = _run(model, rep, tok, need)
        assert loss.item() == loss2.item(), 'the reference forward is not deterministic'
        logits = z_all[:, :, cols]
        with torch.no_grad():
            f0 = image[0] if isinstance(image, list) else image
            arrays['feats_sample'] = model.image_encoder(f0)[:, ::17, ::29].numpy()
    lp = torch.log_softmax(z_all[:, :-1].float(), dim=-1).gather(2, torch.from_numpy(tok[:, 1:, None]))[..., 0]
    meta = {k: v for k, v in cfg.items() if k != 'caps'}
    meta.update(seed=seed, img_seed=img_seed, cap_seed=cap_seed, reference_commit='faae4fb9', torch=torch.__version__,
                generator='oracle/make_score_golden.py', seconds=round(time.time() - t0, 2))
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + '.npz'), meta=np.array(json.dumps(meta)), vocab_cols=cols.numpy(),
                        caption_tokens=tok, need_predict=need, image_index=index, vl_l_loss=np.float32(loss.item()),
                        token_logprobs=lp.numpy().astype(np.float32), logits=logits.numpy().astype(np.float32), **arrays)
    print('%-22s N=%d T=%d loss=%.6f (%.1fs)' % (name, tok.shape[0], tok.shape[1], loss.item(), time.time() - t0))


if __name__ == '__main__':
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for n in sys.argv[1:] or list(CASES):
        run_case(n, CASES[n])
