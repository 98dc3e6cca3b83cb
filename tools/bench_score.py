"""Caption scoring throughput: `model.score` (one teacher-forced pass) against the route that existed before it -- a
teacher-forced generate with step logits, one image row per caption, then log-softmax and gather in torch.

Workloads (synthetic weights and pixels):
  (a) GIT_BASE 224: 64 images x 5 captions of 12-20 tokens;
  (b) GIT_BASE at the VQAv2 geometry (480-crop model, respect-ratio 640): 16 ragged images x (one question + each of 8
      candidate answers).
The two routes are timed in alternating rounds with CUDA events; the script asserts that their token log-probabilities
agree and prints captions scored per second for each, with the card's name and power limit.

    python tools/bench_score.py [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class Tok:
    cls_token_id, sep_token_id = 101, 102


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or 'unknown'
    except Exception:
        power = 'unknown'
    return name, power


def workload(kind, seed=5):
    from generativeimage2text_b200.synthetic import synthetic_images
    g = np.random.Generator(np.random.PCG64(seed))
    rows = []
    if kind == 'a':
        param = {}
        images = synthetic_images(64, 0, 11).cuda()
        for b in range(64):
            for _ in range(5):
                L = int(g.integers(12, 21))
                rows.append(([101] + list(g.integers(1000, 29000, size=L - 2)) + [102], [0] + [1] * (L - 1), b))
    else:
        param = {'test_crop_size': 480, 'test_respect_ratio_max': 640}
        hws = [[480, 640], [640, 480], [480, 480], [480, 560]]
        images = [synthetic_images(1, 0, 40 + b, hws[b % 4])[0].cuda() for b in range(16)]
        for b in range(16):
            q = list(g.integers(1000, 29000, size=int(g.integers(4, 9))))
            for _ in range(8):
                a = list(g.integers(1000, 29000, size=int(g.integers(1, 4))))
                rows.append(([101] + q + a + [102], [0] * (1 + len(q)) + [1] * (len(a) + 1), b))
    T = max(len(r[0]) for r in rows)
    tok = torch.zeros((len(rows), T), dtype=torch.long)
    need = torch.zeros((len(rows), T), dtype=torch.long)
    for n, (t, m, _) in enumerate(rows):
        tok[n, :len(t)] = torch.tensor(t)
        need[n, :len(m)] = torch.tensor(m)
    index = torch.tensor([r[2] for r in rows])
    return param, images, tok, need, index


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    from generativeimage2text_b200.model import get_git_model, AutoRegressiveBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    name, power = card()
    results = {'card': name, 'power_limit': power}
    for kind in ('a', 'b'):
        param, images, tok, need, index = workload(kind)
        N, T = tok.shape
        m = get_git_model(Tok(), param)
        m.load_state_dict(synthetic_state_dict(param, 0, 'perturbed'), strict=False)
        m = m.cuda().eval()
        m.decoder = AutoRegressiveBeamSearch(102, max_steps=T, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
        batch = {'image': images, 'caption_tokens': tok, 'need_predict': need, 'image_index': index}
        rep = images[index.cuda()] if torch.is_tensor(images) else [images[i] for i in index.tolist()]
        tok_d = tok.cuda()

        def run_score():
            return m.score(batch)['token_logprobs']

        def run_generate():
            z = m({'image': rep}, forced_tokens=tok, return_step_logits=True)['step_logits']   # [T - 1, N, V]
            return torch.log_softmax(z, dim=-1).gather(2, tok_d[:, 1:].T[..., None])[..., 0].T

        a, b = run_score(), run_generate()                 # warm-up (engine creation, weight upload, graphs)
        torch.cuda.synchronize()
        valid = (need[:, 1:] == 1).cuda()
        diff = (a - b).abs()[valid].max().item()
        assert diff < 0.25, 'score and teacher-forced generate disagree by %.3f' % diff
        times = {'score': [], 'generate': []}
        for _ in range(args.rounds):
            for key, fn in (('score', run_score), ('generate', run_generate)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        med = {k: float(np.median(v)) for k, v in times.items()}
        results['workload_' + kind] = {
            'captions': N, 'positions': T, 'images': len(images), 'max_abs_logprob_diff': round(diff, 5),
            'score_ms': round(med['score'], 2), 'generate_ms': round(med['generate'], 2),
            'score_captions_per_s': round(N / med['score'] * 1e3, 1),
            'generate_captions_per_s': round(N / med['generate'] * 1e3, 1)}
        print('workload %s on %s (power limit %s): %d captions x %d positions: score %.2f ms (%.0f captions/s), '
              'teacher-forced generate %.2f ms (%.0f captions/s); max |logprob difference| %.4f'
              % (kind, name, power, N, T, med['score'], N / med['score'] * 1e3, med['generate'],
                 N / med['generate'] * 1e3, diff))
        m.release()
    print(json.dumps(results))
    out = os.environ.get('BENCH_SCORE_OUT')
    if out:
        with open(out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
