"""Ragged batches for the VQA models: how much does one call of mixed-size images gain over one call per image?

GIT_BASE with the VQAv2 geometry (test_crop_size 480, test_respect_ratio_max 640) and the default decoder
(GeneratorWithBeamSearch, beam 4, max_len 40).  16 synthetic images of MinMaxResizeForTest sizes from a seeded list of
aspect ratios, two questions of 4-8 prefix tokens per image: 32 rows, 128 decoder rows under beam 4.  Two ways to answer
them are timed in alternation, each a whole round ending in a device synchronise:
  ragged    : ONE `model(batch)` call with the 16 images as a ragged list (every image repeated once per question) and one
              prefix per row;
  per-image : 16 calls, each image expanded once per question with one prefix per row (the TSV driver's question batch
              at batch_size=1).
Both must give the same outputs (asserted, exact).  Prints one JSON line with questions/s of both, the card's name and its
power limit (read-only nvidia-smi query in the same run):

    python tools/bench_ragged.py [--steps K] [--warmup W]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MAX_STEPS = 40


class Tok:
    cls_token_id, sep_token_id = 101, 102


def gpu_card(index):
    """(name, power limit in W) of the card (read-only query)."""
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(',')
        return out[0].strip(), float(out[1])
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5, help='timed rounds of each way (alternating)')
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()

    import torch
    import __graft_entry__
    __graft_entry__.build()
    from generativeimage2text_b200.inference import MinMaxResizeForTest
    from generativeimage2text_b200.model import get_git_model, GeneratorWithBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images

    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    param = {'test_crop_size': 480, 'test_respect_ratio_max': 640}
    model = get_git_model(Tok(), param)
    model.load_state_dict(synthetic_state_dict(param, 0, 'init'), strict=True)
    model = model.to(dev).eval()
    model.decoder = GeneratorWithBeamSearch(102, max_steps=MAX_STEPS, beam_size=4, length_penalty=0.6)
    rnd = random.Random(2024)
    resize = MinMaxResizeForTest(480, 640)
    sizes = [resize.get_size((1000, int(1000 * rnd.uniform(0.5, 2.0)))) for _ in range(16)]   # (h, w) of (w, h) inputs
    images = [synthetic_images(1, 0, 100 + b, hw)[0].to(dev) for b, hw in enumerate(sizes)]
    prefixes = [[[101] + [rnd.randrange(1000, 30000) for _ in range(rnd.randrange(3, 8))] for _ in range(2)] for _ in images]

    def pad(ps):
        t = torch.zeros((len(ps), max(len(p) for p in ps)), dtype=torch.long)
        for r, p in enumerate(ps):
            t[r, :len(p)] = torch.tensor(p)
        return {'prefix': t.to(dev), 'prefix_len': torch.tensor([len(p) for p in ps])}
    rows = [p for ps in prefixes for p in ps]
    ragged_batch = dict(image=[im for im in images for _ in range(2)], **pad(rows))
    per_image = [dict(image=im[None].expand(2, -1, -1, -1), **pad(ps)) for im, ps in zip(images, prefixes)]

    def ragged():
        return [model(ragged_batch)]

    def one_per_image():
        return [model(b) for b in per_image]

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    for _ in range(args.warmup):
        ragged()
        one_per_image()
    t_r, t_p = [], []
    for _ in range(args.steps):
        s, out_r = timed(ragged)
        t_r.append(s)
        s, out_p = timed(one_per_image)
        t_p.append(s)
    # the same outputs: row 2b + i of the ragged call == row i of image b's call (EOS padding aside)
    pr, lr = out_r[0]['predictions'].cpu(), out_r[0]['logprobs'].cpu().reshape(-1)
    for b, o in enumerate(out_p):
        pp, lp = o['predictions'].cpu(), o['logprobs'].cpu().reshape(-1)
        for i in range(2):
            a, c = pr[2 * b + i], pp[i]
            w = min(a.numel(), c.numel())
            assert torch.equal(a[:w], c[:w]) and bool((a[w:] == 102).all()) and bool((c[w:] == 102).all()), (b, i)
            assert torch.equal(lr[2 * b + i], lp[i]), (b, i)
    sec_r, sec_p = statistics.median(t_r), statistics.median(t_p)
    name, power = gpu_card(0)
    n_q = len(rows)
    print(json.dumps({
        'metric': 'questions/s (beam=4, max_len=%d) GIT_BASE VQAv2 geometry 480/640, 16 images x 2 questions' % MAX_STEPS,
        'unit': 'questions/s', 'ragged_call': n_q / sec_r, 'per_image_calls': n_q / sec_p, 'speedup': sec_p / sec_r,
        'median_ms_ragged_call': sec_r * 1e3, 'median_ms_per_image_calls': sec_p * 1e3,
        'ms_ragged_rounds': [round(t * 1e3, 2) for t in t_r], 'ms_per_image_rounds': [round(t * 1e3, 2) for t in t_p],
        'image_tokens': [(h // 16) * (w // 16) + 1 for h, w in sizes], 'outputs_equal': True, 'steps': args.steps,
        'warmup': args.warmup, 'gpu': name, 'power_limit_w': power}), flush=True)


if __name__ == '__main__':
    main()
