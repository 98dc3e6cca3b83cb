"""n sequences per image (num_return_sequences) against the same call with every image repeated n times.

Two workloads, random-init weights, synthetic 224x224 images, max_len 40:
  scst : GIT_BASE, 64 images x n = 5, greedy decoder sampling at temperature 0.7 (320 sequences; the reference's
         self-critical training asks for five samples per image, layers/decoder.py:894-906);
  beam : GIT_LARGE, 32 images x n = 2, GeneratorWithBeamSearch beam 4, sampled at top_k 50 / top_p 0.9 (256 rows).
For each, the n-sequence call and the repeated-image call run in alternating rounds with the same uniforms, timed with CUDA
events (each round ends in a device synchronise); the outputs of both are asserted bit-identical every round.  Reported per
arm: median ms per call, sequences/s, the decode loop's ms per step (last_decode_timing) and the rest of the call (encode +
prefill + set-up).  Prints one JSON line with the card's name and its power limit (read-only nvidia-smi query in the same run):

    python tools/bench_return_sequences.py [--steps K] [--warmup W] [--workload scst|beam|both]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MAX_STEPS = 40
LARGE = {'image_encoder_type': 'CLIPViT_L_14', 'visual_feature_size': 1024}


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


def run(name, param, B, n, decoder, sp, u, rounds, warmup, dev):
    import torch
    from generativeimage2text_b200.model import get_git_model
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    model = get_git_model(Tok(), param)
    model.load_state_dict(synthetic_state_dict(param, 0, 'init'), strict=True)
    model = model.to(dev).eval()
    model.decoder = decoder
    x = synthetic_images(B, 0, 1234).to(dev)
    sp = dict(sp, uniforms=u.to(dev))
    arms = {'n_sequences': lambda: model({'image': x}, search_param=dict(sp, num_return_sequences=n)),
            'repeated_images': lambda: model({'image': x.repeat_interleave(n, 0)}, search_param=sp)}
    times = {k: [] for k in arms}
    dec = {k: [] for k in arms}
    for i in range(warmup + rounds):
        outs = {}
        for arm, fn in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            outs[arm] = fn()
            t1.record()
            torch.cuda.synchronize()
            if i >= warmup:
                times[arm].append(t0.elapsed_time(t1))
                dec[arm].append(model.last_decode_timing()[:2])
        a, b = outs['n_sequences'], outs['repeated_images']
        assert torch.equal(a['predictions'], b['predictions']) and torch.equal(a['logprobs'], b['logprobs']), name
    res = {'images': B, 'sequences_per_image': n, 'rows': int(u.shape[1]), 'rounds': rounds}
    for arm in arms:
        call = statistics.median(times[arm])
        dms = statistics.median(d for d, _ in dec[arm])
        res[arm] = {'call_ms_median': round(call, 3), 'call_ms': [round(t, 3) for t in times[arm]],
                    'sequences_per_s': round(B * n / call * 1e3, 1),
                    'decode_ms_median': round(dms, 3), 'step_launches': sorted({s for _, s in dec[arm]}),
                    'decode_ms_per_step': round(statistics.median(d / s for d, s in dec[arm]), 4),
                    'rest_of_call_ms': round(statistics.median(t - d for t, (d, _) in zip(times[arm], dec[arm])), 3)}
    model.release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=7, help='timed rounds of each arm (alternating)')
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--workload', choices=['scst', 'beam', 'both'], default='both')
    args = ap.parse_args()

    import torch
    import __graft_entry__
    __graft_entry__.build()
    from generativeimage2text_b200.model import AutoRegressiveBeamSearch, GeneratorWithBeamSearch

    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(7)
    card, watts = gpu_card(0)
    res = {'card': card, 'power_limit_w': watts, 'max_len': MAX_STEPS, 'weights': 'random-init (synthetic_state_dict init)'}
    if args.workload in ('scst', 'both'):
        dec = AutoRegressiveBeamSearch(102, max_steps=MAX_STEPS, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
        res['scst_base_64x5_greedy_sampled_T0.7'] = run(
            'scst', {}, 64, 5, dec, {'do_sample': True, 'temperature': 0.7}, torch.rand((MAX_STEPS, 320), generator=g),
            args.steps, args.warmup, dev)
    if args.workload in ('beam', 'both'):
        dec = GeneratorWithBeamSearch(102, max_steps=MAX_STEPS, beam_size=4, length_penalty=0.6)
        res['large_32x2_beam4_sampled_k50_p0.9'] = run(
            'beam', LARGE, 32, 2, dec, {'do_sample': True, 'top_k': 50, 'top_p': 0.9},
            torch.rand((MAX_STEPS, 256, 2), generator=g), args.steps, args.warmup, dev)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
