"""Sampled beam search against the deterministic one at bench.py config 3's shape: GIT_LARGE, 32 synthetic 224x224 images per
call, GeneratorWithBeamSearch (beam 4, per-node 2, length_penalty 0.6, max_len 40) -- 128 decoder rows.

Two runs in one command:
  calls   : `model(batch)` with search_param {'do_sample': True, 'top_k', 'top_p'} (seeded uniforms) and without, timed in
            alternating rounds with CUDA events (each round ends in a device synchronise), profiler off.  The two arms
            decode different captions, so they may run different numbers of steps: the step launches of each are reported
            and the per-step decode time is the fairer comparison.
  kernels : torch.profiler (CUDA activity) over a few calls of each arm with programmatic dependent launch off: the
            per-step selection kernel of each, beam_sample_kernel against beam_row_topk_kernel (mean device time per
            launch), and the bookkeeping kernels.
Prints one JSON line with both, the card's name and its power limit (read-only nvidia-smi query in the same run):

    python tools/bench_beam_sample.py [--steps K] [--warmup W] [--top-k 50] [--top-p 0.9] [--temperature 1.0]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=6, help='timed rounds of each arm (alternating)')
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--top-k', type=int, default=50)
    ap.add_argument('--top-p', type=float, default=0.9)
    ap.add_argument('--temperature', type=float, default=1.0)
    ap.add_argument('--profile-calls', type=int, default=2)
    args = ap.parse_args()

    import torch
    import __graft_entry__
    __graft_entry__.build()
    from generativeimage2text_b200.model import get_git_model, GeneratorWithBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images

    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    B, beam = 32, 4
    model = get_git_model(Tok(), LARGE)
    model.load_state_dict(synthetic_state_dict(LARGE, 0, 'init'), strict=True)
    model = model.to(dev).eval()
    model.decoder = GeneratorWithBeamSearch(102, max_steps=MAX_STEPS, beam_size=beam, length_penalty=0.6)
    model.decoder.temperature = args.temperature
    batch = {'image': synthetic_images(B, 0, 1234).to(dev)}
    gen = torch.Generator(device=dev)

    def sampled():
        gen.manual_seed(7)
        return model(batch, search_param={'do_sample': True, 'top_k': args.top_k, 'top_p': args.top_p, 'generator': gen})

    def deterministic():
        return model(batch)
    arms = {'sampled': sampled, 'deterministic': deterministic}

    times = {k: [] for k in arms}
    steps = {}
    for i in range(args.warmup + args.steps):
        for name, fn in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            out = fn()
            t1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[name].append(t0.elapsed_time(t1))
                dec_ms, n_steps, _ = model.last_decode_timing()
                steps.setdefault(name, []).append((dec_ms, n_steps))
            assert out['predictions'].shape == (B, MAX_STEPS)
    again = sampled()
    assert torch.equal(again['predictions'], sampled()['predictions'])      # same generator seed -> same captions

    from torch.profiler import profile, ProfilerActivity
    kern = {}
    # without programmatic dependent launch: a kernel launched early would count its wait for the previous one
    model.set_engine_option('use_pdl', 0)
    sampled(), deterministic()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profile_calls):
            sampled()
            deterministic()
        torch.cuda.synchronize()
    model.set_engine_option('use_pdl', 1)
    for ev in prof.key_averages():
        if ev.key in ('beam_sample_kernel', 'beam_row_topk_kernel') or ev.key.startswith(('void gitb200::beam_sample_kernel',
                                                                                          'void gitb200::beam_row_topk_kernel',
                                                                                          'gitb200::beam_')):
            t = getattr(ev, 'device_time_total', None)
            if t is None:
                t = ev.cuda_time_total
            kern[ev.key] = {'launches': ev.count, 'mean_us': t / max(ev.count, 1)}

    card, watts = gpu_card(0)
    res = {'workload': 'GIT_LARGE, %d synthetic 224x224 images per call, beam %d / per-node 2 / length_penalty 0.6, max_len %d, '
                       'random-init weights; sampled: top_k %d, top_p %g, temperature %g' % (
                           B, beam, MAX_STEPS, args.top_k, args.top_p, args.temperature),
           'card': card, 'power_limit_w': watts, 'rounds': args.steps}
    for name in arms:
        dec = steps[name]
        res[name] = {'call_ms_median': statistics.median(times[name]), 'call_ms': [round(t, 3) for t in times[name]],
                     'decode_ms_median': statistics.median(d for d, _ in dec),
                     'step_launches': sorted({n for _, n in dec}),
                     'decode_ms_per_step': statistics.median(d / n for d, n in dec)}
    res['selection_kernels'] = kern
    print(json.dumps(res))


if __name__ == '__main__':
    main()
