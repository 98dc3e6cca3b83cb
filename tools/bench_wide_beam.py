"""Beam sizes 4, 5, 6 and 8 at bench.py config 3's shape: GIT_LARGE, 32 synthetic 224x224 images per call, random-init
weights, GeneratorWithBeamSearch (per-node 2, length_penalty 0.6, max_len 40) -- 128 to 256 decoder rows.

Two runs in one command:
  calls   : `model(batch)` at each beam size, timed in rounds that alternate between the beam sizes, with CUDA events (each
            call ends in a device synchronise), profiler off.  The beam sizes decode different captions, so they may run
            different numbers of steps: the per-step decode time is reported next to the call time.
  kernels : torch.profiler (CUDA activity) over a few calls of each beam size with programmatic dependent launch off: mean
            device time per launch of beam_row_topk_kernel at candidate capacity 8 (beam 4) and 16 (beams 5 .. 8), of
            beam_update_kernel and of decode_attn_kernel<beam>.
Prints one JSON line with both, the card's name and its power limit (read-only nvidia-smi query in the same run):

    python tools/bench_wide_beam.py [--steps K] [--warmup W] [--beams 4,5,6,8]
"""
import argparse
import json
import os
import re
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_beam_sample import LARGE, MAX_STEPS, Tok, gpu_card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5, help='timed rounds (each round runs every beam size once)')
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--beams', default='4,5,6,8')
    ap.add_argument('--profile-calls', type=int, default=2)
    args = ap.parse_args()
    beams = [int(b) for b in args.beams.split(',')]

    import torch
    import __graft_entry__
    __graft_entry__.build()
    from generativeimage2text_b200.model import get_git_model, GeneratorWithBeamSearch
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images

    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    B = 32
    model = get_git_model(Tok(), LARGE)
    model.load_state_dict(synthetic_state_dict(LARGE, 0, 'init'), strict=True)
    model = model.to(dev).eval()
    decoders = {k: GeneratorWithBeamSearch(102, max_steps=MAX_STEPS, beam_size=k, length_penalty=0.6) for k in beams}
    batch = {'image': synthetic_images(B, 0, 1234).to(dev)}

    def call(k):
        model.decoder = decoders[k]
        return model(batch)

    times = {k: [] for k in beams}
    steps = {k: [] for k in beams}
    first = {}
    for i in range(args.warmup + args.steps):
        for k in beams:
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            out = call(k)
            t1.record()
            torch.cuda.synchronize()
            assert out['predictions'].shape == (B, MAX_STEPS)
            if k not in first:
                first[k] = out['predictions'].clone()
            assert torch.equal(out['predictions'], first[k])            # every round decodes the same captions
            if i >= args.warmup:
                times[k].append(t0.elapsed_time(t1))
                dec_ms, n_steps, _ = model.last_decode_timing()
                steps[k].append((dec_ms, n_steps))

    from torch.profiler import profile, ProfilerActivity
    kern = {}
    # without programmatic dependent launch: a kernel launched early would count its wait for the previous one
    model.set_engine_option('use_pdl', 0)
    for k in beams:
        call(k)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_calls):
                call(k)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            m = re.match(r'(?:void )?gitb200::(beam_row_topk_kernel|beam_update_kernel|decode_attn_kernel)<([^>]*)>', ev.key)
            if m:
                t = getattr(ev, 'device_time_total', None)
                if t is None:
                    t = ev.cuda_time_total
                kern.setdefault('beam%d' % k, {})['%s<%s>' % m.groups()] = {'launches': ev.count,
                                                                          'mean_us': round(t / max(ev.count, 1), 3)}
    model.set_engine_option('use_pdl', 1)

    card, watts = gpu_card(0)
    res = {'workload': 'GIT_LARGE, %d synthetic 224x224 images per call, per-node 2 / length_penalty 0.6, max_len %d, '
                       'random-init weights' % (B, MAX_STEPS),
           'card': card, 'power_limit_w': watts, 'rounds': args.steps}
    for k in beams:
        med = statistics.median(times[k])
        res['beam%d' % k] = {'call_ms_median': round(med, 3), 'captions_per_s': round(B / med * 1e3, 1),
                             'call_ms': [round(t, 3) for t in times[k]],
                             'step_launches': sorted({n for _, n in steps[k]}),
                             'decode_ms_per_step': round(statistics.median(d / n for d, n in steps[k]), 4)}
    res['kernels'] = kern
    print(json.dumps(res))


if __name__ == '__main__':
    main()
