"""Writes tests/golden/beam_sample_checks.json: what the original GenerativeImage2Text code's GeneratorWithBeamSearch.search
returns with do_sample=True on the toy steps of tests/test_beam_sample_host.py, with torch.multinomial replaced by the draw
the engine makes (beam_sample_oracle.two_draws: two sequential index-order inverse-CDF lookups) fed the same uniforms -- the way
make_reference_golden.py pins the greedy sampling branch.  Regenerate with the original tree importable (oracle/ref_shim.py,
GIT_REFERENCE_ROOT):

    python oracle/make_beam_sample_golden.py
"""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import ref_shim  # noqa: E402
import beam_sample_oracle as bso  # noqa: E402
import test_beam_sample_host as T  # noqa: E402


def run_case(ref_decoder, case, seen):
    beam, B, temperature, top_k, top_p, steps, seed, eos_bias = case
    eos = 2
    u = T.case_uniforms(case)
    start = torch.tensor([[1]] * B)
    dec = ref_decoder.GeneratorWithBeamSearch(eos, max_steps=steps, beam_size=beam, per_node_beam_size=2,
                                              length_penalty=0.6, temperature=temperature)
    calls = {'t': start.shape[1], 'last': 0}
    real_multinomial, real_filter = torch.multinomial, ref_decoder.top_k_top_p_filtering

    def fake_multinomial(probs, num_samples):
        assert num_samples == 2
        t = calls['t']
        calls['t'] += 1
        calls['last'] = t
        words = bso.two_draws(probs, u[t])
        seen['eos_drawn'] |= bool((words == eos).any())
        return words

    def watch_filter(logits, top_k=0, top_p=1.0, filter_value=-float('Inf'), min_tokens_to_keep=1):
        before = logits.clone()
        out = real_filter(logits, top_k=top_k, top_p=top_p, filter_value=filter_value, min_tokens_to_keep=min_tokens_to_keep)
        if top_p and top_p < 1.0:
            # the keep-three rule decides where the nucleus alone would keep fewer than three tokens
            k_only = bso.top_k_top_p_filter(before, top_k, None)
            probs = torch.softmax(k_only, dim=-1).sort(dim=-1, descending=True)[0]
            seen['keep_three_decides'] |= bool((probs[:, 0] + probs[:, 1] > top_p).any())
        return out
    torch.multinomial, ref_decoder.top_k_top_p_filtering = fake_multinomial, watch_filter
    try:
        pred, lp = dec.search(start, T.toy_step(seed=seed, eos_bias=eos_bias), do_sample=True, top_k=top_k, top_p=top_p)
    finally:
        torch.multinomial, ref_decoder.top_k_top_p_filtering = real_multinomial, real_filter
    if calls['last'] + 1 < steps:
        seen['ended_early'] = True
    else:
        seen['ran_to_max_steps'] = True
    seen['batch_gt_1'] |= B > 1
    seen['beam_%d' % beam] = True
    return {'case': list(case), 'predictions': pred.tolist(), 'logprobs': lp.double().tolist()}


def main():
    if not ref_shim.reference_available():
        raise SystemExit('the original code is not importable at %s (set GIT_REFERENCE_ROOT)' % ref_shim.REFERENCE_ROOT)
    _, ref_decoder = ref_shim._import_reference()
    seen = dict.fromkeys(('eos_drawn', 'ended_early', 'ran_to_max_steps', 'keep_three_decides', 'batch_gt_1', 'beam_2',
                          'beam_3', 'beam_4'), False)
    out = {'cases': [run_case(ref_decoder, case, seen) for case in T.CASES], 'seen': seen}
    with open(T.GOLDEN, 'w') as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write('\n')
    print('%s: %d bytes; %s' % (T.GOLDEN, os.path.getsize(T.GOLDEN), seen))


if __name__ == '__main__':
    main()
