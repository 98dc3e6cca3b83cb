"""Writes tests/golden/return_sequences_checks.json: what the original GenerativeImage2Text code returns with
num_return_sequences = n (layers/decoder.py:232-237, 1093-1096; trie_decoder.py:51-55) on the cases of
tests/test_return_sequences_host.py -- a random-init GIT_BASE, distinct synthetic images, the greedy decoder (deterministic
and sampling), the trie decoder and GeneratorWithBeamSearch (deterministic and sampling) -- with torch.multinomial replaced
by the draws the engine makes fed the same uniforms (git_oracle.inverse_cdf_draw, beam_sample_oracle.two_draws), the way
make_beam_sample_golden.py pins sampled beam search.  Regenerate with the original tree importable (oracle/ref_shim.py,
GIT_REFERENCE_ROOT):

    python oracle/make_return_sequences_golden.py
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
import git_oracle  # noqa: E402
import test_return_sequences_host as T  # noqa: E402


def run_case(model, ref_decoder, td, case):
    search, B, n, temperature, top_k, top_p, _ = case
    eos = ref_shim.Tok.sep_token_id
    u = T.case_uniforms(case)
    if search in ('greedy', 'sample'):
        model.decoder = ref_decoder.AutoRegressiveBeamSearch(eos_index=eos, max_steps=T.MAX_STEPS, beam_size=1,
                                                             per_node_beam_size=1, fix_missing_prefix=True)
    elif search == 'trie':
        model.decoder = td.TrieAutoRegressiveBeamSearch(eos, max_steps=T.MAX_STEPS, beam_size=1,
                                                        trie=td.TokenTrie.construct(T.trie_sequences()))
    else:
        model.decoder = ref_decoder.GeneratorWithBeamSearch(eos_index=eos, max_steps=T.MAX_STEPS, beam_size=T.BEAM,
                                                            length_penalty=0.6, temperature=temperature)
    param = {'num_return_sequences': n}
    if search == 'sample':
        param.update(do_sample=True, temperature=temperature)
    elif search == 'beam_sample':
        param.update(do_sample=True, top_k=top_k, top_p=top_p)
    calls = {'t': 1}

    def fake_multinomial(probs, num_samples):
        t = calls['t']
        calls['t'] += 1
        if num_samples == 2:
            return bso.two_draws(probs, u[t])
        return git_oracle.inverse_cdf_draw(probs, u[t])[:, None]
    images = T.case_images(case)
    real = torch.multinomial
    torch.multinomial = fake_multinomial
    try:
        with torch.no_grad():
            feats = model.image_encoder(images)
            out = model.infer({'image': images}, feats, None, param)
    finally:
        torch.multinomial = real
    return {'case': list(case), 'predictions': out['predictions'].tolist(), 'logprobs': out['logprobs'].double().tolist()}


def main():
    if not ref_shim.reference_available():
        raise SystemExit('the original code is not importable at %s (set GIT_REFERENCE_ROOT)' % ref_shim.REFERENCE_ROOT)
    _, ref_decoder = ref_shim._import_reference()
    import generativeimage2text.trie_decoder as td
    model = ref_shim.load_reference_model({}, 'stock', state_dict=T.state_dict())
    out = {'cases': [run_case(model, ref_decoder, td, case) for case in T.CASES]}
    with open(T.GOLDEN, 'w') as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write('\n')
    print('%s: %d bytes' % (T.GOLDEN, os.path.getsize(T.GOLDEN)))


if __name__ == '__main__':
    main()
