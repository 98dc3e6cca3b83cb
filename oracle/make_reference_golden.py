"""Writes tests/golden/reference_checks.json: what the original GenerativeImage2Text code returns on the inputs of the tests
that compare this project with it (tests/test_oracle_vs_reference.py, test_tsv_io.py, test_preprocess_oracle.py,
test_torch_common.py, test_inference_host.py).  Those tests compare against this file, so they run anywhere; regenerate it
with the original tree importable (oracle/ref_shim.py, GIT_REFERENCE_ROOT):

    python oracle/make_reference_golden.py

Small results are stored as values; large arrays as the SHA-256 of their bytes (the tests compare bit for bit anyway).
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
from golden_io import REFERENCE_CHECKS as OUT, digest, file_digest  # noqa: E402


def oracle_checks(out):
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    import test_oracle_vs_reference as T
    layout = {}
    for name, param in (('base', {}), ('vatex', {'num_image_with_embedding': 6})):
        ref = ref_shim.load_reference_model(param, 'greedy', 40)
        rsd = ref.state_dict()
        layout[name] = {'keys': list(rsd.keys()), 'shapes': [list(v.shape) for v in rsd.values()],
                        'tied': rsd['textual.output.weight'].data_ptr() == rsd['textual.embedding.words.weight'].data_ptr()}
    out['state_dict_layout'] = layout
    fresh = {}
    sd = synthetic_state_dict({}, seed=7, variant='init')
    img = synthetic_images(1, 0, seed=99)
    for search in ('greedy', 'beam'):
        ref = ref_shim.load_reference_model({}, search, 10, state_dict=sd)
        with torch.no_grad():
            r = ref({'image': img})
        fresh[search] = {'predictions': r['predictions'].tolist(), 'logprobs': r['logprobs'].double().tolist()}
    out['fresh_seed'] = fresh
    ref_shim._import_reference()
    import generativeimage2text.trie_decoder as td
    eos = 2
    seqs = T._toy_trie_sequences(eos)
    trie = []
    for seed in range(4):
        step = T._toy_step(seed=seed)
        dec = td.TrieAutoRegressiveBeamSearch(eos, max_steps=12, beam_size=1, trie=td.TokenTrie.construct(seqs))
        rp, rl = dec.search(torch.tensor([[1]]), step)
        trie.append({'predictions': rp.tolist(), 'logprobs': rl.double().tolist()})
    out['trie_search'] = trie
    _, ref_decoder = ref_shim._import_reference()
    import git_oracle
    steps = 14
    start = torch.tensor([[1]] * 4)
    u = torch.rand((steps, 4), generator=torch.Generator().manual_seed(5))
    sample = {}
    for temperature in (1.0, 0.7):
        runs = []
        for seed in range(3):
            step = T._toy_step(seed=seed)
            dec = ref_decoder.AutoRegressiveBeamSearch(eos, max_steps=steps, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
            calls = {'t': start.shape[1]}

            def fake_multinomial(probs, num_samples):
                t = calls['t']
                calls['t'] += 1
                return git_oracle.inverse_cdf_draw(probs, u[t])[:, None]
            real = torch.multinomial
            torch.multinomial = fake_multinomial
            try:
                rp, rl = dec.search(start, step, do_sample=True, temperature=temperature)
            finally:
                torch.multinomial = real
            runs.append({'predictions': rp.tolist(), 'logprobs': rl.double().tolist()})
        sample[repr(temperature)] = runs
    out['sample_search'] = sample


def tsv_checks(out, tmp):
    import test_tsv_io as T
    ref_shim._import_reference()
    import generativeimage2text.tsv_io as rio
    rows = T._rows(23, 7)
    b = os.path.join(tmp, 'ref.tsv')
    rio.tsv_writer(iter(rows), b)
    t = rio.TSVFile(b)
    reads = {str(i): {'row': list(t[i]), 'key': t.get_key(i)} for i in (0, 22, 9)}
    p1, p2 = os.path.join(tmp, 'p.0.2.tsv'), os.path.join(tmp, 'p.1.2.tsv')
    rio.tsv_writer(iter(rows[:10]), p1)
    rio.tsv_writer(iter(rows[10:]), p2)
    o2 = os.path.join(tmp, 'm_ref.tsv')
    orig = rio.parallel_map
    rio.parallel_map = lambda f, tasks, num_worker=0: [f(x) for x in tasks]
    os.environ['GIT_TMP_FOLDER'] = os.path.join(tmp, 'tmp')
    os.makedirs(os.path.join(os.environ['GIT_TMP_FOLDER'], tmp.lstrip('/')), exist_ok=True)
    try:
        rio.concat_tsv_files([p1, p2], o2)
    finally:
        rio.parallel_map = orig
    out['tsv'] = {'len': len(t), 'files': [file_digest(f) for f in T._files(b)], 'reads': reads,
                  'concat': file_digest(o2), 'concat_lineidx_8b': file_digest(T._files(o2)[2])}


def transform_checks(out):
    from PIL import Image
    import test_preprocess_oracle as T
    import test_inference_host as H
    ref_shim._import_reference()
    import generativeimage2text.inference as rinf
    res = {}
    for key, param in (('default', {}), ('minmax_480_640', {'test_crop_size': 480, 'test_respect_ratio_max': 640})):
        t = rinf.get_image_transform(param)
        per = []
        for hw in [(480, 640), (1000, 300), (200, 200), (300, 1000), (480, 600)]:
            want = t(Image.fromarray(T._img(hw[0], hw[1], 3))).numpy()
            e = {'shape': list(want.shape), 'digest': digest(want)}
            if 'test_respect_ratio_max' in param:
                mm = rinf.MinMaxResizeForTest(param['test_crop_size'], param['test_respect_ratio_max'])
                e['minmax_size'] = list(mm.get_size((hw[1], hw[0])))
            per.append(e)
        res[key] = per
    out['image_transform'] = res
    mm = {}
    for mn, mx in [(480, 640), (420, 560), (224, 224)]:
        a = rinf.MinMaxResizeForTest(mn, mx)
        mm['%d_%d' % (mn, mx)] = {'sizes': [list(a.get_size((w, h))) for h, w in H.SHAPES], 'repr': repr(a)}
    out['minmax_resize'] = mm


def loader_checks(out):
    import test_torch_common as T
    from generativeimage2text_b200.synthetic import synthetic_state_dict
    ref_shim._import_reference()
    import generativeimage2text.torch_common as rtc
    param = {'num_image_with_embedding': 6}
    ckpt, _ = T._messy_checkpoint(param)
    ref = ref_shim.load_reference_model(param, 'stock')
    ref.load_state_dict(synthetic_state_dict(param, 11, 'init'), strict=False)
    rtc.load_state_dict(ref, ckpt)
    rsd = ref.state_dict()
    out['loader'] = {'keys': list(rsd.keys()), 'digests': [digest(v) for v in rsd.values()]}
    pos = {}
    for patch, width, after in [(16, 768, 480), (14, 1024, 420), (16, 768, 160)]:
        g = 224 // patch
        pe = torch.randn(g * g + 1, width, generator=torch.Generator().manual_seed(5))
        a = rtc.resize_2d_pos_embed(pe, 224, patch, after)
        a3 = rtc.resize_2d_pos_embed(pe[None], 224, patch, after)
        pos['%d_%d_%d' % (patch, width, after)] = {'shape': list(a.shape), 'digest': digest(a), 'digest_batched': digest(a3)}
    out['resize_2d_pos_embed'] = pos


def main():
    import tempfile
    if not ref_shim.reference_available():
        raise SystemExit('the original code is not importable at %s (set GIT_REFERENCE_ROOT)' % ref_shim.REFERENCE_ROOT)
    out = {}
    oracle_checks(out)
    with tempfile.TemporaryDirectory() as tmp:
        tsv_checks(out, tmp)
    transform_checks(out)
    loader_checks(out)
    with open(OUT, 'w') as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write('\n')
    print('%s: %d bytes' % (OUT, os.path.getsize(OUT)))


if __name__ == '__main__':
    main()
