"""CPU: host side of ragged batches (a list of [3, H_b, W_b] images of their own sizes in one call) -- input validation,
what the model packs and hands to the C ABI (through a stub library), the TSV driver's batching for respect-ratio models
(with a stand-in model), and the reference goldens of one reference call per image against the CPU oracle."""
import ctypes
import json

import numpy as np
import pytest
import torch

import git_oracle
from helpers import load_golden
from generativeimage2text_b200 import model as M
from generativeimage2text_b200 import _lib

EOS = 102
RATIO = {'test_crop_size': 160, 'test_respect_ratio_max': 224}
HWS = [(160, 208), (208, 160), (160, 160), (160, 224)]


class Tok:
    cls_token_id, sep_token_id = 101, 102

    def __call__(self, text, **kw):
        return {'input_ids': [1000 + len(w) for w in text.split()]}

    def decode(self, ids, skip_special_tokens=True):
        return ' '.join(str(i) for i in ids if not (skip_special_tokens and i in (0, 101, 102)))


def _imgs(hws):
    return [torch.full((3, h, w), float(b)) for b, (h, w) in enumerate(hws)]


def test_image_batch_reads_lists_of_3d_images_as_ragged_and_frames_keep_their_meaning():
    m = M.get_git_model(Tok(), RATIO)
    assert m._image_batch(_imgs(HWS)).sizes == HWS
    video = m._image_batch([torch.zeros(2, 3, 16, 16), torch.zeros(2, 3, 16, 16)])   # video frames
    assert video.sizes is None and (video.B, video.frames) == (2, 2)
    bare = m._image_batch(torch.zeros(2, 3, 16, 16))
    assert bare.sizes is None and (bare.B, bare.frames) == (2, 0)
    with pytest.raises(ValueError, match='mixed'):
        m._image_batch([torch.zeros(3, 16, 16), torch.zeros(1, 3, 16, 16)])


def test_image_batch_ragged_validation_errors():
    m = M.get_git_model(Tok(), RATIO)
    with pytest.raises(ValueError, match=r'\[3, H, W\]'):
        m._image_batch([torch.zeros(3, 32, 32), torch.zeros(4, 32, 32)])
    with pytest.raises(ValueError, match='smaller than one patch'):
        m._image_batch([torch.zeros(3, 32, 32), torch.zeros(3, 15, 64)])


def test_image_batch_packing_offsets_token_counts_and_size_array():
    m = M.get_git_model(Tok(), RATIO)
    imgs = _imgs(HWS)
    img = m._image_batch(imgs)
    x = img.x
    assert img.B == 4 and img.frames == 0 and img.sizes == HWS
    assert x.dim() == 1 and x.dtype == torch.float32 and x.numel() == sum(3 * h * w for h, w in HWS)
    off = 0
    for b, (h, w) in enumerate(HWS):                       # image b: [3, h, w] back to back after the ones before it
        assert torch.equal(x[off:off + 3 * h * w].view(3, h, w), imgs[b])
        off += 3 * h * w
    assert img.tokens == [131, 131, 101, 141]                 # grids 10x13, 13x10, 10x10, 10x14 + the class token
    stub = _StubLib()
    m._set_image_sizes(stub, 'eng', img)
    [(name, (eng, arr, n))] = stub.calls
    assert name == 'gitb200_set_image_sizes' and eng == 'eng'
    assert n == 4 and list(arr) == [160, 208, 208, 160, 160, 160, 160, 224]


class _StubLib:
    """Records the ABI calls of one `submit`; every call succeeds."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn


class _Stream:
    cuda_stream = 0


def test_submit_hands_sizes_and_packed_pixels_to_the_abi(monkeypatch):
    m = M.get_git_model(Tok(), RATIO).eval()
    m.decoder = M.GeneratorWithBeamSearch(EOS, max_steps=6, beam_size=4, length_penalty=0.6)
    stub = _StubLib()
    monkeypatch.setattr(m, '_ensure_engine', lambda slot=0: (stub, None))
    monkeypatch.setattr(_lib, 'load', lambda: stub)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda dev=None: _Stream())
    m._slots[0]['engine'] = ctypes.c_void_p(1)
    try:
        _check_submit(m, stub)
    finally:
        m._slots[0]['engine'] = None          # a stub handle: nothing for the real library to destroy


def _check_submit(m, stub):
    imgs = _imgs(HWS)
    m({'image': imgs})
    names = [c[0] for c in stub.calls]
    assert 'gitb200_set_input_size' not in names
    assert names.index('gitb200_set_image_sizes') < names.index('gitb200_generate_async')
    _, (eng, arr, n) = stub.calls[names.index('gitb200_set_image_sizes')]
    assert n == 4 and list(arr) == [v for hw in HWS for v in hw]
    _, gen = stub.calls[names.index('gitb200_generate_async')]
    assert gen[2] == 4 and gen[3] == 0                         # batch = number of images, frames = 0 (no temporal embedding)
    # a uniform batch keeps its one-size call
    stub.calls.clear()
    m({'image': torch.zeros(2, 3, 160, 208)})
    names = [c[0] for c in stub.calls]
    assert 'gitb200_set_input_size' in names and 'gitb200_set_image_sizes' not in names


def test_coalesced_submit_launches_a_ragged_batch_on_its_own(monkeypatch):
    m = M.get_git_model(Tok(), RATIO).eval()
    seen = []
    monkeypatch.setattr(m, '_submit_coalesced', lambda *a, **k: seen.append('coalesced'))
    monkeypatch.setattr(m, '_ensure_engine', lambda slot=0: (_ for _ in ()).throw(RuntimeError('engine')))
    with pytest.raises(RuntimeError, match='engine'):
        m.submit({'image': _imgs(HWS)}, coalesce=4)
    assert seen == []
    m.submit({'image': torch.zeros(2, 3, 160, 160)}, coalesce=4)
    assert seen == ['coalesced']


# ---- the TSV driver with a stand-in model ------------------------------------------------------------------------------
class _FakeTransform:
    """ImageTransform stand-in: a 'decoded image' is (h, w, id); the result carries the id in its pixels."""
    minmax = object()

    def batch(self, imgs):
        return [torch.full((1, 3, h, w), float(i)) for h, w, i in imgs]

    def __call__(self, img):
        return self.batch([img])[0][0]


class _FakeModel:
    """Returns, per row, [image id, prefix tokens...]: what was sent where is visible in the output."""

    def __init__(self):
        self.calls = []
        self.decoder = M.GeneratorWithBeamSearch(EOS, max_steps=20, beam_size=4, length_penalty=0.6)

    def eval(self):
        return self

    def cuda(self):
        return self

    def _rows(self, batch):
        image = batch['image']
        if isinstance(image, list):
            ids = [int(im[0, 0, 0]) if im.dim() == 3 else int(im[0, 0, 0, 0]) for im in image]
        else:
            ids = [int(v) for v in image[:, 0, 0, 0]]
        self.calls.append((type(image).__name__, len(ids)))
        out = []
        for r, i in enumerate(ids):
            if 'prefix_len' in batch:
                pre = batch['prefix'][r, :int(batch['prefix_len'][r])].tolist()
            elif 'prefix' in batch:
                pre = batch['prefix'][0].tolist()
            else:
                pre = []
            out.append([500 + i] + pre[1:])
        w = max(len(o) for o in out)
        return {'predictions': torch.tensor([o + [EOS] * (w - len(o)) for o in out])}

    def __call__(self, batch):
        return self._rows(batch)

    def submit(self, batch, depth=2):
        out = self._rows(batch)

        class H:
            def result(self):
                return out
        return H()


def _run_tsv(tmp_path, monkeypatch, bs, questions):
    from generativeimage2text_b200 import inference as inf
    from generativeimage2text_b200.tsv_io import tsv_writer
    shapes = [(300, 200), (200, 300), (250, 250), (180, 400), (400, 260)]
    tsv_writer([('k%d' % i, '%d,%d,%d' % (h, w, i)) for i, (h, w) in enumerate(shapes)], str(tmp_path / 'img.tsv'))
    qtsv = None
    if questions:
        qtsv = str(tmp_path / 'q.tsv')
        tsv_writer([('k%d' % i, json.dumps([{'question': 'a ' * (i + 1), 'question_id': 10 * i + j} for j in range(1 + i % 2)]))
                    for i in range(len(shapes))], qtsv)
    monkeypatch.setattr(inf, 'get_image_transform', lambda param, device=None: _FakeTransform())
    monkeypatch.setattr(inf, 'pilimg_from_base64', lambda s: tuple(int(v) for v in (s.decode() if isinstance(s, bytes) else s).split(',')))
    monkeypatch.setattr(torch.cuda, 'set_device', lambda *a: None)
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    fm = _FakeModel()
    out = str(tmp_path / ('out%d.tsv' % bs))
    inf.test_git_inference_single_tsv(str(tmp_path / 'img.tsv'), 'x', qtsv, out, tokenizer=Tok(), param=RATIO,
                                      batch_size=bs, model=fm)
    return open(out).read().splitlines(), fm.calls


def test_tsv_captions_of_ratio_models_go_out_in_ragged_batches(tmp_path, monkeypatch):
    lines1, calls1 = _run_tsv(tmp_path, monkeypatch, 1, False)
    lines3, calls3 = _run_tsv(tmp_path, monkeypatch, 3, False)
    assert calls1 == [('Tensor', 1)] * 5                         # batch_size=1: today's one-image calls
    assert calls3 == [('list', 3), ('list', 2)]                   # ragged lists of batch_size images
    assert lines1 == lines3
    assert [json.loads(l.split('\t')[1])[0]['caption'] for l in lines3] == ['500', '501', '502', '503', '504']
    assert [l.split('\t')[0] for l in lines3] == ['k0', 'k1', 'k2', 'k3', 'k4']


def test_tsv_questions_of_ratio_models_go_out_with_their_images(tmp_path, monkeypatch):
    lines1, calls1 = _run_tsv(tmp_path, monkeypatch, 1, True)
    lines2, calls2 = _run_tsv(tmp_path, monkeypatch, 2, True)
    # batch_size=1: today's calls -- one call per question for a single question, one call per image for several
    assert calls1 == [('Tensor', 1), ('Tensor', 2), ('Tensor', 1), ('Tensor', 2), ('Tensor', 1)]
    assert calls2 == [('list', 3), ('list', 3), ('list', 1)]      # images 0+1, 2+3, 4 with all their questions
    want = []
    for i in range(5):
        for j in range(1 + i % 2):
            want.append({'answer': ' '.join(['%d' % (500 + i)] + ['1001'] * (i + 1)), 'question_id': 10 * i + j})
    assert [json.loads(l) for l in lines2] == want
    assert [json.loads(l) for l in lines1] == want


# ---- reference goldens of one reference call per image -----------------------------------------------------------------
@pytest.mark.parametrize('name', ['base_ragged_greedy', 'base_ragged_beam'])
def test_oracle_reproduces_the_ragged_goldens(name):
    from generativeimage2text_b200.synthetic import synthetic_state_dict, synthetic_images
    g = load_golden(name)
    meta = g['meta']
    assert [tuple(hw) for hw in meta['image_hws']] == HWS
    sd = synthetic_state_dict(meta['param'], meta['seed'], meta['variant'])
    cols = torch.from_numpy(g['vocab_cols'])
    for b, hw in enumerate(meta['image_hws']):
        image = synthetic_images(1, 0, meta['img_seed'] + b, hw)
        trace = []
        out = git_oracle.generate(sd, meta['param'], {'image': image}, meta['search'], meta['max_steps'], cached=True,
                                  raw_trace=trace)
        assert np.array_equal(out['predictions'].numpy(), g['predictions_%d' % b]), (name, b)
        np.testing.assert_allclose(out['logprobs'].numpy().reshape(-1), g['logprobs_%d' % b].reshape(-1), rtol=0, atol=1e-4)
        if meta['search'] == 'greedy':
            for i, z in enumerate(trace):
                np.testing.assert_allclose(z[:, cols].numpy(), g['step_logits_%d' % b][i], rtol=0, atol=1e-3)
