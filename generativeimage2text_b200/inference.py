"""The callers either side of the hot path -- host-side mirror of the reference's `generativeimage2text/inference.py`
(same function / class names and argument meaning; SURVEY.md section 8f-2/3):

  * `get_image_transform(param)` / `MinMaxResizeForTest` (reference inference.py:29-64, 111-132): the size rules are
    host arithmetic on two integers; the pixels (bicubic resize with Pillow's antialiasing, crop, /255, CLIP
    normalisation) are produced on the GPU by libgitb200.so (`gitb200_preproc_run`), bit-identical to the reference's
    PIL / torchvision pipeline.  There is no CPU transform: without a CUDA device the call raises.
  * `test_git_inference_single_image` (inference.py:67-109) and `test_git_inference_single_tsv` (:134-225), the latter
    batched: rows are decoded by a thread pool, transformed on the GPU `batch_size` at a time and captioned with
    several batches in flight (`model.submit`), where the reference runs batch 1 (:201-212).  Output rows are the
    reference's: `key \\t json([{'caption': ...}])`, or `json({'answer', 'question_id'})` on the question path.
    Multi-GPU: the reference's rank slicing (:152-169); the parts are merged by one gather when `torch.distributed` is
    initialised, else by the reference's part files + concat (:213-225).
"""
import base64
import ctypes
import io
import json
import logging
import os
import os.path as op
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib
from .sharding import get_mpi_rank, get_mpi_size, get_mpi_local_rank, shard_range
from .tsv_io import TSVFile, tsv_writer, tsv_reader, concat_tsv_files

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)     # reference inference.py:125-128
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def json_dump(obj):
    """reference common.py:223-226."""
    return json.dumps(obj, sort_keys=True, separators=(',', ':'))


def pilimg_from_base64(imagestring):
    """reference common.py:213-221 (None when the payload does not decode)."""
    try:
        from PIL import Image
        return Image.open(io.BytesIO(base64.b64decode(imagestring))).convert('RGB')
    except Exception:
        return None


def load_image_by_pil(file_name):
    """reference process_image.py:4-13."""
    from PIL import Image
    if isinstance(file_name, bytes):
        return Image.open(io.BytesIO(file_name)).convert('RGB')
    return Image.open(file_name).convert('RGB')


def load_from_yaml_file(file_name):
    import yaml
    with open(file_name, 'r') as fp:
        data = yaml.safe_load(fp)
    while isinstance(data, dict) and '_base_' in data:       # reference tsv_io.py:97-107: per-path merge into the base
        base = load_from_yaml_file(op.join(op.dirname(file_name), data.pop('_base_')))
        assert isinstance(base, dict)
        _merge_paths(base, data)
        data = base
    return data or {}


def _merge_paths(base, child):
    """Every leaf path of `child` overrides the same path of `base` (nested dicts are merged, not replaced; lists and
    scalars are leaves) -- what the reference's get_all_path / dict_update_path_value loop does (tsv_io.py:102-106)."""
    for k, v in child.items():
        if isinstance(v, dict) and isinstance(base.get(k), dict):
            _merge_paths(base[k], v)
        else:
            base[k] = v


class MinMaxResizeForTest(object):
    """Size rule of reference inference.py:29-64: the shorter edge goes to `min_size` unless the longer edge would pass
    `max_size`; aspect ratio kept (truncating division)."""

    def __init__(self, min_size, max_size):
        self.min_size = min_size
        self.max_size = max_size

    def get_size(self, image_size):
        """(width, height) of the decoded image -> (out_h, out_w)."""
        w, h = image_size
        short, long_ = float(min(w, h)), float(max(w, h))
        target = self.min_size
        if long_ / short * target > self.max_size:            # the longer edge would overshoot: shrink the target
            target = int(round(self.max_size * short / long_))
        if min(w, h) == target:                               # already there: no resampling at all
            return (h, w)
        if w < h:
            return (int(target * h / w), target)
        return (target, int(target * w / h))

    def __repr__(self):
        return 'MinMaxResizeForTest({}, {})'.format(self.min_size, self.max_size)


def _as_rgb_array(img):
    """PIL image / uint8 HWC array / uint8 HWC tensor -> contiguous uint8 [H, W, 3] numpy array."""
    if isinstance(img, torch.Tensor):
        img = img.cpu().numpy()
    if not isinstance(img, np.ndarray):
        img = np.asarray(img.convert('RGB'))
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('expected a decoded RGB image (uint8 [H, W, 3]); got %s %s' % (img.dtype, img.shape))
    return np.ascontiguousarray(img)


class ImageTransform(object):
    """`get_image_transform(param)`: callable on one decoded image like the reference's `Compose`, but the result is a
    CUDA tensor (the reference's callers do `.cuda()` next, a no-op then); `batch()` transforms many images per call."""

    def __init__(self, param, device=None):
        param = param or {}
        self.crop_size = param.get('test_crop_size', 224)
        self.respect_ratio_max = param.get('test_respect_ratio_max')
        # the reference tests `'test_respect_ratio_max' in param` (inference.py:113), not the value's truthiness
        self.minmax = MinMaxResizeForTest(self.crop_size, self.respect_ratio_max) if 'test_respect_ratio_max' in param else None
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None and torch.cuda.is_available() \
            else (torch.device(device) if device is not None else None)
        self._handle = None
        self._mean = (ctypes.c_float * 3)(*CLIP_MEAN)
        self._std = (ctypes.c_float * 3)(*CLIP_STD)
        self._stage = None
        self._copied = None          # event: the previous batch's bytes have left the pinned staging buffer

    # -- size rules (host) -------------------------------------------------------------------------------------
    def geometry(self, h, w):
        """-> (resize_h, resize_w, crop_top, crop_left, out_h, out_w) for a decoded h x w image."""
        if self.minmax is not None:
            oh, ow = self.minmax.get_size((w, h))
            return oh, ow, 0, 0, oh, ow
        s = self.crop_size
        # torchvision Resize(int): shorter edge -> s, longer edge -> int(s * long / short)
        short, long_ = (w, h) if w <= h else (h, w)
        new_long = int(s * long_ / short)
        rh, rw = (new_long, s) if w <= h else (s, new_long)
        # torchvision CenterCrop(s)
        top, left = int(round((rh - s) / 2.0)), int(round((rw - s) / 2.0))
        return rh, rw, top, left, s, s

    # -- pixels (GPU) ------------------------------------------------------------------------------------------
    def _ensure(self):
        if self.device is None or self.device.type != 'cuda':
            raise RuntimeError('the image transform runs on CUDA devices only (libgitb200.so, sm_90a); there is no CPU path')
        if self._handle is None:
            h = ctypes.c_void_p()
            lib = _lib.load()
            if lib.gitb200_preproc_create(self.device.index or 0, ctypes.byref(h)) != 0:
                raise RuntimeError('gitb200_preproc_create failed: %s' % (lib.gitb200_preproc_last_error(None) or b'').decode())
            self._handle = h
        return _lib.load()

    def batch(self, imgs):
        """Decoded images -> fp32 CUDA tensor [B, 3, S, S] (fixed crop) or, with `test_respect_ratio_max`, a list of
        [1, 3, oh, ow] tensors (sizes differ per image)."""
        lib = self._ensure()
        arrs = [_as_rgb_array(im) for im in imgs]
        n = len(arrs)
        if n == 0:
            raise ValueError('empty batch')
        descs = (_lib.ImageDesc * n)()
        src_bytes = 0
        out_elems = 0
        geo = []
        for i, a in enumerate(arrs):
            h, w = a.shape[:2]
            rh, rw, top, left, oh, ow = self.geometry(h, w)
            descs[i] = _lib.ImageDesc(src_bytes, h, w, rh, rw, top, left, oh, ow, out_elems)
            geo.append((oh, ow, out_elems))
            src_bytes += (a.size + 15) // 16 * 16
            out_elems += 3 * oh * ow
        if self._copied is not None:
            self._copied.synchronize()
        if self._stage is None or self._stage.numel() < src_bytes:
            self._stage = torch.empty(max(src_bytes, 1 << 20), dtype=torch.uint8).pin_memory()
        stage = self._stage.numpy()
        for i, a in enumerate(arrs):
            stage[descs[i].src_offset:descs[i].src_offset + a.size] = a.reshape(-1)
        out = torch.empty(out_elems, dtype=torch.float32, device=self.device)
        stream = torch.cuda.current_stream(self.device)
        rc = lib.gitb200_preproc_run(self._handle, self._stage.data_ptr(), src_bytes, 1, descs, n, self._mean, self._std,
                                     out.data_ptr(), out_elems, stream.cuda_stream)
        if rc != 0:
            raise RuntimeError('gitb200_preproc_run failed: %s' % lib.gitb200_preproc_last_error(self._handle).decode())
        if self._copied is None:
            self._copied = torch.cuda.Event()
        self._copied.record(stream)
        if self.minmax is None:
            return out.view(n, 3, self.crop_size, self.crop_size)
        return [out[off:off + 3 * oh * ow].view(1, 3, oh, ow) for oh, ow, off in geo]

    def __call__(self, img):
        r = self.batch([img])
        return r[0] if self.minmax is None else r[0][0]

    def launch_count(self):
        return int(_lib.load().gitb200_preproc_launch_count(self._handle)) if self._handle is not None else 0

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.load().gitb200_preproc_destroy(self._handle)
                self._handle = None
        except Exception:
            pass


def get_image_transform(param, device=None):
    """reference inference.py:111-132."""
    return ImageTransform(param, device)


def _default_tokenizer():
    from transformers import BertTokenizer
    return BertTokenizer.from_pretrained('bert-base-uncased', do_lower_case=True)


def _prefix_ids(tokenizer, prefix, max_text_len=40):
    """reference inference.py:92-101."""
    enc = tokenizer(prefix, padding='do_not_pad', truncation=True, add_special_tokens=False, max_length=max_text_len)
    payload = enc['input_ids']
    if len(payload) > max_text_len - 2:
        payload = payload[-(max_text_len - 2):]
    return [tokenizer.cls_token_id] + payload


def _build_model(model_name, param, tokenizer, checkpoint):
    from .model import get_git_model
    from .torch_common import torch_load, load_state_dict
    model = get_git_model(tokenizer, param)
    if checkpoint is None:
        checkpoint = torch_load(f'output/{model_name}/snapshot/model.pt')['model']
    elif isinstance(checkpoint, str):
        checkpoint = torch_load(checkpoint)['model']
    load_state_dict(model, checkpoint)
    return model


def test_git_inference_single_image(image_path, model_name, prefix, tokenizer=None, checkpoint=None, param=None):
    """reference inference.py:67-109.  `tokenizer` / `checkpoint` (a state dict or a path) / `param` default to what
    the reference loads (bert-base-uncased, output/{model}/snapshot/model.pt, aux_data/models/{model}/parameter.yaml)."""
    if param is None:
        param = {}
        if op.isfile(f'aux_data/models/{model_name}/parameter.yaml'):
            param = load_from_yaml_file(f'aux_data/models/{model_name}/parameter.yaml')
    tokenizer = tokenizer or _default_tokenizer()
    if isinstance(image_path, str):
        image_path = [image_path]
    img = [load_image_by_pil(i) if isinstance(i, (str, bytes)) else i for i in image_path]
    transforms = get_image_transform(param)
    model = _build_model(model_name, param, tokenizer, checkpoint)
    model.cuda()
    model.eval()
    img = [transforms(i).unsqueeze(0).cuda() for i in img]
    input_ids = _prefix_ids(tokenizer, prefix)
    with torch.no_grad():
        result = model({'image': img, 'prefix': torch.tensor(input_ids).unsqueeze(0).cuda()})
    cap = tokenizer.decode(result['predictions'][0].tolist(), skip_special_tokens=True)
    logging.info('output: {}'.format(cap))
    return cap


def write_rows_sharded(rows, out_tsv, rank=None, world_size=None, poll_s=0.2):
    """Write this rank's prediction rows and merge the ranks' parts into `out_tsv` (row order = rank order, as the
    rows were sharded by `shard_range`).  Returns the number of rows this rank produced.

    * one process: rows go straight to `out_tsv` (reference inference.py:163-164, 212);
    * `torch.distributed` initialised: ONE gather of the finished rows to rank 0, which writes `out_tsv`;
    * ranks without a process group (plain mpirun, as the reference is launched): the reference's scheme
      (inference.py:159-162, 213-225) -- every rank writes `{out_tsv}.{rank}.{world}.tsv`, rank 0 waits for all parts
      and concatenates them -- except that a part appears under its final name only once complete."""
    rank = get_mpi_rank() if rank is None else rank
    world_size = get_mpi_size() if world_size is None else world_size
    if world_size <= 1:
        n = 0

        def counted():
            nonlocal n
            for r in rows:
                n += 1
                yield r
        tsv_writer(counted(), out_tsv)
        return n
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        mine = list(rows)
        gathered = [None] * world_size if rank == 0 else None
        torch.distributed.gather_object(mine, gathered, dst=0)
        if rank == 0:
            tsv_writer((r for part in gathered for r in part), out_tsv)
        return len(mine)

    def part(r):
        return '{}.{}.{}.tsv'.format(out_tsv, r, world_size)
    n = 0

    def counted():
        nonlocal n
        for r in rows:
            n += 1
            yield r
    tmp = part(rank)[:-4] + '.partial.tsv'
    tsv_writer(counted(), tmp)
    for ext in ('.lineidx', '.lineidx.8b', '.tsv'):      # the .tsv last: it is what rank 0 polls for
        os.replace(op.splitext(tmp)[0] + ext, op.splitext(part(rank))[0] + ext)
    if rank == 0:
        parts = [part(i) for i in range(world_size)]
        while True:
            not_ready = [t for t in parts if not op.isfile(t)]
            if not not_ready:
                break
            logging.info('waiting {}'.format(','.join(not_ready)))
            time.sleep(poll_s)
        concat_tsv_files(parts, out_tsv)
    return n


def test_git_inference_single_tsv(image_tsv, model_name, question_tsv, out_tsv, tokenizer=None, checkpoint=None,
                                  param=None, batch_size=64, depth=4, decode_workers=8, model=None):
    """reference inference.py:134-225, batched (see module docstring).  Returns the number of rows this rank wrote."""
    if param is None:
        param = {}
        if op.isfile(f'output/{model_name}/parameter.yaml'):
            param = load_from_yaml_file(f'output/{model_name}/parameter.yaml')
    tokenizer = tokenizer or _default_tokenizer()
    image_tsv = TSVFile(image_tsv)
    question_tsv = TSVFile(question_tsv) if question_tsv else None
    torch.cuda.set_device(get_mpi_local_rank())
    transforms = get_image_transform(param)
    if model is None:
        model = _build_model(model_name, param, tokenizer, checkpoint)
    model.eval()
    model.cuda()

    rank, world_size = get_mpi_rank(), get_mpi_size()

    curr_start, curr_end = shard_range(len(image_tsv), rank, world_size)
    pool = ThreadPoolExecutor(max_workers=max(1, decode_workers))

    def decode_row(i):
        key, col = image_tsv[i][:2]
        img = pilimg_from_base64(col)
        if img is None:     # the reference crashes inside its transform on such a row (inference.py:204); name the row
            raise ValueError('row %d (key %r) of the image tsv does not decode to an image' % (i, key))
        return key, img

    def caption_rows():
        """Batches of decoded rows -> GPU transform -> model.submit with `depth` batches in flight.  With
        `test_respect_ratio_max` every image has its own size: batches of more than one image go out as ragged lists."""
        variable = transforms.minmax is not None
        bs = max(1, batch_size)
        pending = []

        def drain(item):
            keys, handle = item
            preds = handle.result()['predictions'].tolist()
            for key, p in zip(keys, preds):
                yield key, json_dump([{'caption': tokenizer.decode(p, skip_special_tokens=True)}])
        idx = list(range(curr_start, curr_end))
        for b0 in range(0, len(idx), bs):
            rows = list(pool.map(decode_row, idx[b0:b0 + bs]))
            keys = [k for k, _ in rows]
            t = transforms.batch([im for _, im in rows])
            x = t if not variable else (t[0] if bs == 1 else [im[0] for im in t])
            pending.append((keys, model.submit({'image': x}, depth=depth)))
            if len(pending) >= depth:
                yield from drain(pending.pop(0))
        while pending:
            yield from drain(pending.pop(0))

    def question_rows_ragged(group):
        """Up to `group` consecutive images with all their questions in ONE ragged call: the image repeated once per
        question, one prefix per row (as the per-image question batch below)."""
        idx = list(range(curr_start, curr_end))
        for b0 in range(0, len(idx), group):
            images, questions, ids = [], [], []
            for i in idx[b0:b0 + group]:
                image_key, image_col = image_tsv[i][:2]
                q_key, q_info = question_tsv[i][:2]
                assert image_key == q_key
                img = transforms(pilimg_from_base64(image_col))
                for q in json.loads(q_info):
                    images.append(img)
                    questions.append(q)
                    ids.append(_prefix_ids(tokenizer, q['question']))
            if not ids:
                continue
            with torch.no_grad():
                if len(ids) == 1:
                    result = model({'image': images, 'prefix': torch.tensor(ids[0]).unsqueeze(0).cuda()})
                else:
                    width = max(len(i) for i in ids)
                    pad = torch.zeros((len(ids), width), dtype=torch.long)
                    for r, i in enumerate(ids):
                        pad[r, :len(i)] = torch.tensor(i)
                    result = model({'image': images, 'prefix': pad.cuda(), 'prefix_len': torch.tensor([len(i) for i in ids])})
            for q, p in zip(questions, result['predictions'].tolist()):
                answer = tokenizer.decode(p, skip_special_tokens=True)
                yield json_dump({'answer': answer, 'question_id': q['question_id']}),

    def question_rows():
        if transforms.minmax is not None and batch_size > 1:
            yield from question_rows_ragged(batch_size)
            return
        for i in range(curr_start, curr_end):
            image_key, image_col = image_tsv[i][:2]
            q_key, q_info = question_tsv[i][:2]
            assert image_key == q_key
            img = transforms(pilimg_from_base64(image_col)).unsqueeze(0)
            questions = json.loads(q_info)
            ids = [_prefix_ids(tokenizer, q['question']) for q in questions]
            if len(questions) > 1 and max(len(i) for i in ids) < model.decoder.max_steps:
                # all questions of an image in ONE call (one prefix per row; the reference loops with batch 1,
                # inference.py:201-212): each row is generated exactly as its own batch-1 call would be
                width = max(len(i) for i in ids)
                pad = torch.zeros((len(ids), width), dtype=torch.long)
                for r, i in enumerate(ids):
                    pad[r, :len(i)] = torch.tensor(i)
                with torch.no_grad():
                    result = model({'image': img.expand(len(ids), -1, -1, -1), 'prefix': pad.cuda(),
                                    'prefix_len': torch.tensor([len(i) for i in ids])})
                preds = result['predictions'].tolist()
            else:
                preds = []
                for input_ids in ids:
                    with torch.no_grad():
                        result = model({'image': img, 'prefix': torch.tensor(input_ids).unsqueeze(0).cuda()})
                    preds.append(result['predictions'][0].tolist())
            for q, p in zip(questions, preds):
                answer = tokenizer.decode(p, skip_special_tokens=True)
                yield json_dump({'answer': answer, 'question_id': q['question_id']}),

    gen_rows = question_rows if question_tsv else caption_rows
    with torch.no_grad():
        n_rows = write_rows_sharded(gen_rows(), out_tsv, rank, world_size)
    pool.shutdown()
    return n_rows


def convert_tsv_to_vqa_json(predict_file, out_json):
    """reference inference.py:227-229."""
    result = [json.loads(s) for s, in tsv_reader(predict_file)]
    with open(out_json, 'w') as fp:
        fp.write(json_dump(result))
