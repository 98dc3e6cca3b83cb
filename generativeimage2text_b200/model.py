"""Drop-in for the reference's model factory: `get_git_model(tokenizer, param)`
(reference generativeimage2text/model.py:9-61).

The returned `torch.nn.Module` carries parameters under the reference's own state-dict keys (so
`torch_common.load_state_dict`, reference torch_common.py:93-145, and `.cuda()/.eval()` work unchanged) and
its `forward(batch)` accepts the reference's batch dict and returns `{'predictions', 'logprobs'}`
(reference layers/decoder.py:838-877, 977-1011) -- but no PyTorch op touches the hot path: pixels go in,
token ids come out of libgitb200.so (hand-written sm_90a kernels).  PyTorch only owns the parameter
storage, the CUDA stream and the output tensors.
"""
import collections
import ctypes
import numbers
import warnings

import torch
from torch import nn

from . import _lib
from .synthetic import ENCODER_CFG, VOCAB, HIDDEN, DEC_LAYERS, DEC_HEADS, FFN, MAX_POS, state_spec


class AutoRegressiveBeamSearch(object):
    """Search *configuration* mirroring the reference class of the same name (layers/decoder.py:208-222).
    The engine implements its greedy form (beam_size = per_node_beam_size = 1, the reference's
    commented-out greedy decoder, model.py:27-33) on the device."""

    def __init__(self, eos_index, max_steps=50, beam_size=5, per_node_beam_size=2, fix_missing_prefix=False):
        assert fix_missing_prefix, 'should always true'          # reference layers/decoder.py:222
        self._eos_index = eos_index
        self.max_steps = max_steps
        self.beam_size = beam_size
        self.per_node_beam_size = per_node_beam_size or beam_size
        self.fix_missing_prefix = fix_missing_prefix
        if not (self.beam_size == 1 and self.per_node_beam_size == 1):
            raise NotImplementedError(
                'AutoRegressiveBeamSearch is implemented for beam_size=1/per_node_beam_size=1 (greedy); '
                'use GeneratorWithBeamSearch for beam search (the reference default)')


class GeneratorWithBeamSearch(object):
    """Search configuration mirroring reference layers/decoder.py:1056-1081 (the shipped default:
    beam 4, per-node 2, length_penalty 0.6, model.py:34-40); the engine runs beam sizes 2 .. 8 with per-node 2.  The
    constructor takes temperature 1 only; sampled beam search
    (search_param={'do_sample': True, ...}) divides the logits by the `temperature` attribute, the value the reference's
    search reads (layers/decoder.py:1097, 1140-1142), so `decoder.temperature = 0.7` sets it."""

    def __init__(self, eos_index, max_steps, beam_size, per_node_beam_size=2, length_penalty=1,
                 repetition_penalty=1, temperature=1):
        self._eos_index = eos_index
        self.max_steps = max_steps
        self.beam_size = beam_size
        self.per_node_beam_size = per_node_beam_size or beam_size
        self.length_penalty = length_penalty
        self.repetition_penalty = repetition_penalty
        self.temperature = temperature
        assert self.per_node_beam_size > 1
        assert self.length_penalty > 0, "`length_penalty` should be strictely positive."
        assert self.repetition_penalty >= 1.0, "`repetition_penalty` should be >= 1."
        assert self.temperature > 0, "`temperature` should be strictely positive."
        if repetition_penalty != 1:
            raise NotImplementedError('repetition_penalty is not implemented')
        if temperature != 1:
            raise NotImplementedError('temperature is not a constructor argument here: sampled beam search reads the '
                                      'decoder\'s `temperature` attribute (decoder.temperature = T)')


class BeamSampleArgumentError(TypeError, NotImplementedError):
    """Sampled beam search called without an integer top_k.  The reference raises TypeError there (`top_k > 0` with its
    default None, layers/decoder.py:1355); a sampling call this package cannot run raises NotImplementedError.  The error
    is both, so callers written against either keep working."""


def _beam_filter(search_param):
    """(top_k, top_p) of a sampled GeneratorWithBeamSearch call as the engine takes them.  The reference tests `top_k > 0`
    (layers/decoder.py:1355) and `top_p and top_p < 1.0` (:1359): top_k must be an integer (0: no top-k filter), a false
    top_p means no nucleus filter."""
    top_k, top_p = search_param.get('top_k'), search_param.get('top_p')
    if isinstance(top_k, bool) or not isinstance(top_k, int):
        raise BeamSampleArgumentError('sampled beam search needs an integer top_k (0: no top-k filter), got %r' % (top_k,))
    return top_k, (float(top_p) if top_p else 1.0)


class TokenNode(object):
    """Reference trie_decoder.py:220-222."""

    def __init__(self):
        self.children = {}


class TokenTrie(object):
    """Mirror of the reference's vocabulary trie (trie_decoder.py:224-258): same methods; `to_csr()` is what the engine
    takes (include/gitb200.h gitb200_set_trie)."""

    def __init__(self):
        self.root = TokenNode()
        self.curr = self.root

    @classmethod
    def construct(cls, all_tokens):
        ret = cls()
        for ts in all_tokens:
            ret.insert(ts)
        return ret

    def insert(self, tokens):
        cur = self.root
        for t in tokens:
            cur = cur.children.setdefault(int(t), TokenNode())

    def get_valid(self, tokens):
        r = self.root
        for t in tokens:
            r = r.children.get(int(t))
            if r is None:
                return []
        return list(r.children.keys())

    def reset(self):
        self.curr = self.root

    def get_curr_valid(self):
        return list(self.curr.children.keys())

    def move(self, t):
        assert t in self.curr.children
        self.curr = self.curr.children[t]

    def to_csr(self):
        """(child_begin [n_nodes + 1], child_token [n_edges], child_node [n_edges]) as int32 lists; node 0 = root,
        nodes numbered breadth first, a node's edges in insertion order."""
        nodes, begin, tok, child = [self.root], [0], [], []
        index = {id(self.root): 0}
        i = 0
        while i < len(nodes):
            for t, c in nodes[i].children.items():
                if id(c) not in index:
                    index[id(c)] = len(nodes)
                    nodes.append(c)
                tok.append(int(t))
                child.append(index[id(c)])
            begin.append(len(tok))
            i += 1
        return begin, tok, child


class TrieAutoRegressiveBeamSearch(object):
    """Search configuration mirroring reference trie_decoder.py:27-42 (the decoder model.py:42-48 keeps commented out):
    greedy decoding restricted to the token sequences of `trie`.  The reference holds one trie cursor and constrains row 0
    only; the engine gives every row of a batch its own cursor (each row = a batch-1 call of the reference)."""

    def __init__(self, eos_index, max_steps=50, beam_size=5, trie=None):
        self._eos_index = eos_index
        self.max_steps = max_steps
        assert beam_size == 1                                      # reference trie_decoder.py:38
        self.beam_size = beam_size
        self.per_node_beam_size = 1
        self.trie = trie


class _Pending(object):
    """Handle of an enqueued `model(batch)` (see GitB200CaptioningModel.submit)."""

    def __init__(self, model, slot, sp, P, tokens, logprobs, step_logits, keep, row_lens=None):
        self.model, self.slot, self.sp, self.P = model, slot, sp, P
        self.row_lens = row_lens          # per-row prefix lengths (host list) of a prefix batch
        self.tokens, self.logprobs, self.step_logits, self._keep = tokens, logprobs, step_logits, keep
        self._out = None

    def result(self):
        if self._out is None:
            self._out = self.model._finish(self)
            self._keep = None
        return self._out


def greedy_width(pred, eos):
    """Number of columns the reference's greedy loop produces for these rows ALONE: it stops right after the first step
    in which every row holds EOS (layers/decoder.py:316-320); rows that finished earlier are EOS-forced (:347-351), which
    adds 0 to their logprob and nothing to `num_valid` (:433-438), so extra columns never change a row's result."""
    all_eos = (pred == eos).all(dim=0)
    hit = torch.nonzero(all_eos)
    return int(hit[0]) + 1 if hit.numel() else pred.shape[1]


# One call's images as the engine takes them (GitB200CaptioningModel._image_batch): x = the pixels on the device, B images,
# frames (0: a bare tensor), sizes = [(H_b, W_b)] of a ragged batch or None, tokens = image tokens L_b of each image.
_Images = collections.namedtuple('_Images', 'x B frames sizes tokens')


class _Group(object):
    """Batches submitted one by one that share ONE engine launch (dynamic batching): one encoder pass over all their
    images and one decode chain over all their rows.  The decode chain is ~45 latency-bound kernels per step whose
    duration barely depends on the row count, so k batches in one chain cost little more than one."""

    def __init__(self, model, key, depth, want):
        self.model, self.key, self.depth, self.want = model, key, depth, want
        self.images, self.rows = [], []
        self.pending, self.out = None, None

    def add(self, img):
        self.images.append(img)
        self.rows.append(img.B)
        return len(self.rows) - 1

    def launch(self):
        if self.pending is not None or self.out is not None:
            return
        m = self.model
        if m._open_group is self:
            m._open_group = None
        img = self.images[0]
        if len(self.images) > 1:   # along the batch axis: [frames, B, 3, H, W] of several frames, else [B, 3, H, W]
            x = torch.cat([im.x for im in self.images], dim=1 if img.frames > 1 else 0)
            img = img._replace(x=x, B=sum(self.rows), tokens=img.tokens[:1] * sum(self.rows))
        self.images = None
        self.pending = m.submit({'image': img}, depth=self.depth)

    def result(self):
        if self.out is None:
            self.launch()
            self.out = self.pending.result()
            self.pending = None
        return self.out


class _Member(object):
    """Handle of one batch inside a _Group: `.result()` is what `model(batch)` would have returned for it."""

    def __init__(self, group, index):
        self.group, self.index = group, index
        self._out = None

    def result(self):
        if self._out is not None:
            return self._out
        g = self.group
        out = g.result()
        r0 = sum(g.rows[:self.index])
        r1 = r0 + g.rows[self.index]
        pred, lp = out['predictions'][r0:r1], out['logprobs'][r0:r1]
        m = g.model
        if isinstance(m.decoder, AutoRegressiveBeamSearch) and pred.shape[1] > 1 and len(g.rows) > 1:
            if bool((pred[:, 1] == m.eos_index).all()):
                # this batch alone would have taken the reference's empty-caption exit (layers/decoder.py:279-291)
                warnings.warn('Empty captions predicted. You may want to increase beam size or ensure your step '
                              'function is working properly.', RuntimeWarning)
                pred, lp = pred[:, 1:2], lp.reshape(-1)[:, None]
            else:
                pred = pred[:, :greedy_width(pred, m.eos_index)]
        self._out = {'predictions': pred, 'logprobs': lp}
        return self._out


class _Holder(nn.Module):
    """Attribute container so that parameters get the reference's dotted names."""


def _set_path(root, dotted, param):
    parts = dotted.split('.')
    mod = root
    for p in parts[:-1]:
        if not hasattr(mod, p):
            mod.add_module(p, _Holder())
        mod = getattr(mod, p)
    mod.register_parameter(parts[-1], param)


class GitB200CaptioningModel(nn.Module):
    """Parameter shell + engine handle. See module docstring."""

    def __init__(self, tokenizer, param):
        super().__init__()
        self.param = dict(param or {})
        enc_type = self.param.get('image_encoder_type', 'CLIPViT_B_16')
        enc = ENCODER_CFG[enc_type]
        self.image_size = self.param.get('test_crop_size', 224)
        self.num_image_with_embedding = self.param.get('num_image_with_embedding')
        self.sos_index = tokenizer.cls_token_id
        self.eos_index = tokenizer.sep_token_id
        self.tokenizer = tokenizer
        if self.param.get('visual_feature_size', 768) != enc['width']:
            raise ValueError('visual_feature_size must equal the encoder width (grid features are not projected)')
        words = None
        for key, shape, (kind, scale) in state_spec(self.param):
            if kind == 'tied':
                p = words                                         # reference layers/decoder.py:503-505
            else:
                t = torch.empty(shape, dtype=torch.float32)
                if kind == 'normal':
                    t.normal_(0.0, scale)
                elif kind == 'ones':
                    t.fill_(1.0)
                else:
                    t.zero_()
                p = nn.Parameter(t, requires_grad=False)
                if key == 'textual.embedding.words.weight':
                    words = p
            if key.startswith('img_temperal_embedding.'):
                continue
            _set_path(self, key, p)
        n_emb = self.num_image_with_embedding or 0
        if n_emb:
            self.img_temperal_embedding = nn.ParameterList(
                nn.Parameter(torch.zeros(1, 1, enc['width']), requires_grad=False) for _ in range(n_emb))
        # the shipped default decoder (reference model.py:34-40)
        self.decoder = GeneratorWithBeamSearch(eos_index=self.eos_index, max_steps=1024, beam_size=4,
                                               length_penalty=0.6)
        self._cfg = _lib.Config(
            image_size=self.image_size, patch=enc['patch'], enc_width=enc['width'], enc_layers=enc['layers'],
            enc_heads=enc['heads'], dec_hidden=HIDDEN, dec_layers=DEC_LAYERS, dec_heads=DEC_HEADS, dec_ffn=FFN,
            vocab=VOCAB, max_positions=MAX_POS, num_frames_emb=n_emb, sos_id=self.sos_index, eos_id=self.eos_index)
        # engine slots: slot 0 serves `model(batch)`; `submit()` round-robins over `n_slots` engines, each on its own
        # stream, so the encoder of one batch overlaps the latency-bound decode loop of the previous one
        # (all slots share slot 0's device copy of the parameters: gitb200_share_weights)
        import os
        self.n_slots = max(1, min(8, int(os.environ.get('GITB200_SLOTS', '4'))))
        self._options = {}
        self._slots = [dict(engine=None, sig=None, stream=None, pending=None) for _ in range(self.n_slots)]
        self._engine_device = None
        self._next_slot = 0
        self._open_group = None      # batches waiting to be launched together (submit(..., coalesce=k))
        self._param_cache = None

    # ---------------------------------------------------------------- engine plumbing
    def _device(self):
        return self.textual.embedding.words.weight.device

    def _weights_signature(self):
        # (storage address, in-place version) of every parameter; the (name, tensor) list itself is cached and dropped by
        # anything that can re-seat parameters (`_apply`: .cuda()/.to()/.float(); load_state_dict)
        if self._param_cache is None:
            self._param_cache = list(self.state_dict(keep_vars=True).items())
        return tuple((v.data_ptr(), v._version) for _, v in self._param_cache)

    def _apply(self, fn, *args, **kwargs):
        self._param_cache = None
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        self._param_cache = None
        return super().load_state_dict(*args, **kwargs)

    @property
    def _engine(self):
        return self._slots[0]['engine']

    def _ensure_engine(self, slot=0):
        dev = self._device()
        if dev.type != 'cuda':
            raise RuntimeError('the gitb200 engine runs on CUDA devices only (sm_90a); call model.cuda() first. '
                               'There is no CPU path.')
        lib = _lib.load()
        if self._engine_device is not None and self._engine_device != dev:
            self.release()
        self._engine_device = dev
        sl = self._slots[slot]
        stream = torch.cuda.current_stream(dev).cuda_stream
        if sl['engine'] is None:
            h = ctypes.c_void_p()
            _lib.check(lib.gitb200_create(ctypes.byref(self._cfg), dev.index or 0, ctypes.byref(h)), None, 'create')
            sl['engine'], sl['sig'], sl['trie_key'] = h, None, None
            import os
            for opt in ('use_graph', 'use_pdl', 'use_mega', 'debug_layers', 'parity'):
                v = os.environ.get('GITB200_' + opt.upper())      # debugging switches, e.g. GITB200_USE_MEGA=0
                if v is not None:
                    _lib.check(lib.gitb200_set_option(h, opt.encode(), int(v)), h, 'set_option')
            for opt, v in self._options.items():                  # set_engine_option() calls made so far
                _lib.check(lib.gitb200_set_option(h, opt.encode(), int(v)), h, 'set_option')
        sig = self._weights_signature()
        if slot > 0:
            # one device copy of the parameters: slot 0 owns it, the other slots borrow it
            if self._slots[0]['engine'] is None or self._slots[0]['sig'] != sig:
                self._ensure_engine(0)
            if sl['sig'] is None:
                _lib.check(lib.gitb200_share_weights(sl['engine'], self._slots[0]['engine']), sl['engine'], 'share_weights')
            sl['sig'] = sig
            return lib, stream
        if sig != sl['sig']:
            eng = sl['engine']
            for other in self._slots:         # the slots share this copy: nothing may be in flight while it is rewritten
                if other['pending'] is not None:
                    other['pending'].result()
            if self._param_cache is None:
                self._param_cache = list(self.state_dict(keep_vars=True).items())
            for key, p in self._param_cache:
                t = p.detach()
                if t.dtype != torch.float32 or not t.is_contiguous():
                    t = t.float().contiguous()
                shape = (ctypes.c_int64 * t.dim())(*t.shape)
                _lib.check(lib.gitb200_set_weight(eng, key.encode(), t.data_ptr(), shape, t.dim(), _lib.F32,
                                                  stream), eng, 'set_weight(%s)' % key)
            _lib.check(lib.gitb200_finalize_weights(eng, stream), eng, 'finalize_weights')
            sl['sig'] = sig
        return lib, stream

    def release(self):
        for sl in reversed(self._slots):   # borrowers before the owner of the weights
            if sl['engine'] is not None:
                _lib.load().gitb200_destroy(sl['engine'])
                sl['engine'], sl['sig'], sl['pending'], sl['trie_key'] = None, None, None, None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def set_engine_option(self, name, value):
        """Engine switches (0/1): 'use_graph', 'use_pdl', 'use_mega' (persistent one-kernel decode
        step for greedy batches of <= 64), and 'parity' -- the fp32-grade
        verification mode (every GEMM as a three-term bf16 split product through the same wgmma kernels, fp32
        attention and K/V caches): logits within 1e-3 of the fp32 reference at ~3x the GEMM work."""
        self._options[name] = int(value)
        if name == 'parity':
            self.release()          # operand formats differ: engines are re-created (and weights re-packed) on next use
            return
        for k in range(self.n_slots):
            if k == 0 or self._slots[k]['engine'] is not None:
                lib, _ = self._ensure_engine(k)
                _lib.check(lib.gitb200_set_option(self._slots[k]['engine'], name.encode(), int(value)), self._slots[k]['engine'], 'set_option')

    def last_decode_timing(self):
        """(device ms of the last call's decode loop, step launches in it, whether each was one decode_mega_kernel
        launch) -- CUDA events on the engine's stream (include/gitb200.h gitb200_last_decode_ms); bench.py's roofline."""
        lib = _lib.load()
        ms, steps, one = ctypes.c_float(), ctypes.c_int32(), ctypes.c_int32()
        h = self._slots[0]['engine']
        _lib.check(lib.gitb200_last_decode_ms(h, ctypes.byref(ms), ctypes.byref(steps), ctypes.byref(one)), h, 'last_decode_ms')
        return ms.value, steps.value, bool(one.value)

    def launch_count(self):
        lib = _lib.load()
        return sum(int(lib.gitb200_launch_count(sl['engine'])) for sl in self._slots if sl['engine'] is not None)

    def _search_struct(self):
        d = self.decoder
        if isinstance(d, (AutoRegressiveBeamSearch, TrieAutoRegressiveBeamSearch)):
            return _lib.Search(mode=_lib.SEARCH_GREEDY, max_steps=d.max_steps, beam_size=1, per_node_beam=1,
                               length_penalty=1.0)
        if isinstance(d, GeneratorWithBeamSearch):
            return _lib.Search(mode=_lib.SEARCH_BEAM, max_steps=d.max_steps, beam_size=d.beam_size,
                               per_node_beam=d.per_node_beam_size, length_penalty=float(d.length_penalty))
        raise TypeError('model.decoder must be an AutoRegressiveBeamSearch, TrieAutoRegressiveBeamSearch or GeneratorWithBeamSearch '
                        'of this package')

    def _image_batch(self, image):
        """Checks one call's 'image' argument and puts its pixels on the device as the engine reads them -> _Images.
        A list of [3, H_b, W_b] tensors is a ragged batch (B single images of their own sizes, back to back), a list of
        [B, 3, H, W] tensors is video frames ([frames, B, 3, H, W]) and a bare [B, 3, H, W] tensor has frames = 0 (no
        temporal embedding)."""
        p = ENCODER_CFG[self.param.get('image_encoder_type', 'CLIPViT_B_16')]['patch']
        dev = self._device()

        def to_dev(t):
            return t.to(device=dev, dtype=torch.float32, non_blocking=True)
        frames = 0
        if isinstance(image, (list, tuple)):
            if not image:
                raise ValueError('an image list must not be empty')
            dims = [im.dim() for im in image]
            if 3 in dims and any(n != 3 for n in dims):
                raise ValueError('a ragged batch is a list of [3, H, W] images; it cannot be mixed with [B, 3, H, W] frames')
            if dims[0] == 3:
                sizes = []
                for b, im in enumerate(image):
                    if im.shape[0] != 3:
                        raise ValueError('image %d of a ragged batch must be [3, H, W] (got %s)' % (b, tuple(im.shape)))
                    if im.shape[1] < p or im.shape[2] < p:
                        raise ValueError('image %d (%s) is smaller than one patch' % (b, tuple(im.shape[1:])))
                    sizes.append((int(im.shape[1]), int(im.shape[2])))
                x = torch.cat([to_dev(im).reshape(-1) for im in image])
                return _Images(x, len(sizes), 0, sizes, [(h // p) * (w // p) + 1 for h, w in sizes])
            frames = len(image)
            ims = [to_dev(im) for im in image]
            if any(im.shape != ims[0].shape for im in ims):
                raise ValueError('all frames of a batch must share one size')
            x = ims[0].contiguous() if frames == 1 else torch.stack(ims, dim=0).contiguous()
        else:
            x = to_dev(image).contiguous()
        if x.dim() != (4 if frames <= 1 else 5) or x.shape[-3] != 3:
            raise ValueError('images must be [B, 3, H, W] tensors (got %s)' % (tuple(x.shape),))
        H, W = int(x.shape[-2]), int(x.shape[-1])
        if H < p or W < p:
            raise ValueError('input %s is smaller than one patch' % ((H, W),))
        B = int(x.shape[-4])
        return _Images(x, B, frames, None, [(H // p) * (W // p) + 1] * B)

    @staticmethod
    def _set_image_sizes(lib, eng, img):
        """Hands the sizes of `img` to engine `eng`: every image's own size for the next call only, or the one size of
        them all (sticky; inputs of another size than test_crop_size, reference inference.py:29-64, get the positional
        embedding re-sampled to their patch grid, reference layers/CLIP/model.py:245-251)."""
        if img.sizes is None:
            _lib.check(lib.gitb200_set_input_size(eng, int(img.x.shape[-2]), int(img.x.shape[-1])), eng, 'set_input_size')
        else:
            hw = (ctypes.c_int32 * (2 * img.B))(*[v for s in img.sizes for v in s])
            _lib.check(lib.gitb200_set_image_sizes(eng, hw, img.B), eng, 'set_image_sizes')

    # ---------------------------------------------------------------- the reference surface
    @torch.no_grad()
    def forward(self, batch, forced_tokens=None, return_step_logits=False, search_param=None):
        """`model(batch)` of the reference in eval mode: CaptioningModel.forward -> infer.

        batch: {'image': FloatTensor[B,3,H,W] | [FloatTensor[B,3,H,W]] * frames, 'prefix'?: LongTensor[1,P]}
               (extension: 'prefix': LongTensor[B,P] + optional 'prefix_len': [B] = one prefix per image;
               extension: 'image': [FloatTensor[3,H_b,W_b]] * B = B single images of their own sizes (ragged batch): row b is
               what `model({'image': image[b][None]})` returns, no temporal embedding)
        forced_tokens / return_step_logits are parity-test hooks (teacher forcing, raw per-step logits).
        search_param: the dict CaptioningModel.infer forwards to decoder.search (layers/decoder.py:999-1003); understood:
               {'do_sample': True, 'temperature': T, 'top_k': ., 'top_p': .} with the greedy decoder -- top_k / top_p are
               accepted and ignored exactly like the reference (its filter call is commented out, :372) -- plus
               'uniforms': FloatTensor[max_steps, B] or 'generator': torch.Generator for the random numbers;
               {'do_sample': True, 'top_k': int, 'top_p': .} with GeneratorWithBeamSearch (the temperature is the
               decoder's `temperature` attribute; num_keep_best only 1) plus 'uniforms': FloatTensor[max_steps,
               B * beam_size, 2] or 'generator';
               'num_return_sequences': n (an int >= 1, every decoder): B images give B * n sequences in image-major order
               (row b * n + i belongs to image b; per-image prefixes apply to all n), each searching on its own, and every
               B above counts sequences: 'uniforms' [max_steps, B * n] (beam: [max_steps, B * n * beam_size, 2]),
               forced_tokens [B * n, max_steps], predictions / logprobs / step_logits B * n (* beam) rows.  Each image is
               encoded and its K/V cached once; the result is bit for bit that of the call with every image repeated n
               times (greedy without sampling: with use_mega 0, since n > 1 runs on the kernel chain).
        """
        return self.submit(batch, forced_tokens, return_step_logits, slot=0, _caller_stream=True,
                           search_param=search_param).result()

    @torch.no_grad()
    def submit(self, batch, forced_tokens=None, return_step_logits=False, slot=None, depth=2, _caller_stream=False,
               coalesce=1, search_param=None):
        """Enqueue `model(batch)` without waiting: returns a handle whose `.result()` gives the reference's output
        dict.  Successive submits rotate over `depth` engines / streams (each engine: one call in flight).

        coalesce = k > 1 (dynamic batching): k successive batches of one shape are launched as ONE engine call -- one
        encoder pass, one decode chain over all their rows -- as soon as the k-th arrives or a result is asked for; every
        handle still returns exactly its own batch's reference output (greedy width and empty-caption exit included)."""
        if self.training:
            raise NotImplementedError('training (loss / SCST branches) is out of scope: call model.eval()')
        if 'image' not in batch:
            raise NotImplementedError("batch without 'image' is not supported")
        if 'context' in batch:
            raise NotImplementedError("'context' batches are not produced by the reference inference path")
        search_param = dict(search_param or {})
        n_seq = _sequences_per_image(search_param.pop('num_return_sequences', 1))
        constrained = bool(search_param) or isinstance(self.decoder, TrieAutoRegressiveBeamSearch)
        image = batch['image']
        # (copies / casts, if any, run on the caller's stream; a coalesced group hands over its images as one _Images)
        img = image if isinstance(image, _Images) else self._image_batch(image)
        x, B, frames = img.x, img.B, img.frames
        # a ragged batch is launched on its own (never coalesced)
        if (int(coalesce) > 1 and img.sizes is None and slot is None and not _caller_stream and forced_tokens is None and not return_step_logits
                and 'prefix' not in batch and 'prefix_len' not in batch and not constrained and n_seq == 1):
            return self._submit_coalesced(img, depth, int(coalesce))
        if self._open_group is not None:
            self._open_group.launch()         # keep the submission order
        if slot is None:
            depth = max(1, min(int(depth), self.n_slots))
            slot = self._next_slot % depth
            self._next_slot = (slot + 1) % depth
        sl = self._slots[slot]
        if sl['pending'] is not None:
            sl['pending'].result()
        lib, _ = self._ensure_engine(slot)
        eng = sl['engine']
        dev = self._device()
        cur = torch.cuda.current_stream(dev)
        if _caller_stream:
            stream = cur                      # synchronous path: the caller's stream (stream 0 -> engine-owned stream)
        else:
            # every slot on its own stream: work submitted earlier on the caller's stream must not order the batches in
            # flight behind each other (only the inputs' producer is waited for)
            if sl['stream'] is None:
                sl['stream'] = torch.cuda.Stream(device=dev)
            stream = sl['stream']
            stream.wait_stream(cur)           # inputs produced on the caller's stream
        sp = self._search_struct()
        prefix, P = None, 0
        row_prefix, row_lens_dev, row_lens = None, None, None
        if 'prefix' in batch and B > 1 and len(batch['prefix']) == B:
            # one prefix per image (question batches) -- beyond the reference, which asserts a single prefix and batch 1
            # (layers/decoder.py:985-989): row r is generated exactly as a batch-1 call with batch['prefix'][r, :len_r]
            row_prefix = batch['prefix'].to(device=dev, dtype=torch.long).contiguous()
            if row_prefix.dim() != 2:
                raise ValueError("a per-image 'prefix' must be a [B, P] tensor")
            if 'prefix_len' in batch:
                row_lens = [int(v) for v in batch['prefix_len']]
            else:
                row_lens = [row_prefix.shape[1]] * B
            if len(row_lens) != B or min(row_lens) < 1 or max(row_lens) > row_prefix.shape[1] or max(row_lens) >= sp.max_steps:
                raise ValueError("'prefix_len' must hold B lengths in [1, P] below the decoder's max_steps")
            if forced_tokens is not None:
                raise ValueError('teacher forcing is not available for per-image prefixes')
            if n_seq > 1:           # every sequence of image b starts from image b's prefix
                row_prefix = row_prefix.repeat_interleave(n_seq, 0)
                row_lens = [n for n in row_lens for _ in range(n_seq)]
            row_lens_dev = torch.tensor(row_lens, dtype=torch.int32, device=dev)
        elif 'prefix' in batch:
            assert len(batch['prefix']) == 1, 'not supported'      # reference layers/decoder.py:988
            if B != 1:
                raise AssertionError('not supported: one shared prefix needs batch size 1 (pass a [B, P] prefix for one per image)')
            prefix = batch['prefix'].to(device=dev, dtype=torch.long).contiguous().view(-1)
            P = prefix.numel()
        S = B * n_seq                         # sequences: row b * n_seq + i belongs to image b
        tokens = torch.empty((S, sp.max_steps), dtype=torch.long, device=dev)
        logprobs = torch.empty((S,), dtype=torch.float32, device=dev)
        forced = None
        if forced_tokens is not None:
            forced = forced_tokens.to(device=dev, dtype=torch.long).contiguous()
            assert tuple(forced.shape) == (S, sp.max_steps)
        step_logits = None
        if return_step_logits:
            rows = S * (sp.beam_size if sp.mode == _lib.SEARCH_BEAM else 1)
            step_logits = torch.zeros((sp.max_steps - max(P, 1), rows, VOCAB), dtype=torch.float32, device=dev)
        uniforms = self._sampling_setup(search_param, sp, S, dev)
        for t in (x, prefix, forced, row_prefix, row_lens_dev, uniforms):
            if t is not None and stream is not cur:
                t.record_stream(stream)
        self._set_image_sizes(lib, eng, img)
        if row_prefix is not None:
            _lib.check(lib.gitb200_set_row_prefixes(eng, row_prefix.data_ptr(), S, int(row_prefix.shape[1]), row_lens_dev.data_ptr()),
                       eng, 'set_row_prefixes')
        self._trie_setup(lib, sl)
        if uniforms is not None and sp.mode == _lib.SEARCH_BEAM:
            top_k, top_p = _beam_filter(search_param)
            _lib.check(lib.gitb200_set_beam_sampling(eng, uniforms.data_ptr(), int(uniforms.shape[0]), int(uniforms.shape[1]),
                                                     float(self.decoder.temperature), top_k, top_p), eng, 'set_beam_sampling')
        elif uniforms is not None:
            _lib.check(lib.gitb200_set_sampling(eng, uniforms.data_ptr(), int(uniforms.shape[0]), S,
                                                float(search_param.get('temperature', 1))), eng, 'set_sampling')
        if n_seq > 1:
            _lib.check(lib.gitb200_set_sequences_per_image(eng, n_seq), eng, 'set_sequences_per_image')
        _lib.check(lib.gitb200_generate_async(
            eng, x.data_ptr(), B, frames, prefix.data_ptr() if prefix is not None else None, P,
            ctypes.byref(sp), forced.data_ptr() if forced is not None else None, tokens.data_ptr(),
            logprobs.data_ptr(), step_logits.data_ptr() if step_logits is not None else None,
            stream.cuda_stream), eng, 'generate')
        pend = _Pending(self, slot, sp, P, tokens, logprobs, step_logits, (x, prefix, forced, row_prefix, row_lens_dev, uniforms), row_lens)
        sl['pending'] = pend
        return pend

    # ---------------------------------------------------------------- caption scoring
    def _score_args(self, batch):
        """Host-side checks of a score() batch (before any engine is touched) -> (_Images, B, tokens, need_predict,
        image_index), the last three as CPU tensors."""
        for key in ('context', 'bi_valid_mask_caption'):
            if key in batch:
                raise NotImplementedError("score(): %r batches are not supported" % key)
        for key in ('image', 'caption_tokens', 'need_predict'):
            if key not in batch:
                raise ValueError("score(): batch needs %r" % key)
        img = self._image_batch(batch['image'])
        B = img.B
        tokens = torch.as_tensor(batch['caption_tokens']).detach().cpu()
        need = torch.as_tensor(batch['need_predict']).detach().cpu()
        if tokens.dim() != 2 or tokens.dtype.is_floating_point:
            raise ValueError("score(): 'caption_tokens' must be an integer [N, T] tensor")
        N, T = tokens.shape
        if not 2 <= T <= MAX_POS:
            raise ValueError('score(): T = %d positions; 2 <= T <= %d' % (T, MAX_POS))
        if N < 1:
            raise ValueError('score(): no captions')
        if tuple(need.shape) != (N, T):
            raise ValueError("score(): 'need_predict' is %s, 'caption_tokens' %s" % (tuple(need.shape), (N, T)))
        if bool(((need != 0) & (need != 1)).any()):
            raise ValueError("score(): 'need_predict' must hold 0 / 1")
        if int(tokens.min()) < 0 or int(tokens.max()) >= VOCAB:
            raise ValueError('score(): token ids must lie in [0, %d)' % VOCAB)
        index = batch.get('image_index')
        if index is not None:
            index = torch.as_tensor(index).detach().cpu()
            if tuple(index.shape) != (N,) or index.dtype.is_floating_point:
                raise ValueError("score(): 'image_index' must be an integer [N] tensor")
            if int(index.min()) < 0 or int(index.max()) >= B:
                raise ValueError("score(): 'image_index' must lie in [0, %d)" % B)
        elif N != B:
            raise ValueError("score(): %d captions for %d images need an 'image_index'" % (N, B))
        if not bool(((need[:, 1:] == 1) & (tokens[:, 1:] != 0)).any()):
            raise ValueError('score(): no position to predict (need_predict == 1 with a non-zero target)')
        return img, B, tokens.long(), need.long(), index

    @torch.no_grad()
    def score(self, batch):
        """Teacher-forced scoring of given captions in one pass (the reference's training-branch forward,
        layers/decoder.py:916-972, with dropout off).

        batch: {'image': as for `model(batch)` (tensor, list of frames, or ragged list of [3, H_b, W_b] images),
                'caption_tokens': LongTensor[N, T] (CLS .. SEP, 0-padded), 'need_predict': [N, T] of 0 / 1,
                'image_index'?: LongTensor[N] = the image of each caption (default: caption n, image n)}.
        Returns {'token_logprobs': fp32 [N, T-1] = log_softmax(logits[n, t])[caption_tokens[n, t+1]],
                 'vl_l_loss': fp32 scalar = the reference's SmoothLabelCrossEntropyLoss (eps 0.1) over the positions with
                 need_predict[n, t+1] == 1 and a non-zero target}.
        Captions of one image share its encoder pass.  The arguments are checked on the host (token ids, shapes, indices)."""
        img, _, tokens, need, index = self._score_args(batch)
        N, T = tokens.shape
        lib, _ = self._ensure_engine(0)
        sl = self._slots[0]
        if sl['pending'] is not None:
            sl['pending'].result()
        eng = sl['engine']
        dev = self._device()
        tok_d = tokens.to(dev).contiguous()
        need_d = need.to(dev).contiguous()
        idx_d = index.to(device=dev, dtype=torch.int32).contiguous() if index is not None else None
        lp = torch.empty((N, T - 1), dtype=torch.float32, device=dev)
        loss = torch.empty((1,), dtype=torch.float32, device=dev)
        self._set_image_sizes(lib, eng, img)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gitb200_score(eng, img.x.data_ptr(), img.B, img.frames, tok_d.data_ptr(), need_d.data_ptr(),
                                     idx_d.data_ptr() if idx_d is not None else None, N, T, lp.data_ptr(), loss.data_ptr(),
                                     stream), eng, 'score')
        return {'token_logprobs': lp, 'vl_l_loss': loss[0]}

    def _sampling_setup(self, search_param, sp, B, dev):
        """search_param of the reference's decoder.search (layers/decoder.py:224-232, 1083-1092) -> the uniforms the engine
        draws with (None: a deterministic search).  B counts sequences: submit takes num_return_sequences out first and
        passes B * n (a num_return_sequences above 1 that reaches this point raises)."""
        if not search_param:
            return None
        if isinstance(self.decoder, GeneratorWithBeamSearch):
            return self._beam_sampling_setup(search_param, sp, B, dev)
        unknown = set(search_param) - {'do_sample', 'temperature', 'top_k', 'top_p', 'num_return_sequences', 'uniforms',
                                       'generator', 'only_return_best'}
        if unknown:
            raise TypeError('unknown search_param keys: %s' % sorted(unknown))
        if not isinstance(self.decoder, AutoRegressiveBeamSearch):
            raise NotImplementedError('search_param (sampling) is implemented for AutoRegressiveBeamSearch and '
                                      'GeneratorWithBeamSearch only')
        if search_param.get('num_return_sequences', 1) != 1 or not search_param.get('only_return_best', True):
            raise NotImplementedError('num_return_sequences > 1 / only_return_best=False are not implemented')
        temperature = float(search_param.get('temperature', 1))
        if not search_param.get('do_sample', False):
            assert temperature == 1, 'temperature needs do_sample'         # reference layers/decoder.py:259-261
            return None
        if not temperature > 0:
            raise ValueError('temperature must be positive')
        u = search_param.get('uniforms')
        if u is None:
            u = torch.rand((sp.max_steps, B), dtype=torch.float32, device=dev, generator=search_param.get('generator'))
        u = u.to(device=dev, dtype=torch.float32).contiguous()
        if u.dim() != 2 or u.shape[0] < sp.max_steps or u.shape[1] != B:
            raise ValueError("'uniforms' must be a [>= max_steps, B] tensor")
        return u

    def _beam_sampling_setup(self, search_param, sp, B, dev):
        """GeneratorWithBeamSearch.search(input_ids, step, num_keep_best, do_sample, top_k, top_p, num_return_sequences)
        (reference layers/decoder.py:1083-1092); its temperature is the decoder's `temperature` attribute (:1097).  -> uniforms
        [max_steps, B * beam_size, 2], or None when do_sample is off (top_k / top_p are then unused, as in the reference)."""
        if 'temperature' in search_param:
            raise TypeError("GeneratorWithBeamSearch.search() got an unexpected keyword argument 'temperature' (sampled "
                            "beam search divides by the decoder's `temperature` attribute)")
        unknown = set(search_param) - {'do_sample', 'top_k', 'top_p', 'uniforms', 'generator', 'num_keep_best',
                                       'num_return_sequences'}
        if unknown:
            raise NotImplementedError('search_param keys not implemented for GeneratorWithBeamSearch: %s' % sorted(unknown))
        for key in ('num_keep_best', 'num_return_sequences'):
            if search_param.get(key, 1) != 1:
                raise NotImplementedError('%s > 1 is not implemented' % key)
        if not search_param.get('do_sample', False):
            return None
        _beam_filter(search_param)
        temperature = self.decoder.temperature
        if not (isinstance(temperature, (int, float)) and 0 < temperature < float('inf')):
            raise ValueError('decoder.temperature must be a positive number (got %r)' % (temperature,))
        rows = B * sp.beam_size
        u = search_param.get('uniforms')
        if u is None:
            u = torch.rand((sp.max_steps, rows, 2), dtype=torch.float32, device=dev, generator=search_param.get('generator'))
        u = u.to(device=dev, dtype=torch.float32).contiguous()
        if u.dim() != 3 or u.shape[0] < sp.max_steps or u.shape[1] != rows or u.shape[2] != 2:
            raise ValueError("'uniforms' must be a [>= max_steps, B * beam_size, 2] tensor")
        return u

    def _trie_setup(self, lib, sl):
        """Hand the decoder's trie to the engine (or remove the one it holds) -- once per (engine, trie object)."""
        d = self.decoder
        trie = d.trie if isinstance(d, TrieAutoRegressiveBeamSearch) else None
        key = id(trie) if trie is not None else None
        if sl.get('trie_key') == key:
            return
        eng = sl['engine']
        if trie is None:
            _lib.check(lib.gitb200_set_trie(eng, None, None, None, 0, 0), eng, 'set_trie')
        else:
            begin, tok, child = trie.to_csr()
            arr = lambda v: (ctypes.c_int32 * max(len(v), 1))(*v)
            _lib.check(lib.gitb200_set_trie(eng, arr(begin), arr(tok), arr(child), len(begin) - 1, len(tok)), eng, 'set_trie')
        sl['trie_key'] = key

    def _submit_coalesced(self, img, depth, want):
        key = (img.frames,) + tuple(img.x.shape[-3:]) + (id(self.decoder), depth, want)
        g = self._open_group
        if g is not None and g.key != key:
            g.launch()
            g = None
        if g is None:
            g = self._open_group = _Group(self, key, depth, want)
        member = _Member(g, g.add(img))
        if len(g.rows) >= want:
            g.launch()
        return member

    def _finish(self, pend):
        lib = _lib.load()
        sl = self._slots[pend.slot]
        out_len = ctypes.c_int32(0)
        rc = lib.gitb200_generate_finish(sl['engine'], ctypes.byref(out_len))
        sl['pending'] = None                  # finished either way: the engine takes the next call
        _lib.check(rc, sl['engine'], 'generate_finish')
        sp, P, tokens, logprobs = pend.sp, pend.P, pend.tokens, pend.logprobs
        n = out_len.value
        if pend.row_lens is not None:
            # per-image prefixes: row r = what a batch-1 call with its prefix returns (prefix stripped), EOS-padded to the
            # longest row; greedy width as the reference's loop would leave it for the rows together
            full = tokens[:, :n] if sp.mode == _lib.SEARCH_GREEDY else tokens
            width = full.shape[1] - min(pend.row_lens)
            pred = torch.full((full.shape[0], width), self.eos_index, dtype=torch.long, device=full.device)
            for r, pl in enumerate(pend.row_lens):
                pred[r, :full.shape[1] - pl] = full[r, pl:]
            out = {'predictions': pred, 'logprobs': logprobs if sp.mode == _lib.SEARCH_GREEDY else logprobs[:, None]}
            if pend.step_logits is not None:
                out['step_logits'] = pend.step_logits
            return out
        if sp.mode == _lib.SEARCH_GREEDY:
            if n < 0:   # every first token was EOS (reference layers/decoder.py:279-291)
                warnings.warn('Empty captions predicted. You may want to increase beam size or ensure your step '
                              'function is working properly.', RuntimeWarning)
                pred = tokens[:, max(P, 1):max(P, 1) + 1]
                lp = logprobs[:, None]
            else:
                pred = tokens[:, :n]
                lp = logprobs
                if P:
                    pred = pred[:, P:]                              # reference layers/decoder.py:1004-1006
                if not bool(torch.isfinite(lp).all()):              # reference layers/decoder.py:419-426
                    warnings.warn('Infinite log probs encountered. Some final captions may not make sense. This can '
                                  'happen when the beam size is larger than the number of valid (non-zero probability) '
                                  'transitions that the step function produces.', RuntimeWarning)
        else:
            pred = tokens[:, P:] if P else tokens
            lp = logprobs[:, None]
        out = {'predictions': pred, 'logprobs': lp}
        if pend.step_logits is not None:
            out['step_logits'] = pend.step_logits
        return out

    # ---------------------------------------------------------------- parity hooks (intermediate activations)
    @torch.no_grad()
    def encode_image(self, image):
        """Image features as the decoder sees them: [B, frames*L, d] fp32 (reference layers/decoder.py:846-857); for a ragged
        list of [3, H_b, W_b] images, a list of [1, L_b, d] (image b alone, as `encode_image(image[b][None])` gives it)."""
        lib, stream = self._ensure_engine()
        img = self._image_batch(image)
        if img.sizes is not None:
            M = max(img.tokens)
        else:
            nf = max(img.frames, 1)
            if img.frames and self.num_image_with_embedding:
                nf = min(nf, self.num_image_with_embedding)
            M = nf * img.tokens[0]
        width = ENCODER_CFG[self.param.get('image_encoder_type', 'CLIPViT_B_16')]['width']
        feats = torch.empty((img.B, M, width), dtype=torch.float32, device=img.x.device)
        self._m_tokens = M
        self._set_image_sizes(lib, self._engine, img)
        _lib.check(lib.gitb200_encode(self._engine, img.x.data_ptr(), img.B, img.frames, feats.data_ptr(), stream),
                   self._engine, 'encode')
        if img.sizes is not None:
            return [feats[b:b + 1, :n] for b, n in enumerate(img.tokens)]
        return feats

    @torch.no_grad()
    def prefill(self, batch_size, beam=1):
        """visual_projection output [B, M, 768] fp32 after the last encode_image; fills the image K/V cache."""
        lib, stream = self._ensure_engine()
        out = torch.empty((batch_size, self._m_tokens, HIDDEN), dtype=torch.float32, device=self._device())
        _lib.check(lib.gitb200_prefill(self._engine, batch_size, beam, out.data_ptr(), stream), self._engine, 'prefill')
        return out

    @torch.no_grad()
    def decoding_step(self, tokens, pos, beam_idx=None):
        """Raw last-position logits [rows, V] for one new token per row at text position `pos`."""
        lib, stream = self._ensure_engine()
        tokens = tokens.to(device=self._device(), dtype=torch.long).contiguous()
        rows = tokens.numel()
        logits = torch.empty((rows, VOCAB), dtype=torch.float32, device=self._device())
        bi = None
        if beam_idx is not None:
            bi = beam_idx.to(device=self._device(), dtype=torch.int32).contiguous()
        _lib.check(lib.gitb200_decode_step(self._engine, tokens.data_ptr(), bi.data_ptr() if bi is not None else None,
                                           rows, int(pos), logits.data_ptr(), stream), self._engine, 'decode_step')
        return logits


def _sequences_per_image(n):
    """The num_return_sequences of a search_param (reference layers/decoder.py:229-237, 1091-1096): an int >= 1."""
    if isinstance(n, bool) or not isinstance(n, numbers.Integral) or int(n) < 1:
        raise ValueError('num_return_sequences must be an integer >= 1 (got %r)' % (n,))
    return int(n)


def get_git_model(tokenizer, param):
    """Same signature and `param` keys as reference model.py:9 (`image_encoder_type`, `test_crop_size`,
    `visual_feature_size`, `num_image_with_embedding`); reads only `tokenizer.cls_token_id/sep_token_id`."""
    return GitB200CaptioningModel(tokenizer, param)
