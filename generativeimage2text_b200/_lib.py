"""ctypes binding of libgitb200.so (include/gitb200.h).  Fails loudly when the library is missing or does
not export the declared symbols: there is no CPU or PyTorch fallback for the hot path."""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libgitb200.so')
ABI_VERSION = 12

c_void_p, c_int, c_int64, c_float, c_char_p = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_char_p
c_ll = ctypes.c_longlong


class Config(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        'image_size', 'patch', 'enc_width', 'enc_layers', 'enc_heads', 'dec_hidden', 'dec_layers', 'dec_heads',
        'dec_ffn', 'vocab', 'max_positions', 'num_frames_emb', 'sos_id', 'eos_id')]


class Search(ctypes.Structure):
    _fields_ = [('mode', ctypes.c_int32), ('max_steps', ctypes.c_int32), ('beam_size', ctypes.c_int32),
                ('per_node_beam', ctypes.c_int32), ('length_penalty', ctypes.c_float)]


class ImageDesc(ctypes.Structure):
    _fields_ = [('src_offset', ctypes.c_int64), ('src_h', ctypes.c_int32), ('src_w', ctypes.c_int32),
                ('resize_h', ctypes.c_int32), ('resize_w', ctypes.c_int32), ('crop_top', ctypes.c_int32),
                ('crop_left', ctypes.c_int32), ('out_h', ctypes.c_int32), ('out_w', ctypes.c_int32),
                ('dst_offset', ctypes.c_int64)]


class GemmDesc(ctypes.Structure):
    """gitb200_gemm_desc: one launch of the GEMM kernel as its launcher sees it (gitb200_op_gemm_ex)."""
    _fields_ = ([('a', c_void_p), ('b', c_void_p), ('bias', c_void_p), ('resid', c_void_p), ('out', c_void_p * 3),
                 ('lse_target', c_void_p), ('skip', c_void_p)] +
                [(n, ctypes.c_int64) for n in ('lda', 'ldb', 'ld_resid', 'ldo', 'batch_stride', 'split_stride')] +
                [(n, ctypes.c_int32) for n in ('M', 'N', 'K', 'act', 'out_bf16', 'split3', 'transposed', 'k_splits', 'bn',
                                               'seg_n', 'rows_per_batch', 'row_offset')])


SEARCH_GREEDY, SEARCH_BEAM = 0, 1
F32, BF16, I64 = 0, 1, 2

# name -> (restype, argtypes); must list every symbol include/gitb200.h declares
SIGNATURES = {
    'gitb200_create': (c_int, [ctypes.POINTER(Config), c_int, ctypes.POINTER(c_void_p)]),
    'gitb200_destroy': (None, [c_void_p]),
    'gitb200_last_error': (c_char_p, [c_void_p]),
    'gitb200_abi_version': (c_int, []),
    'gitb200_set_weight': (c_int, [c_void_p, c_char_p, c_void_p, ctypes.POINTER(c_int64), c_int, c_int, c_void_p]),
    'gitb200_finalize_weights': (c_int, [c_void_p, c_void_p]),
    'gitb200_share_weights': (c_int, [c_void_p, c_void_p]),
    'gitb200_set_input_size': (c_int, [c_void_p, c_int, c_int]),
    'gitb200_set_image_sizes': (c_int, [c_void_p, ctypes.POINTER(ctypes.c_int32), c_int]),
    'gitb200_encode': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'gitb200_prefill': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'gitb200_decode_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'gitb200_generate': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, ctypes.POINTER(Search), c_void_p,
                                 c_void_p, c_void_p, ctypes.POINTER(ctypes.c_int32), c_void_p, c_void_p]),
    'gitb200_generate_host': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, ctypes.POINTER(Search),
                                      c_void_p, c_void_p, ctypes.POINTER(ctypes.c_int32), c_void_p]),
    'gitb200_generate_async': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, ctypes.POINTER(Search), c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    'gitb200_generate_host_async': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, ctypes.POINTER(Search),
                                            c_void_p, c_void_p, c_void_p]),
    'gitb200_generate_finish': (c_int, [c_void_p, ctypes.POINTER(ctypes.c_int32)]),
    'gitb200_last_decode_ms': (c_int, [c_void_p, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
    'gitb200_set_row_prefixes': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    'gitb200_set_trie': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int]),
    'gitb200_set_sampling': (c_int, [c_void_p, c_void_p, c_int, c_int, c_float]),
    'gitb200_set_beam_sampling': (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_float]),
    'gitb200_set_sequences_per_image': (c_int, [c_void_p, c_int]),
    'gitb200_launch_count': (c_int64, [c_void_p]),
    'gitb200_set_option': (c_int, [c_void_p, c_char_p, c_int64]),
    'gitb200_preproc_create': (c_int, [c_int, ctypes.POINTER(c_void_p)]),
    'gitb200_preproc_destroy': (None, [c_void_p]),
    'gitb200_preproc_last_error': (c_char_p, [c_void_p]),
    'gitb200_preproc_launch_count': (c_int64, [c_void_p]),
    'gitb200_preproc_set_option': (c_int, [c_void_p, c_char_p, c_int64]),
    'gitb200_preproc_run': (c_int, [c_void_p, c_void_p, c_int64, c_int, ctypes.POINTER(ImageDesc), c_int,
                                    ctypes.POINTER(c_float), ctypes.POINTER(c_float), c_void_p, c_int64, c_void_p]),
    'gitb200_preproc_coeffs': (c_int, [c_int, c_int, ctypes.POINTER(ctypes.c_int32), c_void_p, c_void_p, c_int]),
    'gitb200_debug_timeline': (c_int, [c_int, c_void_p, c_int]),
    'gitb200_debug_read': (c_ll, [c_void_p, c_char_p, c_void_p, c_ll]),
    'gitb200_op_gemm': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                c_int, c_int, c_int, c_void_p]),
    'gitb200_op_layernorm': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p,
                                     c_int, c_int, c_void_p]),
    'gitb200_op_gemm_ex': (c_int, [ctypes.POINTER(GemmDesc), ctypes.POINTER(c_int), c_void_p]),
    'gitb200_op_layernorm_ex': (c_int, [c_void_p, c_int, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p,
                                        c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_int,
                                        c_void_p]),
    'gitb200_op_lse_combine': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    'gitb200_op_attention': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_ll,
                                     c_ll, c_ll, c_void_p]),
    'gitb200_op_attention_ex': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll,
                                        c_ll, c_ll, c_ll, ctypes.POINTER(ctypes.c_int32), c_int, c_void_p]),
    'gitb200_score': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                               c_void_p, c_void_p]),
    'gitb200_op_text_attention': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                          c_int, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32), c_int, c_int,
                                          c_void_p]),
    'gitb200_op_decode_attention': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_int, c_int, c_int, ctypes.POINTER(ctypes.c_int32), c_int, c_int,
                                            c_int, c_int, c_int, c_void_p]),
    'gitb200_op_beam_sample': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_float, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
}

_lib = None


def load():
    """dlopen libgitb200.so and bind every declared entry point."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'libgitb200.so is not built (%s). Run `python -c "import __graft_entry__ as g; g.build()"` or '
            '`python -m generativeimage2text_b200.build`; the GIT hot path has no CPU fallback.' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError = missing export
        fn.restype = res
        fn.argtypes = args
    got = lib.gitb200_abi_version()
    if got != ABI_VERSION:
        raise RuntimeError('libgitb200.so ABI %d != binding ABI %d: rebuild the library' % (got, ABI_VERSION))
    _lib = lib
    return lib


def last_error(handle=None):
    msg = load().gitb200_last_error(handle)
    return msg.decode() if msg else ''


def check(rc, handle=None, what=''):
    if rc != 0:
        raise RuntimeError('gitb200 %s failed: %s' % (what, last_error(handle)))
