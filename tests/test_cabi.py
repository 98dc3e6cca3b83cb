"""CPU: the C-ABI library builds, loads, and exports exactly the symbols include/gitb200.h declares
(no compute calls -- there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, 'include', 'gitb200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(gitb200_[a-z0-9_]+)\s*\(', src)))


def test_library_builds_and_exports_declared_symbols():
    from generativeimage2text_b200 import build, _lib
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    names = _declared()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), 'missing export %s' % n
    assert sorted(_lib.SIGNATURES) == names, 'ctypes binding and header disagree'
    assert _lib.load().gitb200_abi_version() == _lib.ABI_VERSION


def test_struct_layouts_match_header():
    from generativeimage2text_b200 import _lib
    assert ctypes.sizeof(_lib.Config) == 14 * 4
    assert ctypes.sizeof(_lib.Search) == 5 * 4
    assert ctypes.sizeof(_lib.GemmDesc) == 9 * 8 + 6 * 8 + 12 * 4    # gitb200_gemm_desc: pointers, int64, int32


def test_no_cpu_fallback():
    """Without a CUDA device the product path must fail loudly, never compute on the CPU."""
    import torch
    from generativeimage2text_b200.model import get_git_model, AutoRegressiveBeamSearch

    class Tok:
        cls_token_id, sep_token_id = 101, 102
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    m = get_git_model(Tok(), {}).eval()
    m.decoder = AutoRegressiveBeamSearch(102, max_steps=8, beam_size=1, per_node_beam_size=1, fix_missing_prefix=True)
    with pytest.raises(RuntimeError):
        m({'image': torch.zeros(1, 3, 224, 224)})
    h = ctypes.c_void_p()
    rc = _lib_create(h)
    assert rc != 0


def _lib_create(h):
    from generativeimage2text_b200 import _lib
    from generativeimage2text_b200.model import get_git_model

    class Tok:
        cls_token_id, sep_token_id = 101, 102
    cfg = get_git_model(Tok(), {})._cfg
    return _lib.load().gitb200_create(ctypes.byref(cfg), 0, ctypes.byref(h))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, 'generativeimage2text_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py'):
            src = open(os.path.join(pkg, fn)).read()
            assert 'git_oracle' not in src and 'ref_shim' not in src and 'import oracle' not in src, fn
