"""Builds the in-tree CUDA library (libgitb200.so) with nvcc for sm_90a (H100).

nvcc cross-compiles without a GPU, so the library can be built on a machine without one; it is a build product
(git-ignored) next to this file.
"""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libgitb200.so')
SOURCES = ['gitb200.cu']
HEADER = os.path.join(HERE, '..', 'include', 'gitb200.h')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC', '-shared']


def _nvcc():
    for c in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if c and os.path.exists(c):
            return c
    raise RuntimeError('nvcc not found: libgitb200.so cannot be built (there is no CPU implementation)')


def deps():
    """Every file the library is compiled from: all of csrc/ (sources and the headers they include) and the C header."""
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [HEADER]


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in deps())


def build(force=False, verbose=False):
    """Compile csrc/*.cu -> libgitb200.so (no-op when up to date). Returns the library path."""
    if not force and not is_stale():
        return LIB
    flags = list(NVCC_FLAGS)
    if os.environ.get('GITB200_TIMELINE'):      # debug build with the in-situ decode-step timeline (tools/step_timeline2.py)
        flags.append('-DGITB200_TIMELINE')
    cmd = [_nvcc()] + flags + [os.path.join(CSRC, s) for s in SOURCES] + ['-o', LIB]
    if verbose:
        cmd.insert(1, '-Xptxas=-v')
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed:\n%s\n%s' % (' '.join(cmd), r.stderr[-4000:]))
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == '__main__':
    print(build(force=True, verbose=True))
