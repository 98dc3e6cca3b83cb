"""Reading tests/golden/reference_checks.json (written by oracle/make_reference_golden.py) and the digests it stores: the
SHA-256 of an array's dtype, shape and bytes, or of a file's bytes."""
import hashlib
import json
import os

import numpy as np
import torch

REFERENCE_CHECKS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_checks.json')


def digest(x):
    """SHA-256 of an array's dtype, shape and bytes (C order)."""
    a = x.detach().contiguous().cpu().numpy() if isinstance(x, torch.Tensor) else np.ascontiguousarray(x)
    h = hashlib.sha256()
    h.update(('%s%s' % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return h.hexdigest()


def file_digest(path):
    with open(path, 'rb') as f:
        return hashlib.sha256(f.read()).hexdigest()


def load_reference_checks():
    with open(REFERENCE_CHECKS) as f:
        return json.load(f)
