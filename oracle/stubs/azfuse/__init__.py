"""Test-infrastructure stub for the absent `azfuse` package (blob-storage file layer).

Only used by oracle/ref_shim.py so that the reference can be imported offline.
Mirrors the handful of static methods the reference calls (torch_common.py:41-45,
tsv_io.py). Not part of the product."""
import os


class File(object):
    isfile = staticmethod(os.path.isfile)
    open = staticmethod(open)
    get_file_size = staticmethod(os.path.getsize)

    @staticmethod
    def prepare(paths):
        return None

    @staticmethod
    def clear_cache(path):
        return None
