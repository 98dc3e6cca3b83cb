"""TSV container I/O on both sides of the hot path -- host-side mirror of the reference's
`generativeimage2text/tsv_io.py` (SURVEY.md section 8f-3): same class / function names, same on-disk format.

Format (reference tsv_io.py:354-375): `<name>.tsv` holds one row per line, columns separated by TAB; `<name>.lineidx`
holds the byte offset of every row as decimal text, one per line; `<name>.lineidx.8b` holds the same offsets as
little-endian int64.  Image TSVs are `key \\t base64(jpeg)`; prediction TSVs are `key \\t json` (inference.py:212).

Differences in mechanism, not in results: rows are served from one read-only mmap of the .tsv and a numpy view of the
.lineidx.8b (the reference seeks a file handle per access, tsv_io.py:281-293); `concat_tsv_files` shifts the offsets
with numpy instead of a process pool (tsv_io.py:71-96).  No azfuse: plain local files.
"""
import mmap
import os
import os.path as op
import shutil
import threading

import numpy as np


def _lineidx_names(tsv_file):
    base = op.splitext(tsv_file)[0]
    return base + '.lineidx', base + '.lineidx.8b'


def tsv_reader(tsv_file_name, sep='\t'):
    """Rows as lists of stripped columns (reference tsv_io.py:98-101)."""
    with open(tsv_file_name, 'r') as fp:
        for line in fp:
            yield [x.strip() for x in line.split(sep)]


def tsv_writer(values, tsv_file_name, sep='\t'):
    """Write rows + both line indices (reference tsv_io.py:354-375).  Columns may be bytes or anything str()-able."""
    lineidx, lineidx_8b = _lineidx_names(tsv_file_name)
    assert values is not None
    sep = sep.encode()
    idx = 0
    folder = op.dirname(tsv_file_name)
    if folder:
        os.makedirs(folder, exist_ok=True)
    with open(tsv_file_name, 'wb') as fp, open(lineidx, 'w') as fpidx, open(lineidx_8b, 'wb') as fp8b:
        for value in values:
            assert value is not None
            v = sep.join(c if type(c) == bytes else str(c).encode() for c in value) + b'\n'
            fp.write(v)
            fpidx.write(str(idx) + '\n')
            fp8b.write(idx.to_bytes(8, 'little'))
            idx += len(v)


def generate_lineidx(tsv_file):
    """(Re)build `.lineidx` / `.lineidx.8b` for an existing TSV by scanning for newlines."""
    lineidx, lineidx_8b = _lineidx_names(tsv_file)
    size = op.getsize(tsv_file)
    if size == 0:
        offsets = np.zeros((0,), dtype='<i8')
    else:
        chunks = [np.zeros((1,), dtype='<i8')]
        step = 64 << 20                                     # scan 64 MiB at a time: image TSVs run to hundreds of GB
        with open(tsv_file, 'rb') as fp, mmap.mmap(fp.fileno(), 0, access=mmap.ACCESS_READ) as m:
            for lo in range(0, size, step):
                view = np.frombuffer(m, dtype=np.uint8, count=min(step, size - lo), offset=lo)
                chunks.append(np.flatnonzero(view == 10).astype('<i8') + (lo + 1))
                del view
        starts = np.concatenate(chunks)
        offsets = starts[starts < size]
    offsets.astype('<i8').tofile(lineidx_8b)
    with open(lineidx, 'w') as fp:
        fp.write(''.join('%d\n' % o for o in offsets.tolist()))
    return len(offsets)


def concat_files(ins, out):
    with open(out, 'wb') as fp_out:
        for f in ins:
            with open(f, 'rb') as fp_in:
                shutil.copyfileobj(fp_in, fp_out, 1024 * 1024 * 10)


def concat_tsv_files(tsvs, out_tsv):
    """Byte-concatenate TSV parts and rebuild the merged `.lineidx.8b` by shifting each part's offsets by the bytes
    before it (reference tsv_io.py:22-31, 61-96; like the reference, only the 8-byte index is produced)."""
    if len(tsvs) == 1 and tsvs[0] == out_tsv:
        return
    concat_files(tsvs, out_tsv)
    sizes = np.cumsum([0] + [op.getsize(t) for t in tsvs])[:-1]
    parts = []
    for off, t in zip(sizes.tolist(), tsvs):
        parts.append(np.fromfile(_lineidx_names(t)[1], dtype='<i8') + off)
    merged = np.concatenate(parts) if parts else np.zeros((0,), dtype='<i8')
    merged.astype('<i8').tofile(_lineidx_names(out_tsv)[1])


_OPEN_LOCK = threading.Lock()


class TSVFile(object):
    """Random access to the rows of a TSV through its `.lineidx.8b` (reference tsv_io.py:121-352).

    `tsv[i]` -> list of stripped columns of row i; `len(tsv)`; iteration; `get_key(i)`; `seek_first_columns()`.
    `row_bytes(i)` gives the undecoded row (a zero-copy memoryview of the mmap) for the batched loader."""

    def __init__(self, tsv_file, cache_policy=None):
        self.tsv_file = tsv_file
        self.lineidx, self.lineidx_8b = _lineidx_names(tsv_file)
        self.cache_policy = cache_policy
        self._fp = None
        self._mfp = None
        self._offsets = None
        self._size = None
        self.pid = None

    # -- index ---------------------------------------------------------------------------------------------------
    def _ensure_lineidx_loaded(self):
        if self._offsets is None:
            if op.isfile(self.lineidx_8b):
                self._offsets = np.fromfile(self.lineidx_8b, dtype='<i8')
            elif op.isfile(self.lineidx):
                with open(self.lineidx, 'r') as fp:
                    self._offsets = np.asarray([int(x) for x in fp.read().split()], dtype='<i8')
            else:
                raise FileNotFoundError('no line index next to %s (expected %s; generate_lineidx() builds one)'
                                        % (self.tsv_file, self.lineidx_8b))
        return self._offsets

    @property
    def tsv_file_size(self):
        if self._size is None:
            self._size = op.getsize(self.tsv_file)
        return self._size

    def num_rows(self):
        return len(self._ensure_lineidx_loaded())

    def __len__(self):
        return self.num_rows()

    def get_offset(self, idx):
        return int(self._ensure_lineidx_loaded()[idx])

    def get_row_offsets(self, i):
        off = self._ensure_lineidx_loaded()
        n = len(off)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError(i)
        start = int(off[i])
        end = int(off[i + 1]) if i < n - 1 else self.tsv_file_size
        return start, end

    def get_row_len(self, i):
        start, end = self.get_row_offsets(i)
        return end - start

    # -- data ----------------------------------------------------------------------------------------------------
    def _ensure_tsv_opened(self):
        if self._mfp is not None and self.pid == os.getpid():
            return
        # threads of one process (the TSV driver decodes rows on a thread pool) open the file once: without the lock a
        # second opener replaced self._fp and closed the file another thread was about to map
        with _OPEN_LOCK:
            if self._mfp is not None and self.pid != os.getpid():     # forked worker: re-open (reference tsv_io.py:345-350)
                self.close_fp()
            if self._mfp is None:
                fp = open(self.tsv_file, 'rb')
                self._mfp = mmap.mmap(fp.fileno(), 0, access=mmap.ACCESS_READ) if self.tsv_file_size else b''
                self._fp = fp
                self.pid = os.getpid()

    def row_bytes(self, i):
        self._ensure_tsv_opened()
        start, end = self.get_row_offsets(i)
        return memoryview(self._mfp)[start:end]

    def seek(self, idx):
        return [s.strip() for s in bytes(self.row_bytes(idx)).decode().split('\t')]

    def __getitem__(self, index):
        return self.seek(index)

    def seek_first_column(self, idx):
        row = self.row_bytes(idx)
        b = bytes(row[:256])
        cut = b.find(b'\t')
        if cut < 0:
            b = bytes(row)
            cut = b.find(b'\t')
            assert cut >= 0
        return b[:cut].decode()

    def get_key(self, idx):
        return self.seek_first_column(idx)

    def seek_first_columns(self):
        return [self.seek_first_column(i) for i in range(len(self))]

    def __iter__(self):
        for i in range(len(self)):
            yield self.seek(i)

    # -- lifetime ------------------------------------------------------------------------------------------------
    def close_fp(self):
        if self._mfp is not None and not isinstance(self._mfp, bytes):
            try:
                self._mfp.close()
            except BufferError:      # a row_bytes() view is still alive; the map goes with it
                pass
        self._mfp = None
        if self._fp:
            self._fp.close()
            self._fp = None

    def close(self):
        self.close_fp()

    def release(self):
        self.close_fp()
        self._offsets = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def __str__(self):
        return "TSVFile(tsv_file='{}')".format(self.tsv_file)

    __repr__ = __str__
