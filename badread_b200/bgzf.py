"""
BGZF (SAM specification §4.1) on the GPU, both ways.

Output of `simulate --gzip`: FASTQ records compressed on the GPUs (Engine.bgzf_compress, csrc/bb_bgzf.cuh) and written as
BGZF, which gzip, zlib and htslib read.  Members hold BGZF_CHUNK bytes at fixed offsets of the whole FASTQ stream: the
writer carries the tail of every buffer into the next one, so the compressed bytes depend neither on the batch size nor
on the number of GPUs.

Input (`decompress`): a whole BGZF file, BAM for the model builders, inflated on one GPU, one warp per member
(csrc/bb_inflate.cuh).  `gunzip` takes any gzip stream, BGZF or not: one that is not BGZF is decoded in parallel chunks
(csrc/bb_gunzip.cuh).
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import BB_BGZF_CHUNK as BGZF_CHUNK
from .engine import run_each

# the empty member that ends a BGZF file (SAM specification §4.1.2)
EOF_MEMBER = bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')


def decompress(data, device=0):
    """The inflated bytes (a bytearray) of the BGZF stream `data` (bytes-like), inflated on GPU `device`.  Raises ValueError
    with the library's message for input that is not BGZF or a member that is corrupt (named by index and offset)."""
    L = _lib.lib()
    src = np.frombuffer(memoryview(data).cast('B'), dtype=np.uint8)
    src_ptr = src.ctypes.data_as(ctypes.c_void_p) if src.size else None
    n_out = ctypes.c_int64(0)
    rc = L.bb_bgzf_decompress(device, src_ptr, src.size, None, 0, ctypes.byref(n_out))
    out = bytearray(n_out.value)
    if rc == _lib.BB_ERR_CAPACITY:
        rc = L.bb_bgzf_decompress(device, src_ptr, src.size, (ctypes.c_char * len(out)).from_buffer(out), len(out),
                                  ctypes.byref(n_out))
    if rc == _lib.BB_ERR_ARG:
        raise ValueError(L.bb_model_error().decode(errors='replace'))
    if rc != _lib.BB_OK:
        raise RuntimeError('bgzf.decompress: ' + L.bb_model_error().decode(errors='replace'))
    return out


def gunzip(data, device=0, chunk_bytes=0):
    """(the inflated bytes as a bytearray, the stats as a dict) of the gzip stream `data` (bytes-like, any number of
    members, BGZF or not), inflated on GPU `device` (bb_gzip_decompress); chunk_bytes: compressed bytes per chunk, 0 for
    the default.  Raises ValueError with the library's message for a corrupt stream (the member named by index and
    offset)."""
    L = _lib.lib()
    src = np.frombuffer(memoryview(data).cast('B'), dtype=np.uint8)
    src_ptr = src.ctypes.data_as(ctypes.c_void_p) if src.size else None
    n_out, stats = ctypes.c_int64(0), _lib.GzipStats()
    out = bytearray(4 * src.size)   # (a guess: a larger stream is inflated again into the room it asks for)

    def call(buf):
        ptr = (ctypes.c_char * len(buf)).from_buffer(buf) if buf else None
        return L.bb_gzip_decompress(device, src_ptr, src.size, ptr, len(buf), ctypes.byref(n_out), chunk_bytes,
                                    ctypes.byref(stats))
    rc = call(out)
    if rc == _lib.BB_ERR_CAPACITY:
        out = bytearray(n_out.value)
        rc = call(out)
    if rc == _lib.BB_ERR_ARG:
        raise ValueError(L.bb_model_error().decode(errors='replace'))
    if rc != _lib.BB_OK:
        raise RuntimeError('bgzf.gunzip: ' + L.bb_model_error().decode(errors='replace'))
    del out[n_out.value:]
    return out, stats.as_dict()


def chunk_runs(n_chunks, n_engines):
    """Chunks [0, n_chunks) dealt out over at most n_engines in contiguous runs of ceil(n_chunks / runs) chunks (the last
    ones shorter, possibly empty): the byte bounds [(start, end)] of the runs, at least one."""
    n_runs = max(1, min(n_engines, n_chunks))
    per, end = -(-n_chunks // n_runs) * BGZF_CHUNK, n_chunks * BGZF_CHUNK
    return [(min(k * per, end), min((k + 1) * per, end)) for k in range(n_runs)]


def _newlines(buf):
    return int(np.count_nonzero(np.frombuffer(buf, dtype=np.uint8) == 10))


class BGZFWriter(object):
    """Compresses whole FASTQ records with `engines` and writes the members to the binary stream `out` in stream order.
    With several engines the whole chunks of a buffer are dealt out over them in contiguous runs, one host thread each."""

    def __init__(self, engines, out):
        self.engines = list(engines)
        self.out = out
        self.tail = b''        # input after the last whole chunk
        self.tail_mod4 = 0     # index mod 4 of the FASTQ line the tail's first byte belongs to

    def write(self, records):
        """records: a bytes-like object of whole FASTQ records (it starts with a header line and ends with the newline
        of a quality line)."""
        data = memoryview(records).cast('B')
        if len(self.tail) + len(data) < BGZF_CHUNK:
            self.tail += bytes(data)
            return
        mod4 = 0
        if self.tail:   # the chunk that spans the previous buffer's tail and this buffer's head
            need = BGZF_CHUNK - len(self.tail)
            members, _ = self.engines[0].bgzf_compress(self.tail + bytes(data[:need]), self.tail_mod4, final=False)
            self.out.write(members)
            mod4 = _newlines(data[:need]) & 3
            data = data[need:]
        n_chunks = len(data) // BGZF_CHUNK
        parts = self._parts(data, n_chunks, mod4)
        results = [None] * len(parts)

        def work(k):
            results[k] = self.engines[k].bgzf_compress(parts[k][0], parts[k][1], final=False)[0]

        run_each(len(parts), work)
        for members in results:
            self.out.write(members)
        self.tail = bytes(data[n_chunks * BGZF_CHUNK:])
        self.tail_mod4 = -_newlines(self.tail) & 3   # the records end with a quality line: line index 0 mod 4 follows

    def _parts(self, data, n_chunks, mod4):
        """The whole chunks of data as [(slice, line index mod 4 at its start)], one contiguous run per engine."""
        runs = chunk_runs(n_chunks, len(self.engines))
        lines = [0] * len(runs)

        def count(k):   # the newlines of run k come before run k + 1; counted side by side
            lines[k + 1] = _newlines(data[runs[k][0]:runs[k][1]])

        run_each(len(runs) - 1, count)
        return [(data[a:b], (mod4 + sum(lines[:k + 1])) & 3) for k, (a, b) in enumerate(runs)]

    def close(self):
        """Compresses the tail and ends the file with the end-of-file member."""
        if self.tail:
            members, _ = self.engines[0].bgzf_compress(self.tail, self.tail_mod4, final=True)
            self.out.write(members)
            self.tail = b''
        self.out.write(EOF_MEMBER)
