"""
Unaligned BAM output of `simulate --bam` (SAM specification v1.6 §4.2), built and compressed on the GPUs.

The file is the BAM header in a BGZF member of its own, then the record stream: one unaligned record per read the FASTQ
would hold, in the same order (csrc/bb_bam_out.cuh), compressed in members of BGZF_CHUNK bytes at fixed offsets of the
record stream (a deflate block per seq and qual field, bgzf_k_compress_bam in csrc/bb_bgzf.cuh), then the end-of-file
member.  So the bytes depend neither on the batch size nor on the number of GPUs.

With one GPU the records are built on the device from the batch's output buffers and compressed there, the rest of the
stream carried on the device from batch to batch: the bases and qualities cross PCIe only as compressed members.  With
several GPUs each builds the records of its own reads; they are copied back, merged in read-index order, and their whole
chunks dealt out over the GPUs in contiguous runs, as BGZFWriter does for FASTQ.
"""
import struct

import numpy as np

from ._lib import BB_BGZF_CHUNK as BGZF_CHUNK
from .bgzf import EOF_MEMBER, chunk_runs
from .engine import run_each
from .planner import bam_layout_sharded
from .version import __version__


def header_bytes():
    """The uncompressed BAM header: magic, @HD and @PG lines (no CL field, so that the bytes do not depend on the command
    line), no reference sequences."""
    text = (f'@HD\tVN:1.6\tSO:unknown\n@PG\tID:badread\tPN:badread\tVN:{__version__}\n').encode()
    return b'BAM\x01' + struct.pack('<i', len(text)) + text + struct.pack('<i', 0)


class BAMWriter(object):
    """Writes the BAM file of a simulation to the binary stream `out`: the header member now, the records of every batch
    (write_batch), then the rest of the stream and the end-of-file member (close)."""

    def __init__(self, engines, out):
        self.engines = list(engines)
        self.out = out
        self.stream_len = 0                            # bytes of the record stream laid out so far
        self.tail = b''                                # multi-GPU: the bytes after the last whole chunk ...
        self.tail_fields = np.zeros((0, 2), np.int64)  # ... and the seq / qual fields in them
        members, _ = self.engines[0].bam_compress(header_bytes(), 0, np.zeros((0, 2), np.int64), final=True)
        self.out.write(members)

    def write_batch(self, planned, results, bases_so_far, target_bases):
        """The records of a finished batch (planned[g], results[g] of GPU g; results from Engine.run_batch_results) for
        the reads that FASTQ output would emit.  Returns (records, bases) emitted."""
        lay = bam_layout_sharded(planned, results, 0, bases_so_far, target_bases, self.stream_len)
        if len(self.engines) == 1:
            eng = self.engines[0]
            eng.bam_build(lay.recs, lay.text)
            self.out.write(eng.bam_compress_device(final=False))
        else:
            base = self.stream_len
            merged = np.empty(lay.stream_len, np.uint8)

            def build(g):
                mine = lay.shard == g
                if mine.any():
                    self.engines[g].bam_build(lay.recs[mine], lay.text)
                    self.engines[g].bam_fetch_records(merged, lay.stream_off[mine] - base)

            run_each(len(self.engines), build)
            self._write_host(merged, lay.fields)
        self.stream_len += lay.stream_len
        return lay.n_emitted, lay.bases

    def _write_host(self, records, fields):
        """Whole chunks of the merged record stream, dealt out over the engines in contiguous runs; the rest is carried."""
        base = self.stream_len - len(self.tail)   # stream offset of the tail's first byte
        data = np.concatenate([np.frombuffer(self.tail, np.uint8), records]) if self.tail else records
        fields = np.concatenate([self.tail_fields, fields]) if len(self.tail_fields) else fields
        n_chunks = len(data) // BGZF_CHUNK
        runs = chunk_runs(n_chunks, len(self.engines))
        parts = [None] * len(runs)

        def work(k):
            a, b = runs[k]
            if b > a:
                parts[k] = bytes(self.engines[k].bam_compress(data[a:b], base + a, fields)[0])

        run_each(len(runs), work)
        for p in parts:
            if p:
                self.out.write(p)
        end = n_chunks * BGZF_CHUNK
        self.tail = data[end:].tobytes()
        self.tail_fields = fields[fields[:, 0] > base + end] if len(fields) else fields

    def close(self):
        """Compresses the rest of the record stream and ends the file with the end-of-file member."""
        if len(self.engines) == 1:
            self.out.write(self.engines[0].bam_compress_device(final=True))
        elif self.tail:
            base = self.stream_len - len(self.tail)
            self.out.write(self.engines[0].bam_compress(self.tail, base, self.tail_fields, final=True)[0])
            self.tail = b''
        self.out.write(EOF_MEMBER)
