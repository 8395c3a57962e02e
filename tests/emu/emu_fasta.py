"""ctypes front end of tests/emu/emu_fasta.cpp: the FASTA parser's device code under the warp emulator.
TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_fasta.so'


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_fasta.cpp', HERE / 'cuda_emu.h', csrc / 'bb_fasta.cuh']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # 64 threads per tile (two warps: the cross-warp step of the block scan runs) and 16 in the scan CTA (so that
        # its threads take several tiles each on small inputs)
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique',
                        '-DFASTA_THREADS=64', '-DFASTA_SCAN_THREADS=16', '-o', str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
        L.emu_fasta_parse.restype = ctypes.c_int
        L.emu_fasta_parse.argtypes = [ctypes.c_char_p, i64, i32, vp, vp, vp]
        L.emu_fasta_gather.restype = ctypes.c_int
        L.emu_fasta_gather.argtypes = [vp, i64, vp, vp, i32, vp]
        _lib = L
    return _lib


def parse(data, tile):
    """Passes 1 to 3 on the emulator -> (kept bytes as a uint8 array, header starts, ends, kept offsets)."""
    L = lib()
    data = bytes(data)
    totals = np.zeros(2, np.int64)
    rc = L.emu_fasta_parse(data, len(data), int(tile), None, None, totals.ctypes.data)
    if rc:
        raise RuntimeError(f'emu_fasta_parse failed ({rc})')
    kept = np.zeros(max(int(totals[0]), 1), np.uint8)
    hdr = np.zeros(max(3 * int(totals[1]), 1), np.int64)
    rc = L.emu_fasta_parse(data, len(data), int(tile), kept.ctypes.data, hdr.ctypes.data, totals.ctypes.data)
    if rc:
        raise RuntimeError(f'emu_fasta_parse failed ({rc})')
    nh = int(totals[1])
    return kept[:int(totals[0])], hdr[:nh], hdr[nh:2 * nh], hdr[2 * nh:3 * nh]


def gather(src, lo, hi):
    """fasta_k_gather on the emulator: the concatenation of src[lo[r]:hi[r]]."""
    L = lib()
    src = np.ascontiguousarray(np.frombuffer(bytes(src), np.uint8) if not isinstance(src, np.ndarray) else src)
    lo = np.asarray(lo, np.int64)
    if lo.size and not (np.all(lo >= 0) and np.all(np.asarray(hi) >= lo) and np.all(np.asarray(hi) <= len(src))):
        raise ValueError('gather: a range outside the source')
    off = np.concatenate([[0], np.cumsum(np.asarray(hi, np.int64) - lo)]).astype(np.int64)
    out = np.zeros(max(int(off[-1]), 1), np.uint8)
    srcp = src if src.size else np.zeros(1, np.uint8)
    lop = lo if lo.size else np.zeros(1, np.int64)
    rc = L.emu_fasta_gather(srcp.ctypes.data, src.size, lop.ctypes.data, off.ctypes.data, len(lo), out.ctypes.data)
    if rc:
        raise RuntimeError(f'emu_fasta_gather failed ({rc})')
    return out[:int(off[-1])]


def load(data, tile):
    """What bb_fasta_parse, bb_fasta_headers and bb_fasta_reference do, on the emulator: -> (names, [contig bases],
    depths, circular, hairpin_left, hairpin_right) as misc.load_fasta_arrays returns them."""
    from badread_b200.misc import fasta_contigs
    kept, start, end, kept_off = parse(data, tile)
    text = gather(data, start + 1, end)
    text_off = np.concatenate([[0], np.cumsum(end - start - 1)]).astype(np.int64)
    bounds = list(kept_off) + [kept.size]
    headers = [(bytes(text[text_off[k]:text_off[k + 1]]).decode('latin-1'), (int(bounds[k]), int(bounds[k + 1])))
               for k in range(len(start))]
    names, ranges, depths, circular, hp_left, hp_right = fasta_contigs(headers)
    ref = gather(kept, [r[0] for r in ranges], [r[1] for r in ranges])
    off = np.concatenate([[0], np.cumsum([r[1] - r[0] for r in ranges])]).astype(np.int64)
    seqs = [ref[off[i]:off[i + 1]] for i in range(len(names))]
    return names, seqs, depths, circular, hp_left, hp_right
