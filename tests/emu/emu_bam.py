"""ctypes front end of tests/emu/emu_bam.cpp: the BAM record kernel and the compressor's BAM mode under the warp
emulator.  TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_bam.so'
CHUNK = 65280


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_bam.cpp', HERE / 'cuda_emu.h', csrc / 'bb_bam_out.cuh', csrc / 'bb_bgzf.cuh', csrc / 'bb_crc32.cuh']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # the emulator's state stays private to this library (the other emulator libraries have their own)
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique', '-o',
                        str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
        L.emu_bam_record_size.restype = i64
        L.emu_bam_record_size.argtypes = [i32, i32, i32]
        L.emu_bam_records.restype = ctypes.c_int
        L.emu_bam_records.argtypes = [ctypes.c_int, vp, vp, vp, ctypes.c_int, vp, vp, vp, vp, i64, vp]
        L.emu_bam_compress.restype = ctypes.c_int
        L.emu_bam_compress.argtypes = [vp, i64, i64, vp, i64, ctypes.c_int, vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i64)]
        _lib = L
    return _lib


def record_size(name_len, l_seq, co_len):
    return int(lib().emu_bam_record_size(name_len, l_seq, co_len))


def records(recs, text, sources, stream_base=0, carry=0):
    """bb_bam_build's kernel on the emulator: recs (planner.BAM_RECORD_DTYPE) built back to back after `carry` bytes;
    sources: [(seq, qual)] uint8 arrays, the batch output concatenated in that order.  Returns (record bytes after the
    carry, fields as an (2 n, 2) int64 array)."""
    L = lib()
    recs = np.ascontiguousarray(recs)
    n = len(recs)
    sizes = [record_size(int(r['name_len']), int(r['out_len']), int(r['co_len'])) for r in recs]
    pos = np.asarray(np.cumsum([0] + sizes)[:-1] + carry, dtype=np.int64)
    total = int(sum(sizes))
    out = np.zeros(carry + total + 1, np.uint8)
    fields = np.zeros((2 * max(n, 1), 2), np.int64)
    text = np.ascontiguousarray(np.frombuffer(bytes(text), np.uint8) if not isinstance(text, np.ndarray) else text)
    text = text if text.size else np.zeros(1, np.uint8)
    seqs = [np.ascontiguousarray(s, dtype=np.uint8) for s, _ in sources]
    quals = [np.ascontiguousarray(q, dtype=np.uint8) for _, q in sources]
    base = np.concatenate([[0], np.cumsum([s.size for s in seqs])]).astype(np.int64)
    sp = (ctypes.c_void_p * len(seqs))(*[s.ctypes.data for s in seqs])
    qp = (ctypes.c_void_p * len(quals))(*[q.ctypes.data for q in quals])
    rc = L.emu_bam_records(n, recs.ctypes.data, pos.ctypes.data, text.ctypes.data, len(seqs), sp, qp, base.ctypes.data,
                           out.ctypes.data, int(stream_base), fields.ctypes.data)
    if rc:
        raise RuntimeError(f'emu_bam_records failed ({rc})')
    return out[carry:carry + total].tobytes(), fields[:2 * n]


def compress(data, stream_base, fields, final=True):
    """bb_bam_compress on the emulator -> (members, bytes consumed)."""
    L = lib()
    data = bytes(data)
    f = np.ascontiguousarray(fields, dtype=np.int64).reshape(-1, 2)
    fp = f if len(f) else np.zeros((1, 2), np.int64)
    cap = len(data) + 31 * (len(data) // CHUNK + 1)
    out = np.zeros(cap, dtype=np.uint8)
    n_out, n_used = ctypes.c_int64(0), ctypes.c_int64(0)
    rc = L.emu_bam_compress(data, len(data), int(stream_base), fp.ctypes.data, len(f), int(bool(final)), out.ctypes.data, cap,
                            ctypes.byref(n_out), ctypes.byref(n_used))
    if rc:
        raise RuntimeError(f'emu_bam_compress failed ({rc})')
    return out[:n_out.value].tobytes(), int(n_used.value)
