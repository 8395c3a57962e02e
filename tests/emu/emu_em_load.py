"""ctypes front end of tests/emu/emu_em_load.cpp: the error model loader's device code under the warp emulator.
TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_em_load.so'


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_em_load.cpp', HERE / 'cuda_emu.h', csrc / 'bb_em_load.cuh',
            HERE.parent.parent / 'include' / 'badread_b200.h']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # 64 threads per tile (two warps: the cross-warp step of the block scan runs) and 16 in the scan CTA (so that
        # its threads take several tiles each on small inputs); no contraction, as nvcc's -fmad=false
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique',
                        '-ffp-contract=off', '-DEML_THREADS=64', '-DEML_SUMS_THREADS=16', '-o', str(LIB), str(srcs[0])],
                       check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
        L.emu_em_load.restype = ctypes.c_int
        L.emu_em_load.argtypes = [ctypes.c_char_p, i64, i32, ctypes.c_int, vp]
        L.emu_em_fetch.restype = ctypes.c_int
        L.emu_em_fetch.argtypes = [vp] * 9
        L.emu_em_parse_prob.restype = ctypes.c_int
        L.emu_em_parse_prob.argtypes = [ctypes.c_char_p, i64, vp, vp]
        L.emu_em_pysum.restype = ctypes.c_double
        L.emu_em_pysum.argtypes = [vp, i64]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data if a is not None else None


def load(text, tile=16384, dense=True):
    """The loader's passes over the model text -> (info dict, tables dict as ErrorModel._tables holds them, rowinfo).
    info['fallback'] != 0: no tables (None); info['capacity']: the pool outgrew its limit."""
    L = lib()
    text = bytes(text)
    c = np.zeros(7, np.int64)
    rc = L.emu_em_load(text, len(text), int(tile), int(bool(dense)), c.ctypes.data)
    if rc:
        raise RuntimeError(f'emu_em_load failed ({rc})')
    info = dict(zip(('k', 'n_rows', 'n_entries', 'n_alts', 'pool_bytes', 'fallback', 'capacity'), (int(x) for x in c)))
    if info['fallback'] or info['capacity']:
        return info, None, None
    k, nr, ne = info['k'], info['n_rows'], info['n_entries']
    t = {'row_off': np.zeros(nr + 1, np.int32), 'cum': np.zeros(ne, np.float64), 'flags': np.zeros(ne, np.uint8),
         'slots': np.zeros(ne * k, np.uint32), 'pool': np.zeros(max(info['pool_bytes'], 1), np.uint8),
         'probs': np.zeros(ne, np.float64), 'kmer_codes': np.zeros(nr, np.int64)}
    if dense and k <= 12:
        t['kmer_to_row'] = np.zeros(4 ** k, np.int32)
    rowinfo = np.zeros((nr, 5), np.float64)
    L.emu_em_fetch(_p(t.get('kmer_to_row')), _p(t['kmer_codes']), _p(t['row_off']), _p(t['cum']), _p(t['probs']),
                   _p(t['flags']), _p(t['slots']), _p(t['pool']), _p(rowinfo))
    return info, t, rowinfo


def parse_prob(s):
    """eml_parse_prob -> float, or None off the fast path.  s must be the whole number."""
    b = s.encode('latin-1')
    out = ctypes.c_double(0.0)
    end = ctypes.c_int64(0)
    ok = lib().emu_em_parse_prob(b, len(b), ctypes.addressof(out), ctypes.addressof(end))
    return out.value if ok and end.value == len(b) else None


def pysum(values):
    x = np.ascontiguousarray(values, dtype=np.float64)
    return lib().emu_em_pysum(x.ctypes.data if x.size else None, x.size)
