"""ctypes front end of tests/emu/emu_qscores.cpp: get_qscores under the warp emulator with the tables of the shared
qscore table builder (badread_b200/csrc/bb_qscore_tables.h), CIGAR keys of any length.  TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

from emu import emu as E

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_qscores.so'


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_qscores.cpp', HERE / 'cuda_emu.h'] + sorted(csrc.glob('*.cuh')) + sorted(csrc.glob('*.h'))
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # the emulator's state stays private to this library (libemu_align.so, loaded next to it, has its own)
        subprocess.run(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique', '-o',
                        str(LIB), str(srcs[0])], check=True)
    E.build()
    return LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        L.emu_qscores_cigars.restype = ctypes.c_int
        L.emu_qscores_cigars.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int32] + \
            [ctypes.c_void_p] * 5 + [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
        _lib = L
    if E._lib is None:
        E._lib = ctypes.CDLL(str(E.LIB))
    return _lib


def get_qscores_cigars(seq, frag, upper, qscore_model, seed, read_index):
    """get_qscores on the device code: the alignment task pipeline (emu_align.cpp), then bb_k_qscores_pair with the tables
    bb_upload_qscore_model_cigars builds -> (quality string, '=' columns, alignment columns).  qscore_model: a QScoreModel
    or its to_device_tables() dict.  A key the builder rejects raises ValueError with its message."""
    L = _load()
    t = qscore_model.to_device_tables() if hasattr(qscore_model, 'to_device_tables') else qscore_model
    q = seq.encode('latin-1') if isinstance(seq, str) else bytes(seq)
    f = frag.encode('latin-1') if isinstance(frag, str) else bytes(frag)
    n = len(q)
    ops = np.zeros(n + 8, dtype=np.uint8)
    dcnt = np.zeros(n + 8, dtype=np.uint32)
    out5 = np.zeros(5, dtype=np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    E._lib.emu_set_quad(0)
    E._lib.emu_set_hist(1)
    rc = E._lib.emu_tasks_align(q, n, f, len(f), int(upper), p(ops), p(dcnt), p(out5))
    if rc or out5[4] or out5[2]:
        raise RuntimeError(f'task pipeline under the emulator failed (flags 0x{int(out5[4]):x}, overflow {int(out5[2])})')
    arr = {name: np.ascontiguousarray(t[name]) for name in ('key_chars', 'key_off', 'row_off', 'scores', 'cum')}
    qual = np.zeros(n, dtype=np.uint8)
    err = ctypes.create_string_buffer(512)
    rc = L.emu_qscores_cigars(p(ops), p(dcnt), n, int(t['kmer_size']), int(t['n_keys']),
                              *(p(arr[k]) for k in ('key_chars', 'key_off', 'row_off', 'scores', 'cum')),
                              seed, read_index, p(qual), err, len(err))
    if rc == 2:
        raise ValueError(err.value.decode())
    if rc:
        raise RuntimeError(f'emu_qscores_cigars failed ({rc})')
    return bytes(qual).decode('latin-1'), int(out5[0]), n + int(out5[1])
