"""ctypes front end of tests/emu/emu_bgzf.cpp: the BGZF compressor's device code under the warp emulator.
TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_bgzf.so'
CHUNK = 65280


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_bgzf.cpp', HERE / 'cuda_emu.h', csrc / 'bb_bgzf.cuh']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # the emulator's state stays private to this library (the other emulator libraries have their own)
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique', '-o',
                        str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None


def compress(data, line_mod4=0, final=True):
    """bb_bgzf_compress on the emulator -> (members, bytes consumed)."""
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        L.emu_bgzf_compress.restype = ctypes.c_int
        L.emu_bgzf_compress.argtypes = [ctypes.c_char_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                        ctypes.c_int64, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]
        _lib = L
    data = bytes(data)
    cap = len(data) + 31 * (len(data) // CHUNK + 1)
    out = np.zeros(cap, dtype=np.uint8)
    n_out, n_used = ctypes.c_int64(0), ctypes.c_int64(0)
    rc = _lib.emu_bgzf_compress(data, len(data), int(line_mod4), int(bool(final)), out.ctypes.data_as(ctypes.c_void_p), cap,
                                ctypes.byref(n_out), ctypes.byref(n_used))
    if rc:
        raise RuntimeError(f'emu_bgzf_compress failed ({rc})')
    return out[:n_out.value].tobytes(), int(n_used.value)
