"""ctypes front end of tests/emu/emu_plot.cpp: the window series kernel of `badread_b200 plot` under the warp emulator.
TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_plot.so'
THREADS = 64        # two warps: the cross-warp step of the block scan runs


def build():
    root = HERE.parent.parent
    srcs = [HERE / 'emu_plot.cpp', HERE / 'cuda_emu.h', root / 'badread_b200' / 'csrc' / 'bb_plot.cuh']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique',
                        '-ffp-contract=off', f'-DWS_THREADS={THREADS}', '-o', str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        vp = ctypes.c_void_p
        L.emu_window_series.restype = ctypes.c_int
        L.emu_window_series.argtypes = [ctypes.c_int32] + [vp] * 9 + [ctypes.c_int64, ctypes.c_int, vp, vp]
        _lib = L
    return _lib


def window_series(flat, window, qual=False, items=8):
    """(identities, mean qscores or None) of every alignment of a flat set, one after the other."""
    p = lambda a: np.ascontiguousarray(a).ctypes.data   # noqa: E731
    points = int(np.maximum(np.diff(flat.read_off) - window, 0).sum())
    ident = np.zeros(max(points, 1), np.float64)
    mq = np.zeros(max(points, 1), np.float64)
    arrays = [np.ascontiguousarray(x) for x in (flat.read, flat.qual, flat.ref, flat.read_off, flat.ref_off, flat.ops,
                                                 flat.op_read0, flat.op_ref0, flat.ops_off)]
    rc = lib().emu_window_series(flat.n, *(a.ctypes.data for a in arrays), window, items, p(ident), p(mq) if qual else None)
    if rc:
        raise RuntimeError(f'emu_window_series failed ({rc})')
    return ident[:points], (mq[:points] if qual else None)
