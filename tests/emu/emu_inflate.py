"""ctypes front end of tests/emu/emu_inflate.cpp: the BGZF inflater's device code under the warp emulator.
TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_inflate.so'


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_inflate.cpp', HERE / 'cuda_emu.h', csrc / 'bb_inflate.cuh', csrc / 'bb_crc32.cuh']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique', '-o',
                        str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None


def decompress(data):
    """bb_bgzf_decompress on the emulator -> the inflated bytes (a bytearray); ValueError with the library's message for
    input that is not BGZF or a corrupt member."""
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        L.emu_bgzf_decompress.restype = ctypes.c_int
        L.emu_bgzf_decompress.argtypes = [ctypes.c_char_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
                                          ctypes.POINTER(ctypes.c_int64), ctypes.c_char_p, ctypes.c_int]
        _lib = L
    data = bytes(data)
    msg = ctypes.create_string_buffer(512)
    n_out = ctypes.c_int64(0)
    rc = _lib.emu_bgzf_decompress(data, len(data), None, 0, ctypes.byref(n_out), msg, 512)
    out = bytearray(n_out.value)
    if rc == -4:
        rc = _lib.emu_bgzf_decompress(data, len(data), (ctypes.c_char * len(out)).from_buffer(out), len(out),
                                      ctypes.byref(n_out), msg, 512)
    if rc == -2:
        raise ValueError(msg.value.decode(errors='replace'))
    if rc:
        raise RuntimeError(f'emu_bgzf_decompress failed ({rc})')
    return out
