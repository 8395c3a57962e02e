"""ctypes front end of tests/emu/emu_gunzip.cpp: the gzip inflater's device code and driver under the warp emulator.
TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_gunzip.so'
STATS = ('members', 'chunks', 'absorbed', 'first_candidate', 'repaired', 'chained', 'reruns', 'bgzf')


class Stats(ctypes.Structure):
    """bb_gzip_stats (include/badread_b200.h)."""
    _fields_ = [(f, ctypes.c_int64) for f in STATS[:-1]] + [('bgzf', ctypes.c_int32), ('reserved', ctypes.c_int32)]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f in STATS}


# a build whose bit readers cover 128 KiB and move forward after 64 KiB, so that a test stream of a few MB moves them
SMALL_SPAN = ('-DGZ_SPAN=(1<<17)', '-DGZ_REBASE=(1<<16)')


def build(defines=()):
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_gunzip.cpp', HERE / 'cuda_emu.h', csrc / 'bb_gunzip.cuh', csrc / 'bb_inflate.cuh', csrc / 'bb_crc32.cuh',
            HERE.parent.parent / 'include' / 'badread_b200.h']
    lib = HERE / ('libemu_gunzip_small_span.so' if defines else LIB.name)
    if not lib.is_file() or any(lib.stat().st_mtime < s.stat().st_mtime for s in srcs):
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique', *defines,
                        '-o', str(lib), str(srcs[0])], check=True)
    return lib


_libs = {}


def gunzip(data, chunk_bytes=0, defines=()):
    """bb_gzip_decompress's chunked inflater on the emulator -> (the inflated bytes, the stats as a dict); ValueError
    with the library's message for a corrupt stream.  defines: a build with other constants (SMALL_SPAN)."""
    key = tuple(defines)
    if key not in _libs:
        L = ctypes.CDLL(str(build(key)))
        L.emu_gzip_decompress.restype = ctypes.c_int
        L.emu_gzip_decompress.argtypes = [ctypes.c_char_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
                                          ctypes.POINTER(ctypes.c_int64), ctypes.c_int64, ctypes.POINTER(Stats),
                                          ctypes.c_char_p, ctypes.c_int]
        _libs[key] = L
    _lib = _libs[key]
    data = bytes(data)
    msg = ctypes.create_string_buffer(512)
    n_out, stats = ctypes.c_int64(0), Stats()
    out = bytearray(max(4 * len(data), 64))
    rc = _lib.emu_gzip_decompress(data, len(data), (ctypes.c_char * len(out)).from_buffer(out), len(out),
                                  ctypes.byref(n_out), chunk_bytes, ctypes.byref(stats), msg, 512)
    if rc == -4:
        out = bytearray(n_out.value)
        rc = _lib.emu_gzip_decompress(data, len(data), (ctypes.c_char * len(out)).from_buffer(out) if out else None, len(out),
                                      ctypes.byref(n_out), chunk_bytes, ctypes.byref(stats), msg, 512)
    if rc == -2:
        raise ValueError(msg.value.decode(errors='replace'))
    if rc:
        raise RuntimeError(f'emu_gzip_decompress failed ({rc}): {msg.value.decode(errors="replace")}')
    return bytes(out[:n_out.value]), stats.as_dict()
