"""ctypes front end of tests/emu/emu_large_k.cpp: the device code of error models with k up to 16 under the warp
emulator - the 128-bit-key counting kernel of `error_model`, K1 with the hash-table k-mer index
(badread_b200/csrc/bb_em_tables.h) and the error loop behind it.  TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_large_k.so'


def build():
    csrc = HERE.parent.parent / 'badread_b200' / 'csrc'
    srcs = [HERE / 'emu_large_k.cpp', HERE / 'cuda_emu.h'] + sorted(csrc.glob('*.cuh')) + sorted(csrc.glob('*.h'))
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # the emulator's state stays private to this library (libemu_align.so may be loaded next to it)
        subprocess.run(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique', '-o',
                        str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None
vp = ctypes.c_void_p


def _load():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        L.emu_count_kmers_wide.restype = ctypes.c_int
        L.emu_count_kmers_wide.argtypes = [ctypes.c_int, ctypes.c_int32] + [vp] * 8 + [ctypes.c_int64, vp, vp, vp,
                                                                                      ctypes.POINTER(ctypes.c_int64),
                                                                                      ctypes.c_int64, vp, vp, vp,
                                                                                      ctypes.POINTER(ctypes.c_int64)]
        L.emu_build_kidx_hash.restype = ctypes.c_int
        L.emu_build_kidx_hash.argtypes = [vp] * 5 + [ctypes.c_int, ctypes.c_int, ctypes.c_int32, vp, ctypes.c_uint64,
                                                     ctypes.c_uint64, vp, vp, ctypes.c_char_p, ctypes.c_int]
        L.emu_error_loop_kmers.restype = ctypes.c_int
        L.emu_error_loop_kmers.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint64, ctypes.c_uint64,
                                           ctypes.c_int, ctypes.c_int32] + [vp] * 6 + [vp, vp, ctypes.c_int]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(vp)


def count_kmers_wide(flat, k, cap=None):
    """bb_count_kmer_alternatives_wide under the emulator, with the return value of model_builders._count('kmers_wide')."""
    L = _load()
    if cap is None:
        cap = 1 << 12
        while cap < 2 * int(flat.ref_off[-1]) + 16:
            cap <<= 1
    ovf_cap = 1 << 16
    while True:
        keys = np.empty(2 * cap, dtype=np.uint64)
        first = np.empty(cap, dtype=np.uint64)
        counts = np.empty(cap, dtype=np.uint32)
        ovf = [np.empty(ovf_cap, dtype=np.int32) for _ in range(3)]
        n, m = ctypes.c_int64(0), ctypes.c_int64(0)
        rc = L.emu_count_kmers_wide(k, flat.n, _p(flat.read), _p(flat.read_off), _p(flat.ref), _p(flat.ref_off), _p(flat.ops),
                                    _p(flat.op_read0), _p(flat.op_ref0), _p(flat.ops_off), cap, _p(keys), _p(first),
                                    _p(counts), ctypes.byref(n), ovf_cap, _p(ovf[0]), _p(ovf[1]), _p(ovf[2]), ctypes.byref(m))
        if rc == -4:
            if m.value > ovf_cap:
                ovf_cap = int(m.value) + 16
            else:
                cap <<= 1
            continue
        if rc:
            raise RuntimeError(f'emu_count_kmers_wide failed ({rc})')
        return keys[:2 * n.value].reshape(n.value, 2), first[:n.value], counts[:n.value].reshape(n.value, 1), \
            np.zeros(94, dtype=np.uint64), [o[:m.value] for o in ovf]


def build_kidx_hash(ref, literals, segments, k, kmer_codes, seed, read_index):
    """K1 with the hash-table index for one read.  segments: [(kind, src, len)] (0 = reference slice, 1 = its reverse
    complement, 2 = literal bytes).  Returns (padded fragment, row per position).  Codes the table builder rejects
    raise ValueError with its message."""
    L = _load()
    r = np.frombuffer((ref.encode('latin-1') if isinstance(ref, str) else bytes(ref)) or b'\0', dtype=np.uint8)
    lit = np.frombuffer((literals.encode('latin-1') if isinstance(literals, str) else bytes(literals)) or b'\0', dtype=np.uint8)
    kind = np.asarray([s[0] for s in segments], dtype=np.int32)
    src = np.asarray([s[1] for s in segments], dtype=np.int64)
    ln = np.asarray([s[2] for s in segments], dtype=np.int32)
    n = int(ln.sum()) + 2 * k
    frag = np.zeros(n + 8, dtype=np.uint8)
    kidx = np.full(n + 8, -9, dtype=np.int32)
    codes = np.ascontiguousarray(kmer_codes, dtype=np.int64)
    err = ctypes.create_string_buffer(512)
    rc = L.emu_build_kidx_hash(_p(r), _p(lit), _p(kind), _p(src), _p(ln), len(segments), k, len(codes), _p(codes), seed,
                               read_index, _p(frag), _p(kidx), err, len(err))
    if rc == 2:
        raise ValueError(err.value.decode())
    return bytes(frag[:n]).decode('latin-1'), kidx[:max(0, n - k + 1)].tolist()


def error_loop_kmers(fragment, target_identity, seed, read_index, error_model):
    """The error loop of one read with the model's hash-table index -> (joined read, stats) as emu.error_loop."""
    L = _load()
    t = error_model.to_device_tables()
    f = fragment.encode('latin-1') if isinstance(fragment, str) else bytes(fragment)
    k = int(t['k'])
    cap = 2 * (len(f) + 2 * k) + 64
    joined = np.zeros(cap, dtype=np.uint8)
    out8 = np.zeros(8, dtype=np.int32)
    arr = {name: np.ascontiguousarray(t[name]) for name in ('kmer_codes', 'row_off', 'cum', 'flags', 'slots', 'pool')}
    rounds = L.emu_error_loop_kmers(f, len(f), float(target_identity), seed, read_index, k, len(arr['row_off']) - 1,
                                    *(_p(arr[n]) for n in ('kmer_codes', 'row_off', 'cum', 'flags', 'slots', 'pool')),
                                    _p(out8), _p(joined), cap)
    if rounds < 0:
        raise RuntimeError(f'error loop under the emulator failed ({rounds})')
    if out8[7]:
        raise RuntimeError(f'error loop flags 0x{int(out8[7]):x}')
    stats = {'loop_count': int(out8[0]), 'change_count': int(out8[1]), 'n_alignments': int(out8[2]),
             'untrimmed_len': int(out8[3]), 'start_trim': int(out8[4]), 'end_trim': int(out8[5]), 'rounds': int(rounds)}
    return bytes(joined[:out8[3]]).decode('latin-1'), stats
