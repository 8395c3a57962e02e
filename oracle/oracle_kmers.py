"""
oracle_kmers.py - ctypes front end of oracle/badread_oracle_kmers.c: the CPU oracle for error models of any k up to
16, whose k-mers are looked up through the rows' sorted codes instead of a dense kmer_to_row[4^k].

TEST INFRASTRUCTURE ONLY.  `make_oracle(error_model, qscore_model)` returns oracle.Oracle for a model with a dense
index (k <= 12, the random model) and OracleKmers otherwise; both have the same sequence_fragment.
"""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

from . import oracle as O

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB_PATH = HERE / 'libbadread_oracle_kmers.so'


def build():
    srcs = [HERE / 'badread_oracle_kmers.c', HERE / 'badread_oracle.c']
    if not LIB_PATH.is_file() or any(LIB_PATH.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # the flags of oracle/Makefile: every FP64 operation of the loop individually rounded
        subprocess.run(['gcc', '-O2', '-fPIC', '-std=c11', '-Wall', '-Wextra', '-fvisibility=hidden', '-ffp-contract=off',
                        '-shared', '-o', str(LIB_PATH), str(srcs[0]), '-lm', '-lpthread'], check=True)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB_PATH))
        c = ctypes
        vp, i32, i64, dbl = c.c_void_p, c.c_int32, c.c_int64, c.c_double
        P = c.POINTER
        L.bo_rng_create.restype = vp
        L.bo_rng_create.argtypes = [c.c_int, c.c_uint64, c.c_uint64]
        L.bo_rng_destroy.argtypes = [vp]
        L.bo_free.argtypes = [vp]
        L.bo_em_kmers_create.restype = vp
        L.bo_em_kmers_create.argtypes = [c.c_int, i32, vp, vp, vp, vp, vp, vp, i64]
        L.bo_em_kmers_destroy.argtypes = [vp]
        L.bo_qm_create.restype = vp
        L.bo_qm_create.argtypes = [c.c_int, i32, vp, vp, vp, vp, vp]
        L.bo_qm_destroy.argtypes = [vp]
        L.bo_sequence_fragment_kmers.restype = c.c_int
        L.bo_sequence_fragment_kmers.argtypes = [vp, vp, vp, vp, i64, dbl, c.c_int, P(vp), P(vp), P(i64), P(i64), P(i64),
                                                 vp]
        L.bo_tree_arm.argtypes = [c.c_int]
        L.bo_tree_take.restype = i64
        L.bo_tree_take.argtypes = [P(vp)]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class OracleKmers(object):
    """oracle.Oracle's sequence_fragment for an error model indexed by its rows' k-mer codes (any k from 3 to 16)."""

    def __init__(self, error_model, qscore_model):
        L = lib()
        t = error_model.to_device_tables()
        codes = np.ascontiguousarray(t['kmer_codes'], dtype=np.int64)
        self._em = L.bo_em_kmers_create(t['k'], len(t['row_off']) - 1, _ptr(codes), _ptr(t['row_off']), _ptr(t['cum']),
                                        _ptr(t['flags']), _ptr(t['slots']), _ptr(t['pool']), t['pool'].size)
        if not self._em:
            raise ValueError(f"error model: k = {t['k']} outside 3..16 or two rows with the same k-mer")
        self.k = t['k']
        q = qscore_model.to_device_tables()
        self._qm = L.bo_qm_create(q['kmer_size'], q['n_keys'], _ptr(q['key_chars']), _ptr(q['key_off']),
                                  _ptr(q['row_off']), _ptr(q['scores']), _ptr(q['cum']))

    def __del__(self):
        L = lib()
        if getattr(self, '_em', None):
            L.bo_em_kmers_destroy(self._em)
            self._em = None
        if getattr(self, '_qm', None):
            L.bo_qm_destroy(self._qm)
            self._qm = None

    def sequence_fragment(self, fragment, target_identity, seed, read_index=0, mode=O.RNG_PHILOX, pow_mode=None,
                          with_stats=False):
        """simulate.sequence_fragment -> (seq, qual, actual_identity[, stats]), as oracle.Oracle.sequence_fragment."""
        L = lib()
        if pow_mode is None:
            pow_mode = 0 if mode == O.RNG_MT else 1
        rng = L.bo_rng_create(mode, ctypes.c_uint64(seed), ctypes.c_uint64(read_index))
        frag = O._bytes(fragment)
        seq, qual = ctypes.c_void_p(), ctypes.c_void_p()
        n, m, c = ctypes.c_int64(0), ctypes.c_int64(0), ctypes.c_int64(0)
        stats = np.zeros(4, dtype=np.int64)
        if with_stats:
            L.bo_tree_arm(1)
        L.bo_sequence_fragment_kmers(self._em, self._qm, rng, frag, len(frag), target_identity, pow_mode,
                                     ctypes.byref(seq), ctypes.byref(qual), ctypes.byref(n), ctypes.byref(m),
                                     ctypes.byref(c), _ptr(stats))
        tree = O._take_tree(L) if with_stats else None
        s = ctypes.string_at(seq, n.value).decode('latin-1')
        q = ctypes.string_at(qual, n.value).decode('latin-1')
        L.bo_free(seq)
        L.bo_free(qual)
        L.bo_rng_destroy(rng)
        ident = m.value / c.value if c.value else 0.0
        if with_stats:
            return s, q, ident, {'matches': m.value, 'columns': c.value, 'loop_count': int(stats[0]),
                                 'change_count': int(stats[1]), 'n_alignments': int(stats[2]),
                                 'untrimmed_len': int(stats[3]), 'tree': tree}
        return s, q, ident


def make_oracle(error_model, qscore_model):
    """oracle.Oracle when the error model has a dense index (or is the random model), else OracleKmers."""
    t = error_model.to_device_tables()
    if t['type'] == 0 or 'kmer_to_row' in t:
        return O.Oracle(error_model, qscore_model)
    return OracleKmers(error_model, qscore_model)
