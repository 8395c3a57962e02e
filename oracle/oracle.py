"""
oracle.py - ctypes front end of the CPU oracle (oracle/badread_oracle.c).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs. Nothing under badread_b200/ imports this module.

The oracle consumes the same flat model tables the product uploads to the GPU
(ErrorModel.to_device_tables / QScoreModel.to_device_tables), so a parity test feeds both sides identical
inputs: fragments, target identities, seed, read indices.
"""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB_PATH = HERE / 'libbadread_oracle.so'
RNG_MT, RNG_PHILOX = 0, 1


def build(force=False):
    src = HERE / 'badread_oracle.c'
    if force or not LIB_PATH.is_file() or LIB_PATH.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(['make', '-C', str(HERE), '-s'], check=True)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not LIB_PATH.is_file():
            build()
        L = ctypes.CDLL(str(LIB_PATH))
        c = ctypes
        vp, i32, i64, u64, dbl = c.c_void_p, c.c_int32, c.c_int64, c.c_uint64, c.c_double
        P = c.POINTER
        L.bo_rng_create.restype = vp
        L.bo_rng_create.argtypes = [c.c_int, u64, u64]
        L.bo_rng_destroy.argtypes = [vp]
        L.bo_rng_u32.restype = c.c_uint32
        L.bo_rng_u32.argtypes = [vp]
        L.bo_rng_random.restype = dbl
        L.bo_rng_random.argtypes = [vp]
        L.bo_rng_randbelow.restype = c.c_uint32
        L.bo_rng_randbelow.argtypes = [vp, c.c_uint32]
        L.bo_rng_stream.argtypes = [vp, c.c_uint32, c.c_uint32]
        L.bo_philox.argtypes = [vp, vp, vp]
        L.bo_set_traceback_limit.argtypes = [i64]
        L.bo_get_traceback_limit.restype = i64
        L.bo_align_path.restype = i64
        L.bo_align_path.argtypes = [vp, i64, vp, i64, c.c_int, P(vp), P(i64)]
        L.bo_free.argtypes = [vp]
        L.bo_em_create.restype = vp
        L.bo_em_create.argtypes = [c.c_int, c.c_int, vp, i64, i32, vp, vp, vp, vp, vp, i64]
        L.bo_em_destroy.argtypes = [vp]
        L.bo_qm_create.restype = vp
        L.bo_qm_create.argtypes = [c.c_int, i32, vp, vp, vp, vp, vp]
        L.bo_qm_destroy.argtypes = [vp]
        L.bo_sequence_fragment.restype = c.c_int
        L.bo_sequence_fragment.argtypes = [vp, vp, vp, vp, i64, dbl, c.c_int, P(vp), P(vp), P(i64), P(i64), P(i64), vp]
        L.bo_get_qscores.restype = c.c_int
        L.bo_get_qscores.argtypes = [vp, vp, vp, i64, vp, i64, vp, P(i64), P(i64)]
        L.bo_add_errors_to_kmer.restype = c.c_int
        L.bo_add_errors_to_kmer.argtypes = [vp, vp, vp, vp, vp]
        L.bo_sequence_batch.restype = i64
        L.bo_block_steps_reset.argtypes = []
        L.bo_block_steps.argtypes = []
        L.bo_block_steps.restype = i64
        L.bo_sequence_batch.argtypes = [vp, vp, u64, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, c.c_int]
        L.bo_sequence_batch_stats.restype = i64
        L.bo_sequence_batch_stats.argtypes = [vp, vp, u64, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, c.c_int, vp, vp, vp]
        L.bo_tree_arm.argtypes = [c.c_int]
        L.bo_tree_take.restype = i64
        L.bo_tree_take.argtypes = [P(vp)]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _bytes(s):
    return s.encode('latin-1') if isinstance(s, str) else bytes(s)


TREE_FIELDS = ('depth', 'q0', 'nn', 't0', 'mm', 'best', 'is_leaf', 'target_has_non_acgt')


def _tree_from(ptr, n, L=None):
    """bo_tree_take's entries as a list of TREE_FIELDS tuples (and the buffer released by library L)."""
    if not n:
        return []
    flat = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_int64)), shape=(n * len(TREE_FIELDS),))
    tree = [tuple(int(x) for x in row) for row in flat.reshape(n, len(TREE_FIELDS))]
    (L or lib()).bo_free(ptr)
    return tree


def _take_tree(L=None):
    """The tree the last final alignment of this thread recorded in library L (this oracle's by default)."""
    L = L or lib()
    ptr = ctypes.c_void_p()
    n = L.bo_tree_take(ctypes.byref(ptr))
    return _tree_from(ptr, n, L)


def align_path(query, target, naive=False, with_tree=False):
    """edlib.align(query, target, task='path') -> (expanded ops string or None, edit distance[, tree]).

    with_tree: also the Hirschberg tree of the alignment - every call of obtain_alignment (naive_obtain with
    naive=True) with both sides non-empty, in call order, as (depth, q0, nn, t0, mm, best, is_leaf,
    target_has_non_acgt)."""
    L = lib()
    q, t = _bytes(query), _bytes(target)
    out = ctypes.c_void_p()
    dist = ctypes.c_int64(0)
    if with_tree:
        L.bo_tree_arm(1)
    n = L.bo_align_path(q, len(q), t, len(t), 1 if naive else 0, ctypes.byref(out), ctypes.byref(dist))
    tree = _take_tree() if with_tree else None
    if n < 0:
        ops = None
    else:
        ops = ctypes.string_at(out, n).decode('ascii')
        L.bo_free(out)
    return (ops, dist.value, tree) if with_tree else (ops, dist.value)


def set_traceback_limit(v):
    lib().bo_set_traceback_limit(int(v))


class Rng(object):
    def __init__(self, mode, seed, read_index=0):
        self._h = lib().bo_rng_create(mode, ctypes.c_uint64(seed), ctypes.c_uint64(read_index))

    def __del__(self):
        if getattr(self, '_h', None):
            lib().bo_rng_destroy(self._h)
            self._h = None

    def u32(self):
        return lib().bo_rng_u32(self._h)

    def random(self):
        return lib().bo_rng_random(self._h)

    def randbelow(self, n):
        return lib().bo_rng_randbelow(self._h, n)

    def stream(self, purpose, index):
        lib().bo_rng_stream(self._h, purpose, index)


class Oracle(object):
    """Holds C copies of the model tables; sequence_fragment / get_qscores for one read or a batch."""

    def __init__(self, error_model, qscore_model):
        L = lib()
        t = error_model.to_device_tables()
        if t['type'] == 0:
            self._em = L.bo_em_create(1, 0, None, 0, 0, None, None, None, None, None, 0)
        else:
            self._em = L.bo_em_create(t['k'], 1, _ptr(t['kmer_to_row']), t['kmer_to_row'].size, len(t['row_off']) - 1,
                                      _ptr(t['row_off']), _ptr(t['cum']), _ptr(t['flags']), _ptr(t['slots']),
                                      _ptr(t['pool']), t['pool'].size)
        self.k = t['k']
        q = qscore_model.to_device_tables()
        self._qm = L.bo_qm_create(q['kmer_size'], q['n_keys'], _ptr(q['key_chars']), _ptr(q['key_off']),
                                  _ptr(q['row_off']), _ptr(q['scores']), _ptr(q['cum']))

    def __del__(self):
        L = lib()
        if getattr(self, '_em', None):
            L.bo_em_destroy(self._em)
            self._em = None
        if getattr(self, '_qm', None):
            L.bo_qm_destroy(self._qm)
            self._qm = None

    def sequence_fragment(self, fragment, target_identity, seed, read_index=0, mode=RNG_PHILOX, pow_mode=None,
                          with_stats=False):
        """simulate.sequence_fragment -> (seq, qual, actual_identity[, stats]).

        stats['tree'] is the Hirschberg tree of the final alignment (the untrimmed read against the padded fragment;
        see align_path's with_tree); the window alignments of the error loop are not in it."""
        L = lib()
        if pow_mode is None:
            pow_mode = 0 if mode == RNG_MT else 1
        rng = L.bo_rng_create(mode, ctypes.c_uint64(seed), ctypes.c_uint64(read_index))
        frag = _bytes(fragment)
        seq, qual = ctypes.c_void_p(), ctypes.c_void_p()
        n, m, c = ctypes.c_int64(0), ctypes.c_int64(0), ctypes.c_int64(0)
        stats = np.zeros(4, dtype=np.int64)
        if with_stats:
            L.bo_tree_arm(1)
        L.bo_sequence_fragment(self._em, self._qm, rng, frag, len(frag), target_identity, pow_mode, ctypes.byref(seq),
                               ctypes.byref(qual), ctypes.byref(n), ctypes.byref(m), ctypes.byref(c), _ptr(stats))
        tree = _take_tree() if with_stats else None
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

    def get_qscores(self, seq, frag, seed, read_index=0, mode=RNG_PHILOX):
        L = lib()
        rng = L.bo_rng_create(mode, ctypes.c_uint64(seed), ctypes.c_uint64(read_index))
        s, f = _bytes(seq), _bytes(frag)
        qual = np.zeros(len(s), dtype=np.uint8)
        m, c = ctypes.c_int64(0), ctypes.c_int64(0)
        L.bo_get_qscores(self._qm, rng, s, len(s), f, len(f), _ptr(qual), ctypes.byref(m), ctypes.byref(c))
        L.bo_rng_destroy(rng)
        return bytes(qual).decode('latin-1'), m.value, c.value

    def add_errors_to_kmer(self, kmer, rng):
        L = lib()
        out = np.zeros(64 * 260, dtype=np.uint8)
        off = np.zeros(self.k + 1, dtype=np.int32)
        kb = _bytes(kmer)
        L.bo_add_errors_to_kmer(self._em, rng._h, kb, _ptr(out), _ptr(off))
        return [bytes(out[off[j]:off[j + 1]]).decode('latin-1') for j in range(self.k)]

    def sequence_batch(self, fragments, target_identities, seed, read_indices, n_threads=1, with_stats=False):
        """Philox-mode batch over independent reads with `n_threads` host threads (the timed CPU baseline).
        Returns (list of (seq, qual, matches, columns), total_bases).  with_stats: every read's tuple gains a fifth
        item, the stats dict of sequence_fragment(..., with_stats=True) without 'matches' / 'columns' (the tree
        included)."""
        L = lib()
        n = len(fragments)
        frs = [_bytes(f) for f in fragments]
        off = np.zeros(n + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(f) for f in frs])
        blob = np.frombuffer(b''.join(frs), dtype=np.uint8) if off[-1] else np.zeros(1, dtype=np.uint8)
        ti = np.asarray(target_identities, dtype=np.float64)
        ri = np.asarray(read_indices, dtype=np.uint64)
        seq_ptrs = (ctypes.c_void_p * n)()
        qual_ptrs = (ctypes.c_void_p * n)()
        out_len = np.zeros(n, dtype=np.int64)
        matches = np.zeros(n, dtype=np.int64)
        cols = np.zeros(n, dtype=np.int64)
        if with_stats:
            stats = np.zeros((max(n, 1), 4), dtype=np.int64)
            tree_ptrs = (ctypes.c_void_p * n)()
            tree_len = np.zeros(n, dtype=np.int64)
            total = L.bo_sequence_batch_stats(self._em, self._qm, ctypes.c_uint64(seed), _ptr(ri), _ptr(blob), _ptr(off),
                                              n, _ptr(ti), seq_ptrs, qual_ptrs, _ptr(out_len), _ptr(matches), _ptr(cols),
                                              n_threads, _ptr(stats), tree_ptrs, _ptr(tree_len))
        else:
            total = L.bo_sequence_batch(self._em, self._qm, ctypes.c_uint64(seed), _ptr(ri), _ptr(blob), _ptr(off), n,
                                        _ptr(ti), seq_ptrs, qual_ptrs, _ptr(out_len), _ptr(matches), _ptr(cols), n_threads)
        out = []
        for r in range(n):
            s = ctypes.string_at(seq_ptrs[r], int(out_len[r])).decode('latin-1')
            q = ctypes.string_at(qual_ptrs[r], int(out_len[r])).decode('latin-1')
            L.bo_free(seq_ptrs[r])
            L.bo_free(qual_ptrs[r])
            if with_stats:
                st = {'loop_count': int(stats[r, 0]), 'change_count': int(stats[r, 1]), 'n_alignments': int(stats[r, 2]),
                      'untrimmed_len': int(stats[r, 3]), 'tree': _tree_from(tree_ptrs[r], int(tree_len[r]))}
                out.append((s, q, int(matches[r]), int(cols[r]), st))
            else:
                out.append((s, q, int(matches[r]), int(cols[r])))
        return out, int(total)


def block_steps_reset():
    """Zeroes the counter of 64-row block updates of the path passes (see badread_oracle.c, work accounting)."""
    lib().bo_block_steps_reset()


def block_steps():
    return int(lib().bo_block_steps())
