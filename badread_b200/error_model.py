"""
ErrorModel - host side of the k-mer error model, same plugin surface as
/root/reference/badread/error_model.py:86-160 (constructor arguments, `kmer_size`, `type`, `alternatives`,
`probabilities`, `add_errors_to_kmer`) plus `to_device_tables()`, the flat arrays that
`bb_upload_error_model` ships to HBM once.

Table layout (shared by the CUDA path and the CPU oracle):
  kmer_to_row[4^k]  row of each ACGT k-mer, -1 if the model has no line for it (then: one random change,
                    error_model.py:143-144; the same happens for k-mers holding non-ACGT characters).  Only for
                    k <= DENSE_MAX_K: larger models (up to MAX_K) are indexed by `kmer_codes` alone, which the library
                    turns into a hash table (bb_upload_error_model_kmers)
  kmer_codes[n_rows] the 2-bit code of each row's k-mer (base j in bits 2*(k-1-j), A C G T = 0 1 2 3)
  row_off[n_rows+1] entry range of each row
  per entry:        cum    list(itertools.accumulate(probs)) - what random.choices builds (error_model.py:156)
                    flags  bit0: ''.join(alt) == kmer (the `continue` at simulate.py:300)
                           bit1: the "random change" remainder entry.  The reference appends
                                 (None, 1.0 - sum(probs)) to the row IN PLACE on every visit while that
                                 remainder is > 0 (error_model.py:151-154); with CPython >= 3.12's compensated
                                 sum() one append makes the row a fixed point, so the steady-state row is static.
                    slots  k encoded slot strings: len | chars << 8 for len <= 3, else len | pool_offset << 8
The slot strings come from align_kmers (error_model.py:179-229), run for the whole file by the host helper
`bb_host_align_kmers` (csrc/bb_host.cpp).

Derived from Badread (Copyright 2018 Ryan Wick, rrwick@gmail.com, https://github.com/rrwick/Badread), which is free
software under the GNU General Public License version 3 or later; this file mirrors the named parts of the
reference's interface and is distributed under the same licence (see LICENSE and NOTICE at the repository root).
"""
import ctypes
import itertools
import os
import pathlib
import random
import sys

import numpy as np

from . import _lib
from .misc import get_open_func, get_random_base, get_random_different_base, random_chance

BUILTIN_MODELS = ('nanopore2018', 'nanopore2020', 'nanopore2023', 'pacbio2016', 'pacbio2021')
MODEL_DIR = pathlib.Path(os.path.dirname(os.path.realpath(__file__))) / 'models'
_CODE = {'A': 0, 'C': 1, 'G': 2, 'T': 3}
DENSE_MAX_K = 12   # largest k with a dense kmer_to_row[4^k] (64 MB at k = 12)
MAX_K = 16         # a k-mer's code fits 32 bits; the mutate kernel keeps 16 slots per candidate in shared memory


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def decode_slot(enc, pool):
    length = int(enc) & 0xff
    if length <= 3:
        return ''.join(chr((int(enc) >> (8 * (i + 1))) & 0xff) for i in range(length))
    off = int(enc) >> 8
    return bytes(pool[off:off + length]).decode('latin-1')


class ErrorModel(object):

    def __init__(self, model_type_or_filename, output=sys.stderr):
        self.kmer_size = None
        self._alternatives = None
        self._probabilities = None
        self._tables = None
        self._kmers = []
        self._probs_loaded = []
        if model_type_or_filename == 'random':
            print('\nUsing a random error model', file=output)
            self.type = 'random'
            self.kmer_size = 1
            self._alternatives, self._probabilities = {}, {}
        elif model_type_or_filename in BUILTIN_MODELS:
            self._load_builtin(model_type_or_filename, output)
        else:
            self.load_from_file(model_type_or_filename, output)

    # ------------------------------------------------------------------------------------------ loading
    def _load_builtin(self, name, output):
        """Built-in models ship as precompiled tables (models/<name>.error.npz, produced from the reference's
        model text by tools/compile_models.py); loading them skips the ~425k load-time alignments."""
        path = MODEL_DIR / f'{name}.error.npz'
        print(f'\nLoading error model from {path}', file=output)
        if not path.is_file():
            sys.exit(f'Error: built-in error model {name} is not installed ({path} missing) - '
                     f'run tools/compile_models.py or pass a model filename')
        self.type = 'model'
        with np.load(str(path)) as z:
            self.kmer_size = int(z['k'])
            self._tables = {key: np.ascontiguousarray(z[key]) for key in
                            ('kmer_to_row', 'row_off', 'cum', 'flags', 'slots', 'pool', 'probs', 'kmer_codes') if key in z}
        print(f'\r  done: loaded error distributions for {len(self._tables["row_off"]) - 1} '
              f'{self.kmer_size}-mers', file=output)

    def load_from_file(self, filename, output):
        """error_model.py:111-133."""
        print('\nLoading error model from {}'.format(filename), file=output)
        self.type = 'model'
        rows = {}
        with get_open_func(filename)(filename, 'rt') as model_file:
            for line in model_file:
                kmer = line.split(',', 1)[0]
                if self.kmer_size is None:
                    self.kmer_size = len(kmer)
                else:
                    assert self.kmer_size == len(kmer)
                alternatives = [x.split(',') for x in line.strip().split(';') if x]
                assert alternatives[0][0] == kmer
                rows[kmer] = ([x[0] for x in alternatives], [float(x[1]) for x in alternatives])
        self._build_tables(rows)
        print(f'\r  done: loaded error distributions for {len(rows)} {self.kmer_size}-mers', file=output)

    def _build_tables(self, rows):
        k = self.kmer_size
        if k is None:
            sys.exit('Error: the error model file holds no k-mers')
        assert k > 2  # error_model.py:188
        if k > MAX_K:
            sys.exit(f'Error: error models with k > {MAX_K} are not supported by badread_b200 (this model has k = {k})')
        kmers = list(rows.keys())
        for kmer in kmers:
            if any(c not in _CODE for c in kmer):
                sys.exit(f'Error: error model k-mer {kmer} is not ACGT-only (unsupported by badread_b200)')
        n_alts = sum(len(rows[kmer][0]) for kmer in kmers)
        kmer_bytes = bytearray()
        alt_bytes = bytearray()
        alt_off = np.zeros(n_alts + 1, dtype=np.int32)
        a = 0
        for kmer in kmers:
            for alt in rows[kmer][0]:
                assert len(alt) > 1 and kmer[0] == alt[0] and kmer[-1] == alt[-1]  # error_model.py:189,195
                kmer_bytes += kmer.encode('ascii')
                alt_bytes += alt.encode('ascii')
                a += 1
                alt_off[a] = len(alt_bytes)
        kmer_arr = np.frombuffer(bytes(kmer_bytes), dtype=np.uint8)
        alt_arr = np.frombuffer(bytes(alt_bytes), dtype=np.uint8)
        slots_all = np.zeros(n_alts * k, dtype=np.uint32)
        same_all = np.zeros(n_alts, dtype=np.uint8)
        pool = np.zeros(max(len(alt_bytes), 16), dtype=np.uint8)
        pool_len = ctypes.c_int64(0)
        rc = _lib.lib().bb_host_align_kmers(k, n_alts, _ptr(kmer_arr), _ptr(alt_arr), _ptr(alt_off), _ptr(slots_all),
                                            _ptr(same_all), _ptr(pool), len(pool), ctypes.byref(pool_len))
        if rc != 0:
            sys.exit('Error: could not align the error model alternatives')
        # rows -> entries, appending the "random change" remainder (error_model.py:151-154).  One append makes the row a
        # fixed point only with CPython >= 3.12's compensated sum() (SURVEY.md 8a a2, measured for all 16 384 rows of
        # every shipped model); older interpreters may append again on later visits, which a static table cannot follow.
        assert sys.version_info >= (3, 12), 'the static remainder entry assumes CPython >= 3.12 (compensated sum())'
        row_off = [0]
        cum, flags, slot_rows, probs_flat = [], [], [], []
        kmer_to_row = np.full(4 ** k, -1, dtype=np.int32) if k <= DENSE_MAX_K else None
        kmer_codes = np.zeros(len(kmers), dtype=np.int64)
        a = 0
        for r, kmer in enumerate(kmers):
            probs = list(rows[kmer][1])
            n = len(probs)
            entry_slots = [slots_all[(a + i) * k:(a + i + 1) * k] for i in range(n)]
            entry_flags = [int(same_all[a + i]) for i in range(n)]
            a += n
            random_change_prob = 1.0 - sum(probs)
            if random_change_prob > 0.0:
                probs.append(random_change_prob)
                entry_slots.append(np.full(k, 0xFFFFFFFF, dtype=np.uint32))
                entry_flags.append(2)
            cum.extend(itertools.accumulate(probs))
            probs_flat.extend(probs)
            flags.extend(entry_flags)
            slot_rows.extend(entry_slots)
            row_off.append(len(cum))
            code = 0
            for c in kmer:
                code = code * 4 + _CODE[c]
            if kmer_to_row is not None:
                kmer_to_row[code] = r
            kmer_codes[r] = code
        self._tables = {
            'row_off': np.asarray(row_off, dtype=np.int32),
            'cum': np.asarray(cum, dtype=np.float64),
            'flags': np.asarray(flags, dtype=np.uint8),
            'slots': np.ascontiguousarray(np.concatenate(slot_rows).astype(np.uint32)),
            'pool': np.ascontiguousarray(pool[:max(int(pool_len.value), 1)]),
            'probs': np.asarray(probs_flat, dtype=np.float64),
            'kmer_codes': kmer_codes,
        }
        if kmer_to_row is not None:
            self._tables['kmer_to_row'] = kmer_to_row

    def save_tables(self, path):
        t = self._tables
        np.savez_compressed(str(path), k=np.int32(self.kmer_size), **t)

    # ------------------------------------------------------------------------------------------ surface
    def to_device_tables(self):
        """Flat arrays for bb_upload_error_model(_kmers) / the oracle. 'random' has no tables.  `index` says how the
        k-mers are found: 'dense' (kmer_to_row[4^k], k <= 12) or 'hash' (kmer_codes only, for the library's hash
        table)."""
        if self.type == 'random':
            return {'k': 1, 'type': 0, 'index': None}
        t = dict(self._tables)
        t['k'] = self.kmer_size
        t['type'] = 1
        t['index'] = 'dense' if 'kmer_to_row' in t else 'hash'
        return t

    def _kmer_of_row(self, r):
        code = int(self._tables['kmer_codes'][r])
        k = self.kmer_size
        return ''.join('ACGT'[(code >> (2 * (k - 1 - j))) & 3] for j in range(k))

    def _materialise_dicts(self):
        """`alternatives` / `probabilities` as the reference holds them right after loading
        (error_model.py:129-130): the remainder entry is not part of the loaded lists."""
        alts, probs = {}, {}
        t = self._tables
        k = self.kmer_size
        for r in range(len(t['row_off']) - 1):
            kmer = self._kmer_of_row(r)
            e0, e1 = int(t['row_off'][r]), int(t['row_off'][r + 1])
            row_alts, row_probs = [], []
            for e in range(e0, e1):
                if t['flags'][e] & 2:
                    continue
                row_alts.append([decode_slot(s, t['pool']) for s in t['slots'][e * k:(e + 1) * k]])
                row_probs.append(float(t['probs'][e]))
            alts[kmer], probs[kmer] = row_alts, row_probs
        self._alternatives, self._probabilities = alts, probs

    @property
    def alternatives(self):
        if self._alternatives is None:
            self._materialise_dicts()
        return self._alternatives

    @property
    def probabilities(self):
        if self._probabilities is None:
            self._materialise_dicts()
        return self._probabilities

    def add_errors_to_kmer(self, kmer):
        """error_model.py:135-160 for a single k-mer on the host with the `random` module (plugin surface for
        callers and tests; the simulation itself samples these tables on the GPU)."""
        if self.type == 'random':
            return add_one_random_change(kmer)
        if kmer not in self.alternatives:
            return add_one_random_change(kmer)
        alts = self.alternatives[kmer]
        probs = self.probabilities[kmer]
        random_change_prob = 1.0 - sum(probs)
        if random_change_prob > 0.0:
            alts.append(None)
            probs.append(random_change_prob)
        alt = random.choices(alts, weights=probs)[0]
        if alt is None:
            return add_one_random_change(kmer)
        return alt


def add_one_random_change(kmer):
    """error_model.py:163-176."""
    result = [x for x in kmer]
    error_type = random.choice(['s', 'i', 'd'])
    error_pos = random.randint(0, len(kmer) - 1)
    if error_type == 's':
        result[error_pos] = get_random_different_base(result[error_pos])
    elif error_type == 'i':
        if random_chance(0.5):
            result[error_pos] = result[error_pos] + get_random_base()
        else:
            result[error_pos] = get_random_base() + result[error_pos]
    else:
        result[error_pos] = ''
    return result


def align_kmers(kmer, alt):
    """error_model.py:179-229 for one pair (same slot list the table builder produces)."""
    assert len(kmer) > 2
    assert len(alt) > 1
    assert kmer[0] == alt[0] and kmer[-1] == alt[-1]
    k = len(kmer)
    kmer_arr = np.frombuffer(kmer.encode('ascii'), dtype=np.uint8)
    alt_arr = np.frombuffer(alt.encode('ascii'), dtype=np.uint8)
    alt_off = np.asarray([0, len(alt)], dtype=np.int32)
    slots = np.zeros(k, dtype=np.uint32)
    same = np.zeros(1, dtype=np.uint8)
    pool = np.zeros(len(alt) + 16, dtype=np.uint8)
    pool_len = ctypes.c_int64(0)
    rc = _lib.lib().bb_host_align_kmers(k, 1, _ptr(kmer_arr), _ptr(alt_arr), _ptr(alt_off), _ptr(slots), _ptr(same),
                                        _ptr(pool), len(pool), ctypes.byref(pool_len))
    assert rc == 0
    return [decode_slot(s, pool) for s in slots]
