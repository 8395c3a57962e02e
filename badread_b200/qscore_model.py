"""
QScoreModel and get_qscores - host side of the qscore model, same plugin surface as
/root/reference/badread/qscore_model.py:178-287 (`scores`, `probabilities`, `kmer_size`, `type`, `get_qscore`)
plus `to_device_tables()` for `bb_upload_qscore_model_cigars`, and the module-level `get_qscores(seq, frag, model)`
(qscore_model.py:32-75) which runs on the GPU through the C ABI.

Device table layout: the CIGAR keys over {=,X,I,D}, of any length, as key_chars / key_off; row_off / scores / cum
per key, cum = list(itertools.accumulate(probabilities)) as random.choices builds it (qscore_model.py:283).  `keys`
also gives each key of at most 31 symbols packed two bits per symbol ('='=0, 'X'=1, 'I'=2, 'D'=3) under a leading 1
bit, the form bb_upload_qscore_model takes; a longer key has no packed form and is 0 there.

Derived from Badread (Copyright 2018 Ryan Wick, rrwick@gmail.com, https://github.com/rrwick/Badread), which is free
software under the GNU General Public License version 3 or later; this file mirrors the named parts of the
reference's interface and is distributed under the same licence (see LICENSE and NOTICE at the repository root).
"""
import ctypes
import itertools
import os
import pathlib
import random
import statistics
import sys

import numpy as np

from . import settings
from .misc import get_open_func

BUILTIN_MODELS = ('nanopore2018', 'nanopore2020', 'nanopore2023', 'pacbio2016', 'pacbio2021')
MODEL_DIR = pathlib.Path(os.path.dirname(os.path.realpath(__file__))) / 'models'
_SYMBOL = {'=': 0, 'X': 1, 'I': 2, 'D': 3}
PACKED_KEY_SYMBOLS = 31    # the most a uint64 holds under its leading 1 bit


def pack_cigar(cigar):
    key = 1
    for c in cigar:
        key = (key << 2) | _SYMBOL[c]
    return key


class QScoreModel(object):

    def __init__(self, model_type_or_filename, output=sys.stderr):
        self.scores, self.probabilities = {}, {}
        self.kmer_size = 1
        self.type = None
        if model_type_or_filename == 'random':
            self.set_up_random_model(output)
        elif model_type_or_filename == 'ideal':
            self.set_up_ideal_model(output)
        elif model_type_or_filename in BUILTIN_MODELS:
            self._load_builtin(model_type_or_filename, output)
        else:
            self.load_from_file(model_type_or_filename, output)
        # qscore_model.py:205-207: the 1-mer cigars must exist or get_qscore could fail
        assert '=' in self.scores
        assert 'X' in self.scores
        assert 'I' in self.scores

    def set_up_random_model(self, output):
        print('\nUsing a random qscore model', file=output)
        self.type = 'random'
        self.kmer_size = 1
        for c in ['=', 'X', 'I']:
            self.scores[c], self.probabilities[c] = \
                uniform_dist_scores_and_probs(settings.RANDOM_QSCORE_MIN, settings.RANDOM_QSCORE_MAX)

    def set_up_ideal_model(self, output):
        print('\nUsing an ideal qscore model', file=output)
        self.type = 'ideal'
        self.kmer_size = 9
        ranks = {'X': (settings.IDEAL_QSCORE_RANK_1_MIN, settings.IDEAL_QSCORE_RANK_1_MAX),
                 'I': (settings.IDEAL_QSCORE_RANK_1_MIN, settings.IDEAL_QSCORE_RANK_1_MAX),
                 '=': (settings.IDEAL_QSCORE_RANK_2_MIN, settings.IDEAL_QSCORE_RANK_2_MAX),
                 '===': (settings.IDEAL_QSCORE_RANK_3_MIN, settings.IDEAL_QSCORE_RANK_3_MAX),
                 '=====': (settings.IDEAL_QSCORE_RANK_4_MIN, settings.IDEAL_QSCORE_RANK_4_MAX),
                 '=======': (settings.IDEAL_QSCORE_RANK_5_MIN, settings.IDEAL_QSCORE_RANK_5_MAX),
                 '=========': (settings.IDEAL_QSCORE_RANK_6_MIN, settings.IDEAL_QSCORE_RANK_6_MAX)}
        for cigar, (lo, hi) in ranks.items():
            self.scores[cigar], self.probabilities[cigar] = uniform_dist_scores_and_probs(lo, hi)

    def _load_builtin(self, name, output):
        """Built-in models ship as models/<name>.qscore.npz (tools/compile_models.py)."""
        path = MODEL_DIR / f'{name}.qscore.npz'
        print(f'\nLoading qscore model from {path}', file=output)
        if not path.is_file():
            sys.exit(f'Error: built-in qscore model {name} is not installed ({path} missing) - '
                     f'run tools/compile_models.py or pass a model filename')
        self.type = 'model'
        with np.load(str(path)) as z:
            self.kmer_size = int(z['kmer_size'])
            keys = bytes(z['key_chars']).decode('ascii')
            key_off, row_off = z['key_off'], z['row_off']
            scores, probs = z['scores'], z['probs']
        for i in range(len(key_off) - 1):
            cigar = keys[key_off[i]:key_off[i + 1]]
            self.scores[cigar] = [int(x) for x in scores[row_off[i]:row_off[i + 1]]]
            self.probabilities[cigar] = [float(x) for x in probs[row_off[i]:row_off[i + 1]]]
        print(f'\r  done: loaded qscore distributions for {len(key_off) - 1} alignments', file=output)

    def load_from_file(self, filename, output):
        """qscore_model.py:246-271."""
        print('\nLoading qscore model from {}'.format(filename), file=output)
        self.type = 'model'
        count = 0
        with get_open_func(filename)(filename, 'rt') as model_file:
            for line in model_file:
                parts = line.strip().split(';')
                try:
                    if parts[0] == 'overall':
                        continue
                    cigar = parts[0]
                    k = len(cigar.replace('D', ''))
                    if k > self.kmer_size:
                        self.kmer_size = k
                    scores_and_probs = [x.split(':') for x in parts[2].split(',') if x]
                    self.scores[cigar] = [int(x[0]) for x in scores_and_probs]
                    self.probabilities[cigar] = [float(x[1]) for x in scores_and_probs]
                    count += 1
                except (IndexError, ValueError):
                    sys.exit(f'Error: {filename} does not seem to be a valid qscore model file')
        print(f'\r  done: loaded qscore distributions for {count} alignments', file=output)

    def save_tables(self, path):
        keys = list(self.scores.keys())
        key_off, row_off = [0], [0]
        scores, probs = [], []
        for cigar in keys:
            key_off.append(key_off[-1] + len(cigar))
            scores.extend(self.scores[cigar])
            probs.extend(self.probabilities[cigar])
            row_off.append(len(scores))
        np.savez_compressed(str(path), kmer_size=np.int32(self.kmer_size),
                            key_chars=np.frombuffer(''.join(keys).encode('ascii'), dtype=np.uint8),
                            key_off=np.asarray(key_off, dtype=np.int32), row_off=np.asarray(row_off, dtype=np.int32),
                            scores=np.asarray(scores, dtype=np.uint8), probs=np.asarray(probs, dtype=np.float64))

    def to_device_tables(self):
        """Flat arrays for bb_upload_qscore_model_cigars and the oracle (key strings, any length); `keys` holds the
        packed form of bb_upload_qscore_model, 0 for a key longer than 31 symbols."""
        keys = list(self.scores.keys())
        packed, key_chars, key_off, row_off = [], [], [0], [0]
        scores, cum = [], []
        for cigar in keys:
            if any(c not in _SYMBOL for c in cigar) or len(cigar) == 0:
                sys.exit(f'Error: qscore model CIGAR {cigar!r} holds symbols other than =XID')
            s, p = self.scores[cigar], self.probabilities[cigar]
            if len(s) == 0 or len(s) != len(p) or min(s) < 0 or max(s) > 93:
                sys.exit(f'Error: qscore model row {cigar} is malformed')
            packed.append(pack_cigar(cigar) if len(cigar) <= PACKED_KEY_SYMBOLS else 0)
            key_chars.append(cigar)
            key_off.append(key_off[-1] + len(cigar))
            scores.extend(s)
            cum.extend(itertools.accumulate(p))
            row_off.append(len(scores))
        return {'kmer_size': int(self.kmer_size), 'n_keys': len(keys),
                'keys': np.asarray(packed, dtype=np.uint64),
                'key_chars': np.frombuffer(''.join(key_chars).encode('ascii'), dtype=np.uint8).copy(),
                'key_off': np.asarray(key_off, dtype=np.int32), 'row_off': np.asarray(row_off, dtype=np.int32),
                'scores': np.asarray(scores, dtype=np.uint8), 'cum': np.asarray(cum, dtype=np.float64)}

    def get_qscore(self, cigar):
        """qscore_model.py:273-287 on the host with the `random` module (plugin surface; the simulation samples
        the same tables on the GPU)."""
        while True:
            assert len(cigar.replace('D', '')) % 2 == 1
            if cigar in self.scores:
                qscore = random.choices(self.scores[cigar], weights=self.probabilities[cigar])[0]
                break
            cigar = cigar[1:-1].strip('D')
        return qscore_val_to_char(qscore)


def get_qscores(seq, frag, qscore_model):
    """qscore_model.py:32-75 on the GPU: returns (qual, actual_identity, identity_by_qscores)."""
    from .engine import default_engine, next_read_index
    assert len(seq) > 0
    eng = default_engine(qscore_model=qscore_model)
    # every call draws from the Philox streams of a fresh read index (successive calls are independent, like the
    # reference's advancing `random` stream; sequence_fragment() numbers its reads from the same counter)
    qual, matches, columns = eng.get_qscores(seq, frag, read_index=next_read_index())
    actual_identity = matches / columns if columns else 0.0
    identity_by_qscores = 1.0 - statistics.mean(qscore_char_to_error_prob(q) for q in qual)
    return qual, actual_identity, identity_by_qscores


def uniform_dist_scores_and_probs(bottom_q, top_q):
    count = top_q - bottom_q + 1
    return list(range(bottom_q, top_q + 1)), [1 / count] * count


def qscore_char_to_val(q):
    return ord(q) - 33


def qscore_val_to_char(q):
    return chr(q + 33)


def qscore_val_to_error_prob(q):
    return 10.0 ** (-q / 10.0)


def qscore_char_to_error_prob(q):
    return qscore_val_to_error_prob(qscore_char_to_val(q))


def align_sequences_from_edlib_cigar(seq, frag, cigar, gap_char='-'):
    """qscore_model.py:290-311."""
    import re
    aligned_seq, aligned_frag, full_cigar = [], [], []
    seq_pos, frag_pos = 0, 0
    for part in re.findall(r'\d+[IDX=]', cigar):
        kind, size = part[-1], int(part[:-1])
        if kind in '=X':
            aligned_seq.append(seq[seq_pos:seq_pos + size])
            aligned_frag.append(frag[frag_pos:frag_pos + size])
            seq_pos += size
            frag_pos += size
        elif kind == 'I':
            aligned_seq.append(seq[seq_pos:seq_pos + size])
            aligned_frag.append(gap_char * size)
            seq_pos += size
        else:
            aligned_seq.append(gap_char * size)
            aligned_frag.append(frag[frag_pos:frag_pos + size])
            frag_pos += size
        full_cigar.append(kind * size)
    return ''.join(aligned_seq), ''.join(aligned_frag), ''.join(full_cigar)
