"""
The counting kernels of the model builders on the GPU against the count made from the definition
(tests/model_counts_ref.py; tests/test_model_counts.py pins it to the unmodified reference and runs the same comparisons
under the emulator, which runs one thread at a time): model files and decoded raw entries under real contention, at
scale, through the capacity paths of the table and of the overflow list, from a BAM of several hundred BGZF members, and
against the unmodified reference's digests of tests/golden/golden_model_stress.json.  Run with -s for, per data set, the
windows counted, the distinct keys, the overflow windows and how often the table was doubled.

Data sets (all from seeds, sizes as generated; the window and key counts are what the definitional count reports and do
not depend on the device):
  edges         21 hand-built alignments: read k-mers of max_len and max_len + 1 bases at k = 3, 7, 12, 13, 16; CIGAR windows
                of 29 and 30 symbols; qualities '!' and '~'; N in the read; fewer reference bases than k, fewer read
                bases than the window; alignments starting / ending with I and with D; D next to I; two D runs in a row
  hot           3 000 error-free alignments of 200 bases over homopolymers and dinucleotide repeats, one quality value:
                0.58 M error-model windows per k, 2.94 M CIGAR windows at k = 9, fewer than a hundred distinct keys; 300 + 300
                alignments with one inserted C / G give alternatives and CIGARs with equal counts
  diverse       400 alignments of 1 250 reference bases with 25-30 % errors: 0.49 M error-model windows and 2.5 M CIGAR
                windows (k = 9); 257 116 distinct error-model keys at k = 12, 136 659 distinct CIGARs at k = 9 / max_del = 6
  long          one alignment of 150 kb with a single M run of 100 kb, alone and in the middle of diverse
  many          70 000 alignments of 102-105 columns: 7.2 M windows per pass
"""
import ctypes
import json
import types

import numpy as np
import pytest

import model_counts_ref as R
from test_model_counts import (ERROR_KS, QSCORE_KS, STRESS, Case, check_error_model, check_qscore_model, decode_cigar_entries,
                               decode_kmer_entries, run_builder)
from test_model_builders_alignments import bam_bytes, bgzf, paf_to_records

pytestmark = pytest.mark.gpu

WHICH = {'kmers': ('bb_count_kmer_alternatives', 11), 'kmers_wide': ('bb_count_kmer_alternatives_wide', 11),
         'cigars': ('bb_count_cigar_qscores', 13)}        # entry point, position of table_cap among its arguments


@pytest.fixture(scope='module')
def mb():
    from badread_b200 import model_builders
    return model_builders


@pytest.fixture(scope='module')
def cases(tmp_path_factory):
    made = {}

    def get(name):
        if name not in made:
            if name == 'diverse_long':
                div, d = R.diverse(400), R.Dataset()
                d.refs.update(div.refs)
                d.extend(R.long_alignment())
                half = len(div.paf) // 2
                d.reads, d.paf = div.reads[:half] + d.reads + div.reads[half:], div.paf[:half] + d.paf + div.paf[half:]
            else:
                d = {'edges': R.edges, 'hot': R.hot, 'long': R.long_alignment, 'many': R.many, 'stress': R.stress_mix,
                     'diverse': lambda: R.diverse(400), 'diverse_big': lambda: R.diverse(1500, seed=18),
                     'capacity': lambda: R.edges().extend(R.diverse(100, seed=17))}[name]()
            made[name] = Case(d, tmp_path_factory.mktemp(name))
        return made[name]
    return get


@pytest.fixture
def calls(monkeypatch):
    """(entry point, table_cap, return code) of every count call the library gets."""
    from badread_b200 import _lib
    L, seen = _lib.lib(), []
    for name, cap_at in WHICH.values():
        def wrapped(*a, _inner=getattr(L, name), _name=name, _cap_at=cap_at):
            rc = _inner(*a)
            seen.append((_name, int(a[_cap_at]), rc))
            return rc
        monkeypatch.setattr(L, name, wrapped)
    return seen


def doublings(calls):
    return sum(1 for a, b in zip(calls, calls[1:]) if b[1] == 2 * a[1])


def _decoded(which, raw, k):
    entries = decode_cigar_entries(raw) if which == 'cigars' else decode_kmer_entries(raw, k)
    return entries, raw[3].tolist(), sorted(zip(*(o.tolist() for o in raw[4])))


RUNS = [('edges', 'error', k) for k in ERROR_KS] + [('edges', 'qscore', kd) for kd in QSCORE_KS] + \
    [('hot', 'error', 7), ('hot', 'error', 13), ('hot', 'qscore', (9, 6)),
     ('diverse', 'error', 12), ('diverse', 'error', 16), ('diverse', 'qscore', (9, 6)),
     ('long', 'error', 7), ('long', 'qscore', (9, 6)), ('diverse_long', 'error', 7), ('diverse_long', 'qscore', (5, 3)),
     ('many', 'error', 7), ('many', 'qscore', (1, 6))]


@pytest.mark.parametrize('data,which,param', RUNS, ids=[f'{d}-{w}-{p}' for d, w, p in RUNS])
def test_device_counts_the_definition(mb, cases, calls, data, which, param):
    """The model file equals the definitional one and every entry the count call returned - count or histogram, first
    occurrence, `overall`, overflow list - equals the definitional dicts.  On `hot` every thread of every CTA adds to the
    same few words, and the order of the tied alternatives is the atomicMin's alone; on `diverse` the table takes some
    hundred thousand distinct keys; `long` has one thread spread a 100 kb run and a CTA loop 600 times over its windows;
    `many` has more CTAs than 65 535 and alignment numbers beyond 16 bits in the stamps."""
    case = cases(data)
    if which == 'error':
        n_keys, n_ovf = check_error_model(mb, case, param)
        windows = case.error(param)[2]
    else:
        n_keys, n_ovf = check_qscore_model(mb, case, *param)
        windows = case.qscore(*param)[3]
    print(f'\n{data} {which} {param}: {len(case.alns)} alignments, {windows} windows, {n_keys} distinct keys in the table, '
          f'{n_ovf} overflow windows, table doubled {doublings(calls)} times from {calls[0][1]} slots')


def test_default_table_growth(mb, cases, calls):
    """The qscore table is not sized from the input: it starts at 2^18 slots whatever comes.  The 136 659 distinct CIGARs
    of `diverse` (k = 9, max_del = 6; 2.5 M windows) fit it, so there the default call never grows.  The 317 207 of 1 500 such
    alignments (9.3 M windows) do not: the default call goes through "table full, double, count again" by itself and must end with
    the entries of a call that started large enough."""
    flat = cases('diverse_big').flat
    got = _decoded('cigars', mb._count('cigars', flat, 9, 6), 9)
    n, grown = len(got[0]), doublings(calls)
    print(f'\n1 500 diverse alignments, qscore (9, 6): {n} distinct CIGAR keys, table doubled {grown} times from {calls[0][1]} slots')
    assert calls[0][1] == 1 << 18 and calls[-1][1] == (1 << 18) << grown
    assert n > 1 << 18 and grown >= 1
    assert got == _decoded('cigars', mb._count('cigars', flat, 9, 6, cap=1 << 20), 9)


CAPACITY = [('kmers', 12, 0), ('kmers_wide', 16, 0), ('cigars', 9, 6)]


@pytest.mark.parametrize('which,k,max_del', CAPACITY, ids=[c[0] for c in CAPACITY])
def test_capacity_paths_give_the_same_entries(mb, cases, calls, which, k, max_del):
    """A table of 16 and of 256 slots and an overflow list of 0 and of 1 entries: CTAs give up in the middle of the grid
    while others insert, the host doubles the table, sizes the list from the reported count and counts again - and ends
    with the entries of the generously sized run, one for one (the edges and 100 diverse alignments)."""
    case = cases('capacity')
    want = _decoded(which, mb._count(which, case.flat, k, max_del), k)
    assert want[2], 'the data set has overflow windows'
    for cap, ovf_cap in ((16, 0), (256, 1)):
        del calls[:]
        got = _decoded(which, mb._count(which, case.flat, k, max_del, cap=cap, ovf_cap=ovf_cap), k)
        assert got == want, (cap, ovf_cap)
        assert calls[0][1] == cap and doublings(calls) >= 4 and calls[-1][2] == 0
        print(f'\n{which} from {cap} slots / {ovf_cap} overflow entries: {len(calls)} calls, table doubled {doublings(calls)} times, '
              f'{len(want[0])} keys, {len(want[2])} overflow windows')


def _direct_call(which, flat, k, max_del, cap, ovf_cap):
    """One call of the entry point itself -> (return code, n_entries, n_ovf, bb_model_error())."""
    from badread_b200 import _lib
    L = _lib.lib()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    keys = np.empty(cap * (2 if which == 'kmers_wide' else 1), dtype=np.uint64)
    first, counts = np.empty(cap, dtype=np.uint64), np.empty(cap * (94 if which == 'cigars' else 1), dtype=np.uint32)
    ovf = [np.empty(max(ovf_cap, 1), dtype=np.int32) for _ in range(3)]
    overall = np.zeros(94, dtype=np.uint64)
    n, m = ctypes.c_int64(0), ctypes.c_int64(0)
    head = [0, k] + ([max_del] if which == 'cigars' else []) + [flat.n, p(flat.read)] + ([p(flat.qual)] if which == 'cigars' else [])
    rc = getattr(L, WHICH[which][0])(*head, p(flat.read_off), p(flat.ref), p(flat.ref_off), p(flat.ops), p(flat.op_read0),
                                     p(flat.op_ref0), p(flat.ops_off), cap, p(keys), p(first), p(counts), ctypes.byref(n),
                                     *([p(overall)] if which == 'cigars' else []), ovf_cap, p(ovf[0]), p(ovf[1]), p(ovf[2]),
                                     ctypes.byref(m))
    return rc, n.value, m.value, L.bb_model_error().decode()


@pytest.mark.parametrize('which,k,max_del', CAPACITY, ids=[c[0] for c in CAPACITY])
def test_entry_points_report_which_capacity_was_too_small(mb, cases, which, k, max_del):
    """The designed status returns of one call each: a table that cannot take the keys, and an overflow list of one entry
    with a table that can - the latter with the true number of overflow windows, which is what the host sizes the list
    from."""
    from badread_b200 import _lib
    flat = cases('capacity').flat
    n_ovf = len(mb._count(which, flat, k, max_del)[4][0])
    assert n_ovf > 1
    rc, _, _, message = _direct_call(which, flat, k, max_del, 16, 1 << 16)
    assert (rc, message) == (_lib.BB_ERR_CAPACITY, 'bb_count_*: table too small')
    rc, _, m, message = _direct_call(which, flat, k, max_del, 1 << 19, 1)
    assert (rc, m, message) == (_lib.BB_ERR_CAPACITY, n_ovf, 'bb_count_*: overflow list too small')


@pytest.mark.parametrize('data,which,k,max_del', [('hot', 'kmers', 7, 0), ('hot', 'cigars', 9, 6), ('diverse', 'kmers_wide', 13, 0),
                                                  ('diverse', 'cigars', 9, 6)])
def test_two_runs_give_the_same_entries(mb, cases, data, which, k, max_del):
    """Nothing in the counts or in `first` depends on which CTA ran when (the order of the compacted output may)."""
    flat = cases(data).flat
    assert _decoded(which, mb._count(which, flat, k, max_del), k) == _decoded(which, mb._count(which, flat, k, max_del), k)


def test_models_from_a_bam_of_the_diverse_set(mb, cases, tmp_path):
    """`diverse` as a BAM whose BGZF members hold 2 000 to 4 321 bytes (several hundred of them, records straddling them),
    inflated on the GPU; both models built from it without --reads equal the definitional files."""
    case = cases('diverse')
    reads = {name: (seq, qual) for name, (seq, qual) in case.reads.items()}
    with open(case.args.alignment) as f:
        records = paf_to_records(f.read().splitlines(), reads)
    stream = bgzf(bam_bytes(records, case.refs), sizes=[3000, 2000, 4321])
    assert stream.count(b'\x1f\x8b\x08\x04') >= 300
    (tmp_path / 'reads.bam').write_bytes(stream)
    args = dict(vars(case.args), alignment=str(tmp_path / 'reads.bam'), reads=None)
    args = types.SimpleNamespace(**args)
    assert run_builder(mb, 'error', args, k_size=7, max_alt=25) == R.error_model_text(case.error(7)[0], 25)
    hist, _, overall, _ = case.qscore(9, 6)
    assert run_builder(mb, 'qscore', args, k_size=9, max_del=6, min_occur=2, max_output=100000) == \
        R.qscore_model_text(hist, overall, 2, 100000)


@pytest.mark.parametrize('name,which,kw', R.STRESS_MODELS, ids=[m[0] for m in R.STRESS_MODELS])
def test_device_writes_the_references_files_for_the_stress_mix(mb, cases, name, which, kw):
    """The unmodified reference's files for the hot + diverse + edges mix (oracle/make_golden_model_stress.py), by digest."""
    with open(STRESS) as f:
        want = json.load(f)[name]
    assert R.stress_digest(run_builder(mb, which, cases('stress').args, **kw)) == want
