"""The return codes and bb_model_error() messages of the loader and model-builder entry points (CPU tier: every case is
answered before the library touches a device).  Invalid arguments are refused before any CUDA call; the BGZF host walk
answers input that is not BGZF and an output buffer that is too small; a successful call clears the message; the
message is per thread; and a message longer than 255 bytes comes back whole."""
import ctypes
import threading
import zlib

import numpy as np
import pytest

from emu import emu_inflate as EI
from test_model_builders_alignments import bgzf_member

VP = ctypes.c_void_p


@pytest.fixture(scope='module')
def L():
    from badread_b200 import _lib
    return _lib.lib()


def _message(L):
    return L.bb_model_error().decode()


def _n_out():
    return ctypes.c_int64(-1)


# one call per entry point with an argument it refuses, and the name its message starts with
INVALID = [
    ('bb_bgzf_decompress', lambda L: L.bb_bgzf_decompress(0, None, -1, None, 0, ctypes.byref(_n_out())), 'bb_bgzf_decompress'),
    ('bb_gzip_decompress', lambda L: L.bb_gzip_decompress(0, None, -1, None, 0, ctypes.byref(_n_out()), 0, None),
     'bb_gzip_decompress'),
    ('bb_fastq_parse', lambda L: L.bb_fastq_parse(0, None, -1, 0, None, None, None), 'bb_fastq_parse'),
    ('bb_flat_build', lambda L: L.bb_flat_build(None, None, 0, None, None, None, None, 0, None, None, None), 'bb_flat_build'),
    ('bb_flat_fetch', lambda L: L.bb_flat_fetch(None, 0, 0, 0, None), 'bb_flat_fetch'),
    ('bb_window_series', lambda L: L.bb_window_series(0, -1, *[None] * 9, 1, 0, 0, 0, None, None, None), 'bb_window_series'),
    ('bb_count_kmer_alternatives', lambda L: L.bb_count_kmer_alternatives(0, 7, 0, *[None] * 8, 16, None, None, None, None, 0,
                                                                         None, None, None, None), 'bb_count_*'),
    ('bb_count_kmer_alternatives_wide', lambda L: L.bb_count_kmer_alternatives_wide(0, 13, 0, *[None] * 8, 16, None, None, None,
                                                                                   None, 0, None, None, None, None), 'bb_count_*'),
    ('bb_count_cigar_qscores', lambda L: L.bb_count_cigar_qscores(0, 9, 6, 0, *[None] * 9, 16, None, None, None, None, None, 0,
                                                                 None, None, None, None), 'bb_count_*'),
    ('bb_aln_parse', lambda L: L.bb_aln_parse(None, 0, 0, 0, None), 'bb_aln_parse'),
]


@pytest.mark.parametrize('call,prefix', [c[1:] for c in INVALID], ids=[c[0] for c in INVALID])
def test_invalid_argument(L, call, prefix):
    from badread_b200 import _lib
    assert call(L) == _lib.BB_ERR_ARG
    assert _message(L) == f'{prefix}: invalid argument'


@pytest.mark.parametrize('data', [b'not BGZF at all', zlib.compress(b'ACGT' * 100), bgzf_member(b'ACGT' * 100)[:-3]],
                         ids=['text', 'zlib', 'truncated'])
def test_bgzf_refusal_is_the_emulators(L, data):
    from badread_b200 import _lib
    with pytest.raises(ValueError) as emu_err:
        EI.decompress(data)
    out = ctypes.create_string_buffer(1 << 12)
    rc = L.bb_bgzf_decompress(0, data, len(data), out, len(out), ctypes.byref(_n_out()))
    assert rc == _lib.BB_ERR_ARG
    assert _message(L) == str(emu_err.value)


def test_bgzf_capacity_from_the_host_walk(L):
    from badread_b200 import _lib
    raw = b'ACGT' * 1000 + b'\n'
    data = bgzf_member(raw[:3000]) + bgzf_member(raw[3000:])
    n_out = _n_out()
    assert L.bb_bgzf_decompress(0, data, len(data), None, 0, ctypes.byref(n_out)) == _lib.BB_ERR_CAPACITY
    assert n_out.value == len(raw)
    assert _message(L) == f'bb_bgzf_decompress: {len(raw)} bytes of output, capacity 0'


def _window_series_empty(L):
    off = np.zeros(1, dtype=np.int64)
    p = off.ctypes.data_as(VP)
    n_points = ctypes.c_int64(-1)
    rc = L.bb_window_series(0, 0, None, None, None, p, p, None, None, None, p, 100, 0, 0, 0, None, None, ctypes.byref(n_points))
    return rc, n_points.value


def _paf_parse(L, text):
    from badread_b200 import _lib
    handle = VP()
    rc = L.bb_aln_parse(text, len(text), _lib.BB_ALN_PAF, 0, ctypes.byref(handle))
    if handle.value:
        L.bb_aln_free(handle)
    return rc


PAF = b'read1\t100\t0\t10\t+\tchr1\t1000\t5\t15\t10\t10\t60\tcg:Z:10M\tAS:i:10\n'


def test_success_clears_the_message(L):
    from badread_b200 import _lib
    L.bb_flat_fetch(None, 0, 0, 0, None)
    assert _message(L) == 'bb_flat_fetch: invalid argument'
    assert _window_series_empty(L) == (_lib.BB_OK, 0)
    assert _message(L) == ''
    L.bb_aln_parse(None, 0, 0, 0, None)
    assert _message(L) != ''
    assert _paf_parse(L, PAF) == _lib.BB_OK
    assert _message(L) == ''


def test_the_message_is_per_thread(L):
    from badread_b200 import _lib
    assert _paf_parse(L, PAF) == _lib.BB_OK
    seen = []

    def fail():
        seen.append(L.bb_gzip_decompress(0, None, -1, None, 0, ctypes.byref(_n_out()), 0, None))
        seen.append(_message(L))

    t = threading.Thread(target=fail)
    t.start()
    t.join()
    assert seen == [_lib.BB_ERR_ARG, 'bb_gzip_decompress: invalid argument']
    assert _message(L) == ''


def test_a_long_message_is_reported_whole(L):
    """A read name of 300 characters in the message of a SAM record whose CIGAR has an N."""
    from badread_b200 import _lib
    name = 'r' * 150 + 'x' * 150
    sam = f'@SQ\tSN:chr1\tLN:1000\n{name}\t0\tchr1\t1\t60\t5M1N5M\t*\t0\t0\tACGTACGTAC\tIIIIIIIIII\tAS:i:10\n'.encode()
    handle = VP()
    assert L.bb_aln_parse(sam, len(sam), 0, 0, ctypes.byref(handle)) == _lib.BB_ERR_ARG
    assert not handle.value
    assert _message(L) == (f'Error: the CIGAR of read {name} has an N operation '
                           '(skipped regions and padding are not supported)')
