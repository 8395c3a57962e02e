"""
Descriptor checks of bb_batch_upload.  A batch is checked as a whole before its reads are dealt out over the workers,
so every kind of invalid descriptor gives the same status and message whether the batch stays on one worker (< 64
reads per worker) or is split, with the bad read dealt to a worker other than 0.  A batch uploaded before the models
gets BB_ERR_STATE.  After each refusal the same context still runs valid batches to the oracle's reads.
"""
import ctypes

import numpy as np
import pytest

from conftest import load_models

pytestmark = pytest.mark.gpu

SEED = 91
BB_ERR_STATE, BB_ERR_ARG = -3, -2
REF_LEN = 5000
N_WORKERS = 2              # pinned by the fixtures (BADREAD_B200_SUBBATCHES); 2 workers form no head batch
SMALL, SPLIT = 8, 64 * N_WORKERS + 2   # < 64 reads per worker stay on worker 0; the split count is even


def _dna(rnd, n):
    return np.frombuffer(b'ACGT', dtype=np.uint8)[rnd.randint(0, 4, n)].tobytes().decode('ascii')


def _reads(n, seed):
    """n literal reads of at least 403 bases; the last one, which the cases break, is much shorter (300 bases here, 310
    with its reference segment), so a split batch deals it last: to worker 1 (longest first, round robin over an even
    count).  _upload checks that."""
    rnd = np.random.RandomState(seed)
    return [(_dna(rnd, 400 + 3 * (n - i) if i < n - 1 else 300), 0.9, 1000 + i) for i in range(n)]


def _batch(reads):
    from badread_b200.engine import FragmentBatch
    batch = FragmentBatch()
    for frag, ident, ri in reads[:-1]:
        batch.add_literal_read(ri, frag, ident)
    frag, ident, ri = reads[-1]   # the read the cases break: a literal and a reference segment
    batch.add_literal_segment(frag)
    batch.add_ref_segment(REF_LEN - 10, 10, False)
    batch.end_read(ri, ident)
    return batch


def _break(kind, so, seg):
    last = len(so) - 2          # the last read's segments: [so[last], so[last + 1])
    lit, ref = so[last], so[last] + 1
    if kind == 'seg_off':
        so[last + 1] = so[last] - 1
    elif kind == 'negative_len':
        seg['len'][lit] = -1
    elif kind == 'negative_src':
        seg['src'][ref] = -5
    elif kind == 'kind':
        seg['kind'][lit] = 7
    elif kind == 'literal_range':
        seg['len'][lit] += 1
    elif kind == 'reference_range':
        seg['src'][ref] = REF_LEN - 9


CASES = {
    'seg_off': 'seg_off must be non-decreasing',
    'negative_len': 'negative segment',
    'negative_src': 'negative segment',
    'kind': 'unknown segment kind',
    'literal_range': 'literal segment out of range',
    'reference_range': 'reference segment out of range',
}


def _upload(eng, batch, kind=None):
    """(status, bb_last_error) of bb_batch_upload with the descriptors broken as `kind` says."""
    ri, so, segs, lit, lit_len, ti = batch._build_arrays()   # fresh arrays: the batch's cached ones stay intact
    so = so.copy()
    seg = np.frombuffer(segs, dtype=np.dtype([('src', np.int64), ('len', np.int32), ('kind', np.int32)]))
    if kind:
        _break(kind, so, seg)
    if len(ri) == SPLIT and kind != 'seg_off':   # where bb_batch_upload deals the broken read: longest first, round robin
        lens = [int(seg['len'][so[r]:so[r + 1]].sum()) for r in range(len(ri))]
        order = sorted(range(len(ri)), key=lambda r: -lens[r])   # stable, as the library's
        assert order.index(len(ri) - 1) % N_WORKERS != 0, 'the broken read must go to a worker other than 0'
    rc = eng._lib.bb_batch_upload(eng._ctx, len(ri), ri.ctypes.data, so.ctypes.data, ctypes.cast(segs, ctypes.c_void_p),
                                  lit.ctypes.data, lit_len, ti.ctypes.data)
    msg = eng._lib.bb_last_error(eng._ctx)
    return rc, msg.decode() if msg else ''


def _fragment(ref, frag):
    return frag + ref[REF_LEN - 10:]


def _engine(mp):
    from badread_b200.engine import Engine
    mp.setenv('BADREAD_B200_SUBBATCHES', str(N_WORKERS))
    mp.delenv('BADREAD_B200_HEAD_WORKER', raising=False)
    return Engine(device=0, seed=SEED)


@pytest.fixture(scope='module')
def setup():
    from oracle import oracle as O
    em, qm = load_models('nanopore2023', 'nanopore2023')
    ref = _dna(np.random.RandomState(5), REF_LEN)
    with pytest.MonkeyPatch.context() as mp:
        eng = _engine(mp)
    yield eng, em, qm, ref, O.Oracle(em, qm)
    eng.close()


def _check_run(eng, orc, ref, reads):
    res, _ = eng.sequence_batch(_batch(reads))
    for i, (frag, ident, ri) in enumerate(reads):
        full = _fragment(ref, frag) if i == len(reads) - 1 else frag
        s, q, _ = orc.sequence_fragment(full, ident, SEED, read_index=ri)
        assert res.read(i) == (s, q), f'read {i} differs from the oracle'


def test_models_first(monkeypatch):
    eng = _engine(monkeypatch)
    try:
        for n in (SMALL, SPLIT):
            rc, msg = _upload(eng, _batch(_reads(n, n)))
            assert (rc, msg) == (BB_ERR_STATE, 'upload the error and qscore models first')
    finally:
        eng.close()


@pytest.mark.parametrize('kind', sorted(CASES))
def test_invalid_descriptor_same_on_both_paths(setup, kind):
    eng, em, qm, ref, orc = setup
    eng.upload_reference(ref.encode('ascii'))
    eng.set_error_model(em)
    eng.set_qscore_model(qm)
    small, split = _reads(SMALL, 1), _reads(SPLIT, 2)
    got = [_upload(eng, _batch(reads), kind) for reads in (small, split)]
    assert got[0] == got[1] == (BB_ERR_ARG, CASES[kind])
    for reads in (small, split):   # the same context still runs both batches, valid, on one worker and split
        _check_run(eng, orc, ref, reads)
