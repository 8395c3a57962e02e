"""The return codes and bb_last_error() messages of the context entry points.

CPU tier: every entry point that takes a context refuses a null one with BB_ERR_ARG before it touches a device, and
bb_create without a device says so.  Both run in a child process that sees no CUDA device, so a call that reached the
device would fail with BB_ERR_CUDA instead.

GPU tier: one call per refusal on a fresh engine, each checked byte for byte, and then a seeded batch on the same engine
gives the reads a fresh engine gives."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import load_models

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
BB_OK, BB_ERR_CUDA, BB_ERR_ARG, BB_ERR_STATE, BB_ERR_CAPACITY = 0, -1, -2, -3, -4

# every entry point that takes a bb_ctx * (bb_comm_init_all and bb_allreduce_bases_all take an array of them)
CONTEXT_CALLS = ['bb_upload_reference', 'bb_download_reference', 'bb_fasta_parse', 'bb_last_gzip_stats', 'bb_fasta_headers',
                 'bb_fasta_reference', 'bb_upload_error_model', 'bb_upload_error_model_kmers', 'bb_load_error_model_file',
                 'bb_download_error_model', 'bb_upload_qscore_model', 'bb_upload_qscore_model_cigars', 'bb_synchronize',
                 'bb_bgzf_compress', 'bb_batch_upload', 'bb_batch_run', 'bb_last_run_retries', 'bb_last_run_work',
                 'bb_last_run_ms', 'bb_trace_dump', 'bb_fetch_last_batch_results', 'bb_fetch_last_batch', 'bb_sequence_batch',
                 'bb_bam_build', 'bb_bam_compress_device', 'bb_bam_fetch_records', 'bb_bam_compress', 'bb_align_path',
                 'bb_get_qscores', 'bb_comm_init_rank', 'bb_comm_init_all', 'bb_allreduce_bases', 'bb_allreduce_bases_all']

# Run with no CUDA device visible: each call with a null context (every other argument null or 0), then bb_create.
_CHILD = r'''
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from badread_b200 import _lib
L = _lib.lib()
out = {}
for name in json.loads(sys.argv[2]):
    fn = getattr(L, name)
    out[name] = fn(*[None if t is not ctypes.c_int and t is not ctypes.c_int32 and t is not ctypes.c_int64
                     and t is not ctypes.c_uint64 else 0 for t in fn.argtypes])
out['bb_destroy'] = L.bb_destroy(None)
out['bb_launch_count'] = L.bb_launch_count(None)
out['error_before'] = L.bb_last_error(None).decode()
ctx = ctypes.c_void_p()
out['bb_create'] = L.bb_create(ctypes.byref(ctx), 0, 1)
out['create_ctx'] = ctx.value
out['error_after'] = L.bb_last_error(None).decode()
print(json.dumps(out))
'''


@pytest.fixture(scope='module')
def no_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, '-c', _CHILD, ROOT, json.dumps(CONTEXT_CALLS)], env=env, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize('name', CONTEXT_CALLS)
def test_null_context_is_refused(no_device, name):
    assert no_device[name] == BB_ERR_ARG


def test_null_context_getters(no_device):
    assert no_device['bb_destroy'] == BB_OK
    assert no_device['bb_launch_count'] == 0
    assert no_device['error_before'] == ''   # bb_last_error(NULL) is the creation message: none yet


def test_create_without_device(no_device):
    assert no_device['bb_create'] == BB_ERR_CUDA
    assert no_device['create_ctx'] is None
    msg = no_device['error_after']
    assert msg.startswith('no CUDA device available: ') and msg.endswith(' (badread_b200 has no CPU path)'), msg


# ---- GPU tier -----------------------------------------------------------------------------------------------------
SEED = 23
I32, I64 = ctypes.c_int32, ctypes.c_int64


def _refusals(L, ctx):
    """(name, call) for one refusal of each kind; call returns (rc, extra outputs to check)."""
    byref = ctypes.byref

    def fasta_parse_then_out_of_range():
        text = b'>a\nACGT\n'
        nh, tb, nk = I32(), I64(), I64()
        assert L.bb_fasta_parse(ctx, text, len(text), 0, byref(nh), byref(tb), byref(nk)) == BB_OK
        assert (nh.value, nk.value) == (1, 4)
        lo, hi = (I64 * 1)(0), (I64 * 1)(5)
        return L.bb_fasta_reference(ctx, 1, lo, hi), None

    def bgzf_short():
        data = b'ACGT' * 25
        n_out, n_cons = I64(-1), I64(-1)
        rc = L.bb_bgzf_compress(ctx, data, len(data), 0, 1, None, 0, byref(n_out), byref(n_cons))
        return rc, (n_out.value, n_cons.value, L.bb_bgzf_bound(len(data)))

    def bam_fetch():
        n = I64(-1)
        return L.bb_bam_fetch_records(ctx, None, None, 0, byref(n)), n.value

    def qscores():
        s = b'ACGTACGT'
        qual = (ctypes.c_uint8 * len(s))()
        return L.bb_get_qscores(ctx, 0, s, len(s), s, len(s), qual, None, None), None

    def align_empty():
        return L.bb_align_path(ctx, b'A', 0, b'ACGT', 4, None, 0, None, None), None

    return [
        ('bb_fasta_headers', lambda: (L.bb_fasta_headers(ctx, None, 0, None, None, 0), None),
         (BB_ERR_STATE, 'bb_fasta_headers: no FASTA parsed (bb_fasta_parse)', None)),
        ('bb_fasta_reference', lambda: (L.bb_fasta_reference(ctx, 0, None, None), None),
         (BB_ERR_STATE, 'bb_fasta_reference: no FASTA parsed (bb_fasta_parse)', None)),
        ('bb_fasta_reference_range', fasta_parse_then_out_of_range,
         (BB_ERR_ARG, 'bb_fasta_reference: contig out of range', None)),
        ('bb_upload_error_model', lambda: (L.bb_upload_error_model(ctx, 13, 1, None, 0, 0, None, None, None, None, None, 0), None),
         (BB_ERR_ARG, 'error model: k must be 1..12', None)),
        ('bb_download_error_model', lambda: (L.bb_download_error_model(ctx, *[None] * 8), None),
         (BB_ERR_STATE, 'bb_download_error_model: no model installed by bb_load_error_model_file', None)),
        ('bb_upload_qscore_model_cigars', lambda: (L.bb_upload_qscore_model_cigars(ctx, 4, 1, b'M', b'\0' * 8, b'\0' * 8,
                                                                                     b'\0', b'\0' * 8), None),
         (BB_ERR_ARG, 'qscore model: bad arguments', None)),
        ('bb_batch_run', lambda: (L.bb_batch_run(ctx), None), (BB_ERR_STATE, 'bb_batch_run: no batch uploaded', None)),
        ('bb_fetch_last_batch', lambda: (L.bb_fetch_last_batch(ctx, None, None, None, 0, None), None),
         (BB_ERR_STATE, 'bb_fetch_last_batch: nothing to fetch', None)),
        ('bb_last_run_ms', lambda: (L.bb_last_run_ms(ctx, None, None), None), (BB_ERR_STATE, 'no run to time', None)),
        ('bb_last_run_work', lambda: (L.bb_last_run_work(ctx, None, None, 0, None), None),
         (BB_ERR_STATE, 'bb_last_run_work: fetch the batch first', None)),
        ('bb_bam_build', lambda: (L.bb_bam_build(ctx, 0, None, None, 0), None),
         (BB_ERR_STATE, 'bb_bam_build: no fetched batch (bb_fetch_last_batch_results)', None)),
        ('bb_bam_fetch_records', bam_fetch,
         (BB_ERR_STATE, 'bb_bam_fetch_records: no records built since the stream was last compressed or fetched', 0)),
        ('bb_bgzf_compress', bgzf_short,
         (BB_ERR_CAPACITY, 'bb_bgzf_compress: out_cap is less than bb_bgzf_bound of the input', 'bound')),
        ('bb_trace_dump', lambda: (L.bb_trace_dump(ctx, os.devnull.encode()), None),
         (BB_ERR_STATE, 'no trace (set BADREAD_B200_TRACE=1 before bb_create)', None)),
        ('bb_allreduce_bases', lambda: (L.bb_allreduce_bases(ctx, 5, ctypes.byref(I64())), None),
         (BB_ERR_STATE, 'bb_allreduce_bases: no communicator (bb_comm_init_rank)', None)),
        ('bb_get_qscores', qscores, (BB_ERR_STATE, 'upload the qscore model first', None)),
        ('bb_align_path', align_empty, (BB_ERR_ARG, 'bb_align_path: empty sequence', None)),
    ]


def _batch():
    from badread_b200.engine import FragmentBatch
    rnd = np.random.RandomState(SEED)
    batch = FragmentBatch()
    for i, n in enumerate((300, 1500, 4000, 900)):
        batch.add_literal_read(i, np.frombuffer(b'ACGT', dtype=np.uint8)[rnd.randint(0, 4, n)].tobytes().decode(), 0.88)
    return batch


def _reads(eng):
    em, qm = load_models('nanopore2023', 'nanopore2023')
    eng.set_error_model(em)
    eng.set_qscore_model(qm)
    res, _ = eng.sequence_batch(_batch())
    return [res.read(i) for i in range(4)]


@pytest.mark.gpu
def test_create_invalid_device():
    from badread_b200 import _lib
    L = _lib.lib()
    ctx = ctypes.c_void_p()
    assert L.bb_create(ctypes.byref(ctx), -1, 1) == BB_ERR_ARG
    assert ctx.value is None
    assert L.bb_last_error(None).decode() == 'invalid device ordinal'


@pytest.mark.gpu
def test_refusals_then_a_batch(monkeypatch):
    from badread_b200 import _lib
    from badread_b200.engine import Engine
    monkeypatch.delenv('BADREAD_B200_TRACE', raising=False)
    L = _lib.lib()
    eng = Engine(device=0, seed=SEED)
    try:
        for name, call, (rc_want, msg_want, extra_want) in _refusals(L, eng._ctx):
            rc, extra = call()
            assert (rc, L.bb_last_error(eng._ctx).decode()) == (rc_want, msg_want), name
            if extra_want == 'bound':   # *n_out = the bound the call asks for, nothing consumed
                assert extra[0] == extra[2] and extra[1] == 0, (name, extra)
            else:
                assert extra == extra_want, name
        got = _reads(eng)
    finally:
        eng.close()
    fresh = Engine(device=0, seed=SEED)
    try:
        assert got == _reads(fresh)
    finally:
        fresh.close()
