"""The model builders with SAM and BAM alignments on the GPU: the BAM inflated by bb_bgzf_decompress and the windows counted
by the counting kernels give the reference's model files; the command line builds from a BAM alone; the device's
inflated bytes equal the emulator's and gzip's on a multi-megabyte stream of `simulate --gzip`; corrupt members give
BB_ERR_ARG (the same cases tests/test_model_builders_alignments.py runs under the emulator first)."""
import gzip
import os
import subprocess
import sys

import pytest

from emu import emu_inflate as EI
from test_model_builders import _golden
from test_model_builders_alignments import DATA, MODELS, _args, _run, corrupt_cases, inputs  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.realpath(__file__))


@pytest.mark.parametrize('with_reads', [True, False], ids=['reads', 'no_reads'])
@pytest.mark.parametrize('name,kw', MODELS, ids=[m[0] for m in MODELS])
def test_golden_models_from_bam_on_the_device(inputs, with_reads, name, kw):  # noqa: F811
    from badread_b200 import model_builders as mb
    fn = mb.make_error_model if name.startswith('error') else mb.make_qscore_model
    assert _run(fn, _args(inputs.dir / 'reads.bam', with_reads, **kw)) == _golden(name)


@pytest.mark.parametrize('name,kw', [MODELS[1], MODELS[4]], ids=[MODELS[1][0], MODELS[4][0]])
def test_golden_models_from_sam_on_the_device(inputs, name, kw):  # noqa: F811
    from badread_b200 import model_builders as mb
    fn = mb.make_error_model if name.startswith('error') else mb.make_qscore_model
    assert _run(fn, _args(inputs.dir / 'reads.sam', False, **kw)) == _golden(name)


def test_command_line_from_a_bam_alone(inputs):  # noqa: F811
    p = subprocess.run([sys.executable, '-m', 'badread_b200', 'error_model', '--reference', os.path.join(DATA, 'ref.fasta'),
                        '--alignment', str(inputs.dir / 'reads.bam')], cwd=os.path.join(HERE, '..'),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert p.returncode == 0, p.stderr.decode()[-500:]
    assert p.stdout.decode() == _golden('error_model_k7')
    assert b'Loading alignments' in p.stderr and b'Choosing best alignment per read' in p.stderr


def test_device_inflate_equals_emulator_and_gzip(tmp_path):
    """A multi-megabyte FASTQ of `simulate --gzip` (its members compressed on the GPU) inflated on the device."""
    from badread_b200.bgzf import decompress
    from test_gpu_bgzf import _run as simulate_run
    comp = simulate_run(tmp_path, ['--quantity', '80x'], gz=True)
    want = gzip.decompress(comp)
    assert len(want) > 4 << 20
    got = decompress(comp)
    assert bytes(got) == want
    assert EI.decompress(comp) == got
    assert decompress(b'') == bytearray()


def test_device_inflate_of_zlib_members(inputs):  # noqa: F811
    from badread_b200.bgzf import decompress
    from test_model_builders_alignments import bgzf
    for sizes in ([65280], [1, 333, 65280, 4097, 0], [100]):
        stream = bgzf(inputs.raw_bam, sizes)
        assert bytes(decompress(stream)) == inputs.raw_bam


@pytest.mark.parametrize('name,stream', corrupt_cases(), ids=[c[0] for c in corrupt_cases()])
def test_corrupt_members_give_bb_err_arg(name, stream):
    import ctypes
    from badread_b200 import _lib
    with pytest.raises(ValueError) as emu_err:       # the emulator first: the bounds hold on this input
        EI.decompress(stream)
    L = _lib.lib()
    out = (ctypes.c_char * (1 << 20))()
    n_out = ctypes.c_int64(0)
    rc = L.bb_bgzf_decompress(0, stream, len(stream), out, 1 << 20, ctypes.byref(n_out))
    assert rc == _lib.BB_ERR_ARG
    assert L.bb_model_error().decode() == str(emu_err.value)
