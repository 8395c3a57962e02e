"""The BGZF compressor and inflater on the GPU, on the stress inputs and block programs of tests/test_deflate_edges.py:
the device gives the emulator's members and their structure, a 64 MB call of the stress chunks inflates back, the
inflater corpus gives zlib's bytes in one stream, and every corruption the emulator refuses is refused on the device
with the same message (the same member index)."""
import gzip
import random

import numpy as np
import pytest

import deflate_ref as R
from emu import emu_bgzf as B
from emu import emu_inflate as EI
from test_deflate_edges import CHUNK, EOF, check_stream, corpus, corruptions, stress, zlib_inflate

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engine():
    """A context of this module's own, released when the module is done (as in test_gpu_bgzf.py)."""
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=1234)
    yield eng
    eng.close()


def test_stress_inputs_give_the_emulators_members(engine):
    for name, data, mod4 in stress():
        got = bytes(engine.bgzf_compress(data, mod4, final=True)[0])
        assert got == B.compress(data, mod4, final=True)[0], name
        check_stream(data, mod4, got)


def test_64_mb_of_stress_chunks(engine):
    """About 64 MB of the stress inputs' chunks in a seeded order, starting at a random line index: one call inflates
    back, and the members at a seeded sample of chunk indices equal the emulator's."""
    rnd = random.Random(21)
    chunks = [d[i:i + CHUNK] for _, d, _ in stress() for i in range(0, len(d), CHUNK)]
    parts, total = [], 0
    while total < 64 << 20:
        c = rnd.choice(chunks)
        parts.append(c)
        total += len(c)
    data = b''.join(parts)
    mod4 = rnd.randrange(4)
    comp = bytes(engine.bgzf_compress(data, mod4, final=True)[0])
    assert gzip.decompress(comp + EOF) == data
    ms = R.split_bgzf(comp)
    assert len(ms) == -(-len(data) // CHUNK)
    nl = np.cumsum(np.frombuffer(data, dtype=np.uint8) == 10)
    for c in sorted(rnd.sample(range(len(ms)), 24)) + [len(ms) - 1]:
        at = c * CHUNK
        m4 = (mod4 + (int(nl[at - 1]) if at else 0)) & 3
        assert ms[c] == B.compress(data[at:at + CHUNK], m4, final=True)[0], c


def test_inflater_corpus_in_one_stream():
    from badread_b200.bgzf import decompress
    cs = corpus()
    stream = b''.join(m for _, m, _ in cs) + EOF
    want = b''.join(d for _, _, d in cs)
    assert gzip.decompress(stream) == want
    assert bytes(decompress(stream)) == want


def test_refused_corruptions_give_bb_err_arg():
    """Each corruption the emulator refuses, after one good member: BB_ERR_ARG with the emulator's message (member 1)."""
    import ctypes
    from badread_b200 import _lib
    L = _lib.lib()
    good = corpus()[0][1]
    out = (ctypes.c_char * (1 << 18))()
    n_out = ctypes.c_int64(0)
    n = 0
    for name, m in corruptions():
        if zlib_inflate(m) is not None:
            continue
        stream = good + m + EOF
        with pytest.raises(ValueError) as emu_err:
            EI.decompress(stream)
        assert 'member 1 ' in str(emu_err.value), name
        rc = L.bb_bgzf_decompress(0, stream, len(stream), out, len(out), ctypes.byref(n_out))
        assert rc == _lib.BB_ERR_ARG, name
        assert L.bb_model_error().decode() == str(emu_err.value), name
        n += 1
    assert n > 50
