"""
Inputs that make a batch outgrow the limits it is enqueued with, checked on the CPU so that the GPU re-run tests
(test_gpu_rerun.py) rest on a premise a run without a GPU can see:
- reads whose error loop needs four or more rounds (three are enqueued), on the device code under the emulator;
- reads whose joined sequence is far longer than their fragment (the read buffers and the split-score scratch are sized
  for 1.25x and for the expected edits), by the oracle.
"""
import io
import random

import pytest

# k=3, homopolymer slippage: inside a run of A's one base is gained or lost, nothing else.  A gain and a loss in the same
# run cancel, so the read stays close to its fragment and the loop runs until it has changed 90 % of the bases
# (simulate.py:285) - several times the changes its target identity asks for.
SLIP_MODEL = 'AAA,0.1;AAAA,0.45;AA,0.45;\n'

# k=3, every 3-mer gains four bases in the middle seven times in ten: joined reads 1.5x their fragment and more.
INSERT_MODEL = ''.join(f'{a}{b}{c},0.3;{a}{b}TTT{b}{c},0.7;\n' for a in 'ACGT' for b in 'ACGT' for c in 'ACGT')


def model(tmp_path, text, name):
    from badread_b200.error_model import ErrorModel
    path = tmp_path / name
    path.write_text(text)
    return ErrorModel(str(path), io.StringIO())


def slip_fragments():
    """Runs of 30-200 A's between single other bases, with the identity each read is asked for."""
    rnd = random.Random(404)
    out = []
    for n, ident in ((2000, 0.9), (3000, 0.92), (2600, 0.88)):
        frag = ''.join('A' * rnd.randint(30, 200) + rnd.choice('CGT') for _ in range(n // 60))[:n]
        out.append((frag, ident))
    return out


SLIP_SEED, SLIP_FIRST_INDEX = 1234, 61000


def test_slip_model_reads_need_more_than_three_loop_rounds(tmp_path):
    """The error loop of each slip-model read, as the GPU enqueues it round after round, needs at least four rounds: a
    batch of them outgrows the three rounds a run starts with.  Its counts equal the oracle's."""
    from emu import emu as E
    from oracle import oracle as O
    from conftest import load_models
    E.build()
    em = model(tmp_path, SLIP_MODEL, 'slip.txt')
    orc = O.Oracle(em, load_models('random', 'ideal')[1])
    for i, (frag, ident) in enumerate(slip_fragments()):
        joined, st = E.error_loop(frag, ident, SLIP_SEED, SLIP_FIRST_INDEX + i, em)
        seq, _, _, want = orc.sequence_fragment(frag, ident, SLIP_SEED, SLIP_FIRST_INDEX + i, with_stats=True)
        assert (st['loop_count'], st['change_count'], st['n_alignments']) == \
            (want['loop_count'], want['change_count'], want['n_alignments'])
        assert joined[st['start_trim']:len(joined) - st['end_trim']] == seq
        assert st['change_count'] > 2.5 * (1.0 - ident) * len(frag), (i, st['change_count'])
        assert 4 <= st['rounds'] <= 6, (i, st['rounds'])     # one re-run with 3 more rounds covers it


@pytest.mark.parametrize('ident', [0.55, 0.6])
def test_insert_model_reads_outgrow_the_read_buffers(tmp_path, ident):
    """With the insertion model a read at identity 0.55-0.6 comes out more than 1.5x as long as its fragment: beyond
    the 1.25x the read buffers start with, and beyond the split-score rows sized from the expected edits."""
    from oracle import oracle as O
    from conftest import load_models, random_dna
    em = model(tmp_path, INSERT_MODEL, 'insert.txt')
    orc = O.Oracle(em, load_models('random', 'ideal')[1])
    frag = random_dna(random.Random(5), 6000)
    seq, _, _ = orc.sequence_fragment(frag, ident, 1234, 17)
    expect_rows = 3.0 * (1.0 - ident) * len(frag) + 0.02 * len(frag) + 512
    assert len(seq) > 1.5 * len(frag) and len(seq) > expect_rows, (len(seq), len(frag))
