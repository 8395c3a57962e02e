"""The BGZF compressor (csrc/bb_bgzf.cuh) and inflater (csrc/bb_inflate.cuh) under the warp emulator, against the
plain deflate reference in tests/deflate_ref.py, on the inputs FASTQ and zlib never produce.

Compressor: seeded inputs with skewed byte statistics (Fibonacci, geometric and Pareto histograms), every byte value,
one and two symbols, FASTQ lines at the block-start threshold and at the chunk's end, a chunk with as many block
starts as fit, an input whose code-length code needs the 7-bit limit, and a skew sweep across the stored / dynamic
decision.  Every member's structure is checked: block starts by the rule of DESIGN.md, complete codes of at most 15
(7) bits ranked by (frequency, symbol), optimal cost (or within 0.1 % of the optimal 15-bit-limited cost), the header's
fields and run-length symbols, and the stored fallback against the dynamic size the same rules give.

Inflater: block programs with what zlib never writes (distance 32 768, length 258 as code 284 + 31, HLIT 286 / HDIST
30, one or no distance codes, code-length repeats across the literal / distance boundary, stored blocks at every bit
phase, ISIZE 65 536, ...) inflate to zlib's bytes, and a seeded list of corruptions is refused exactly when zlib
refuses it."""
import gzip
import random
import struct
import zlib

import numpy as np
import pytest

import deflate_ref as R
from emu import emu_bgzf as B
from emu import emu_inflate as EI

CHUNK = 65280
MIN_SEG = 1024
EOF = bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')
# limited cost / optimal length-limited cost, at most: literal codes (15 bits) and code-length codes (7 bits, a few
# hundred bits in all, where one bit is 0.3 %)
LIMIT_SLACK = {15: 1.001, 7: 1.01}


# ------------------------------------------------------------------------------------------------ the compressor's rules
def block_starts(chunk, mod4):
    """DESIGN.md §4: a block starts at every line of index 1 or 3 mod 4 that starts in the chunk and has at least
    BGZF_MIN_SEG bytes in it, its newline included; the first block starts at 0."""
    starts, line, i = [0], mod4, chunk.find(b'\n')
    while 0 <= i < len(chunk) - 1:
        line += 1
        a = i + 1
        end = chunk.find(b'\n', a)
        if line & 1 and (end + 1 if end >= 0 else len(chunk)) - a >= MIN_SEG:
            starts.append(a)
        i = end
    return starts


def cl_freq(rle):
    """The code-length code's histogram as the compressor builds it: the run-length symbols, and symbols of frequency 1
    added from the lowest until two are used."""
    f = [0] * 19
    for s, _ in rle:
        f[s] += 1
    for s in range(19):
        if sum(1 for x in f if x) < 2 and not f[s]:
            f[s] = 1
    return f


def trimmed_hclen(cl):
    n = 19
    while n > 4 and not cl[R.CL_ORDER[n - 1]]:
        n -= 1
    return n


def lit_freq(block_bytes):
    f = np.bincount(np.frombuffer(block_bytes, dtype=np.uint8), minlength=257).tolist()
    f[256] = 1
    return f


def reference_dynamic_bits(chunk, mod4):
    """The size in bits (from the member's first byte) of the dynamic member the compressor's rules give, with least-depth
    optimal codes, and whether any block needs a length limit (its literal code more than 15 bits deep, or its
    code-length code more than 7): then the size is not the compressor's."""
    starts = block_starts(chunk, mod4) + [len(chunk)]
    bits, limited = 8 * 18, False
    for a, b in zip(starts, starts[1:]):
        f = lit_freq(chunk[a:b])
        lens = R.huffman_lengths(f)
        if max(lens) > 15:
            limited = True
            continue
        rle = R.rle_greedy(lens + [1, 1])
        cl = R.huffman_lengths(cl_freq(rle))
        limited |= max(cl) > 7
        bits += 17 + 3 * trimmed_hclen(cl) + sum(cl[s] + R.RLE_EXTRA.get(s, 0) for s, _ in rle)
        bits += sum(x * l for x, l in zip(f, lens))
    return bits, limited


WORST = {15: [1.0, 0], 7: [1.0, 0]}       # per length limit: the largest limited / optimal cost ratio, blocks


def check_member(m, chunk, mod4):
    """Structure of one member of the compressor against its rules; returns the parse."""
    p = R.parse_member(m)
    assert p['data'] == chunk
    assert (p['flg'], p['mtime'], p['xfl'], p['os']) == (4, 0, 0, 255)
    assert p['extra'] == [(b'BC', struct.pack('<H', len(m) - 1))] and len(m) <= 65536
    assert p['padding'] == (0, p['padding'][1]) and p['trailing'] == 0
    blocks = p['blocks']
    assert [b['final'] for b in blocks] == [0] * (len(blocks) - 1) + [1]
    ref_bits, ref_limited = reference_dynamic_bits(chunk, mod4)
    if blocks[0]['type'] == 'stored':
        assert len(blocks) == 1 and blocks[0]['len'] == len(chunk) and blocks[0]['pad'] == 5
        if not ref_limited:           # stored only when the dynamic member would not be smaller
            assert ref_bits > 8 * (18 + 4 + len(chunk)), (ref_bits, len(chunk))
        return p
    assert {b['type'] for b in blocks} == {'dynamic'}
    assert [b['out'][0] for b in blocks] == block_starts(chunk, mod4)
    assert p['data_bytes'] <= len(chunk) + 4
    for b in blocks:
        a, e = b['out']
        f = lit_freq(chunk[a:e])
        lens = b['lit_lens']
        assert (b['hlit'], b['hdist'], b['dist_lens']) == (257, 2, [1, 1])
        _check_code(f, lens, 15, 'literal')
        assert b['rle'] == R.rle_greedy(lens + [1, 1])
        cf = cl_freq(b['rle'])
        _check_code(cf, b['cl_lens'], 7, 'code-length')
        assert b['hclen'] == trimmed_hclen(b['cl_lens'])
    if not ref_limited:               # the compressor's size is the one its rules give
        assert blocks[-1]['end'] + 8 * 18 == ref_bits
    return p


def _check_code(f, lens, max_len, what):
    assert all((x > 0) == (l > 0) for x, l in zip(f, lens)), what
    assert max(lens) <= max_len and R.kraft(lens) == 1 << 15, what
    ranked = [lens[s] for _, s in sorted((x, s) for s, x in enumerate(f) if x)]
    assert ranked == sorted(ranked, reverse=True), f'{what}: a rarer (or lower, equally frequent) symbol has a shorter code'
    cost = sum(x * l for x, l in zip(f, lens))
    if max(R.huffman_lengths(f)) <= max_len:
        assert cost == R.huffman_cost(f), what
    else:
        best = R.limited_cost(f, max_len)
        assert best <= cost <= best * LIMIT_SLACK[max_len], (what, cost, best)
        WORST[max_len] = [max(WORST[max_len][0], cost / best), WORST[max_len][1] + 1]


def check_stream(data, mod4, comp):
    """Every member of comp (the members of data, no end-of-file member) checked; returns the parses."""
    ms = R.split_bgzf(comp)
    assert len(ms) == -(-len(data) // CHUNK)
    out = []
    for c, m in enumerate(ms):
        chunk = data[c * CHUNK:(c + 1) * CHUNK]
        out.append(check_member(m, chunk, (mod4 + data.count(b'\n', 0, c * CHUNK)) & 3))
    assert gzip.decompress(comp + EOF) == data
    return out


# ------------------------------------------------------------------------------------------------ compressor inputs
def _fib(k):
    a, b, out = 1, 1, []
    for _ in range(k):
        out.append(a)
        a, b = b, a + b
    return out


def _shuffled(rs, syms, counts):
    arr = np.repeat(np.asarray(syms, dtype=np.uint8), counts)
    rs.shuffle(arr)
    return arr.tobytes()


def _drawn(rs, n, p, syms=None):
    p = np.asarray(p, dtype=np.float64)
    syms = np.arange(len(p)) if syms is None else np.frombuffer(syms, dtype=np.uint8) if isinstance(syms, bytes) \
        else np.asarray(syms)
    return syms[rs.choice(len(p), n, p=p / p.sum())].astype(np.uint8).tobytes()


def _no_newline(rs, k):
    return rs.permutation([s for s in range(256) if s != 10])[:k]


def _fastq(rs, lens, qual_p):
    out = []
    for i, n in enumerate(lens):
        out.append(b'@r%d\n' % i + _drawn(rs, n, [1, 1, 1, 1], b'ACGT') + b'\n+\n' +
                   _drawn(rs, n, qual_p, np.arange(33, 33 + len(qual_p))) + b'\n')
    return b''.join(out)


# Found by a seeded search with the reference (reference_dynamic_bits): Zipf-distributed bytes whose code-length
# code is more than 7 bits deep, and an input whose dynamic member has exactly len + 4 bytes of deflate data.
CL_LIMIT_SEED = 2
EXACT_SEED = 143


def cl_limit_input(seed):
    rs = np.random.RandomState(seed)
    k = int(rs.randint(64, 257))
    syms = rs.permutation(256)[:k]
    syms = syms[syms != 10]
    return _drawn(rs, int(rs.randint(8000, CHUNK)), 1.0 / np.arange(1, len(syms) + 1) ** rs.uniform(0.9, 1.3), syms)


def exact_input(seed):
    rs = np.random.RandomState(seed)
    k = int(rs.randint(2, 12))
    return _drawn(rs, int(rs.randint(16, 400)), rs.uniform(0.05, 1, k), _no_newline(rs, k))


def sweep_input(r, seed=5):
    """8 000 bytes of all 256 values with geometric weights r^i: the stored / dynamic decision flips inside the sweep."""
    rs = np.random.RandomState(seed)
    return _drawn(rs, 8000, r ** np.arange(256), rs.permutation(256))


SWEEP = [1.0, 0.999, 0.998, 0.997, 0.996, 0.995, 0.994, 0.993, 0.99, 0.985, 0.98, 0.97]


def stress_inputs():
    """(name, data, line_mod4): the compressor's seeded stress set, shared with the GPU tier."""
    rs = np.random.RandomState(2026)
    out = []
    # Fibonacci counts 1, 2, 3, 5, ... (k of them): with the end-of-block code every optimal tree is a chain of depth k
    # (21 is the deepest whose bytes fit in a chunk); 1, 1, 2, 3, ...: optimal trees as deep as k + 1 and as shallow as
    # half that, so a least-depth tree fits in 15 bits
    for k in range(17, 22):
        out.append((f'fibonacci_chain_{k}', _shuffled(rs, _no_newline(rs, k), _fib(k + 1)[1:]), 0))
    for k in (20, 22):
        out.append((f'fibonacci_ties_{k}', _shuffled(rs, _no_newline(rs, k), _fib(k)), 0))
    out.append(('fibonacci_two_chunks', _shuffled(rs, _no_newline(rs, 21), _fib(22)[1:]) +
                _shuffled(rs, _no_newline(rs, 20), _fib(21)[1:]), 0))
    for n_sym in (2, 3, 5, 9, 17, 33, 65, 129, 256):
        for r in (0.3, 0.6, 0.85, 0.95):
            n = int(rs.randint(500, 2 * CHUNK))
            out.append((f'geometric_{n_sym}_{r}', _drawn(rs, n, r ** np.arange(n_sym), _no_newline(rs, n_sym)
                                                         if n_sym < 256 else rs.permutation(256)), int(rs.randint(4))))
        for a in (0.8, 1.5, 3.0):
            n = int(rs.randint(500, 2 * CHUNK))
            out.append((f'pareto_{n_sym}_{a}', _drawn(rs, n, np.arange(1, n_sym + 1) ** -a, _no_newline(rs, n_sym)
                                                      if n_sym < 256 else rs.permutation(256)), int(rs.randint(4))))
    out.append(('all_256_values', _drawn(rs, CHUNK - 256, 0.975 ** np.arange(256), rs.permutation(256)) + bytes(range(256)), 0))
    out.append(('single_symbol', b'Q' * 40000, 0))
    out.append(('two_symbols', _drawn(rs, 30000, [0.9, 0.1], b'AB'), 0))
    fib_q = _fib(20)[::-1]
    for n in (1022, 1023, 1024, 1025):            # lines on both sides of the block-start threshold
        out.append((f'fastq_quality_lines_{n}', _fastq(rs, [n] * 80, fib_q), 0))
        out.append((f'fastq_quality_lines_{n}_mod4_2', _fastq(rs, [n] * 40, fib_q), 2))
    for back in (1024, 1023):                     # a sequence line starting BGZF_MIN_SEG or one byte less before the end
        for total in (CHUNK, 5000):
            at = total - back
            out.append((f'line_at_len_minus_{back}_of_{total}',
                        b'X' * (at - 1) + b'\n' + _drawn(rs, back + (CHUNK if total == CHUNK else 0), [4, 2, 1, 1], b'ACGT'), 0))
    rows = [b'\n']                                # as many block starts as fit: lines of 1023 bytes between empty lines
    while sum(map(len, rows)) + 1025 <= CHUNK:
        rows.append(_drawn(rs, 1023, rs.uniform(0.1, 1, 3), b'ACG') + b'\n\n')
    rows.append(b'T' * (CHUNK - sum(map(len, rows))))
    out.append(('most_block_starts', b''.join(rows), 0))
    out.append(('code_length_code_limit', cl_limit_input(CL_LIMIT_SEED), 0))
    out.append(('deflate_data_len_plus_4', exact_input(EXACT_SEED), 0))
    for r in SWEEP:
        out.append((f'skew_sweep_{r}', sweep_input(r), 0))
    return out


_STRESS = None


def stress():
    global _STRESS
    if _STRESS is None:
        _STRESS = stress_inputs()
    return _STRESS


# ------------------------------------------------------------------------------------------------ compressor tests
def test_stress_inputs_reach_the_edges():
    """The stress set reaches what it is for, by the reference: unlimited literal depths 17 and beyond, a code-length code
    over 7 bits, 64 blocks in one chunk, a dynamic member of exactly len + 4 bytes of deflate data."""
    cases = {n: (d, m) for n, d, m in stress()}
    depths = {n: max(R.huffman_lengths(lit_freq(d[:CHUNK]))) for n, (d, _) in cases.items() if n.startswith('fibonacci')}
    assert [depths[f'fibonacci_chain_{k}'] for k in range(17, 22)] == list(range(17, 22)), depths
    assert depths['fibonacci_ties_22'] <= 15, depths
    d = cases['code_length_code_limit'][0]
    lens = R.huffman_lengths(lit_freq(d))
    assert max(lens) <= 15 and max(R.huffman_lengths(cl_freq(R.rle_greedy(lens + [1, 1])))) > 7
    assert len(block_starts(*cases['most_block_starts'])) == 64
    d = cases['deflate_data_len_plus_4'][0]
    bits, limited = reference_dynamic_bits(d, 0)
    assert not limited and (bits + 7) // 8 == 18 + len(d) + 4
    for back, total in ((1024, CHUNK), (1024, 5000), (1023, CHUNK), (1023, 5000)):
        d, m = cases[f'line_at_len_minus_{back}_of_{total}']
        assert block_starts(d[:total], m) == [0] + ([total - back] if back == 1024 else [])


def test_compressor_members_follow_their_rules():
    """Every stress input under the emulator: each member parses to its chunk, with the structure its rules give."""
    types = {}
    for name, data, mod4 in stress():
        comp, used = B.compress(data, mod4, final=True)
        assert used == len(data)
        ps = check_stream(data, mod4, comp)
        types[name] = [p['blocks'][0]['type'] for p in ps]
    assert WORST[15][1] and WORST[7][1], WORST
    print('worst limited / optimal limited cost, blocks:', WORST)
    assert all(set(t) == {'dynamic'} for n, t in types.items() if n.startswith('fibonacci'))
    assert types['all_256_values'] == ['dynamic'] and types['code_length_code_limit'] == ['dynamic']
    assert types['deflate_data_len_plus_4'] == ['dynamic']
    sweep = [types[f'skew_sweep_{r}'][0] for r in SWEEP]
    assert sweep[0] == 'stored' and sweep[-1] == 'dynamic' and sweep == sorted(sweep, reverse=True), sweep


# ------------------------------------------------------------------------------------------------ inflater programs
def _stored(data, **kw):
    return dict(type='stored', data=data, **kw)


def _fixed(tokens, **kw):
    return dict(type='fixed', tokens=tokens, **kw)


def _dynamic(tokens, **kw):
    return dict(type='dynamic', tokens=tokens, **kw)


def _complete(lens_by_len):
    """A complete code: [(length, count)] handed out to consecutive symbols."""
    out = []
    for l, n in lens_by_len:
        out += [l] * n
    assert R.kraft(out) == 1 << 15
    return out


def inflater_programs():
    """(name, program): block programs of what zlib's deflate never writes; every one is valid deflate."""
    rnd = random.Random(11)

    def noise(n):
        return bytes(rnd.getrandbits(8) for _ in range(n))

    P = []
    far = [(258, 32768), (258, 32768, 284)] * 63 + [(257, 32768), (3, 32768)]          # 32 768 bytes of matches
    P.append(('distance_32768_isize_65536', [_stored(noise(32768), final=0), _fixed(far)]))
    P.append(('distance_to_the_first_byte', [_fixed([65, 66, 67, (3, 3), (258, 6), (258, 264, 284), (100, 522)])]))
    P.append(('length_258_both_ways', [_dynamic([7, (258, 1), (258, 1, 284), 9, (258, 2, 284), (258, 2)])]))
    P.append(('overlapping_copies', [_fixed([1, (258, 1), 2, (258, 2), 3, (258, 3), (258, 3, 284)])]))
    # 15-bit codes: literal / length lengths 1 .. 15 (and one more 15) on symbols 65 .., distance lengths likewise
    lit = [0] * 286
    for s, l in zip([65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 75, 256, 257, 265, 284, 285], list(range(1, 16)) + [15]):
        lit[s] = l
    dist = [0] * 30
    for s, l in zip(range(16), list(range(1, 16)) + [15]):
        dist[s] = l
    toks = [65, 75, (3, 1), 70, (258, 2), (11, 5), 74, (258, 129, 284), (250, 200), 66, (3, 250)]
    P.append(('codes_of_15_bits', [_fixed([65] * 300, final=0), _dynamic(toks, lit_lens=lit, dist_lens=dist)]))
    # 9- and 10-bit codes, on either side of the inflater's 9-bit table: literals 0..253 of 8 bits, 254 / 255 of 9, the
    # end-of-block and lengths 257..259 of 10
    lit = _complete([(8, 254), (9, 2), (10, 4)])
    P.append(('codes_of_9_and_10_bits', [_dynamic([0, 254, 255, 253, (3, 2), (4, 3), (5, 4), 255],
                                                  lit_lens=lit, dist_lens=[2, 2, 2, 2])]))
    P.append(('one_distance_code_of_one_bit', [_dynamic([5, 6, (10, 1), (258, 1, 284)], dist_lens=[1])]))
    P.append(('one_distance_code_second_symbol', [_dynamic([5, 6, (10, 2)], dist_lens=[0, 1])]))
    P.append(('no_distance_codes', [_dynamic(list(noise(500)), dist_lens=[0])]))
    lf = [rnd.randint(1, 60) for _ in range(286)]
    df = [rnd.randint(1, 60) for _ in range(30)]
    toks = [rnd.randrange(256) for _ in range(40)] + [(rnd.randint(3, 258), rnd.randint(1, 40)) for _ in range(60)]
    P.append(('hlit_286_hdist_30', [_dynamic(toks, lit_lens=R.limited_lengths(lf, 15), dist_lens=R.limited_lengths(df, 15))]))
    # code 16 across the literal / distance boundary: the last literal / length lengths and the first distance lengths
    # equal; code 16 right after 17 and after 18 (repeating a zero)
    lit = [0] * 65 + [4] * 4 + [0] * 6 + [5] * 8 + [0] * 173 + [5] * 2 + [6] * 28
    dist = [6] * 16 + [5] * 4 + [4] * 10
    assert R.kraft(lit) == R.kraft(dist) == 1 << 15
    lens = lit + dist
    P.append(('repeat_across_the_boundary', [_dynamic([65, 80, (3, 1), (10, 2)], lit_lens=lit, dist_lens=dist)]))
    rle = R.rle_greedy(lens)
    rle2 = []
    for s, x in rle:                                   # every 17 / 18 of at least 6 zeros as a shorter one and a 16
        if s in (17, 18) and (3 if s == 17 else 11) + x >= (6 if s == 17 else 14):
            rle2 += [(s, x - 3), (16, 0)]
        else:
            rle2.append((s, x))
    assert any(a[0] == 17 and b[0] == 16 for a, b in zip(rle2, rle2[1:]))
    assert any(a[0] == 18 and b[0] == 16 for a, b in zip(rle2, rle2[1:]))
    P.append(('repeat_after_17_and_18', [_dynamic([65, 80, (3, 1), (10, 2)], lit_lens=lit, dist_lens=dist, rle=rle2)]))
    lit = [0] * 286                                    # an 18 of exactly 138 zeros
    lit[0], lit[139], lit[278] = 2, 2, 2
    lit[256] = 2
    P.append(('zero_runs_of_138', [_dynamic([0, 139, 0], lit_lens=lit, dist_lens=[0])]))
    P.append(('empty_blocks', [_stored(b'', final=0), _fixed([], final=0), _dynamic([], final=0), _stored(b'x', final=0),
                               _fixed([], final=0), _dynamic([]), ]))
    phases = []
    for p in range(8):                                 # a fixed block of (p - 2) mod 8 9-bit literals before each
        phases += [_fixed([200] * ((p - 2) % 8), final=0), _stored(noise(p + 1), final=0, phase=p)]
    P.append(('stored_at_every_phase', phases[:-1] + [dict(phases[-1], final=1)]))
    a = noise(3000)
    P.append(('matches_across_block_types', [
        _stored(a, final=0), _fixed([(258, 3000), (100, 2900)], final=0),
        _dynamic([9, (258, 3358 + 1), (200, 3000)], final=0), _stored(noise(10), final=0),
        _fixed([(30, 15), (258, 3800, 284)], final=0), _dynamic([(258, 4000), (3, 1)], dist_lens=[1] + [0] * 22 + [1])]))
    P.append(('isize_0_stored', [_stored(b'')]))
    P.append(('isize_0_fixed', [_fixed([])]))
    return P


def big_members(n=24):
    """Members of exactly 65 536 bytes: stored, fixed, dynamic and mixed programs in turn."""
    rnd = random.Random(12)
    out = []
    for i in range(n):
        a = bytes(rnd.getrandbits(8) for _ in range(4096))
        k = i % 4
        if k == 0:
            prog = [_stored(a, final=0), _stored(a[:1000], final=0), _fixed([(258, 5000)] * 234 + [(68, 5000)])]
        elif k == 1:
            prog = [_fixed(list(a[:1000]) + [(258, 1000)] * 250 + [(36, 999)])]
        elif k == 2:
            prog = [_dynamic(list(a[:96]) + [(258, 96)] * 252 + [(258, 2, 284), (166, 1)])]
        else:
            prog = [_stored(a, final=0), _dynamic([(258, 4096)] * 238, final=0), _fixed([(36, 32768)])]
        out.append((f'isize_65536_{i}', prog))
    return out


def zlib_inflate(m):
    """zlib on one gzip member (wbits 31): the bytes, or None where zlib refuses it (or leaves bytes unused)."""
    d = zlib.decompressobj(31)
    try:
        out = d.decompress(m) + d.flush()
    except zlib.error:
        return None
    return out if d.eof and not d.unused_data else None


def corpus():
    """(name, member, bytes) of every program, each checked by zlib and parsed by the reference on the way."""
    out = []
    for name, prog in inflater_programs() + big_members():
        m, data = R.encode(prog)
        out.append((name, m, data))
    return out


def test_reference_parses_zlib_corpus():
    """The reference parses every zlib member of the level / strategy settings the inflater is tested on to zlib's
    bytes, and reports no padding or trailing bytes where zlib writes none."""
    from test_model_builders_alignments import SETTINGS, bgzf_member
    rnd = random.Random(3)
    text = ''.join(rnd.choice(['ACGT', 'AC', 'G', 'TTTTTTTT', 'ACGTTGCA\n']) for _ in range(40000)).encode()
    noise = bytes(rnd.getrandbits(8) for _ in range(70000))
    for level, strategy in SETTINGS:
        for raw in (text, noise):
            for n in (0, 1, 2, 7, 258, 259, 1000, 32768, 32769, 65280):
                p = R.parse_member(bgzf_member(raw[:n], level, strategy))
                assert p['data'] == raw[:n] and p['trailing'] == 0


def test_reference_programs_are_accepted_by_zlib():
    for name, m, data in corpus():
        assert len(data) <= 65536
        assert zlib_inflate(m) == data, name
        assert gzip.decompress(m) == data, name
        assert R.parse_member(m)['data'] == data, name
    progs = dict(inflater_programs())
    p = R.parse_member(R.encode(progs['stored_at_every_phase'])[0])
    assert sorted(b['start'] & 7 for b in p['blocks'] if b['type'] == 'stored') == list(range(8))
    p = R.parse_member(R.encode(progs['repeat_across_the_boundary'])[0])
    at = 0
    for s, x in p['blocks'][0]['rle']:                 # a code 16 fills lengths on both sides of HLIT
        n = 1 if s < 16 else 3 + x if s != 18 else 11 + x
        crossed = s == 16 and at < p['blocks'][0]['hlit'] < at + n
        if crossed:
            break
        at += n
    assert crossed
    assert sum(1 for s, x in R.parse_member(R.encode(progs['zero_runs_of_138'])[0])['blocks'][0]['rle'] if (s, x) == (18, 127)) == 1
    for name in ('codes_of_15_bits',):
        b = R.parse_member(R.encode(progs[name])[0])['blocks'][1]
        assert max(b['lit_lens']) == 15 and max(b['dist_lens']) == 15


@pytest.mark.parametrize('name', [n for n, _ in inflater_programs()])
def test_inflater_programs_give_zlibs_bytes(name):
    m, data = R.encode(dict(inflater_programs())[name])
    assert bytes(EI.decompress(m + EOF)) == zlib_inflate(m) == data


def test_stream_of_65536_byte_members():
    ms = [R.encode(p) for _, p in big_members()]
    assert all(len(d) == 65536 for _, d in ms)
    stream = b''.join(m for m, _ in ms) + EOF
    assert bytes(EI.decompress(stream)) == gzip.decompress(stream) == b''.join(d for _, d in ms)


def test_isize_beyond_65536_refused_by_the_walk():
    m, data = R.encode([_fixed([97] + [(258, 1)] * 254 + [(4, 1)])])
    assert len(data) == 65537 and zlib_inflate(m) == data
    with pytest.raises(ValueError, match=r'member 0 .*ISIZE beyond'):
        EI.decompress(m)


# ------------------------------------------------------------------------------------------------ rejection parity
def _header_bits(b):
    """Bits of a parsed block's header: type, and the stored lengths or the dynamic tables."""
    if b['type'] == 'stored':
        return 3 + b['pad'] + 32
    if b['type'] == 'fixed':
        return 3
    return 17 + 3 * b['hclen'] + sum(b['cl_lens'][s] + R.RLE_EXTRA.get(s, 0) for s, _ in b['rle'])


def corruptions():
    """(name, member): a fixed, seeded list of corrupt (or possibly still valid) variants of the inflater programs."""
    rnd = random.Random(13)
    progs = dict(inflater_programs())
    out = []
    big = progs['hlit_286_hdist_30'][0]
    for h in (287, 288):
        out.append((f'hlit_{h}', [dict(big, lit_lens=big['lit_lens'] + [0] * (h - 286), hlit=h)]))
    for h in (31, 32):
        out.append((f'hdist_{h}', [dict(big, dist_lens=big['dist_lens'] + [0] * (h - 30), hdist=h)]))
    cross = progs['repeat_across_the_boundary'][0]
    rle = R.rle_greedy(cross['lit_lens'] + cross['dist_lens'])
    cl = R.limited_lengths(cl_freq(rle), 7)
    s = min((l, s) for s, l in enumerate(cl) if l)[1]
    out.append(('incomplete_code_length_code', [dict(cross, cl_lens=cl[:s] + [cl[s] + 1] + cl[s + 1:])]))
    lit = list(cross['lit_lens'])
    lit[65] += 1
    out.append(('incomplete_literal_code', [dict(cross, lit_lens=lit)]))
    assert rle[0] == (18, 54)                           # 65 zeros: as 16 (after nothing) and 62 zeros
    out.append(('repeat_first', [_dynamic([1, 2, 3], dist_lens=[0], final=0), dict(cross, rle=[(16, 0), (18, 51)] + rle[1:])]))
    out.append(('repeat_past_the_end', [dict(cross, rle=rle[:-1] + [(18, 127)])]))
    fl, fd = R.canonical(R.FIXED_LIT), R.canonical(R.FIXED_DIST)
    for d in (30, 31):
        w = R.BitWriter()
        w.put(1, 1); w.put(1, 2)
        w.put_code(fl[65], 8); w.put_code(fl[257], 7); w.put_code(fd[d], 5); w.put_code(fl[256], 7)
        out.append((f'fixed_distance_code_{d}', w.bytes(), b'AAAA'))
    for name in ('matches_across_block_types', 'stored_at_every_phase', 'empty_blocks', 'codes_of_15_bits',
                 'distance_32768_isize_65536'):
        d, data = R.deflate(progs[name]), R.program_output(progs[name])
        for k, b in enumerate(R.parse_deflate(d)[1][1:] + [None]):
            cut = b['start'] // 8 if b else len(d) - 1
            out.append((f'truncated_{name}_{k}', d[:cut], data))
    for name in ('hlit_286_hdist_30', 'repeat_across_the_boundary', 'repeat_after_17_and_18', 'codes_of_9_and_10_bits',
                 'codes_of_15_bits', 'stored_at_every_phase', 'empty_blocks', 'one_distance_code_of_one_bit',
                 'no_distance_codes', 'zero_runs_of_138'):
        d, data = R.deflate(progs[name]), R.program_output(progs[name])
        for k, b in enumerate(R.parse_deflate(d)[1]):
            bits = range(b['start'], b['start'] + _header_bits(b))
            for bit in sorted(rnd.sample(bits, min(len(bits), 12))):
                flipped = bytearray(d)
                flipped[bit >> 3] ^= 1 << (bit & 7)
                out.append((f'flip_{name}_{k}_{bit}', bytes(flipped), data))
    d = R.deflate(progs['length_258_both_ways'])
    out.append(('byte_before_the_trailer', d + b'\0', R.program_output(progs['length_258_both_ways'])))
    members = []
    for case in out:
        if len(case) == 2:
            m, _ = R.encode(case[1])
        else:
            m = R.member(case[1], case[2])
        members.append((case[0], m))
    return members


def _emulated(stream):
    try:
        return bytes(EI.decompress(stream)), None
    except ValueError as e:
        return None, str(e)


def test_rejection_parity_with_zlib():
    """Every corruption is refused by the emulated inflater exactly when zlib refuses it; where both accept, the bytes
    are equal."""
    refused = 0
    for name, m in corruptions():
        want = zlib_inflate(m)
        got, err = _emulated(m)
        assert (got is None) == (want is None), (name, err)
        assert got == want, name
        refused += want is None
    assert refused > len(corruptions()) // 2


@pytest.mark.parametrize('name', ['hlit_287', 'hlit_288', 'hdist_31', 'hdist_32', 'incomplete_code_length_code',
                                  'incomplete_literal_code', 'repeat_first', 'repeat_past_the_end', 'fixed_distance_code_30',
                                  'fixed_distance_code_31', 'byte_before_the_trailer'])
def test_named_corruptions_are_refused(name):
    m = dict(corruptions())[name]
    assert zlib_inflate(m) is None
    _, err = _emulated(m)
    assert err and err.startswith('bb_bgzf_decompress: member 0 '), err
    if name == 'byte_before_the_trailer':
        assert err.endswith('bytes between the final deflate block and the trailer')
