"""
Small host-side helpers with the semantics of /root/reference/badread/misc.py that the `simulate` surface needs:
FASTA loading (misc.py:122-153), reverse complement (misc.py:56-71), the random helpers (misc.py:156-182),
identity_from_edlib_cigar (misc.py:228-240) and number formatting (misc.py:192-202).

Derived from Badread (Copyright 2018 Ryan Wick, rrwick@gmail.com, https://github.com/rrwick/Badread), which is free
software under the GNU General Public License version 3 or later; this file mirrors the named parts of the
reference's interface and is distributed under the same licence (see LICENSE and NOTICE at the repository root).
"""
import collections
import contextlib
import gzip
import io
import random
import re
import sys

_MAGIC = (('gz', b'\x1f\x8b\x08'), ('bz2', b'\x42\x5a\x68'), ('zip', b'\x50\x4b\x03\x04'))


def get_compression_type(filename):
    """misc.py:26-46 - sniff the first bytes; bzip2 and zip are rejected with the reference's messages."""
    with open(str(filename), 'rb') as handle:
        start = handle.read(max(len(m) for _, m in _MAGIC))
    kind = 'plain'
    for name, magic in _MAGIC:
        if start.startswith(magic):
            kind = name
    if kind == 'bz2':
        sys.exit('Error: cannot use bzip2 format - use gzip instead')
    if kind == 'zip':
        sys.exit('Error: cannot use zip format - use gzip instead')
    return kind


def get_open_func(filename):
    return gzip.open if get_compression_type(filename) == 'gz' else open


_COMP_TABLE = bytearray([ord('N')] * 256)
for _a, _b in zip(b'ATGCatgcRYSWKMBVDHNryswkmbvdhn.-?', b'TACGtacgYRSWMKVBHDNyrswmkvbhdn.-?'):
    _COMP_TABLE[_a] = _b
_COMP_TABLE = bytes(_COMP_TABLE)


def reverse_complement(seq):
    """misc.py:70-71; characters outside REV_COMP_DICT complement to 'N' (misc.py:64-68)."""
    if isinstance(seq, str):
        return seq.encode('latin-1').translate(_COMP_TABLE)[::-1].decode('latin-1')
    return bytes(seq).translate(_COMP_TABLE)[::-1]


def load_fasta(filename):
    """misc.py:122-153: name -> upper-cased sequence, depth=, circular=true, hairpin_left/right=true."""
    seqs = collections.OrderedDict()
    depths, circular, hairpin_left, hairpin_right = {}, {}, {}, {}
    depth_re = re.compile(r'depth=([\d.]+)')
    with get_open_func(filename)(filename, 'rt') as handle:
        name, chunks = '', []
        for line in handle:
            line = line.strip()
            if not line:
                continue
            if line[0] == '>':
                if name:
                    seqs[name.split()[0]] = ''.join(chunks).upper()
                    chunks = []
                name = line[1:]
                short = name.split()[0]
                lowered = name.lower()
                depths[short] = 1.0
                if 'depth=' in lowered:
                    try:
                        depths[short] = float(depth_re.search(lowered).group(1))
                    except (ValueError, AttributeError):
                        depths[short] = 1.0
                circular[short] = 'circular=true' in lowered
                hairpin_left[short] = 'hairpin_left=true' in lowered
                hairpin_right[short] = 'hairpin_right=true' in lowered
            else:
                chunks.append(line)
        if name:
            seqs[name.split()[0]] = ''.join(chunks).upper()
    return seqs, depths, circular, hairpin_left, hairpin_right


_UPPER = None
_DEPTH_RE = re.compile(r'depth=([\d.]+)')


def fasta_contigs(headers):
    """The header semantics of load_fasta (misc.py:122-153), shared by load_fasta_arrays and the GPU loader
    (engine.Engine.load_fasta).  headers: [(text of a header line after its '>', body)] in file order, body being whatever
    the caller finds the contig's bases by.  A header that is empty once stripped names no contig; the name is the first
    token; `depth=`, `circular=true` and `hairpin_left/right=true` are read from the lower-cased header; a repeated name
    keeps its first position and its last body, like the reference's dict.  Returns (names, [body per name], depths,
    circular, hairpin_left, hairpin_right), the last four dicts by name."""
    names, bodies, depths, circular, hp_left, hp_right = [], {}, {}, {}, {}, {}
    for text, body in headers:
        header = text.strip()
        if not header:
            continue
        short = header.split()[0]
        lowered = header.lower()
        depth = 1.0
        if 'depth=' in lowered:
            try:
                depth = float(_DEPTH_RE.search(lowered).group(1))
            except (ValueError, AttributeError):
                depth = 1.0
        if short not in bodies:
            names.append(short)
        bodies[short] = body
        depths[short], circular[short] = depth, 'circular=true' in lowered
        hp_left[short], hp_right[short] = 'hairpin_left=true' in lowered, 'hairpin_right=true' in lowered
    return names, [bodies[n] for n in names], depths, circular, hp_left, hp_right


def load_fasta_arrays(filename):
    """load_fasta (misc.py:122-153) for large references: the whole file is parsed with numpy (no per-line Python, no
    3 Gb Python strings).  Returns (names, [uint8 array per contig, upper-cased], depths, circular, hairpin_left,
    hairpin_right) with the reference's header semantics (fasta_contigs)."""
    global _UPPER
    import numpy as np
    if _UPPER is None:
        _UPPER = np.arange(256, dtype=np.uint8)
        _UPPER[ord('a'):ord('z') + 1] -= 32
    with open(filename, 'rb') as f:
        magic = f.read(2)
    if magic == b'\x1f\x8b':
        with gzip.open(filename, 'rb') as f:
            raw = f.read()
    else:
        with open(filename, 'rb') as f:
            raw = f.read()
    data = np.frombuffer(raw, dtype=np.uint8)
    nl = np.flatnonzero(data == 10)
    starts = np.concatenate([[0], nl + 1])                       # first byte of every line
    starts = starts[starts < data.size]
    ends = np.concatenate([nl, [data.size]])[:starts.size]       # its newline (or the end of the file)
    is_hdr = data[starts] == ord('>')
    hdr_lines = np.flatnonzero(is_hdr)
    headers = []
    for k, li in enumerate(hdr_lines):   # a contig's body: from the end of its header line to the next header line
        hi = starts[hdr_lines[k + 1]] if k + 1 < hdr_lines.size else data.size
        headers.append((raw[starts[li] + 1:ends[li]].decode('latin-1'), (ends[li] + 1, hi)))
    names, bodies, depths, circular, hp_left, hp_right = fasta_contigs(headers)
    keep = (data != 10) & (data != 13) & (data != 32) & (data != 9)
    seqs = [_UPPER[data[lo:hi][keep[lo:hi]]] if hi > lo else np.zeros(0, dtype=np.uint8) for lo, hi in bodies]
    return names, seqs, depths, circular, hp_left, hp_right


RANDOM_SEQ_DICT = {0: 'A', 1: 'C', 2: 'G', 3: 'T'}


def get_random_base(rng=random):
    return RANDOM_SEQ_DICT[rng.randint(0, 3)]


def get_random_different_base(b, rng=random):
    base = get_random_base(rng)
    while b == base:
        base = get_random_base(rng)
    return base


def get_random_sequence(length, rng=random):
    return ''.join([get_random_base(rng) for _ in range(length)])


def random_chance(chance, rng=random):
    assert 0.0 <= chance <= 1.0
    return rng.random() < chance


def float_to_str(v, decimals=1, trim_zeros=False):
    if float(int(v)) == v:
        return str(int(v))
    result = ('%.' + str(decimals) + 'f') % v
    if trim_zeros:
        while result.endswith('0'):
            result = result[:-1]
    return result


def print_in_two_columns(l1p1, l2p1, l3p1, l1p2, l2p2, l3p2, output, space_between=6):
    width = max(len(l1p1), len(l2p1), len(l3p1)) + space_between
    fmt = '{:<' + str(width) + '}'
    print(fmt.format(l1p1) + l1p2, file=output)
    print(fmt.format(l2p1) + l2p2, file=output)
    print(fmt.format(l3p1) + l3p2, file=output)


def str_is_int(s):
    try:
        int(s)
        return True
    except ValueError:
        return False


def str_is_dna_sequence(s):
    return set(s) <= {'A', 'C', 'G', 'T'}


def identity_from_edlib_cigar(cigar):
    """misc.py:228-240: '=' columns over all columns of an extended CIGAR; 0.0 when empty."""
    matches, total = 0, 0
    for part in re.findall(r'\d+[IDX=]', cigar):
        size = int(part[:-1])
        total += size
        if part[-1] == '=':
            matches += size
    try:
        return matches / total
    except ZeroDivisionError:
        return 0.0


def compress_cigar(ops):
    """Expanded per-column ops ('=XID' characters) -> edlib's run-length extended CIGAR string."""
    if isinstance(ops, (bytes, bytearray)):
        ops = ops.decode('ascii')
    out, i = [], 0
    while i < len(ops):
        j = i
        while j < len(ops) and ops[j] == ops[i]:
            j += 1
        out.append(f'{j - i}{ops[i]}')
        i = j
    return ''.join(out)


@contextlib.contextmanager
def captured_output():
    new_out, new_err = io.StringIO(), io.StringIO()
    old_out, old_err = sys.stdout, sys.stderr
    try:
        sys.stdout, sys.stderr = new_out, new_err
        yield sys.stdout, sys.stderr
    finally:
        sys.stdout, sys.stderr = old_out, old_err
