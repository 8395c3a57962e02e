"""A plain deflate (RFC 1951) and gzip (RFC 1952) reference, independent of the kernels in csrc/bb_bgzf.cuh and
csrc/bb_inflate.cuh: a strict member parser that records every block's structure, an encoder of explicit block programs,
and optimal Huffman costs (unlimited from a heap, length-limited by package-merge).  Pure Python and numpy; it is
trusted because it parses zlib's output to zlib's bytes and zlib inflates everything it encodes
(tests/test_deflate_edges.py).  TEST INFRASTRUCTURE."""
import heapq
import struct
import zlib

import numpy as np

CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258)
LEN_EXTRA = (0,) * 8 + (1,) * 4 + (2,) * 4 + (3,) * 4 + (4,) * 4 + (5,) * 4 + (0,)
DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577)
DIST_EXTRA = (0, 0, 0, 0) + tuple(k // 2 for k in range(2, 28))
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32                 # symbols 30 and 31 have codes but are no distance
RLE_EXTRA = {16: 2, 17: 3, 18: 7}
BGZF_HEADER = b'\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0'


class DeflateError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------ codes
def kraft(lens):
    """Kraft sum of the non-zero lengths, as a fraction of 2^15 (exactly 1 << 15 for a complete code)."""
    return sum(1 << (15 - l) for l in lens if l)


def canonical(lens):
    """RFC 1951 §3.2.2: the code of every symbol with a non-zero length, most significant bit first."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    codes = [0] * len(lens)
    for s, l in enumerate(lens):
        if l:
            codes[s] = nxt[l]
            nxt[l] += 1
    return codes


def check_code(lens, what, allow_empty=False):
    """zlib's rule: over-subscribed never; incomplete only as a single code of one bit; no codes only for distances."""
    k, used = kraft(lens), [l for l in lens if l]
    if k > 1 << 15:
        raise DeflateError(f'over-subscribed {what} code')
    if not used:
        if not allow_empty:
            raise DeflateError(f'empty {what} code')
        return
    if k < 1 << 15 and used != [1]:
        raise DeflateError(f'incomplete {what} code')


class _Decoder(object):
    """Table decoder of a canonical code: a list of 2^max_len entries indexed by the next max_len bits, LSB first."""

    def __init__(self, lens):
        self.bits = max(lens) if any(lens) else 1
        self.table = [None] * (1 << self.bits)
        for s, (l, c) in enumerate(zip(lens, canonical(lens))):
            if l:
                rev = int(format(c, f'0{l}b')[::-1], 2)
                self.table[rev::1 << l] = [(s, l)] * (1 << (self.bits - l))


class BitReader(object):
    def __init__(self, data):
        self.data = bytes(data)
        self.n_bits = 8 * len(self.data)
        self.pos = 0

    def peek(self, n):                                   # n <= 25; bits past the end read as zero
        p = self.pos
        return (int.from_bytes(self.data[p >> 3:(p >> 3) + 4], 'little') >> (p & 7)) & ((1 << n) - 1)

    def get(self, n):
        if self.pos + n > self.n_bits:
            raise DeflateError('truncated deflate data')
        v = self.peek(n)
        self.pos += n
        return v

    def sym(self, dec):
        e = dec.table[self.peek(dec.bits)]
        if e is None:
            raise DeflateError('invalid Huffman code')
        if self.pos + e[1] > self.n_bits:
            raise DeflateError('truncated deflate data')
        self.pos += e[1]
        return e[0]


# ------------------------------------------------------------------------------------------------ parser
def parse_deflate(data, limit_out=None):
    """Raw deflate data -> (inflated bytes, blocks, end bit).  Each block is a dict: type ('stored', 'fixed',
    'dynamic'), final, start / end bit, out (first, end) byte of what it produced, and for dynamic blocks hlit, hdist,
    hclen, cl_lens (19, by symbol), rle [(symbol, extra)], lit_lens, dist_lens; stored blocks: len.  Raises DeflateError
    for anything zlib refuses."""
    r = BitReader(data)
    out = bytearray()
    blocks = []
    fixed = (_Decoder(FIXED_LIT), _Decoder(FIXED_DIST))
    while True:
        b = {'start': r.pos, 'out0': len(out)}
        b['final'] = r.get(1)
        bt = r.get(2)
        if bt == 0:
            b['type'] = 'stored'
            b['pad'] = -r.pos & 7
            r.get(b['pad'])
            n, nn = r.get(16), r.get(16)
            if n ^ 0xffff != nn:
                raise DeflateError('stored block length does not match its complement')
            if r.pos + 8 * n > r.n_bits:
                raise DeflateError('truncated deflate data')
            out += r.data[r.pos >> 3:(r.pos >> 3) + n]
            r.pos += 8 * n
            b['len'] = n
        elif bt == 3:
            raise DeflateError('invalid block type')
        else:
            if bt == 1:
                b['type'] = 'fixed'
                lit, dist = fixed
            else:
                b['type'] = 'dynamic'
                hlit, hdist, hclen = r.get(5) + 257, r.get(5) + 1, r.get(4) + 4
                if hlit > 286 or hdist > 30:
                    raise DeflateError('too many length or distance symbols')
                cl = [0] * 19
                for k in range(hclen):
                    cl[CL_ORDER[k]] = r.get(3)
                check_code(cl, 'code-length')
                if kraft(cl) != 1 << 15:
                    raise DeflateError('incomplete code-length code')
                cld = _Decoder(cl)
                lens, rle = [], []
                while len(lens) < hlit + hdist:
                    s = r.sym(cld)
                    x = r.get(RLE_EXTRA[s]) if s >= 16 else 0
                    rle.append((s, x))
                    if s < 16:
                        lens.append(s)
                        continue
                    if s == 16 and not lens:
                        raise DeflateError('repeat of no previous length')
                    v, rep = (lens[-1], 3 + x) if s == 16 else (0, 3 + x if s == 17 else 11 + x)
                    if len(lens) + rep > hlit + hdist:
                        raise DeflateError('code-length repeat past HLIT + HDIST')
                    lens += [v] * rep
                lit_lens, dist_lens = lens[:hlit], lens[hlit:]
                if lit_lens[256] == 0:
                    raise DeflateError('no end-of-block code')
                check_code(lit_lens, 'literal/length')
                check_code(dist_lens, 'distance', allow_empty=True)
                b.update(hlit=hlit, hdist=hdist, hclen=hclen, cl_lens=cl, rle=rle, lit_lens=lit_lens, dist_lens=dist_lens)
                lit, dist = _Decoder(lit_lens), _Decoder(dist_lens)
            while True:
                s = r.sym(lit)
                if s < 256:
                    out.append(s)
                elif s == 256:
                    break
                else:
                    s -= 257
                    if s >= 29:
                        raise DeflateError('invalid literal/length code')
                    n = LEN_BASE[s] + r.get(LEN_EXTRA[s])
                    d = r.sym(dist)
                    if d >= 30:
                        raise DeflateError('invalid distance code')
                    d = DIST_BASE[d] + r.get(DIST_EXTRA[d])
                    if d > len(out):
                        raise DeflateError('distance before the start of the member')
                    for _ in range(n):
                        out.append(out[-d])
                if limit_out is not None and len(out) > limit_out:
                    raise DeflateError('more data than ISIZE')
        b['end'] = r.pos
        b['out'] = (b.pop('out0'), len(out))
        blocks.append(b)
        if b['final']:
            return bytes(out), blocks, r.pos


def parse_member(member, allow_trailing=False):
    """One gzip member -> dict: flg, mtime, xfl, os, extra [(si, bytes)], bsize (BC field or None), blocks, data,
    padding (value, n_bits) after the final block, trailing (bytes between the final block and the trailer), crc,
    isize.  Strict as zlib is (header, codes, repeats, distances, CRC, ISIZE); bytes between the final block and the
    trailer raise DeflateError unless allow_trailing."""
    m = bytes(member)
    if len(m) < 18 or m[:3] != b'\x1f\x8b\x08':
        raise DeflateError('not a gzip member with deflate data')
    flg, mtime, xfl, os_ = m[3], struct.unpack('<I', m[4:8])[0], m[8], m[9]
    if flg & 0xe0:
        raise DeflateError('reserved header flags')
    p, extra, bsize = 10, [], None
    if flg & 4:
        xlen = struct.unpack('<H', m[10:12])[0]
        f, p = 12, 12 + xlen
        while f + 4 <= p:
            si, slen = m[f:f + 2], struct.unpack('<H', m[f + 2:f + 4])[0]
            extra.append((si, m[f + 4:f + 4 + slen]))
            if si == b'BC' and slen == 2:
                bsize = struct.unpack('<H', m[f + 4:f + 6])[0]
            f += 4 + slen
    for bit in (8, 16):                                     # FNAME, FCOMMENT
        if flg & bit:
            p = m.index(b'\0', p) + 1
    if flg & 2:
        p += 2
    if len(m) < p + 8:
        raise DeflateError('truncated member')
    crc, isize = struct.unpack('<II', m[-8:])
    data, blocks, end = parse_deflate(m[p:-8], limit_out=isize)
    n_data = len(m) - 8 - p
    used = (end + 7) // 8
    res = dict(flg=flg, mtime=mtime, xfl=xfl, os=os_, extra=extra, bsize=bsize, blocks=blocks, data=data, crc=crc,
               isize=isize, data_bytes=n_data, padding=(m[p + used - 1] >> (end & 7) if end & 7 else 0, -end & 7),
               trailing=n_data - used)
    if res['trailing'] and not allow_trailing:
        raise DeflateError('bytes between the final block and the trailer')
    if isize != len(data):
        raise DeflateError('ISIZE mismatch')
    if crc != zlib.crc32(data):
        raise DeflateError('CRC-32 mismatch')
    return res


def split_bgzf(stream):
    """The members of a BGZF stream, by their BC fields."""
    out, pos = [], 0
    while pos < len(stream):
        size = struct.unpack('<H', stream[pos + 16:pos + 18])[0] + 1
        assert stream[pos:pos + 4] == b'\x1f\x8b\x08\x04' and stream[pos + 12:pos + 14] == b'BC', pos
        out.append(bytes(stream[pos:pos + size]))
        pos += size
    assert pos == len(stream)
    return out


# ------------------------------------------------------------------------------------------------ costs and lengths
def huffman_cost(freq):
    """Bits of the optimal (unlimited) prefix code of the non-zero frequencies: the sum of a heap-built tree's internal
    node weights.  A lone symbol costs one bit per occurrence."""
    h = [f for f in freq if f]
    if len(h) == 1:
        return h[0]
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        w = heapq.heappop(h) + heapq.heappop(h)
        cost += w
        heapq.heappush(h, w)
    return cost


def huffman_lengths(freq):
    """An optimal code of least depth: leaves ranked by (frequency, symbol), two queues, a leaf taken before an internal
    node of the same weight; the ranks' depths handed out so that the longest lengths go to the lowest ranks.  Lengths
    unlimited."""
    leaves = sorted((f, s) for s, f in enumerate(freq) if f)
    lens = [0] * len(freq)
    if len(leaves) == 1:
        lens[leaves[0][1]] = 1
        return lens
    parent_leaf, parent_node, node_w = [0] * len(leaves), [], []
    li = ni = 0
    for k in range(len(leaves) - 1):
        w = 0
        for _ in range(2):
            if li < len(leaves) and (ni >= k or leaves[li][0] <= node_w[ni]):
                w += leaves[li][0]
                parent_leaf[li] = k
                li += 1
            else:
                w += node_w[ni]
                parent_node.append(k)
                ni += 1
        node_w.append(w)
    depth = [0] * len(node_w)
    for k in range(len(node_w) - 2, -1, -1):
        depth[k] = depth[parent_node[k]] + 1
    ds = sorted((depth[p] + 1 for p in parent_leaf), reverse=True)
    for (_, s), d in zip(leaves, ds):
        lens[s] = d
    return lens


def _package_merge(freq, max_len):
    items = sorted((f, s) for s, f in enumerate(freq) if f)
    n = len(items)
    if n == 1:
        return [1], [items[0][1]], n
    if n > 1 << max_len:
        raise ValueError('too many symbols for the length limit')
    leaves = [(f, np.eye(1, n, i, dtype=np.int64)[0]) for i, (f, _) in enumerate(items)]
    cur = list(leaves)
    for _ in range(max_len - 1):
        pk = [(cur[i][0] + cur[i + 1][0], cur[i][1] + cur[i + 1][1]) for i in range(0, len(cur) - 1, 2)]
        merged, a, b = [], 0, 0
        while a < len(leaves) or b < len(pk):                  # leaves first on ties (stable)
            if b >= len(pk) or (a < len(leaves) and leaves[a][0] <= pk[b][0]):
                merged.append(leaves[a]); a += 1
            else:
                merged.append(pk[b]); b += 1
        cur = merged
    depth = sum(c for _, c in cur[:2 * n - 2])
    return list(depth), [s for _, s in items], n


def limited_lengths(freq, max_len):
    """Optimal code lengths of at most max_len bits (package-merge)."""
    depth, syms, _ = _package_merge(freq, max_len)
    lens = [0] * len(freq)
    for s, d in zip(syms, depth):
        lens[s] = int(d)
    return lens


def limited_cost(freq, max_len):
    """Bits of the optimal code of at most max_len bits."""
    lens = limited_lengths(freq, max_len)
    return sum(f * l for f, l in zip(freq, lens))


# ------------------------------------------------------------------------------------------------ encoder
class BitWriter(object):
    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, v, n):                                 # LSB first
        assert 0 <= v < 1 << n or n == 0 and v == 0, (v, n)
        self.acc |= v << self.n
        self.n += n

    def put_code(self, code, n):                         # Huffman codes go most significant bit first
        self.put(int(format(code, f'0{n}b')[::-1], 2) if n else 0, n)

    def align(self):
        self.n += -self.n & 7

    def bytes(self):
        return self.acc.to_bytes((self.n + 7) // 8, 'little')


def rle_greedy(lens):
    """Code lengths run-length coded the way a simple encoder does: a run of zeros as 18s of up to 138 then one 17
    (3-10), a run of another length as the length once then 16s of up to 6, the rest literally."""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                out.append((18, r - 11))
                run -= r
            if run >= 3:
                out.append((17, run - 3))
                run = 0
        else:
            out.append((v, 0))
            run -= 1
            while run >= 3:
                r = min(run, 6)
                out.append((16, r - 3))
                run -= r
        out += [(v, 0)] * run
    return out


def len_symbol(n):
    k = max(i for i in range(29) if LEN_BASE[i] <= n)
    return k, n - LEN_BASE[k]


def dist_symbol(d):
    k = max(i for i in range(30) if DIST_BASE[i] <= d)
    return k, d - DIST_BASE[k]


def _token_freqs(tokens, n_lit=286, n_dist=30):
    lf, df = [0] * n_lit, [0] * n_dist
    for t in tokens:
        if isinstance(t, int):
            lf[t] += 1
        else:
            lf[t[2] if len(t) == 3 else 257 + len_symbol(t[0])[0]] += 1
            df[dist_symbol(t[1])[0]] += 1
    lf[256] += 1
    return lf, df


def encode_block(w, blk, final):
    """Appends one block of a program to BitWriter w.  blk: dict with 'type' and
    - stored: 'data'; optional 'phase' (asserted bit position mod 8 at the block's start), 'nlen' (override).
    - fixed / dynamic: 'tokens' - ints for literals, (length, distance) for matches, (258, distance, 284) for length
      258 as code 284 with 31 extra bits.
    - dynamic, all optional: 'lit_lens', 'dist_lens' (default: optimal 15-bit lengths of the tokens' histogram; no
      distance codes when there are no matches), 'hlit', 'hdist' (default: the lists' lengths), 'rle' [(symbol, extra)]
      (default rle_greedy), 'cl_lens' (19, by symbol; default optimal 7-bit lengths of the rle's histogram), 'hclen'
      (default: trimmed to the last non-zero entry in CL_ORDER, at least 4)."""
    if 'phase' in blk:
        assert w.n & 7 == blk['phase'], (w.n & 7, blk['phase'])
    w.put(int(final), 1)
    t = blk['type']
    if t == 'stored':
        w.put(0, 2)
        w.align()
        data = bytes(blk['data'])
        w.put(len(data), 16)
        w.put(blk.get('nlen', len(data) ^ 0xffff), 16)
        for c in data:
            w.put(c, 8)
        return
    tokens = blk.get('tokens', [])
    if t == 'fixed':
        w.put(1, 2)
        lit_lens, dist_lens = FIXED_LIT, FIXED_DIST
    else:
        w.put(2, 2)
        lf, df = _token_freqs(tokens)
        lit_lens = blk.get('lit_lens') or limited_lengths(lf, 15)
        if 'dist_lens' in blk:
            dist_lens = blk['dist_lens']
        else:
            dist_lens = limited_lengths(df, 15) if sum(1 for f in df if f) > 1 else [1 if f else 0 for f in df] \
                if any(df) else [0]
        while len(lit_lens) > 257 and not lit_lens[-1] and 'lit_lens' not in blk:
            lit_lens = lit_lens[:-1]
        while len(dist_lens) > 1 and not dist_lens[-1] and 'dist_lens' not in blk:
            dist_lens = dist_lens[:-1]
        lit_lens, dist_lens = list(lit_lens), list(dist_lens)
        hlit, hdist = blk.get('hlit', len(lit_lens)), blk.get('hdist', len(dist_lens))
        rle = blk.get('rle') or rle_greedy(lit_lens + dist_lens)
        if 'cl_lens' in blk:
            cl = blk['cl_lens']
        else:
            cf = [0] * 19
            for s, _ in rle:
                cf[s] += 1
            for s in range(19):                  # a complete code-length code needs two symbols
                if sum(1 for f in cf if f) < 2 and not cf[s]:
                    cf[s] = 1
            cl = limited_lengths(cf, 7)
        hclen = blk.get('hclen')
        if hclen is None:
            hclen = 19
            while hclen > 4 and not cl[CL_ORDER[hclen - 1]]:
                hclen -= 1
        w.put(hlit - 257, 5)
        w.put(hdist - 1, 5)
        w.put(hclen - 4, 4)
        for k in range(hclen):
            w.put(cl[CL_ORDER[k]], 3)
        clc = canonical(cl)
        for s, x in rle:
            w.put_code(clc[s], cl[s])
            if s >= 16:
                w.put(x, RLE_EXTRA[s])
    lc, dc = canonical(lit_lens), canonical(dist_lens)
    for tok in list(tokens) + [256]:
        if isinstance(tok, int):
            assert lit_lens[tok], ('no code for literal', tok)
            w.put_code(lc[tok], lit_lens[tok])
            continue
        n, d = tok[0], tok[1]
        if len(tok) == 3:
            k = tok[2] - 257
            x = n - LEN_BASE[k]
        else:
            k, x = len_symbol(n)
        assert lit_lens[257 + k], ('no code for length symbol', 257 + k)
        w.put_code(lc[257 + k], lit_lens[257 + k])
        w.put(x, LEN_EXTRA[k])
        ds, dx = dist_symbol(d)
        assert dist_lens[ds], ('no code for distance symbol', ds)
        w.put_code(dc[ds], dist_lens[ds])
        w.put(dx, DIST_EXTRA[ds])


def deflate(program):
    """Raw deflate data of a list of blocks (see encode_block); the last block is final unless it says otherwise."""
    w = BitWriter()
    for i, blk in enumerate(program):
        encode_block(w, blk, blk.get('final', i == len(program) - 1))
    return w.bytes()


def tokens_output(tokens):
    """The bytes a list of tokens produces, given nothing before it (distances into a prefix: use expand)."""
    return expand(b'', tokens)


def expand(prefix, tokens):
    out = bytearray(prefix)
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            for _ in range(t[0]):
                out.append(out[-t[1]])
    return bytes(out[len(prefix):])


def program_output(program):
    out = b''
    for blk in program:
        out += bytes(blk['data']) if blk['type'] == 'stored' else expand(out, blk.get('tokens', []))
    return out


def member(deflate_data, data=None, isize=None, crc=None):
    """A BGZF member around raw deflate data; ISIZE and CRC from data unless given."""
    isize = len(data) if isize is None else isize
    crc = zlib.crc32(data) if crc is None else crc
    return BGZF_HEADER + struct.pack('<H', len(deflate_data) + 25) + bytes(deflate_data) + struct.pack('<II', crc, isize)


def encode(program):
    """A BGZF member of a block program, and the bytes it inflates to."""
    data = program_output(program)
    return member(deflate(program), data), data
