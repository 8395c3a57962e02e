"""An independent BAM reader for the tests, written from the SAM specification v1.6 (§4.1 BGZF, §4.2 BAM): it splits the
members with zlib, parses the header and the records, asserts the fixed fields of an unaligned record as `simulate --bam`
writes them, and turns the records back into FASTQ text.  It shares no code with badread_b200.  TEST INFRASTRUCTURE."""
import struct
import zlib

SEQ_CODES = '=ACMGRSVTWYHKDBN'
EOF_MEMBER = bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')


def members(stream):
    """[(member bytes, inflated bytes)] of a BGZF stream, every member checked: gzip magic, FEXTRA with a BC subfield whose
    BSIZE is the member size - 1, deflate data that zlib inflates exactly, CRC-32 and ISIZE."""
    out, pos = [], 0
    stream = bytes(stream)
    while pos < len(stream):
        hdr = stream[pos:pos + 18]
        assert hdr[:4] == b'\x1f\x8b\x08\x04', (pos, hdr)
        xlen, si, slen, bsize = struct.unpack('<H2sHH', hdr[10:18])
        assert (xlen, si, slen) == (6, b'BC', 2), pos
        size = bsize + 1
        assert pos + size <= len(stream), pos
        m = stream[pos:pos + size]
        d = zlib.decompressobj(-15)
        data = d.decompress(m[18:-8]) + d.flush()
        assert d.eof and d.unused_data == b''
        crc, isize = struct.unpack('<II', m[-8:])
        assert crc == zlib.crc32(data) and isize == len(data)
        out.append((m, data))
        pos += size
    return out


def read_bam(stream):
    """(header text, references, records, members) of a whole BAM file, which must end with the EOF member.  Each record
    is a dict of its fields; seq is decoded to letters and qual to Phred values."""
    ms = members(stream)
    assert ms and ms[-1][0] == EOF_MEMBER, 'no end-of-file member'
    data = b''.join(d for _, d in ms)
    assert data[:4] == b'BAM\x01'
    l_text = struct.unpack('<i', data[4:8])[0]
    text = data[8:8 + l_text].decode()
    p = 8 + l_text
    n_ref = struct.unpack('<i', data[p:p + 4])[0]
    p += 4
    refs = []
    for _ in range(n_ref):
        l_name = struct.unpack('<i', data[p:p + 4])[0]
        name = data[p + 4:p + 4 + l_name].rstrip(b'\0').decode()
        l_ref = struct.unpack('<i', data[p + 4 + l_name:p + 8 + l_name])[0]
        refs.append((name, l_ref))
        p += 8 + l_name
    header_end = p
    records = []
    while p < len(data):
        block_size = struct.unpack('<i', data[p:p + 4])[0]
        rec = data[p + 4:p + 4 + block_size]
        assert len(rec) == block_size, 'truncated record'
        records.append(parse_record(rec))
        p += 4 + block_size
    return text, refs, records, ms, header_end


def parse_record(rec):
    (ref_id, pos, l_read_name, mapq, bin_, n_cigar, flag, l_seq, next_ref, next_pos, tlen) = \
        struct.unpack('<iiBBHHHiiii', rec[:32])
    p = 32
    name = rec[p:p + l_read_name]
    assert name.endswith(b'\0')
    p += l_read_name
    cigar = struct.unpack(f'<{n_cigar}I', rec[p:p + 4 * n_cigar])
    p += 4 * n_cigar
    nb = (l_seq + 1) // 2
    packed = rec[p:p + nb]
    p += nb
    seq = ''.join(SEQ_CODES[packed[i // 2] >> 4 if i % 2 == 0 else packed[i // 2] & 15] for i in range(l_seq))
    if l_seq % 2:
        assert packed[-1] & 15 == 0, 'the unused low nibble is not 0'
    qual = rec[p:p + l_seq]
    p += l_seq
    tags = {}
    while p < len(rec):
        tag, typ = rec[p:p + 2].decode(), chr(rec[p + 2])
        p += 3
        assert typ == 'Z', 'only Z tags are written'
        end = rec.index(b'\0', p)
        tags[tag] = (typ, rec[p:end].decode('latin-1'))
        p = end + 1
    return dict(ref_id=ref_id, pos=pos, mapq=mapq, bin=bin_, cigar=cigar, flag=flag, l_seq=l_seq, next_ref=next_ref,
                next_pos=next_pos, tlen=tlen, name=name[:-1].decode('latin-1'), seq=seq, qual=bytes(qual), tags=tags)


def check_unaligned(r):
    """The fixed fields of an unaligned record of `simulate --bam`."""
    assert (r['ref_id'], r['pos'], r['bin'], r['mapq'], r['flag'], r['cigar']) == (-1, -1, 4680, 0, 4, ())
    assert (r['next_ref'], r['next_pos'], r['tlen']) == (-1, -1, 0)
    assert list(r['tags']) == ['CO']


def to_fastq(records):
    """FASTQ text of unaligned records: '@{name} {CO}', the bases, '+', the qualities + 33."""
    out = []
    for r in records:
        check_unaligned(r)
        out.append(f"@{r['name']} {r['tags']['CO'][1]}\n{r['seq']}\n+\n{bytes(q + 33 for q in r['qual']).decode('latin-1')}\n")
    return ''.join(out).encode('latin-1')


def records_only(data):
    """The records of a bare record stream (no header) -> list of dicts."""
    out, p = [], 0
    while p < len(data):
        block_size = struct.unpack('<i', data[p:p + 4])[0]
        out.append(parse_record(data[p + 4:p + 4 + block_size]))
        p += 4 + block_size
    assert p == len(data)
    return out


def n_rule(seq):
    """What a read holds after BAM's 4-bit coding: the letters of =ACMGRSVTWYHKDBN (either case, as upper case), N for
    anything else."""
    return ''.join(c.upper() if c.upper() in SEQ_CODES else 'N' for c in seq)
