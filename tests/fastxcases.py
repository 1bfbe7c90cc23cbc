"""FASTA/FASTQ text parsed on the device (mgb_reads_parse_dev): the texts the simulator and GPU test modules share, the library's
host reader (mgb_reads_load) on the same bytes as the oracle, and the tables of a parse read back as (name, sequence) pairs."""
import ctypes as C
import os
import random
import tempfile

from minigraph_b200 import capi

# the texts of test_reads_loader.py, then one case per rule of the reader
TEXTS = [
    b">r1 comment here\nACGTacgtNN\nGGGG\n\n>r2\tx\nTTTT\r\n>r3\n>r4 empty before\nAC\n",
    b"@q1 c\nACGTAC\nGT\n+\n@@@@>>II\n@q2\nacgtn\n+q2\n>>>@@\n",
    b">a x\r\nACGT\r\nacgt\r\n>b\r\nGG\r\n",                         # CRLF
    b"@a\r\nACGT\r\n+\r\n@@@@\r\n@b\r\nAC\r\n+\r\n>+\r\n",
    b">a\n>b\n\n>c\nAC\n>d\n",                                       # empty records, an empty last one
    b">e\n",
    b">a\tb c\td\nACGT\n>b \t \nGG\n>c\x0bd\nTT\n>e\x0cf\nAA\n",           # comments after tabs and other white space
    b">a\nACGT\n>lastname",                                          # a name at the end without a newline
    b"@x\nAC\n+\n@@\n@y",
    b">a\nACGT\n@b c\nGGTT\n+\n>>@@\n>c\nTT\n",                       # FASTA and FASTQ mixed
    b">a\nAC\nGT\nTT\n>b\nA\n\nC\n",                                  # multi-line
    b"@a\nACG\nTAC\n+\n@@@\n>>>\n@b\nA\n+\n@\n",
    b"@r1\nACGT\n+\n@ABC\n@r2\nACGT\n+\n>ABC\n@r3\nAC\n+\n+A\n@r4\nAC\n+\n@@\n",  # qualities that start with '@', '>', '+'
    b"@r1\nACGTACGT\n+\n@@@",                                        # a quality cut short by the end
    b"junk text\nmore\n>a\nAC\n",                                    # junk before the first header
    b"xyz+\n@q\nAC\n+\n!!\n",
    b">a x>y@z\nAC\n@b c@d>\nGT\n+\n@>@>\n>c\nA>C@G\n",                 # '>' and '@' inside comments, qualities and sequences
    b"", b"\n\n", b"no header at all\n", b">", b"@", b">>>", b"@\n+\n", b"@a\nACGT\n+\n", b">a\r\r\nAC\rGT\n",
    b"@r\nAC\n+\nA\nB\nC\n>x\n", b"@r\nACGT\n+x y\nAB\r\nCD\n@s\n", b"+\n>a\n+\nAC\n", b"@a\n@b\n+\n\n",
    b">a\nac gt\tn-*\n>b\n\x80\xff\x01z\n",
]

_QUAL = b"!\"#$%&'()*+,-./0123456789:;<=>?@ABCDEFGHIJ"


def random_text(rng):
    """pieces of well- and ill-formed records: headers with comments, sequence and quality lines (quality bytes rich in '@>+'),
    CR/LF line ends, junk, records without a quality, qualities of the wrong length and a last line without its newline"""
    out = []
    eol = lambda: rng.choice([b"\n", b"\n", b"\n", b"\r\n", b"\r\r\n"])
    if rng.random() < 0.3:
        out.append(bytes(rng.choice(b"xyz +@>\n\t") for _ in range(rng.randrange(1, 12))))
    for _ in range(rng.randrange(0, 9)):
        fq = rng.random() < 0.6
        name = bytes(rng.choice(b"abcXYZ019_:@>+") for _ in range(rng.randrange(0, 8)))
        head = (b"@" if fq else b">") + name
        if rng.random() < 0.4:
            head += rng.choice([b" ", b"\t", b" \t"]) + bytes(rng.choice(b"cm @>+\t") for _ in range(rng.randrange(0, 8)))
        out.append(head + eol())
        seq = bytes(rng.choice(b"ACGTacgtnN") for _ in range(rng.randrange(0, 40)))
        w = rng.randrange(1, 20)
        for i in range(0, len(seq), w):
            out.append(seq[i:i + w] + eol())
        if rng.random() < 0.15:
            out.append(eol())
        if fq and rng.random() < 0.9:
            out.append(b"+" + (name if rng.random() < 0.3 else b"") + eol())
            ql = len(seq) + (0 if rng.random() < 0.8 else rng.randrange(-3, 4))
            q = bytes(rng.choice(b"@>+" if rng.random() < 0.3 else _QUAL) for _ in range(max(0, ql)))
            qw = rng.randrange(1, 25)
            for i in range(0, len(q), qw):
                out.append(q[i:i + qw] + eol())
    text = b"".join(out)
    if text and rng.random() < 0.25:
        text = text[:rng.randrange(len(text) + 1)]  # cut anywhere
    return text


def random_texts(n, seed):
    rng = random.Random(seed)
    return [random_text(rng) for _ in range(n)]


def host_load(lib, text, max_bases=0):
    """mgb_reads_load() on text written to a file: [(name, sequence)]"""
    fd, fn = tempfile.mkstemp(suffix=".fx")
    try:
        os.write(fd, text)
        os.close(fd)
        r = lib.mgb_reads_load(fn.encode(), max_bases)
        assert r
        c = r.contents
        out = [(c.name[i], C.string_at(c.seq[i], c.len[i])) for i in range(c.n_reads)]
        lib.mgb_reads_free(r)
        return out
    finally:
        os.unlink(fn)


def fastq(names, seqs, rng, width=0):
    """FASTQ text of the reads: 4-line records, or with width > 0 sequence and quality lines of at most width bytes; qualities
    drawn from Q0..Q41 with '@', '>' and '+' (Q31, Q29, Q10) at least a third of the time"""
    out = []
    for nm, s in zip(names, seqs):
        q = bytes(rng.choice(b"@>+") if rng.random() < 0.34 else rng.choice(_QUAL) for _ in range(len(s)))
        out.append(b"@" + nm + b" c\n")
        for x, sep in ((s, b"+\n"), (q, b"")):
            if width:
                out += [x[i:i + width] + b"\n" for i in range(0, len(x), width)] or [b"\n"]
            else:
                out.append(x + b"\n")
            out.append(sep)
    return b"".join(out)


def fasta(names, seqs, width=0):
    out = []
    for nm, s in zip(names, seqs):
        out.append(b">" + nm + b"\n")
        out += [s[i:i + width] + b"\n" for i in range(0, len(s), width)] if width else [s + b"\n"]
    return b"".join(out)


def tables(block_addr, dr, read):
    """the records of an mgb_dev_reads_t as [(name, sequence)], its two offset tables checked; read(addr, nbytes) -> bytes"""
    import numpy as np
    n = dr.n_reads
    off = np.frombuffer(read(block_addr + dr.off[1], 8 * (n + 1)), dtype=np.int64)
    noff = np.frombuffer(read(block_addr + dr.off[3], 8 * (n + 1)), dtype=np.int64)
    assert off[0] == 0 and noff[0] == 0 and off[n] == dr.n_bases and noff[n] == dr.name_bytes, (off, noff)
    seq = read(block_addr + dr.off[0], dr.n_bases)
    name = read(block_addr + dr.off[2], dr.name_bytes)
    return [(name[noff[i]:noff[i + 1]], seq[off[i]:off[i + 1]]) for i in range(n)]


def expect_layout(dr):
    """the block layout the header promises: 256-byte aligned tables in order, sized by the rows"""
    sizes = [dr.n_bases, 8 * (dr.n_reads + 1), dr.name_bytes, 8 * (dr.n_reads + 1)]
    at = 0
    for t, sz in enumerate(sizes):
        assert dr.off[t] == at, (t, list(dr.off))
        at += (sz + 255) & ~255
    assert dr.bytes == at


DR = capi.mgb_dev_reads_t
