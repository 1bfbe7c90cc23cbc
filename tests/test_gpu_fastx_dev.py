"""FASTA/FASTQ text in GPU memory parsed on the device (mgb_reads_parse_dev, minigraph_b200.tensors.parse_cuda_fastx /
iter_cuda_fastx) against the library's host reader mgb_reads_load() on the same bytes: the reader's rule cases, seeded random texts,
the fixtures, the GAF test sets as FASTA and FASTQ mapped end to end against mgb_reads_load() + mgb_map_batch_gaf(), a 6 000-read
file parsed in chunks of a few MB, stream ordering, a second device and refusals."""
import ctypes as C
import os
import random

import pytest

import fastxcases as FX
import gafcases as GC
import mgtest as T
from minigraph_b200 import capi
from minigraph_b200.tensors import iter_cuda_fastx, map_cuda_reads, parse_cuda_fastx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return capi.load_product()


@pytest.fixture(scope="module")
def ix(lib):
    ix = GC.Index(lib, os.path.join(T.FIX, "MT.gfa"), "lr")
    yield ix
    ix.close()


def cuda_bytes(b, device="cuda:0"):
    import torch
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(device) if b else torch.empty(0, dtype=torch.uint8, device=device)


def parse_raw(lib, ix, text, max_bases=0, final=1):
    """the C call with a block torch allocates pre-filled with 0xA5: (rc, [(name, sequence)], used)"""
    import torch
    t = cuda_bytes(text)
    blocks = []

    def alloc(_, nbytes):
        blocks.append(torch.full((max(1, nbytes),), 0xA5, dtype=torch.uint8, device="cuda:0"))
        torch.cuda.synchronize()
        return blocks[-1].data_ptr()

    cb = capi.mgb_dev_alloc_fn(alloc)
    dr = capi.mgb_dev_reads_t()
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.mgb_reads_parse_dev(ix.gi, t.data_ptr(), t.numel(), max_bases, final, stream, cb, None, C.byref(dr))
    if rc < 0:
        assert not blocks and not dr.block
        return rc, None, None
    assert len(blocks) == 1 and dr.block == blocks[0].data_ptr()
    FX.expect_layout(dr)
    host = bytes(blocks[0].cpu().numpy())
    return rc, FX.tables(0, dr, lambda a, n: host[a:a + n]), dr.used


def check(lib, ix, text):
    rc, got, used = parse_raw(lib, ix, text)
    assert rc == 0, lib.mgb_last_error()
    assert got == FX.host_load(lib, text), text[:200]
    assert used == len(text)


def test_reader_cases(lib, ix):
    for text in FX.TEXTS:
        check(lib, ix, text)


def test_random_texts(lib, ix):
    texts = FX.random_texts(300, 11)
    for text in texts:
        check(lib, ix, text)
    check(lib, ix, b"".join(texts + FX.TEXTS) * 3)


def test_fixtures(lib, ix):
    for fn in sorted(os.listdir(T.FIX)):
        if fn.endswith(".fa"):
            check(lib, ix, open(os.path.join(T.FIX, fn), "rb").read())


def test_chunked_and_max_bases(lib, ix):
    texts = [t for t in FX.random_texts(200, 5) if len(t) > 60][:12]
    text = b"junk\n" + b"".join(texts) + FX.TEXTS[12] + FX.TEXTS[1]
    whole = FX.host_load(lib, text)
    for cut in range(0, len(text) + 1, 7):
        out, carry = [], b""
        for piece, final in ((text[:cut], 0), (text[cut:], 1)):
            buf = carry + piece
            rc, recs, used = parse_raw(lib, ix, buf, 0, final)
            assert rc == 0
            out += recs
            carry = buf[used:]
        assert out == whole, cut
    for mb in (1, 5, 16, 40):
        rc, recs, used = parse_raw(lib, ix, text, mb)
        assert recs == FX.host_load(lib, text, mb) and (used == len(text) or text[used:used + 1] in (b">", b"@")), mb


def as_texts(names, seqs, seed):
    rng = random.Random(seed)
    return {"fasta": FX.fasta(names, seqs), "fasta60": FX.fasta(names, seqs, 60), "fastq": FX.fastq(names, seqs, rng),
            "fastq70": FX.fastq(names, seqs, rng, 70)}


def test_gaf_sets_end_to_end(lib, workdir, tmp_path):
    """parse_cuda_fastx -> map_cuda_reads gives the text of mgb_reads_load -> mgb_map_batch_gaf, byte for byte"""
    for kind, preset in (("c2", "lr"), ("c3", "lr"), ("c4", "asm"), ("sv_edge", "lr")):
        gfa, names, seqs = GC.inputs(kind, workdir)
        ix = GC.Index(lib, gfa, preset)
        try:
            for form, text in as_texts(names, seqs, 3).items():
                want_recs = FX.host_load(lib, text)
                assert [s for _, s in want_recs] == seqs, form
                seq, off, got_names, used = parse_cuda_fastx(lib, ix.gi, cuda_bytes(text))
                assert used == len(text) and got_names == [n for n, _ in want_recs]
                rc, want = GC.map_gaf(lib, ix, [n for n, _ in want_recs], [s for _, s in want_recs])
                assert rc == 0
                GC.check(map_cuda_reads(lib, ix.gi, seq, off, got_names, opt=ix.mo), want)
        finally:
            ix.close()


def test_file_in_chunks(lib, workdir, tmp_path):
    """6 000 reads written as FASTQ (and gzip) parsed in chunks of a few MB, with and without max_bases, mapped batch by batch"""
    import gzip
    hap, reads = os.path.join(workdir, "gmt.hap.fa"), os.path.join(workdir, "gfx6000.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, 6000, 5000, "ont", 23)
    names, seqs = T.read_fasta(reads, upper=False)
    text = FX.fastq(names, seqs, random.Random(4), 0)
    fq, fqgz = str(tmp_path / "r.fq"), str(tmp_path / "r.fq.gz")
    open(fq, "wb").write(text)
    with gzip.open(fqgz, "wb") as f:
        f.write(text)
    want = FX.host_load(lib, text)
    assert len(want) == 6000
    gfa = os.path.join(T.FIX, "MT.gfa")
    ix = GC.Index(lib, gfa, "lr")
    try:
        for path, chunk, mb in ((fq, 3 << 20, 0), (fqgz, 5 << 20, 0), (fq, 4 << 20, 4_000_000)):
            got, gaf = [], []
            for seq, off, nm in iter_cuda_fastx(lib, ix.gi, path, chunk, mb):
                s = bytes(seq.cpu().numpy())
                o = off.tolist()
                got += [(nm[i], s[o[i]:o[i + 1]]) for i in range(len(nm))]
                if path == fq and mb == 0:
                    gaf.append(map_cuda_reads(lib, ix.gi, seq, off, nm, opt=ix.mo))
            assert got == want, (path, chunk, mb)
            if gaf:
                rc, w = GC.map_gaf(lib, ix, [n for n, _ in want], [s for _, s in want])
                assert rc == 0
                GC.check(b"".join(gaf), w)
    finally:
        ix.close()


def test_side_stream_and_overwrite(lib, ix, workdir):
    """the text written by a torch kernel on a side stream that is still busy: the parse orders its reads after it; the text is
    overwritten right after the call returns"""
    import torch
    _, names, seqs = GC.inputs("c2", workdir)
    text = FX.fastq(names, seqs, random.Random(8), 50)
    want = FX.host_load(lib, text)
    src = cuda_bytes(text)
    dst = torch.zeros_like(src)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)  # the side stream is busy for a while before it writes the text
        dst.copy_(src)
        seq, off, nm, used = parse_cuda_fastx(lib, ix.gi, dst)
        dst.fill_(ord("@"))
        s = bytes(seq.cpu().numpy())
    o = off.tolist()
    assert used == len(text) and [(nm[i], s[o[i]:o[i + 1]]) for i in range(len(nm))] == want


def test_refusals(lib, ix):
    import torch
    calls = []
    cb = capi.mgb_dev_alloc_fn(lambda _, n: calls.append(n) or None)
    dr = capi.mgb_dev_reads_t()
    host = torch.frombuffer(bytearray(b">a\nAC\n"), dtype=torch.uint8)
    rc = lib.mgb_reads_parse_dev(ix.gi, host.data_ptr(), 6, 0, 1, None, cb, None, C.byref(dr))
    assert rc < 0 and b"not device" in lib.mgb_last_error()
    dev = cuda_bytes(b">a\nAC\n")
    rc = lib.mgb_reads_parse_dev(ix.gi, dev.data_ptr(), -1, 0, 1, None, cb, None, C.byref(dr))
    assert rc < 0 and b"at least 0" in lib.mgb_last_error()
    if torch.cuda.device_count() > 1:
        other = cuda_bytes(b">a\nAC\n", "cuda:1")
        rc = lib.mgb_reads_parse_dev(ix.gi, other.data_ptr(), 6, 0, 1, None, cb, None, C.byref(dr))
        assert rc < 0 and b"not device" in lib.mgb_last_error()
    assert calls == [] and not dr.block
    rc = lib.mgb_reads_parse_dev(ix.gi, dev.data_ptr(), 6, 0, 1, None, cb, None, C.byref(dr))
    assert rc < 0 and b"no block" in lib.mgb_last_error() and len(calls) == 1 and not dr.block
    with pytest.raises(ValueError):
        parse_cuda_fastx(lib, ix.gi, host)
    with pytest.raises(ValueError):
        parse_cuda_fastx(lib, ix.gi, dev.to(torch.int32))
