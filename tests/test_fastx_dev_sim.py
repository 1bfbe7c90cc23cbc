"""FASTA/FASTQ text parsed on the device (mgb_reads_parse_dev), in both simulators of the device code, against the library's host
reader mgb_reads_load() on the same bytes: the reader's rule cases and seeded random texts, chunked parses with carry-over cut at
every byte, max_bases, the refusals, and where oracle/_ref is built the reference's bseq.c on the well-formed texts."""
import ctypes as C
import os

import pytest

import fastxcases as FX
import gafcases as GC
import mgtest as T


@pytest.fixture(scope="module", params=["hostsim", "hostsim32"])
def ctx(request):
    lib = T.load_hostsim() if request.param == "hostsim" else T.load_hostsim32()
    ix = GC.Index(lib, os.path.join(T.FIX, "MT.gfa"), "lr")
    yield lib, ix
    ix.close()


def parse(lib, ix, text, max_bases=0, final=1, calls=None):
    """mgb_reads_parse_dev in a simulator (where "device memory" is host memory), the block pre-filled with 0xA5:
    (rc, [(name, sequence)], used)"""
    buf = C.create_string_buffer(text, max(1, len(text)))
    blocks = []

    def alloc(_, nbytes):
        blocks.append(C.create_string_buffer(b"\xa5" * nbytes, max(1, nbytes)))
        return C.addressof(blocks[-1])

    cb = FX.capi.mgb_dev_alloc_fn(alloc)
    dr = FX.DR()
    rc = lib.mgb_reads_parse_dev(ix.gi, C.addressof(buf), len(text), max_bases, final, None, cb, None, C.byref(dr))
    if calls is not None:
        calls.append(len(blocks))
    if rc < 0:
        assert not blocks and dr.block is None and dr.n_reads == 0
        return rc, None, None
    assert len(blocks) == 1 and dr.block == C.addressof(blocks[0])
    FX.expect_layout(dr)
    return rc, FX.tables(dr.block, dr, C.string_at), dr.used


def check(lib, ix, text):
    rc, got, used = parse(lib, ix, text)
    assert rc == 0, lib.mgb_last_error()
    assert got == FX.host_load(lib, text), text
    assert used == len(text)


def test_reader_cases(ctx):
    lib, ix = ctx
    for text in FX.TEXTS:
        check(lib, ix, text)


def test_random_texts(ctx):
    lib, ix = ctx
    texts = FX.random_texts(300, 11)
    assert sum(len(FX.host_load(lib, t)) for t in texts) > 600
    for text in texts:
        check(lib, ix, text)
    check(lib, ix, b"".join(texts + FX.TEXTS) * 3)  # one text of many chunks: lookups across chunk boundaries


def chunked(lib, ix, text, cut, max_bases=0):
    """the records of text parsed as two buffers cut at byte `cut`, the unparsed tail carried into the second (with max_bases,
    calls on each buffer until it emits nothing)"""
    out, carry = [], b""
    for piece, final in ((text[:cut], 0), (text[cut:], 1)):
        buf = carry + piece
        while True:
            rc, recs, used = parse(lib, ix, buf, max_bases, final)
            assert rc == 0, lib.mgb_last_error()
            assert 0 <= used <= len(buf)
            out += recs
            buf = buf[used:]
            if not recs:
                break
        carry = buf
    assert carry == b"" or not any(c in carry for c in b">@")
    return out


def test_chunked_at_every_byte(ctx):
    lib, ix = ctx
    texts = [t for t in FX.random_texts(200, 5) if len(t) > 60][:12]
    text = b"junk\n" + b"".join(texts) + FX.TEXTS[12] + FX.TEXTS[1]
    assert len(text) > 1500
    whole = FX.host_load(lib, text)
    for cut in range(len(text) + 1):
        assert chunked(lib, ix, text, cut) == whole, cut


def test_max_bases(ctx):
    lib, ix = ctx
    text = FX.TEXTS[0] + FX.TEXTS[12] + FX.TEXTS[1]
    whole = FX.host_load(lib, text)
    for mb in (1, 3, 4, 5, 9, 15, 16, 40, 10 ** 6):
        rc, recs, used = parse(lib, ix, text, mb)
        assert rc == 0
        assert recs == FX.host_load(lib, text, mb), mb
        assert recs == whole[:len(recs)]
        if len(recs) < len(whole):  # used is the next record's header
            assert text[used:used + 1] in (b">", b"@") and FX.host_load(lib, text[used:]) == whole[len(recs):], mb
        else:
            assert used == len(text)
        # calls of at most mb bases each, one after another, give every record
        assert chunked(lib, ix, text, len(text), mb) == whole
    for mb in (1, 3, 7):
        for t in FX.random_texts(60, 3):
            assert parse(lib, ix, t, mb)[1] == FX.host_load(lib, t, mb)


def test_streaming_rules(ctx):
    lib, ix = ctx
    # without final, the last record is held back: its quality (or its next line) may still come
    rc, recs, used = parse(lib, ix, b"junk\n@a\nAC\n+\n@@\n@b\nAC\n+\n@", final=0)
    assert rc == 0 and recs == [(b"a", b"AC")] and used == 16
    rc, recs, used = parse(lib, ix, b"junk>a\nAC\n", final=0)
    assert rc == 0 and recs == [] and used == 4
    rc, recs, used = parse(lib, ix, b"no header\n", final=0)
    assert rc == 0 and recs == [] and used == 10
    for final in (0, 1):
        rc, recs, used = parse(lib, ix, b"", final=final)
        assert rc == 0 and recs == [] and used == 0


def test_refusals(ctx):
    lib, ix = ctx
    calls = []
    dr = FX.DR()
    cb = FX.capi.mgb_dev_alloc_fn(lambda _, n: calls.append(n) or None)
    buf = C.create_string_buffer(b">a\nAC\n")
    for args, why in (((ix.gi, C.addressof(buf), -1, 0, 1, None, cb, None, C.byref(dr)), b"at least 0"),
                      ((ix.gi, None, 6, 0, 1, None, cb, None, C.byref(dr)), b"at least 0"),
                      ((None, C.addressof(buf), 6, 0, 1, None, cb, None, C.byref(dr)), b"an index"),
                      ((ix.gi, C.addressof(buf), 6, 0, 1, None, cb, None, None), b"an index")):
        assert lib.mgb_reads_parse_dev(*args) < 0 and why in lib.mgb_last_error()
    assert calls == []
    # an allocator that returns no block fails the call, after one call to it
    rc = lib.mgb_reads_parse_dev(ix.gi, C.addressof(buf), 6, 0, 1, None, cb, None, C.byref(dr))
    assert rc < 0 and b"no block" in lib.mgb_last_error() and calls == [256 * 4] and dr.block is None


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")
def test_well_formed_texts_match_bseq(ctx, tmp_path):
    from test_reads_loader import ref_load
    lib, ix = ctx
    for k, text in enumerate(FX.TEXTS[:4] + FX.TEXTS[9:13] + [open(os.path.join(T.FIX, "MT-chimp.fa"), "rb").read()]):
        fn = str(tmp_path / ("w%d.fx" % k))
        open(fn, "wb").write(text)
        assert parse(lib, ix, text)[1] == ref_load(fn), k
