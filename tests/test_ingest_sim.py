"""Reads in device memory, in both simulators of the device code: the ingest step (mgb_test_ingest, k_ingest's per-word code run by
its host loop) against a restatement of mg_toupper + pack_read_scalar, mgb_map_batch_dev_gaf() on the GAF test sets, lower case
included, against mgb_map_batch_gaf() on the upper-cased reads, mgb_map_batch_dev() against mg_map_batch_frag() field by field, and
both split over several devices (MGB_DEVICES) against one."""
import os
import random

import pytest

import devreads as DR
import gafcases as GC
import mgtest as T
import reccases as RC


@pytest.fixture(scope="module", params=["hostsim", "hostsim32"])
def lib(request):
    return T.load_hostsim() if request.param == "hostsim" else T.load_hostsim32()


def rand_acgt(rng, n):
    return bytes(rng.choice(b"ACGT") for _ in range(n))


def check_ingest(lib, reads):
    for segmented in (False, True):
        ups, words, raw = DR.ingest(lib, reads, segmented)
        for i, r in enumerate(reads):
            up = DR.toupper(r)
            want_words, want_raw = DR.pack_scalar(up)
            assert ups[i] == up, (segmented, i, len(r))
            assert raw[i] == int(want_raw), (segmented, i, r[:80])
            if not segmented:
                assert words[i] == want_words, (i, len(r))


def test_every_byte_value(lib):
    """each byte 0..255 once inside an A/C/G/T read, and all of them in one read"""
    ctx = b"ACGTTGCA" * 5
    reads = [ctx[:17] + bytes([b]) + ctx for b in range(256)] + [bytes(range(256)), bytes(range(255, -1, -1)) * 3]
    check_ingest(lib, reads)
    _, _, raw = DR.ingest(lib, reads, False)
    flagged = {b for b in range(256) if raw[b]}
    assert flagged == set(range(256)) - set(b"ACGTacgt")


def test_case_n_iupac_and_other_bytes(lib):
    rng = random.Random(5)
    base = rand_acgt(rng, 200)
    reads = [base.lower(), base[:100].lower() + base[100:], base[:50] + b"N" + base[51:], base.replace(b"A", b"n"),
             b"ACGTRYKMSWBDHVN" * 9, b"ACG-T*ACG.T1234\x00\xff\x80", b"z" + base, base + b"{", base + b"`", b"@" + base, b"[" + base]
    check_ingest(lib, reads)
    _, _, raw = DR.ingest(lib, reads, False)
    assert raw[:2] == [0, 0] and all(raw[2:])


def test_lengths_and_source_offsets(lib):
    """lengths around the 32-base words and the 16-byte loads, each read starting at every residue of its offset mod 16"""
    rng = random.Random(7)
    lengths = [0, 1, 31, 32, 33, 63, 64, 65, 1000, 100000]
    residues = set()
    for shift in range(16):
        reads = [rand_acgt(rng, shift)]  # puts the next read at offset shift
        for ln in lengths:
            s = bytearray(rand_acgt(rng, ln))
            if ln and rng.random() < 0.3:
                s[rng.randrange(ln)] = rng.choice(b"acgtnN")
            reads.append(bytes(s))
        at = 0
        for r in reads:
            residues.add(at % 16)
            at += len(r)
        check_ingest(lib, reads)
    assert residues == set(range(16))


def test_refusals(lib):
    import ctypes as C
    off = (C.c_int64 * 3)(0, 5, 3)
    buf = C.create_string_buffer(8)
    rc = lib.mgb_test_ingest(2, b"ACGTACGT", off, 0, buf, (C.c_uint64 * 4)(), (C.c_int32 * 2)())
    assert rc < 0 and b"bad length" in lib.mgb_last_error()


def dev_vs_host(lib, gfa, names, seqs, preset="lr", cigar=True, flag=0, n_seg=None, want=None):
    ix = GC.Index(lib, gfa, preset, cigar, flag)
    try:
        rc, host = GC.map_gaf(lib, ix, names, seqs, n_seg)
        assert rc == 0, lib.mgb_last_error()
        if want is not None:
            GC.check(host, want)
        for reads in (seqs, DR.mixed_case(seqs, 3)):
            rc, got = DR.host_dev_gaf(lib, ix, names, reads, n_seg)
            assert rc == 0, lib.mgb_last_error()
            GC.check(got, host)
    finally:
        ix.close()


def test_gaf_goldens(lib, workdir):
    for name, _, kind, preset in GC.EXISTING:
        if name[:2] in ("c1", "c2", "c4"):
            gfa, names, seqs = GC.inputs(kind, workdir)
            dev_vs_host(lib, gfa, names, seqs, preset, want=GC.golden(name))


def test_gaf_output_options(lib, workdir):
    for name, kind, cigar, flag in (GC.FLAGGED[0], GC.FLAGGED[3], GC.FLAGGED[4]):
        gfa, names, seqs = GC.inputs(kind, workdir)
        dev_vs_host(lib, gfa, names, seqs, "lr", cigar, flag, want=GC.golden(name))


def test_gaf_read_pairs(lib, workdir):
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    dev_vs_host(lib, gfa, names, flat, "sr", False, GC.SHOW_UNMAP, n_seg=n_seg, want=GC.golden(GC.PAIRS))


def test_gaf_refusals_leave_no_text(lib, workdir):
    import ctypes as C
    gfa, names, seqs = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        blob, off = DR.flat(seqs[:3])
        buf = C.create_string_buffer(blob, len(blob))
        for bad, why in (([0, 20, 10, len(blob)], b"decrease"), ([0, 10, 20, len(blob) + 1], b"outside")):
            coff = (C.c_int64 * 4)(*bad)
            out, ln = C.c_void_p(0), C.c_size_t(7)
            rc = lib.mgb_map_batch_dev_gaf(ix.gi, 3, None, 3, C.addressof(buf), len(blob), C.addressof(coff), None, C.byref(ix.mo), None,
                                           C.byref(out), C.byref(ln), None)
            assert rc < 0 and why in lib.mgb_last_error() and not out.value and ln.value == 0
        rc, text = DR.host_dev_gaf(lib, ix, None, [])
        assert rc == 0 and text == b""
        ix.mo.flag |= GC.CAL_COV
        rc, text = DR.host_dev_gaf(lib, ix, None, seqs[:2])
        assert rc < 0 and text is None and b"independent" in lib.mgb_last_error()
    finally:
        ix.close()


def dev_results_vs_host(lib, gfa, names, seqs, preset="lr", cigar=True, flag=0, n_seg=None):
    """mgb_map_batch_dev() on mixed-case reads against mg_map_batch_frag() on the upper-cased ones, field by field; the latter's results"""
    ix = GC.Index(lib, gfa, preset, cigar, flag)
    try:
        want = RC.host_results(lib, ix, names, seqs, n_seg)
        rc, got = DR.host_dev_results(lib, ix, names, DR.mixed_case(seqs, 7), n_seg)
        assert rc == 0, lib.mgb_last_error()
    finally:
        ix.close()
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(want, got)):
        d = T.diff_results(a, b)
        assert d is None, "sequence %d: %s" % (i, d)
    return want


def test_dev_results(lib, workdir):
    for kind, flag in (("c2", 0), ("sv_edge", GC.X)):
        gfa, names, seqs = GC.inputs(kind, workdir)
        want = dev_results_vs_host(lib, gfa, names, seqs, "lr", True, flag)
        assert sum(r is not None and r["n_gc"] > 0 for r in want) > len(seqs) // 2


def test_dev_results_read_pairs(lib, workdir):
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    want = dev_results_vs_host(lib, gfa, names, flat, "sr", False, GC.SHOW_UNMAP, n_seg)
    assert all(want[i] is None for i in range(1, len(flat), 2))
    assert sum(r is not None for r in want) == len(names)


def test_dev_results_empty_batch(lib, workdir):
    gfa, _, _ = GC.inputs("c2", workdir)
    assert dev_results_vs_host(lib, gfa, None, []) == []


def test_dev_several_devices(lib, workdir):
    """MGB_DEVICES: the batch cut into one part per device, each part's span of the reads copied to its device; the results and the
    text of the parts, joined in input order, equal those of one device"""
    gfa, names, seqs = GC.inputs("sv_edge", workdir)
    seqs = DR.mixed_case(seqs, 2)
    out = []
    for devices in (None, "0,0,0"):
        if devices:
            os.environ["MGB_DEVICES"] = devices
        try:
            ix = GC.Index(lib, gfa, "lr", True, GC.X)
        finally:
            os.environ.pop("MGB_DEVICES", None)
        try:
            rc, res = DR.host_dev_results(lib, ix, names, seqs)
            assert rc == 0, lib.mgb_last_error()
            rc, text = DR.host_dev_gaf(lib, ix, names, seqs)
            assert rc == 0, lib.mgb_last_error()
            out.append((res, text))
        finally:
            ix.close()
    (one, one_text), (many, many_text) = out
    assert len(many) == len(one) >= 6
    for i, (a, b) in enumerate(zip(one, many)):
        d = T.diff_results(a, b)
        assert d is None, "sequence %d: %s" % (i, d)
    GC.check(many_text, one_text)
