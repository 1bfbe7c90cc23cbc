"""The ds tables of mgb_map_batch_dev_rec_ds, in both simulators of the device code, where "device memory" is host memory: every
record's ds string and offsets equal the mg_ds_t that mgb_map_batch_dev() gives on the same reads, the eight other tables are byte
for byte those of mgb_map_batch_dev_rec, and the ds:Z field of the GAF text is the one the tables spell.  Covered: the GAF test sets,
secondary chains, read pairs, lower case and N, empty, over-long and unmapped reads, a batch without MG_M_CIGAR, the empty batch,
several devices, every byte alignment of a string in the DS table, and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import devreads as DR
import gafcases as GC
import mgtest as T
import recdscases as RD
import reccases as RC
from minigraph_b200 import capi


@pytest.fixture(scope="module", params=["hostsim", "hostsim32"])
def lib(request):
    return T.load_hostsim() if request.param == "hostsim" else T.load_hostsim32()


def parity(lib, ix, names, seqs, n_seg=None):
    """(the mgb_map_batch_dev results, the eight tables, the ds tables) of the same reads, checked against each other"""
    rc, want = DR.host_dev_results(lib, ix, names, seqs, n_seg)
    assert rc == 0, lib.mgb_last_error()
    rc, plain, _ = RC.host_dev_rec(lib, ix, names, seqs, n_seg)
    assert rc == 0, lib.mgb_last_error()
    rc, tabs, ds, alloc, rec, rec_ds = RD.host_dev_rec_ds(lib, ix, names, seqs, n_seg)
    assert rc == 0, lib.mgb_last_error()
    assert len(alloc.calls) == 1
    RD.check_same_records(tabs, plain)
    RC.check(want, RC.records_to_py(tabs))
    n_ds = RD.check_ds(want, tabs, ds)
    # nothing written past the end of DS (the block was filled with 0xA5 first)
    block = alloc.blocks[-1].raw
    end_ds = rec_ds.off[1] + rec_ds.n_ds
    assert set(block[end_ds:rec_ds.off[2]]) <= {0xA5}
    return want, tabs, ds, n_ds


def mapped(lib, gfa, names, seqs, preset="lr", cigar=True, flag=0, n_seg=None):
    ix = GC.Index(lib, gfa, preset, cigar, flag)
    try:
        return parity(lib, ix, names, seqs, n_seg)
    finally:
        ix.close()


@pytest.mark.parametrize("k", range(len(RC.SETS)))
def test_sets(lib, workdir, k):
    kind, preset, cigar, flag = RC.SETS[k]
    gfa, names, seqs = GC.inputs(kind, workdir)
    want, tabs, ds, n_ds = mapped(lib, gfa, names, seqs, preset, cigar, flag)
    if cigar:
        assert n_ds > len(seqs) // 2 and len(ds["ds_off"]) > 0
    else:  # without MG_M_CIGAR: no ds at all
        assert n_ds == 0 and (ds["ds_csr"] == 0).all() and len(ds["ds"]) == 0 and len(ds["ds_off"]) == 0


def test_secondary_chains(lib, workdir):
    """the tables hold every record whatever the writer's flags: secondary chains with a CIGAR carry their ds"""
    gfa, names, seqs = GC.inputs("stable", workdir)
    want, tabs, ds, _ = mapped(lib, gfa, names, seqs)
    cols = capi.GC_COLUMNS
    gc, csr = tabs["gc"], ds["ds_csr"]
    sec = [k for k in range(len(gc)) if gc[k, cols.index("id")] != gc[k, cols.index("parent")] and gc[k, RD.HAS_CIGAR]]
    assert sec and any(csr[k + 1, 0] > csr[k, 0] for k in sec)


def test_read_pairs(lib, workdir):
    """fragments with segments are not aligned base by base: every ds is empty"""
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    want, tabs, ds, n_ds = mapped(lib, gfa, names, flat, "sr", True, GC.SHOW_UNMAP, n_seg)
    assert len(tabs["gc"]) > 0 and n_ds == 0 and (ds["ds_csr"] == 0).all() and len(ds["ds"]) == 0


def test_mixed_case_and_n(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    _, _, _, n_ds = mapped(lib, gfa, names, DR.mixed_case(RC.with_n(seqs, 3), 5))
    assert n_ds > 0


def test_empty_over_long_and_unmapped_reads(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    reads = [b"", seqs[0][:4000], seqs[1], b"", seqs[2][:3000].lower(), RC.unmapped_read()]
    ix = GC.Index(lib, gfa, "lr")
    ix.mo.max_qlen = 5000
    try:
        want, tabs, ds, n_ds = parity(lib, ix, names[:6], reads)
    finally:
        ix.close()
    assert tabs["seq_info"][:, 0].tolist() == [0, 1, 0, 0, 1, 1] and want[5]["n_gc"] == 0 and n_ds >= 2


def test_every_destination_alignment(lib, workdir):
    """records' strings of lengths that are not multiples of 16 one after another: each of the 16 byte alignments of a string's
    start in DS occurs, with short and long strings"""
    gfa, names, seqs = GC.inputs("c2", workdir)
    gfa3, names3, seqs3 = GC.inputs("c3", workdir)
    _, _, ds, _ = mapped(lib, gfa, names, seqs)
    _, _, ds3, _ = mapped(lib, gfa3, names3, seqs3)
    starts = set()
    for d in (ds, ds3):
        csr = d["ds_csr"]
        lens = np.diff(csr[:, 0])
        starts |= {int(csr[k, 0]) % 16 for k in range(len(lens)) if lens[k] > 0}
        assert any(0 < x % 16 for x in lens) and any(x > 16 * 32 for x in lens)
    assert starts == set(range(16)), sorted(starts)


def test_ds_against_gaf_text(lib, workdir):
    """the ds:Z field that mgb_map_batch_gaf prints for every record is the one the tables spell (reversed after a reverse path)"""
    n_rev = 0
    for kind, flag in (("c3", 0), ("stable", GC.PRINT_2ND)):
        gfa, names, seqs = GC.inputs(kind, workdir)
        ix = GC.Index(lib, gfa, "lr", True, flag)
        try:
            rc, text = GC.map_gaf(lib, ix, names, seqs)
            assert rc == 0, lib.mgb_last_error()
            rc, tabs, ds, _, _, _ = RD.host_dev_rec_ds(lib, ix, names, seqs)
            assert rc == 0, lib.mgb_last_error()
        finally:
            ix.close()
        n, r = RD.check_against_gaf(text, names, tabs, ds, print_2nd=bool(flag))
        assert n > len(seqs) // 2
        n_rev += r
    assert n_rev > 0


def test_several_devices(lib, workdir):
    """MGB_DEVICES: each part tabled on its own, DS and DS_OFF joined behind the parts before and DS_CSR rebased"""
    gfa, names, seqs = GC.inputs("sv_edge", workdir)
    seqs = DR.mixed_case(seqs, 2)
    ix = GC.Index(lib, gfa, "lr", True, GC.X)
    try:
        rc, one, one_ds, _, _, _ = RD.host_dev_rec_ds(lib, ix, names, seqs)
        assert rc == 0, lib.mgb_last_error()
    finally:
        ix.close()
    os.environ["MGB_DEVICES"] = "0,0,0"
    try:
        ix = GC.Index(lib, gfa, "lr", True, GC.X)
    finally:
        del os.environ["MGB_DEVICES"]
    try:
        rc, many, many_ds, alloc, _, _ = RD.host_dev_rec_ds(lib, ix, names, seqs)
        assert rc == 0, lib.mgb_last_error()
        assert len(alloc.calls) == 1
    finally:
        ix.close()
    RD.check_same_records(many, one)
    for k in capi.REC_DS_TABLES:
        assert many_ds[k].tobytes() == one_ds[k].tobytes(), k
    assert len(one_ds["ds"]) > 0


def test_empty_batch(lib, workdir):
    gfa, _, _ = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        rc, tabs, ds, alloc, _, rec_ds = RD.host_dev_rec_ds(lib, ix, None, [])
    finally:
        ix.close()
    assert rc == 0 and len(alloc.calls) == 1
    assert tabs["seq_csr"].tolist() == [[0, 0, 0]] and tabs["cigar_csr"].tolist() == [0]
    assert ds["ds_csr"].tolist() == [[0, 0]] and len(ds["ds"]) == 0 and len(ds["ds_off"]) == 0
    assert rec_ds.n_ds == 0 and rec_ds.n_ds_off == 0


def test_refusals_call_no_allocator(lib, workdir):
    """no mgb_records_ds_t, or a bad batch: refused before any allocation; a NULL block fails the call"""
    gfa, names, seqs = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        alloc = RC.HostAlloc()
        rc, tabs, _, _, _, _ = RD.host_dev_rec_ds(lib, ix, names[:3], seqs[:3], alloc=alloc, ds_out=False)
        assert rc < 0 and tabs is None and b"mgb_records_ds_t" in lib.mgb_last_error() and alloc.calls == []
        alloc = RC.HostAlloc()
        rc, tabs, _, _, _, _ = RD.host_dev_rec_ds(lib, ix, None, seqs[:3], [2, 2], alloc=alloc)
        assert rc < 0 and b"add up" in lib.mgb_last_error() and alloc.calls == []
        alloc = RC.HostAlloc(fail=True)
        rc, tabs, _, _, _, _ = RD.host_dev_rec_ds(lib, ix, names[:3], seqs[:3], alloc=alloc)
        assert rc < 0 and b"allocator" in lib.mgb_last_error() and len(alloc.calls) == 1
    finally:
        ix.close()


def test_records_fields_match_the_plain_call(lib, workdir):
    """mgb_records_t: the same rows and offsets as mgb_map_batch_dev_rec gives; bytes also counts the ds tables"""
    gfa, names, seqs = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        alloc = RC.HostAlloc()
        blob, off = DR.flat(seqs)
        buf = C.create_string_buffer(blob, len(blob))
        coff = (C.c_int64 * len(off))(*[int(x) for x in off])
        plain = capi.mgb_records_t()
        rc = lib.mgb_map_batch_dev_rec(ix.gi, len(seqs), None, len(seqs), C.addressof(buf), len(blob), C.addressof(coff), None,
                                       C.byref(ix.mo), None, alloc.fn, None, C.byref(plain))
        assert rc == 0, lib.mgb_last_error()
        rc, _, _, _, rec, rec_ds = RD.host_dev_rec_ds(lib, ix, None, seqs)
        assert rc == 0, lib.mgb_last_error()
    finally:
        ix.close()
    for f in ("n_seq", "n_rec", "n_lc", "n_a", "n_cigar"):
        assert getattr(rec, f) == getattr(plain, f), f
    assert list(rec.off) == list(plain.off) and rec.bytes == rec_ds.off[2] + ((4 * rec_ds.n_ds_off + 255) & ~255)
    assert rec_ds.off[0] == plain.bytes


def test_header_ds_tables():
    assert capi.REC_DS_TABLES == ("ds_csr", "ds", "ds_off")
    assert C.sizeof(capi.mgb_records_ds_t) == 8 * (2 + 3)
