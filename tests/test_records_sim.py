"""Result tables in device memory (mgb_map_batch_dev_rec), in both simulators of the device code, where "device memory" is host
memory: the tables equal the mg_map_batch_frag() results field by field (div bit for bit) on the GAF test sets, read pairs, lower
case and N; empty, over-long and unmapped reads; the empty batch; the allocator's contract; the refusals of mgb_map_batch_dev."""
import ctypes as C
import os

import pytest

import devreads as DR
import gafcases as GC
import mgtest as T
import reccases as RC
from minigraph_b200 import capi
from minigraph_b200 import tensors


@pytest.fixture(scope="module", params=["hostsim", "hostsim32"])
def lib(request):
    return T.load_hostsim() if request.param == "hostsim" else T.load_hostsim32()


def parity(lib, gfa, names, seqs, preset="lr", cigar=True, flag=0, n_seg=None):
    ix = GC.Index(lib, gfa, preset, cigar, flag)
    try:
        want = RC.host_results(lib, ix, names, seqs, n_seg)
        rc, tabs, alloc = RC.host_dev_rec(lib, ix, names, seqs, n_seg)
        assert rc == 0, lib.mgb_last_error()
        assert len(alloc.calls) == 1
        got = RC.records_to_py(tabs)
        RC.check(want, got)
        return want, tabs
    finally:
        ix.close()


@pytest.mark.parametrize("k", range(len(RC.SETS)))
def test_sets(lib, workdir, k):
    kind, preset, cigar, flag = RC.SETS[k]
    gfa, names, seqs = GC.inputs(kind, workdir)
    want, tabs = parity(lib, gfa, names, seqs, preset, cigar, flag)
    assert sum(r is not None and r["n_gc"] > 0 for r in want) > len(seqs) // 2
    has_cigar = tabs["gc"][:, capi.GC_COLUMNS.index("has_cigar")]
    if cigar:
        assert has_cigar.any() and tabs["cigar_csr"][-1] > 0
    else:
        assert not has_cigar.any() and (tabs["cigar_csr"] == 0).all() and len(tabs["cigar"]) == 0


def test_read_pairs(lib, workdir):
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    want, tabs = parity(lib, gfa, names, flat, "sr", False, GC.SHOW_UNMAP, n_seg)
    csr = tabs["seq_csr"]
    for i in range(1, len(flat), 2):
        assert want[i] is None and tabs["seq_info"][i].tolist() == [0, 0] and (csr[i] == csr[i + 1]).all()
    assert sum(r is not None for r in want) == len(names)


def test_mixed_case_and_n(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    parity(lib, gfa, names, DR.mixed_case(RC.with_n(seqs, 3), 5))


def test_empty_over_long_and_unmapped_reads(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    reads = [b"", seqs[0][:4000], seqs[1], b"", seqs[2][:3000].lower(), RC.unmapped_read()]
    ix = GC.Index(lib, gfa, "lr")
    ix.mo.max_qlen = 5000
    try:
        want = RC.host_results(lib, ix, names[:6], reads)
        rc, tabs, _ = RC.host_dev_rec(lib, ix, names[:6], reads)
        assert rc == 0, lib.mgb_last_error()
    finally:
        ix.close()
    RC.check(want, RC.records_to_py(tabs))
    assert tabs["seq_info"][:, 0].tolist() == [0, 1, 0, 0, 1, 1]
    assert want[5] is not None and want[5]["n_gc"] == 0
    csr = tabs["seq_csr"]
    assert (csr[5] == csr[6]).all() and tabs["seq_info"][5, 1] == want[5]["rep_len"]


def test_several_devices(lib, workdir):
    """MGB_DEVICES: each part tabled on its own, the tables joined in input order with the CSR rows rebased"""
    gfa, names, seqs = GC.inputs("sv_edge", workdir)
    seqs = DR.mixed_case(seqs, 2)
    ix = GC.Index(lib, gfa, "lr", True, GC.X)
    try:
        rc, one, _ = RC.host_dev_rec(lib, ix, names, seqs)
        assert rc == 0, lib.mgb_last_error()
    finally:
        ix.close()
    os.environ["MGB_DEVICES"] = "0,0,0"
    try:
        ix = GC.Index(lib, gfa, "lr", True, GC.X)
    finally:
        del os.environ["MGB_DEVICES"]
    try:
        rc, many, alloc = RC.host_dev_rec(lib, ix, names, seqs)
        assert rc == 0, lib.mgb_last_error()
        assert len(alloc.calls) == 1
    finally:
        ix.close()
    for k in capi.REC_TABLES:
        assert many[k].tobytes() == one[k].tobytes(), k


def test_empty_batch(lib, workdir):
    gfa, _, _ = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        rc, tabs, alloc = RC.host_dev_rec(lib, ix, None, [])
    finally:
        ix.close()
    assert rc == 0 and len(alloc.calls) == 1
    assert tabs["seq_csr"].tolist() == [[0, 0, 0]] and all(len(tabs[k]) == 0 for k in capi.REC_TABLES if k not in ("seq_csr", "cigar_csr"))
    assert tabs["cigar_csr"].tolist() == [0]


def test_allocator_returns_null(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        alloc = RC.HostAlloc(fail=True)
        rc, tabs, _ = RC.host_dev_rec(lib, ix, names[:3], seqs[:3], alloc=alloc)
        assert rc < 0 and tabs is None and b"allocator" in lib.mgb_last_error()
        assert len(alloc.calls) == 1
        rc, tabs, _ = RC.host_dev_rec(lib, ix, names[:3], seqs[:3])  # the index is still usable
        assert rc == 0
    finally:
        ix.close()


def test_refusals_call_no_allocator(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    seqs = seqs[:3]
    tot = sum(len(s) for s in seqs)
    ix = GC.Index(lib, gfa, "lr")
    try:
        cases = [(dict(off=[0, 20, 10, tot]), b"decrease"), (dict(off=[0, 10, 20, tot + 1]), b"outside"),
                 (dict(off=[0, 10, 20, (1 << 31) + 40], seq_bytes=(1 << 31) + 40), b"INT32_MAX"),
                 (dict(n_seg=[2, 2]), b"add up"), (dict(n_seq=2), b"n_seq must be n_frag")]
        for kw, why in cases:
            alloc = RC.HostAlloc()
            rc, tabs, _ = RC.host_dev_rec(lib, ix, None, seqs, alloc=alloc, **kw)
            assert rc < 0 and why in lib.mgb_last_error(), (kw, rc, lib.mgb_last_error())
            assert tabs is None and alloc.calls == []
    finally:
        ix.close()


def test_gc_columns_follow_the_header():
    assert RC.header_gc_columns() == capi.GC_COLUMNS == tensors.GC_COLUMNS
    assert capi.REC_TABLES == ("seq_csr", "seq_info", "gc", "gc_div", "cigar_csr", "lc", "a", "cigar")
    assert C.sizeof(capi.mgb_records_t) == 8 * (5 + 2 + 8)
