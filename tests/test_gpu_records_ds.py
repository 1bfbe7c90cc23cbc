"""The ds tables in GPU memory (mgb_map_batch_dev_rec_ds through minigraph_b200.tensors.map_cuda_reads_to_tensors(ds=True)): every
record's ds string and offsets are those of map_cuda_reads(gaf=False) on the same tensors, the eight other tables are byte for byte
those of the ds=False call, and the ds:Z field of map_cuda_reads(gaf=True) is the one the tables spell.  Covered: the GAF test sets,
L3, read pairs, lower case and N, empty, over-long and unmapped reads, a batch of 6 000 reads, the empty batch and several devices;
ds=False returns what it returned before; only the two totals of the ds tables come back to the host."""
import os

import pytest

import devreads as DR
import gafcases as GC
import mgtest as T
import recdscases as RD
import reccases as RC
from minigraph_b200 import capi
from minigraph_b200.tensors import map_cuda_reads, map_cuda_reads_to_tensors, pack_reads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return capi.load_product()


def as_numpy(t, names):
    return {k: getattr(t, k).cpu().numpy() for k in names}


def stats(lib, ix):
    import ctypes as C
    st = capi.mgb_stats_t()
    lib.mgb_get_stats(ix.gi, C.byref(st))
    return st


def dirty(fn, *args, **kw):
    """fn(*args, **kw) with every block of torch.empty filled with 0xA5 first: a byte the library leaves unwritten cannot pass for
    what it should hold"""
    import torch
    empty = torch.empty
    torch.empty = lambda *a, **k: empty(*a, **k).fill_(0xA5)
    try:
        return fn(*args, **kw)
    finally:
        torch.empty = empty


def gcs_results(lib, seq, off, ix, names, n_seg=None):
    n = off.numel() - 1
    gcs = map_cuda_reads(lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg, gaf=False)
    out = [T.gchains_to_py(gcs[i]) for i in range(n)]
    lib.mgb_free_batch(n, gcs)
    return out


def parity(lib, ix, names, seqs, n_seg=None):
    """the ds=True tables against the ds=False tables and the mg_gchains_t results of the same tensors: (results, tables, ds tables,
    records with a ds)"""
    seq, off = pack_reads(seqs, "cuda:0")
    plain = as_numpy(map_cuda_reads_to_tensors(lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg), capi.REC_TABLES)
    st_plain = stats(lib, ix)
    t = dirty(map_cuda_reads_to_tensors, lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg, ds=True)
    st = stats(lib, ix)
    assert st.out_bytes == st_plain.out_bytes + 16, (st.out_bytes, st_plain.out_bytes)  # the two totals, no ds byte
    tabs, ds = as_numpy(t, capi.REC_TABLES), as_numpy(t, capi.REC_DS_TABLES)
    RD.check_same_records(tabs, plain)
    # nothing written between the end of DS and DS_OFF
    end = t.ds.data_ptr() - t.block.data_ptr() + t.ds.numel()
    o_ds_off = t.ds_off.data_ptr() - t.block.data_ptr()
    assert (t.block[end:o_ds_off] == 0xA5).all()
    want = gcs_results(lib, seq, off, ix, names, n_seg)
    RC.check(want, RC.records_to_py(tabs))
    n_ds = RD.check_ds(want, tabs, ds)
    return want, tabs, ds, n_ds


def mapped(lib, gfa, names, seqs, preset="lr", cigar=True, flag=0, n_seg=None, max_qlen=None):
    ix = GC.Index(lib, gfa, preset, cigar, flag)
    if max_qlen:
        ix.mo.max_qlen = max_qlen
    try:
        return parity(lib, ix, names, seqs, n_seg)
    finally:
        ix.close()


@pytest.mark.parametrize("k", range(len(RC.SETS) + 1))
def test_sets(lib, workdir, k):
    kind, preset, cigar, flag = RC.SETS[k] if k < len(RC.SETS) else ("L3", "lr", True, 0)
    gfa, names, seqs = GC.inputs(kind, workdir)
    _, _, ds, n_ds = mapped(lib, gfa, names, seqs, preset, cigar, flag)
    if cigar:
        assert n_ds > len(seqs) // 2 and len(ds["ds_off"]) > 0
    else:
        assert n_ds == 0 and (ds["ds_csr"] == 0).all() and len(ds["ds"]) == 0 and len(ds["ds_off"]) == 0


def test_secondary_chains_and_gaf_text(lib, workdir):
    """secondary records carry their ds; the ds:Z field of the device's GAF text is the one the tables spell"""
    gfa, names, seqs = GC.inputs("stable", workdir)
    ix = GC.Index(lib, gfa, "lr", True, GC.PRINT_2ND)
    try:
        _, tabs, ds, _ = parity(lib, ix, names, seqs)
        seq, off = pack_reads(seqs, "cuda:0")
        text = map_cuda_reads(lib, ix.gi, seq, off, names, opt=ix.mo)
    finally:
        ix.close()
    cols = capi.GC_COLUMNS
    gc, csr = tabs["gc"], ds["ds_csr"]
    assert any(gc[k, cols.index("id")] != gc[k, cols.index("parent")] and csr[k + 1, 0] > csr[k, 0] for k in range(len(gc)))
    n, n_rev = RD.check_against_gaf(text, names, tabs, ds, print_2nd=True)
    assert n > len(seqs) // 2 and n_rev > 0


def test_read_pairs(lib, workdir):
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    _, tabs, ds, n_ds = mapped(lib, gfa, names, flat, "sr", True, GC.SHOW_UNMAP, n_seg)
    assert len(tabs["gc"]) > 0 and n_ds == 0 and (ds["ds_csr"] == 0).all() and len(ds["ds"]) == 0


def test_mixed_case_n_empty_over_long_and_unmapped(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    reads = DR.mixed_case(RC.with_n(seqs, 3), 5) + [b"", seqs[0] + seqs[1], RC.unmapped_read()]
    want, tabs, _, n_ds = mapped(lib, gfa, None, reads, max_qlen=15000)
    n = len(seqs)
    assert tabs["seq_info"][n:, 0].tolist() == [0, 0, 1] and want[n + 2]["n_gc"] == 0 and n_ds >= n // 2


def test_large_batch(lib, workdir):
    """6 000 reads: the scans run several items per thread"""
    hap, reads = os.path.join(workdir, "gmt.hap.fa"), os.path.join(workdir, "grec6k.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, 6000, 10000, "ont", 11)
    names, seqs = T.read_fasta(reads)
    _, tabs, _, n_ds = mapped(lib, os.path.join(T.FIX, "MT.gfa"), names, seqs)
    assert len(tabs["gc"]) > 5000 and n_ds > 5000


def test_empty_batch(lib, workdir):
    import torch
    gfa, _, _ = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        seq, off = torch.zeros(0, dtype=torch.uint8, device="cuda:0"), torch.zeros(1, dtype=torch.int64, device="cuda:0")
        t = dirty(map_cuda_reads_to_tensors, lib, ix.gi, seq, off, opt=ix.mo, ds=True)
    finally:
        ix.close()
    assert t.seq_csr.tolist() == [[0, 0, 0]] and t.cigar_csr.tolist() == [0] and t.ds_csr.tolist() == [[0, 0]]
    assert t.ds.numel() == 0 and t.ds_off.numel() == 0


def test_ds_false_is_unchanged(lib, workdir):
    """without ds: the tables and nothing else, as before"""
    gfa, names, seqs = GC.inputs("c2", workdir)
    seq, off = pack_reads(seqs, "cuda:0")
    ix = GC.Index(lib, gfa, "lr")
    try:
        t = map_cuda_reads_to_tensors(lib, ix.gi, seq, off, names, opt=ix.mo)
        t2 = map_cuda_reads_to_tensors(lib, ix.gi, seq, off, names, opt=ix.mo, ds=False)
    finally:
        ix.close()
    assert set(vars(t)) == set(vars(t2)) == {"block"} | set(capi.REC_TABLES)
    for k in capi.REC_TABLES:
        assert getattr(t, k).cpu().numpy().tobytes() == getattr(t2, k).cpu().numpy().tobytes(), k


def test_several_devices(lib, workdir):
    import torch
    gfa, names, seqs = GC.inputs("L2", workdir)
    seqs = DR.mixed_case(seqs, 6)
    seq, off = pack_reads(seqs, "cuda:0")
    ix = GC.Index(lib, gfa, "lr")
    try:
        t = map_cuda_reads_to_tensors(lib, ix.gi, seq, off, names, opt=ix.mo, ds=True)
        one, one_ds = as_numpy(t, capi.REC_TABLES), as_numpy(t, capi.REC_DS_TABLES)
    finally:
        ix.close()
    os.environ["MGB_DEVICES"] = "0,1" if torch.cuda.device_count() > 1 else "0,0"
    try:
        ix = GC.Index(lib, gfa, "lr")
    finally:
        del os.environ["MGB_DEVICES"]
    try:
        t = dirty(map_cuda_reads_to_tensors, lib, ix.gi, seq, off, names, opt=ix.mo, ds=True)
        many, many_ds = as_numpy(t, capi.REC_TABLES), as_numpy(t, capi.REC_DS_TABLES)
        RD.check_ds(gcs_results(lib, seq, off, ix, names), many, many_ds)
    finally:
        ix.close()
    RD.check_same_records(many, one)
    for k in capi.REC_DS_TABLES:
        assert many_ds[k].tobytes() == one_ds[k].tobytes(), k
    assert len(one_ds["ds"]) > 0
