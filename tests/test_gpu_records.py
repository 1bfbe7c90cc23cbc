"""Result tables in GPU memory (mgb_map_batch_dev_rec through minigraph_b200.tensors.map_cuda_reads_to_tensors): field by field what
map_cuda_reads(gaf=False) gives on the same tensors, on the GAF test sets, L3, read pairs, lower case and N and a batch of 6 000
reads; stream ordering; tables used by torch right away; several devices; refusals; nothing but the div requests comes back."""
import os

import pytest

import devreads as DR
import gafcases as GC
import mgtest as T
import reccases as RC
from minigraph_b200 import capi
from minigraph_b200.tensors import GC_COLUMNS, map_cuda_reads, map_cuda_reads_to_tensors, pack_reads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return capi.load_product()


def as_numpy(t):
    return {k: getattr(t, k).cpu().numpy() for k in capi.REC_TABLES}


def gcs_results(lib, seq, off, ix, names, n_seg=None):
    n = off.numel() - 1
    gcs = map_cuda_reads(lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg, gaf=False)
    out = [T.gchains_to_py(gcs[i]) for i in range(n)]
    lib.mgb_free_batch(n, gcs)
    return out


def stats(lib, ix):
    import ctypes as C
    st = capi.mgb_stats_t()
    lib.mgb_get_stats(ix.gi, C.byref(st))
    return st


def dirty(fn, *args, **kw):
    """fn(*args, **kw) with every block of torch.empty filled with 0xA5 first (on the current stream): a cell the library leaves
    unwritten cannot pass for a 0"""
    import torch
    empty = torch.empty
    torch.empty = lambda *a, **k: empty(*a, **k).fill_(0xA5)
    try:
        return fn(*args, **kw)
    finally:
        torch.empty = empty


def parity(lib, ix, names, seqs, n_seg=None):
    """the tables and the mg_gchains_t results of the same tensors agree; the tables (numpy) and the results"""
    seq, off = pack_reads(seqs, "cuda:0")
    t = dirty(map_cuda_reads_to_tensors, lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg)
    st = stats(lib, ix)
    tabs = as_numpy(t)
    assert st.out_bytes < 32 * len(tabs["gc"]) + 1024, (st.out_bytes, len(tabs["gc"]))  # no blob came back
    want = gcs_results(lib, seq, off, ix, names, n_seg)
    RC.check(want, RC.records_to_py(tabs))
    return want, tabs


@pytest.mark.parametrize("k", range(len(RC.SETS) + 1))
def test_sets(lib, workdir, k):
    kind, preset, cigar, flag = RC.SETS[k] if k < len(RC.SETS) else ("L3", "lr", True, 0)
    gfa, names, seqs = GC.inputs(kind, workdir)
    ix = GC.Index(lib, gfa, preset, cigar, flag)
    try:
        want, tabs = parity(lib, ix, names, seqs)
    finally:
        ix.close()
    assert sum(r is not None and r["n_gc"] > 0 for r in want) > len(seqs) // 2
    has_cigar = tabs["gc"][:, GC_COLUMNS.index("has_cigar")]
    assert has_cigar.any() == cigar and (tabs["cigar_csr"][-1] > 0) == cigar


def test_read_pairs(lib, workdir):
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    ix = GC.Index(lib, gfa, "sr", False, GC.SHOW_UNMAP)
    try:
        want, tabs = parity(lib, ix, names, flat, n_seg)
    finally:
        ix.close()
    for i in range(1, len(flat), 2):
        assert want[i] is None and tabs["seq_info"][i].tolist() == [0, 0]


def test_mixed_case_n_empty_over_long_and_unmapped(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    reads = DR.mixed_case(RC.with_n(seqs, 3), 5) + [b"", seqs[0] + seqs[1], RC.unmapped_read()]
    ix = GC.Index(lib, gfa, "lr")
    ix.mo.max_qlen = 15000
    try:
        want, tabs = parity(lib, ix, None, reads)
    finally:
        ix.close()
    n = len(seqs)
    assert tabs["seq_info"][n:, 0].tolist() == [0, 0, 1] and want[n + 2]["n_gc"] == 0


def test_empty_batch(lib, workdir):
    """no sequence: both rows of totals are written, all 0"""
    import torch
    gfa, _, _ = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        seq, off = torch.zeros(0, dtype=torch.uint8, device="cuda:0"), torch.zeros(1, dtype=torch.int64, device="cuda:0")
        t = dirty(map_cuda_reads_to_tensors, lib, ix.gi, seq, off, opt=ix.mo)
    finally:
        ix.close()
    assert t.seq_csr.tolist() == [[0, 0, 0]] and t.cigar_csr.tolist() == [0]
    assert all(getattr(t, k).numel() == 0 for k in capi.REC_TABLES if k not in ("seq_csr", "cigar_csr"))


def test_large_batch(lib, workdir):
    """6 000 reads: the scans run several items per thread"""
    hap, reads = os.path.join(workdir, "gmt.hap.fa"), os.path.join(workdir, "grec6k.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, 6000, 10000, "ont", 11)
    names, seqs = T.read_fasta(reads)
    ix = GC.Index(lib, os.path.join(T.FIX, "MT.gfa"), "lr")
    try:
        _, tabs = parity(lib, ix, names, seqs)
    finally:
        ix.close()
    assert len(tabs["gc"]) > 5000


def test_side_stream_and_overwrite(lib, workdir):
    """the reads written by a torch kernel on a side stream that is still busy: the call orders its reads after it; the buffer is
    overwritten right after the call returns, and the tables are used by torch at once"""
    import torch
    gfa, names, seqs = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        src, off = pack_reads(seqs, "cuda:0")
        want = gcs_results(lib, src, off, ix, names)
        dst = torch.zeros_like(src)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            torch.cuda._sleep(200_000_000)  # the side stream is busy for a while before it writes the reads
            torch.bitwise_or(src, 0x20, out=dst)  # lower case
            t = map_cuda_reads_to_tensors(lib, ix.gi, dst, off, names, opt=ix.mo)
            dst.fill_(ord("N"))
            # right after the call, on another stream than the one the block was allocated on
            counts = torch.bincount(t.gc[:, GC_COLUMNS.index("mapq")].long(), minlength=256).cpu().tolist()
        torch.cuda.synchronize()
        RC.check(want, RC.records_to_py(as_numpy(t)))
        mapq = [0] * 256
        for r in want:
            for g in (r or {"gc": []})["gc"]:
                mapq[g["mapq"]] += 1
        assert counts == mapq and sum(mapq) > 0
    finally:
        ix.close()


def test_several_devices(lib, workdir):
    import torch
    gfa, names, seqs = GC.inputs("L2", workdir)
    seqs = DR.mixed_case(seqs, 6)
    ix = GC.Index(lib, gfa, "lr")
    try:
        seq, off = pack_reads(seqs, "cuda:0")
        one = as_numpy(map_cuda_reads_to_tensors(lib, ix.gi, seq, off, names, opt=ix.mo))
    finally:
        ix.close()
    os.environ["MGB_DEVICES"] = "0,1" if torch.cuda.device_count() > 1 else "0,0"
    try:
        ix = GC.Index(lib, gfa, "lr")
    finally:
        del os.environ["MGB_DEVICES"]
    try:
        many = as_numpy(dirty(map_cuda_reads_to_tensors, lib, ix.gi, seq, off, names, opt=ix.mo))
        RC.check(gcs_results(lib, seq, off, ix, names), RC.records_to_py(many))
    finally:
        ix.close()
    for k in capi.REC_TABLES:
        assert many[k].tobytes() == one[k].tobytes(), k


def test_refusals(lib, workdir, monkeypatch):
    import torch
    gfa, names, seqs = GC.inputs("c2", workdir)
    seq, off = pack_reads(seqs[:4], "cuda:0")
    ix = GC.Index(lib, gfa, "lr")
    try:
        with pytest.raises(TypeError):
            map_cuda_reads_to_tensors(lib, ix.gi, seq.to(torch.int32), off, opt=ix.mo)
        with pytest.raises(TypeError):
            map_cuda_reads_to_tensors(lib, ix.gi, seq, off.to(torch.int32), opt=ix.mo)
        with pytest.raises(ValueError):
            map_cuda_reads_to_tensors(lib, ix.gi, seq.cpu(), off, opt=ix.mo)
        with pytest.raises(ValueError):
            map_cuda_reads_to_tensors(lib, ix.gi, seq, off.cpu(), opt=ix.mo)
        import ctypes as C
        calls = []
        cb = capi.mgb_dev_alloc_fn(lambda ctx, n: calls.append(n))  # (would give NULL)
        host = seq.cpu()
        rc = lib.mgb_map_batch_dev_rec(ix.gi, 4, None, 4, host.data_ptr(), host.numel(), off.data_ptr(), None, C.byref(ix.mo), None, cb,
                                       None, C.byref(capi.mgb_records_t()))
        assert rc < 0 and b"not device" in lib.mgb_last_error() and calls == []
        bad = torch.tensor([0, 20, 10, 30, seq.numel()], dtype=torch.int64, device="cuda:0")
        with pytest.raises(RuntimeError, match="decrease"):
            map_cuda_reads_to_tensors(lib, ix.gi, seq, bad, opt=ix.mo)

        class OutOfBlocks(Exception):
            pass

        def no_block(*a, **kw):
            raise OutOfBlocks()
        with monkeypatch.context() as m:
            m.setattr(torch, "empty", no_block)
            with pytest.raises(RuntimeError, match="allocator") as e:
                map_cuda_reads_to_tensors(lib, ix.gi, seq, off, opt=ix.mo)
        assert isinstance(e.value.__cause__, OutOfBlocks)
        t = map_cuda_reads_to_tensors(lib, ix.gi, seq, off, opt=ix.mo)  # the index is still usable
        assert t.seq_info.shape == (4, 2)
    finally:
        ix.close()
