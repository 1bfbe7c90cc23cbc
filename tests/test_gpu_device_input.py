"""Reads that live in GPU memory as CUDA tensors (mgb_map_batch_dev*, minigraph_b200.tensors): the GAF goldens byte for byte,
mg_gchains_t results field by field against the host-string entry points, lower case and N, NULL results, stream ordering,
several devices and refusals."""
import ctypes as C
import os

import pytest

import devreads as DR
import gafcases as GC
import mgtest as T
from minigraph_b200 import capi
from minigraph_b200.tensors import map_cuda_reads, pack_reads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return capi.load_product()


def dev_gaf(lib, ix, names, seqs, n_seg=None):
    seq, off = pack_reads(seqs, "cuda:0")
    return map_cuda_reads(lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg)


def dev_results(lib, ix, names, seqs, n_seg=None):
    seq, off = pack_reads(seqs, "cuda:0")
    gcs = map_cuda_reads(lib, ix.gi, seq, off, names, opt=ix.mo, n_seg=n_seg, gaf=False)
    out = [T.gchains_to_py(gcs[i]) for i in range(len(seqs))]
    lib.mgb_free_batch(len(seqs), gcs)
    return out


def host_frag_results(lib, ix, names, seqs, n_seg):
    n = len(seqs)
    gcs = (C.POINTER(capi.mg_gchains_t) * n)()
    rc = lib.mg_map_batch_frag(ix.gi, len(n_seg), (C.c_int * len(n_seg))(*n_seg), (C.c_int * n)(*[len(s) for s in seqs]),
                               (C.c_char_p * n)(*seqs), (C.c_char_p * len(names))(*names), gcs, C.byref(ix.mo))
    assert rc == 0, lib.mgb_last_error()
    out = [T.gchains_to_py(gcs[i]) for i in range(n)]
    lib.mgb_free_batch(n, gcs)
    return out


def stats(lib, ix):
    st = capi.mgb_stats_t()
    lib.mgb_get_stats(ix.gi, C.byref(st))
    return st


def test_goldens(lib, workdir):
    for name, _, kind, preset in GC.EXISTING:
        if name[:2] in ("c2", "L2", "L4"):
            gfa, names, seqs = GC.inputs(kind, workdir)
            ix = GC.Index(lib, gfa, preset)
            try:
                GC.check(dev_gaf(lib, ix, names, seqs), GC.golden(name))
                st = stats(lib, ix)
                assert st.t_pack_ms == 0 and st.h2d_bytes == 32 * len(seqs), (st.t_pack_ms, st.h2d_bytes)
            finally:
                ix.close()


def test_results_on_sv_graph(lib, workdir):
    gfa, names, seqs = GC.inputs("c3", workdir)
    want = T.map_with_engine(lib, gfa, names, seqs, "lr")[0]
    ix = GC.Index(lib, gfa, "lr")
    try:
        got = dev_results(lib, ix, names, DR.mixed_case(seqs, 9))
    finally:
        ix.close()
    assert sum(r is not None for r in got) > len(seqs) // 2
    for i, (a, b) in enumerate(zip(want, got)):
        d = T.diff_results(a, b)
        assert d is None, "read %d: %s" % (i, d)


def test_read_pairs(lib, workdir):
    gfa, names, n_seg, flat = GC.pair_inputs(workdir)
    ix = GC.Index(lib, gfa, "sr", False, GC.SHOW_UNMAP)
    try:
        want = host_frag_results(lib, ix, names, flat, n_seg)
        got = dev_results(lib, ix, names, flat, n_seg)
        assert all(got[i] is None for i in range(1, len(flat), 2))
        for i, (a, b) in enumerate(zip(want, got)):
            assert T.diff_results(a, b) is None, i
        GC.check(dev_gaf(lib, ix, names, [s.lower() for s in flat], n_seg), GC.golden(GC.PAIRS))
    finally:
        ix.close()


def with_n(seqs, every):
    return [s[:500] + b"N" * 7 + s[507:] if i % every == 0 else s for i, s in enumerate(seqs)]


def test_lower_case_and_n(lib, workdir):
    """a few such reads (the host path packs the others) and more than 64 (the host path sends the whole batch as ASCII)"""
    for kind, every in (("c2", 5), ("L2", 2)):
        gfa, names, seqs = GC.inputs(kind, workdir)
        seqs = with_n(seqs, every)
        ix = GC.Index(lib, gfa, "lr")
        try:
            rc, want = GC.map_gaf(lib, ix, names, seqs)
            assert rc == 0, lib.mgb_last_error()
            mixed = DR.mixed_case(seqs, 4)
            n_odd = sum(m != m.upper() or b"N" in m for m in mixed)
            assert (n_odd > 64) == (kind == "L2")
            GC.check(dev_gaf(lib, ix, names, mixed), want)
        finally:
            ix.close()


def test_empty_and_over_long_reads(lib, workdir):
    gfa, names, seqs = GC.inputs("c2", workdir)
    reads = [b"", seqs[0][:4000], seqs[1], b"", seqs[2][:3000].lower()]
    ix = GC.Index(lib, gfa, "lr")
    ix.mo.max_qlen = 5000
    try:
        got = dev_results(lib, ix, names[:5], reads)
    finally:
        ix.close()
    assert got[0] is None and got[2] is None and got[3] is None
    assert got[1] is not None and got[4] is not None


def test_side_stream_and_overwrite(lib, workdir):
    """the reads written by a torch kernel on a side stream that is still busy: the call orders its reads after it; the buffer is
    overwritten right after the call returns"""
    import torch
    gfa, names, seqs = GC.inputs("c2", workdir)
    ix = GC.Index(lib, gfa, "lr")
    try:
        rc, want = GC.map_gaf(lib, ix, names, seqs)
        assert rc == 0
        src, off = pack_reads(seqs, "cuda:0")
        dst = torch.zeros_like(src)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            torch.cuda._sleep(200_000_000)  # the side stream is busy for a while before it writes the reads
            torch.bitwise_or(src, 0x20, out=dst)  # lower case
            got = map_cuda_reads(lib, ix.gi, dst, off, names, opt=ix.mo)
            dst.fill_(ord("N"))
        GC.check(got, want)
        torch.cuda.synchronize()
        GC.check(got, want)
    finally:
        ix.close()


def test_several_devices(lib, workdir):
    import torch
    gfa, names, seqs = GC.inputs("L2", workdir)
    os.environ["MGB_DEVICES"] = "0,1" if torch.cuda.device_count() > 1 else "0,0"
    try:
        ix = GC.Index(lib, gfa, "lr")
    finally:
        del os.environ["MGB_DEVICES"]
    try:
        GC.check(dev_gaf(lib, ix, names, DR.mixed_case(seqs, 6)), GC.golden("L2_MT_240x10k_ont_s111.lr.gaf.gz"))
        want = T.map_with_engine(lib, gfa, names, seqs, "lr")[0]
        got = dev_results(lib, ix, names, seqs)
        for i, (a, b) in enumerate(zip(want, got)):
            assert T.diff_results(a, b) is None, i
    finally:
        ix.close()


def test_refusals(lib, workdir):
    import torch
    gfa, names, seqs = GC.inputs("c2", workdir)
    seqs = seqs[:4]
    seq, off = pack_reads(seqs, "cuda:0")
    host_seq, host_off = seq.cpu(), off.cpu()
    n, tot = len(seqs), seq.numel()
    bad_off = {"decrease": torch.tensor([0, 20, 10, 30, tot], dtype=torch.int64, device="cuda:0"),
               "outside": torch.tensor([0, 10, 20, 30, tot + 1], dtype=torch.int64, device="cuda:0")}
    ix = GC.Index(lib, gfa, "lr")
    try:
        cases = [(host_seq.data_ptr(), off.data_ptr(), b"not device"), (seq.data_ptr(), host_off.data_ptr(), b"not device"),
                 (seq.data_ptr(), bad_off["decrease"].data_ptr(), b"decrease"), (seq.data_ptr(), bad_off["outside"].data_ptr(), b"outside")]
        for p_seq, p_off, why in cases:
            gcs = (C.POINTER(capi.mg_gchains_t) * n)()
            rc = lib.mgb_map_batch_dev(ix.gi, n, None, n, p_seq, tot, p_off, None, C.byref(ix.mo), None, gcs)
            assert rc < 0 and why in lib.mgb_last_error(), (rc, lib.mgb_last_error())
            assert not any(gcs[i] for i in range(n))
            out, ln = C.c_void_p(0), C.c_size_t(5)
            rc = lib.mgb_map_batch_dev_gaf(ix.gi, n, None, n, p_seq, tot, p_off, None, C.byref(ix.mo), None, C.byref(out), C.byref(ln), None)
            assert rc < 0 and why in lib.mgb_last_error() and not out.value and ln.value == 0
        with pytest.raises(TypeError):
            map_cuda_reads(lib, ix.gi, seq.to(torch.int32), off, opt=ix.mo)
        with pytest.raises(ValueError):
            map_cuda_reads(lib, ix.gi, host_seq, off, opt=ix.mo)
    finally:
        ix.close()
