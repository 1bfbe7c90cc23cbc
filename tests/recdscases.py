"""The ds tables of mgb_map_batch_dev_rec_ds (minigraph_b200.tensors.map_cuda_reads_to_tensors(ds=True)): the calls and checks shared
by the simulator and GPU test modules, and the ds:Z field of the GAF text restated from the tables."""
import ctypes as C

import numpy as np

import devreads as DR
import reccases as RC
from minigraph_b200 import capi

HAS_CIGAR = capi.GC_COLUMNS.index("has_cigar")


def ds_tables_of(base, rec, rec_ds):
    """the ds tables of (rec, rec_ds) in host memory at address base, as numpy arrays"""
    shapes = {"ds_csr": (np.int64, (rec.n_rec + 1, 2)), "ds": (np.uint8, (rec_ds.n_ds,)), "ds_off": (np.int32, (rec_ds.n_ds_off,))}
    out = {}
    for t, name in enumerate(capi.REC_DS_TABLES):
        dtype, shape = shapes[name]
        n = int(np.prod(shape))
        raw = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(base + rec_ds.off[t]) if n else b""
        out[name] = np.frombuffer(raw, dtype=dtype).reshape(shape).copy()
    return out


def host_dev_rec_ds(lib, ix, names, seqs, n_seg=None, alloc=None, ds_out=True):
    """mgb_map_batch_dev_rec_ds in a simulator: (rc, the eight tables, the ds tables, the allocator, mgb_records_t, mgb_records_ds_t);
    the tables are None on failure.  ds_out=False passes a NULL mgb_records_ds_t."""
    blob, off = DR.flat(seqs)
    buf = C.create_string_buffer(blob, max(1, len(blob)))
    coff = (C.c_int64 * len(off))(*[int(x) for x in off])
    n_frag = len(n_seg) if n_seg is not None else len(seqs)
    cnseg = (C.c_int * max(1, n_frag))(*n_seg) if n_seg is not None else None
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    alloc = alloc or RC.HostAlloc()
    rec, rec_ds = capi.mgb_records_t(), capi.mgb_records_ds_t()
    rc = lib.mgb_map_batch_dev_rec_ds(ix.gi, n_frag, cnseg, len(seqs), C.addressof(buf), len(blob), C.addressof(coff), cnames,
                                      C.byref(ix.mo), None, alloc.fn, None, C.byref(rec), C.byref(rec_ds) if ds_out else None)
    if rc < 0:
        return rc, None, None, alloc, rec, rec_ds
    assert rec.block == C.addressof(alloc.blocks[-1]) and rec.bytes <= alloc.calls[-1]
    assert all(o % 256 == 0 for o in list(rec.off) + list(rec_ds.off))
    assert rec_ds.off[0] >= rec.off[capi.REC_TABLES.index("cigar")] + 8 * rec.n_cigar  # after the eight tables
    return rc, RC.tables_of(rec.block, rec), ds_tables_of(rec.block, rec, rec_ds), alloc, rec, rec_ds


def check_ds(want, tabs, ds):
    """every record's ds and offsets in the ds tables equal the mg_ds_t of its mg_gchain_t in want (one mgtest.gchains_to_py() result
    per sequence, or None), an empty ds where it has no CIGAR; the CSR starts at 0, ends with the totals and never decreases.
    Returns the number of records with a ds."""
    csr, text, offs = ds["ds_csr"], ds["ds"], ds["ds_off"]
    n_rec = len(tabs["gc"])
    assert csr.shape == (n_rec + 1, 2)
    assert csr[0].tolist() == [0, 0] and csr[-1].tolist() == [len(text), len(offs)], (csr[0], csr[-1], len(text), len(offs))
    assert (np.diff(csr, axis=0) >= 0).all()
    seq_csr = tabs["seq_csr"]
    n_ds = 0
    for i, r in enumerate(want):
        if r is None:
            continue
        r0 = int(seq_csr[i][0])
        for j, g in enumerate(r["gc"]):
            k = r0 + j
            (b0, o0), (b1, o1) = csr[k].tolist(), csr[k + 1].tolist()
            if g["ds"] is None:
                assert tabs["gc"][k, HAS_CIGAR] == 0 and b0 == b1 and o0 == o1, (i, j)
                continue
            assert text[b0:b1].tobytes() == g["ds"], "sequence %d record %d: ds differs" % (i, j)
            assert offs[o0:o1].tolist() == g["ds_off"], "sequence %d record %d: ds offsets differ" % (i, j)
            n_ds += b1 > b0
    return n_ds


def check_same_records(tabs, plain):
    """the eight tables byte for byte those of mgb_map_batch_dev_rec"""
    for k in capi.REC_TABLES:
        assert tabs[k].tobytes() == plain[k].tobytes(), k


_COMP = b"TVGHEFCDIJMLKNOPQYSAABWXRZ"


def _comp(c):
    if 65 <= c <= 90:
        return _COMP[c - 65]
    if 97 <= c <= 122:
        return _COMP[c - 97] + 32
    return c


def gaf_ds(ds, off, rev):
    """the ds:Z field that format.c prints for a record's ds and offsets; rev: its read has printed a reverse compact path by now,
    and the operations come in reverse order, each in place of the same length"""
    if not rev:
        return bytes(ds)
    if len(off) == 0:
        return b""
    n = len(ds)
    out = bytearray(n - off[0])
    for lo, ok in enumerate(off):
        ek = off[lo + 1] if lo + 1 < len(off) else n
        op, base = ds[ok], n - ek
        out[base] = op
        for j in range(ok + 1, ek):
            c = ds[j]
            if op == ord(":"):
                out[base + j - ok] = c
            elif op == ord("*"):
                out[base + j - ok] = _comp(c)
            else:
                out[base + 1 + (ek - 1 - j)] = ord("]") if c == ord("[") else ord("[") if c == ord("]") else _comp(c)
    return bytes(out)


def check_against_gaf(text, names, tabs, ds, print_2nd=False):
    """every record line of the GAF text (mgb_map_batch_gaf on the same reads, without -S) has the ds:Z field restated from the ds
    tables; returns the number of lines compared and how many of them came after a reverse path (their ds:Z reversed)"""
    lines = {}
    for ln in text.split(b"\n"):
        f = ln.split(b"\t")
        if len(f) > 12 and f[0] != b"*":
            lines.setdefault(f[0], []).append(f)
    gc, csr, seq_csr = tabs["gc"], ds["ds_csr"], tabs["seq_csr"]
    cols = capi.GC_COLUMNS
    i_id, i_parent, i_cnt = cols.index("id"), cols.index("parent"), cols.index("cnt")
    n = n_rev = 0
    for i, name in enumerate(names):
        r0, r1 = int(seq_csr[i][0]), int(seq_csr[i + 1][0])
        printed = [k for k in range(r0, r1) if (print_2nd or gc[k, i_id] == gc[k, i_parent]) and gc[k, i_cnt] > 0]
        got = lines.get(name, [])
        assert len(got) == len(printed), (name, len(got), len(printed))
        rev = False
        for k, f in zip(printed, got):
            rev = rev or f[4] == b"-"
            z = [x[5:] for x in f if x.startswith(b"ds:Z:")]
            if not gc[k, HAS_CIGAR]:
                assert z == []
                continue
            (b0, o0), (b1, o1) = csr[k].tolist(), csr[k + 1].tolist()
            assert z == [gaf_ds(ds["ds"][b0:b1].tobytes(), ds["ds_off"][o0:o1].tolist(), rev)], (name, k)
            n += 1
            n_rev += rev
    return n, n_rev
