"""Result tables in device memory (mgb_map_batch_dev_rec, minigraph_b200.tensors.map_cuda_reads_to_tensors): the tables turned back
into per-read results, the host results they must equal, and the calls shared by the simulator and GPU test modules."""
import ctypes as C
import os
import re
import struct

import numpy as np

import devreads as DR
import gafcases as GC
import mgtest as T
from minigraph_b200 import capi

M32 = 0xffffffff


def records_to_py(t, seqs=None):
    """The tables (a dict of numpy arrays named as capi.REC_TABLES) as mgtest.gchains_to_py() gives every sequence's result (or those
    of the sequences seqs), without ds / ds_off: None where seq_info says there is no result."""
    cols = capi.GC_COLUMNS
    ih = cols.index("has_cigar")
    csr, info = t["seq_csr"], t["seq_info"]
    a_u, cig_u = t["a"].view(np.uint64), t["cigar"].view(np.uint64)
    out = []
    for i in range(len(info)) if seqs is None else seqs:
        has, rep_len = info[i].tolist()
        if not has:
            out.append(None)
            continue
        (r0, l0, a0), (r1, l1, a1) = csr[i].tolist(), csr[i + 1].tolist()
        d = {"n_gc": r1 - r0, "n_lc": l1 - l0, "n_a": a1 - a0, "rep_len": rep_len, "gc": [], "lc": [], "a": []}
        ccsr, div = t["cigar_csr"][r0:r1 + 1].tolist(), t["gc_div"][r0:r1].tolist()
        for k, row in enumerate(t["gc"][r0:r1].tolist()):
            g = dict(zip(cols[:ih], row[:ih]))
            g["hash"] &= M32
            g["div"] = div[k]
            if row[ih]:
                g["cigar_hdr"] = tuple(row[ih + 1:])
                g["cigar"] = cig_u[ccsr[k]:ccsr[k + 1]].tolist()
            else:
                g["cigar_hdr"], g["cigar"] = None, None
            d["gc"].append(g)
        d["lc"] = [(o, c, v & M32, s, e) for o, c, v, s, e in t["lc"][l0:l1].tolist()]
        d["a"] = [tuple(x) for x in a_u[a0:a1].tolist()]
        out.append(d)
    return out


def comparable(r):
    """r without ds / ds_off, every div as its float32 bits"""
    if r is None:
        return None
    r = dict(r)
    r["gc"] = [{k: struct.unpack("<I", struct.pack("<f", v))[0] if k == "div" else v for k, v in g.items() if k not in ("ds", "ds_off")}
               for g in r["gc"]]
    return r


def check(want, got):
    """field by field, div bit for bit"""
    assert len(want) == len(got), (len(want), len(got))
    for i, (a, b) in enumerate(zip(want, got)):
        d = T.diff_results(comparable(a), comparable(b))
        assert d is None, "sequence %d: %s" % (i, d)


def host_results(lib, ix, names, seqs, n_seg=None):
    """mg_map_batch_frag() on host strings, upper-cased: one result per sequence"""
    n = len(seqs)
    n_seg = n_seg if n_seg is not None else [1] * n
    ups = [DR.toupper(s) for s in seqs]
    gcs = (C.POINTER(capi.mg_gchains_t) * max(1, n))()
    cnames = (C.c_char_p * max(1, len(n_seg)))(*names) if names is not None else None
    rc = lib.mg_map_batch_frag(ix.gi, len(n_seg), (C.c_int * max(1, len(n_seg)))(*n_seg), (C.c_int * max(1, n))(*[len(s) for s in ups]),
                               (C.c_char_p * max(1, n))(*ups), cnames, gcs, C.byref(ix.mo))
    assert rc == 0, lib.mgb_last_error()
    out = [T.gchains_to_py(gcs[i]) for i in range(n)]
    lib.mgb_free_batch(n, gcs)
    return out


def header_gc_columns():
    """the MGB_GC_* names of include/mgb200.h in their order, lower case"""
    with open(os.path.join(T.REPO, "include", "mgb200.h")) as f:
        text = f.read()
    body = re.search(r"enum\s*\{[^}]*?(MGB_GC_ID\b[^}]*)\}", text).group(1)
    names = re.findall(r"MGB_GC_(\w+)", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names[-1] == "NCOL"
    return tuple(x.lower() for x in names[:-1])


def tables_of(base, rec):
    """the tables of rec in host memory at address base, as numpy arrays"""
    shapes = {"seq_csr": (np.int64, (rec.n_seq + 1, 3)), "seq_info": (np.int32, (rec.n_seq, 2)), "gc": (np.int32, (rec.n_rec, len(capi.GC_COLUMNS))),
              "gc_div": (np.float32, (rec.n_rec,)), "cigar_csr": (np.int64, (rec.n_rec + 1,)), "lc": (np.int32, (rec.n_lc, 5)),
              "a": (np.int64, (rec.n_a, 2)), "cigar": (np.int64, (rec.n_cigar,))}
    out = {}
    for t, name in enumerate(capi.REC_TABLES):
        dtype, shape = shapes[name]
        n = int(np.prod(shape))
        raw = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(base + rec.off[t]) if n else b""
        out[name] = np.frombuffer(raw, dtype=dtype).reshape(shape).copy()
    return out


class HostAlloc:
    """an allocator for the simulators, where "device memory" is host memory: counts its calls and keeps its blocks, filled with 0xA5
    so that a cell the library leaves unwritten cannot pass for a 0"""

    def __init__(self, fail=False):
        self.calls, self.blocks, self.fail = [], [], fail

        def alloc(ctx, nbytes):
            self.calls.append(nbytes)
            if self.fail:
                return None
            self.blocks.append(C.create_string_buffer(b"\xa5" * nbytes, nbytes))
            return C.addressof(self.blocks[-1])
        self.fn = capi.mgb_dev_alloc_fn(alloc)


def host_dev_rec(lib, ix, names, seqs, n_seg=None, alloc=None, off=None, seq_bytes=None, n_seq=None):
    """mgb_map_batch_dev_rec in a simulator: (rc, tables or None, the allocator).  off / seq_bytes / n_seq replace the batch's own."""
    blob, own_off = DR.flat(seqs)
    off = own_off if off is None else off
    buf = C.create_string_buffer(blob, max(1, len(blob)))
    coff = (C.c_int64 * len(off))(*[int(x) for x in off])
    n_frag = len(n_seg) if n_seg is not None else len(seqs)
    cnseg = (C.c_int * max(1, n_frag))(*n_seg) if n_seg is not None else None
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    alloc = alloc or HostAlloc()
    rec = capi.mgb_records_t()
    rc = lib.mgb_map_batch_dev_rec(ix.gi, n_frag, cnseg, len(seqs) if n_seq is None else n_seq, C.addressof(buf),
                                   len(blob) if seq_bytes is None else seq_bytes, C.addressof(coff), cnames, C.byref(ix.mo), None,
                                   alloc.fn, None, C.byref(rec))
    if rc < 0:
        return rc, None, alloc
    assert rec.block == C.addressof(alloc.blocks[-1]) and rec.bytes <= alloc.calls[-1]
    assert all(o % 256 == 0 for o in rec.off)
    return rc, tables_of(rec.block, rec), alloc


# the parity sets: (inputs, preset, cigar, flag bits beyond the preset's)
SETS = [("c2", "lr", True, 0), ("c3", "lr", True, 0), ("L2", "lr", True, 0), ("sv_edge", "lr", True, GC.X), ("stable", "lr", True, GC.X),
        ("L4", "asm", True, 0), ("sv_edge", "lr", False, GC.X)]


def with_n(seqs, every):
    return [s[:500] + b"N" * 7 + s[507:] if i % every == 0 else s for i, s in enumerate(seqs)]


def unmapped_read(n=3000, seed=3):
    import random
    rng = random.Random(seed)
    return bytes(rng.choice(b"ACGT") for _ in range(n))
