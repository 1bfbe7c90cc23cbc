"""Reads in device memory (mgb_map_batch_dev*, mgb_test_ingest): the host rules they must follow, restated, and calls shared by the
simulator and GPU test modules."""
import ctypes as C
import random

import numpy as np

_CODE = np.full(256, 4, dtype=np.uint8)
_CODE[[ord("A"), ord("C"), ord("G"), ord("T")]] = [0, 1, 2, 3]


def toupper(s):
    """gmap.c:81 mg_toupper: only 'a'..'z' change"""
    a = np.frombuffer(s, dtype=np.uint8).copy()
    a[(a >= 0x61) & (a <= 0x7a)] -= 32
    return a.tobytes()


def pack_scalar(s):
    """mgb_engine.cu pack_read_scalar on an upper-case read: (words, holds a byte other than A/C/G/T)"""
    c = _CODE[np.frombuffer(s, dtype=np.uint8)]
    bad = bool((c == 4).any())
    c = (c & 3).astype(np.uint64)
    c = np.concatenate([c, np.zeros((-len(c)) % 32, dtype=np.uint64)]).reshape(-1, 32)
    words = (c << (2 * np.arange(32, dtype=np.uint64))).sum(axis=1, dtype=np.uint64) if len(c) else np.zeros(0, dtype=np.uint64)
    return [int(w) for w in words], bad


def ingest(lib, reads, segmented):
    """mgb_test_ingest on reads (bytes): (upper-case copies, words per read or None, raw flags)"""
    n = len(reads)
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(r) for r in reads])
    blob = b"".join(reads)
    n_words = sum((len(r) + 31) // 32 for r in reads)
    asc = C.create_string_buffer(max(1, len(blob)))
    pk = (C.c_uint64 * max(1, n_words))()
    raw = (C.c_int32 * max(1, n))()
    coff = (C.c_int64 * (n + 1))(*off.tolist())
    rc = lib.mgb_test_ingest(n, blob, coff, int(segmented), asc, pk, raw)
    assert rc == 0, (rc, lib.mgb_last_error())
    ups = [asc.raw[off[i]:off[i + 1]] for i in range(n)]
    words, at = [], 0
    for r in reads:
        k = (len(r) + 31) // 32
        words.append(None if segmented else list(pk[at:at + k]))
        at += k
    return ups, words, [raw[i] for i in range(n)]


def mixed_case(seqs, seed):
    """copies of upper-case reads with lower case in them: every third read all lower case, the others in random runs"""
    rng = random.Random(seed)
    out = []
    for i, s in enumerate(seqs):
        if i % 3 == 0:
            out.append(s.lower())
            continue
        b = bytearray(s)
        for _ in range(rng.randrange(0, 6)):
            a = rng.randrange(0, max(1, len(b)))
            e = min(len(b), a + rng.randrange(1, 400))
            b[a:e] = bytes(b[a:e]).lower()
        out.append(bytes(b))
    return out


def flat(seqs):
    """the bytes of seqs one after the other and their n + 1 offsets"""
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    return b"".join(seqs), off


def host_dev_gaf(lib, ix, names, seqs, n_seg=None):
    """mgb_map_batch_dev_gaf in a simulator, where "device memory" is host memory"""
    blob, off = flat(seqs)
    buf = C.create_string_buffer(blob, max(1, len(blob)))
    coff = (C.c_int64 * len(off))(*off.tolist())
    n_frag = len(n_seg) if n_seg is not None else len(seqs)
    cnseg = (C.c_int * max(1, n_frag))(*n_seg) if n_seg is not None else None
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    out, ln = C.c_void_p(0), C.c_size_t(0)
    rc = lib.mgb_map_batch_dev_gaf(ix.gi, n_frag, cnseg, len(seqs), C.addressof(buf), len(blob), C.addressof(coff), cnames,
                                   C.byref(ix.mo), None, C.byref(out), C.byref(ln), None)
    text = C.string_at(out, ln.value) if out.value else None
    if out.value:
        C.CDLL(None).free(out)
    return rc, text


def host_dev_results(lib, ix, names, seqs, n_seg=None):
    """mgb_map_batch_dev in a simulator: (rc, one result per sequence as mgtest.gchains_to_py() gives it, None where gcs[i] is NULL)"""
    import mgtest as T
    from minigraph_b200 import capi
    blob, off = flat(seqs)
    buf = C.create_string_buffer(blob, max(1, len(blob)))
    coff = (C.c_int64 * len(off))(*off.tolist())
    n = len(seqs)
    n_frag = len(n_seg) if n_seg is not None else n
    cnseg = (C.c_int * max(1, n_frag))(*n_seg) if n_seg is not None else None
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    gcs = (C.POINTER(capi.mg_gchains_t) * max(1, n))()
    rc = lib.mgb_map_batch_dev(ix.gi, n_frag, cnseg, n, C.addressof(buf), len(blob), C.addressof(coff), cnames, C.byref(ix.mo), None, gcs)
    out = [T.gchains_to_py(gcs[i]) for i in range(n)]
    lib.mgb_free_batch(n, gcs)
    return rc, out
