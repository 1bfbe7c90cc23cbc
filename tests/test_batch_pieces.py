"""A batch of 2048 reads or more goes up and comes back in 4 pieces: the upload packs one piece while the previous one is on the
wire, and the blob download, the assembly, the GAF download and the GAF copy-out follow piece by piece.  2100 reads of 300-1800
bases from the MT fixtures, mapped as one batch and as three batches of 700 (one piece each), give the same results field by field,
and the device GAF text of the whole batch (mgb_map_batch_gaf) is the host writer's over those results.  Once as a packed batch in
which a few reads hold N (those go up as ASCII beside the packed ones), once as a batch of which more than 64 reads hold N (the
whole batch goes up as ASCII)."""
import ctypes as C
import os
import random

import pytest

import gafcases as GC
import mgtest as T
from minigraph_b200 import capi

N_READS, PART = 2100, 700


def windows(rng, seq, n):
    out = []
    for _ in range(n):
        ln = rng.randint(300, 1800)
        p = rng.randrange(len(seq) - ln)
        out.append(seq[p:p + ln])
    return out


def batches():
    rng = random.Random(2100)
    orang = T.read_fasta(os.path.join(T.FIX, "MT-orangA.fa"))[1][0]  # all A/C/G/T
    packed = windows(rng, orang, N_READS)
    for i in rng.sample(range(N_READS), 12):
        b = bytearray(packed[i])
        b[rng.randrange(len(b))] = ord("N")
        packed[i] = bytes(b)
    human = T.read_fasta(os.path.join(T.FIX, "MT-human.fa"))[1][0]  # one N
    ascii_ = windows(rng, human, N_READS)
    assert sum(b"N" in s for s in ascii_) > 64
    return [("packed", packed), ("ascii", ascii_)]


def map_batch(lib, ix, names, seqs):
    n = len(seqs)
    qlens = (C.c_int * n)(*[len(s) for s in seqs])
    cnames = (C.c_char_p * n)(*names)
    gcs = (C.POINTER(capi.mg_gchains_t) * n)()
    assert lib.mg_map_batch(ix.gi, n, qlens, (C.c_char_p * n)(*seqs), cnames, gcs, C.byref(ix.mo)) == 0, lib.mgb_last_error()
    st = capi.mgb_stats_t()
    lib.mgb_get_stats(ix.gi, C.byref(st))
    return gcs, qlens, cnames, st


def host_gaf(lib, ix, gcs, qlens, cnames):
    buf, ln = C.c_void_p(0), C.c_size_t(0)
    lib.mgb_write_gaf_batch(ix.g, len(qlens), gcs, qlens, cnames, ix.mo.flag, 0, C.byref(buf), C.byref(ln), None)
    text = C.string_at(buf, ln.value) if buf else b""
    C.CDLL(None).free(buf)
    return text


def case_pieces(lib):
    ix = GC.Index(lib, os.path.join(T.FIX, "MT.gfa"), "lr")
    try:
        for tag, seqs in batches():
            names = [b"%s%d" % (tag.encode(), i) for i in range(len(seqs))]
            gcs, qlens, cnames, st = map_batch(lib, ix, names, seqs)
            bases = sum(len(s) for s in seqs)
            assert (st.h2d_bytes < bases // 2) == (tag == "packed"), (tag, st.h2d_bytes, bases)
            whole = [T.gchains_to_py(gcs[i]) for i in range(len(seqs))]
            assert sum(1 for r in whole if r and r["n_gc"] > 0) > len(seqs) // 2, tag
            want = host_gaf(lib, ix, gcs, qlens, cnames)
            lib.mgb_free_batch(len(seqs), gcs)
            for p in range(0, len(seqs), PART):
                part, _, _, _ = map_batch(lib, ix, names[p:p + PART], seqs[p:p + PART])
                for i in range(PART):
                    d = T.diff_results(whole[p + i], T.gchains_to_py(part[i]))
                    assert d is None, "%s read %d: %s" % (tag, p + i, d)
                lib.mgb_free_batch(PART, part)
            rc, text = GC.map_gaf(lib, ix, names, seqs)
            assert rc == 0, lib.mgb_last_error()
            GC.check(text, want)
    finally:
        ix.close()


def test_batch_pieces_in_simulator():
    case_pieces(T.load_hostsim())


@pytest.mark.gpu
def test_batch_pieces_on_gpu():
    case_pieces(capi.load_product())
