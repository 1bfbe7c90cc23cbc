"""Parity cases shared by the CPU (hostsim) and GPU (libmgb200) test modules."""
import hashlib
import os

import mgtest as T


class capi_u128(__import__("ctypes").Structure):
    _fields_ = [("x", __import__("ctypes").c_uint64), ("y", __import__("ctypes").c_uint64)]
from minigraph_b200 import capi  # noqa: E402

G = os.path.join(T.REPO, "tests", "golden")


def golden(name):
    with open(os.path.join(G, name), "rb") as f:
        return f.read()


def golden_gz(name):
    import gzip
    with gzip.open(os.path.join(G, name), "rb") as f:
        return f.read()


def case_golden_large(lib, workdir, which=("L2", "L3", "L4")):
    """the larger golden sets (tests/golden/make_golden.sh): 240 x 10 kb reads on test/MT.gfa, 240 x 15 kb on an SV graph as dense as
    the bench's MHC-scale one (1 Mb, 8 haplotypes), 200 x 20 kb HiFi-error reads with the asm preset; GAF text byte for byte"""
    if "L2" in which:
        hap, reads = os.path.join(workdir, "mt.hap.fa"), os.path.join(workdir, "mtL.reads.fa")
        T.sim_mt_haps(hap)
        T.sim_reads(hap, reads, 240, 10000, "ont", 111)
        check_gaf(lib, os.path.join(T.FIX, "MT.gfa"), reads, "lr", golden_gz("L2_MT_240x10k_ont_s111.lr.gaf.gz"))
    if "L3" in which:
        pre, reads = os.path.join(workdir, "svL"), os.path.join(workdir, "svL.reads.fa")
        T.sim_graph(pre, 1000000, 8, 7)
        T.sim_reads(pre + ".hap.fa", reads, 240, 15000, "ont", 105)
        check_gaf(lib, pre + ".gfa", reads, "lr", golden_gz("L3_sv1m_h8_s7_240x15k_ont_s105.lr.gaf.gz"))
    if "L4" in which:
        reads = os.path.join(workdir, "mthL.reads.fa")
        T.sim_reads(os.path.join(T.FIX, "MT-human.fa"), reads, 200, 20000, "hifi", 113, circular=True)
        check_gaf(lib, os.path.join(T.FIX, "MT-human.fa"), reads, "asm", golden_gz("L4_MThuman_200x20k_hifi_s113.asm.gaf.gz"))


def first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            fx, fy = x.split(b"\t"), y.split(b"\t")
            for j, (p, q) in enumerate(zip(fx, fy)):
                if p != q:
                    return "line %d field %d: %r != %r" % (i, j, p[:120], q[:120])
            return "line %d: field count %d != %d" % (i, len(fx), len(fy))
    return "line count %d != %d" % (len(la), len(lb))


def check_gaf(lib, gfa, fasta, preset, want, flag_extra=0):
    names, seqs = T.read_fasta(fasta)
    got, st = T.gaf_with_engine(lib, gfa, names, seqs, preset, flag_extra=flag_extra)
    assert got == want, first_diff(got, want)
    return st


def case_c1(lib, workdir):
    """config 1: test/MT.gfa <- test/MT-orangA.fa, -cx lr; md5 pinned in SURVEY.md section 8c."""
    st = check_gaf(lib, os.path.join(T.FIX, "MT.gfa"), os.path.join(T.FIX, "MT-orangA.fa"), "lr", golden("c1_MT_orangA.lr.gaf"))
    assert hashlib.md5(golden("c1_MT_orangA.lr.gaf")).hexdigest() == "22bf23ebe2039e8353f56f4a324a2eaa"
    check_gaf(lib, os.path.join(T.FIX, "MT.gfa"), os.path.join(T.FIX, "MT-chimp.fa"), "lr", golden("c1_MT_chimp.lr.gaf"))
    return st


def case_c2(lib, workdir):
    hap, reads = os.path.join(workdir, "mt.hap.fa"), os.path.join(workdir, "mt.reads.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, 24, 10000, "ont", 11)
    return check_gaf(lib, os.path.join(T.FIX, "MT.gfa"), reads, "lr", golden("c2_MT_24x10k_ont_s11.lr.gaf"))


def case_c3(lib, workdir):
    pre, reads = os.path.join(workdir, "sv"), os.path.join(workdir, "sv.reads.fa")
    T.sim_graph(pre, 300000, 3, 7)
    T.sim_reads(pre + ".hap.fa", reads, 24, 15000, "ont", 5)
    return check_gaf(lib, pre + ".gfa", reads, "lr", golden("c3_sv300k_h3_s7_24x15k_ont_s5.lr.gaf"))


def case_c4(lib, workdir):
    reads = os.path.join(workdir, "mth.reads.fa")
    T.sim_reads(os.path.join(T.FIX, "MT-human.fa"), reads, 12, 20000, "hifi", 13, circular=True)
    return check_gaf(lib, os.path.join(T.FIX, "MT-human.fa"), reads, "asm", golden("c4_MThuman_12x20k_hifi_s13.asm.gaf"))


def case_edge(lib, workdir):
    """empty, tiny, all-N, unmappable and lower-case-free reads: same objects as the reference (map-algo.c:356-360)."""
    import ctypes as C
    from minigraph_b200 import capi, options
    gfa = os.path.join(T.FIX, "MT.gfa")
    _, hs = T.read_fasta(os.path.join(T.FIX, "MT-human.fa"))
    names = [b"empty", b"tiny", b"allN", b"random", b"short_ok", b"with_N"]
    seqs = [b"", b"ACGT", b"N" * 500, (b"ACGTTGCA" * 200)[:1500], hs[0][1000:1300], hs[0][2900:3300]]
    got, _, _ = T.map_with_engine(lib, gfa, names, seqs, "lr")
    assert got[0] is None                      # qlen == 0 -> no result object
    for r in got[1:4]:
        assert r is not None and r["n_gc"] == 0
    if T.have_ref():
        want, _ = T.map_with_ref(gfa, names, seqs, "lr")
        for i, (a, b) in enumerate(zip(want, got)):
            assert T.diff_results(a, b) is None, (i, T.diff_results(a, b))


def case_struct_random(lib, workdir, n_reads=150, seed=23):
    """field-by-field comparison of mg_gchains_t (incl. anchors, lchains, CIGAR, ds offsets) against the reference library."""
    pre, reads = os.path.join(workdir, "svb"), os.path.join(workdir, "svb.reads.fa")
    T.sim_graph(pre, 400000, 4, 31)
    T.sim_reads(pre + ".hap.fa", reads, n_reads, 12000, "ont", seed)
    names, seqs = T.read_fasta(reads)
    want, mo_r = T.map_with_ref(pre + ".gfa", names, seqs, "lr")
    got, mo_e, st = T.map_with_engine(lib, pre + ".gfa", names, seqs, "lr")
    assert (mo_r.occ_max1, mo_r.lc_max_occ) == (mo_e.occ_max1, mo_e.lc_max_occ)
    for i, (a, b) in enumerate(zip(want, got)):
        d = T.diff_results(a, b)
        assert d is None, "read %d (%s): %s" % (i, names[i], d)
    return st


_mwf = None


def _mwf_types():
    """ctypes view of miniwfa.h:36-51 (mwf_opt_t, mwf_rst_t) and the prototypes of the reference functions used as the checker"""
    global _mwf
    if _mwf is None:
        import ctypes as C
        ref = T.load_ref()

        class mwf_opt_t(C.Structure):
            _fields_ = [("flag", C.c_int32), ("x", C.c_int32), ("o1", C.c_int32), ("e1", C.c_int32), ("o2", C.c_int32), ("e2", C.c_int32),
                        ("step", C.c_int32), ("max_s", C.c_int32), ("max_iter", C.c_int64), ("max_occ", C.c_int32), ("kmer", C.c_int32), ("min_len", C.c_int32)]

        class mwf_rst_t(C.Structure):
            _fields_ = [("s", C.c_int32), ("n_cigar", C.c_int32), ("n_iter", C.c_int64), ("cigar", C.POINTER(C.c_uint32))]
        for f in (ref.mwf_wfa_exact, ref.mwf_wfa_chain):
            f.restype = None
            f.argtypes = [C.c_void_p, C.POINTER(mwf_opt_t), C.c_int32, C.c_char_p, C.c_int32, C.c_char_p, C.POINTER(mwf_rst_t)]
        ref.mwf_opt_init.argtypes = [C.POINTER(mwf_opt_t)]
        _mwf = (mwf_opt_t, mwf_rst_t)
    return _mwf


def case_wfa_fallback(lib, n_cases=12, seed=5):
    """gaps whose exact WFA exceeds the cell cap take the reference's chaining heuristic + low-memory checkpoints
    (miniwfa.c:551-601,776-834): same CIGAR and score as mwf_wfa_exact(max_iter) -> mwf_wfa_chain(step) of the reference"""
    import ctypes as C
    import random
    ref = T.load_ref()
    mwf_opt_t, mwf_rst_t = _mwf_types()
    rng = random.Random(seed)

    def mutate(s, rate):
        out = []
        for c in s:
            u = rng.random()
            if u < rate * 0.4:
                out.append(rng.choice("ACGT"))
            elif u < rate * 0.7:
                continue
            elif u < rate:
                out.append(c)
                out.append(rng.choice("ACGT"))
            else:
                out.append(c)
        return "".join(out)
    n_fallback = 0
    for it in range(n_cases):
        n = rng.choice([300, 900, 2500])
        if it == 0:
            n = 9000  # tl + ql > 16000: beyond the 16-bit ring of tier 3, takes the 32-bit one
        t = "".join(rng.choice("ACGT") for _ in range(n))
        blocks = [mutate(t[i:i + 200], rng.choice([0.02, 0.1, 0.3]) if it else 0.02) if rng.random() < 0.8 or it == 0 else "".join(rng.choice("ACGT") for _ in range(rng.choice([50, 300])))
                  for i in range(0, n, 200)]
        q = "".join(blocks)
        ts, qs = t.encode(), q.encode()
        max_iter, step = rng.choice([(2000, 40), (20000, 25), (50000, 100), (10 ** 8, 5000)])
        if it == 0:
            max_iter, step = 10 ** 8, 5000
        opt = mwf_opt_t()
        ref.mwf_opt_init(C.byref(opt))
        opt.flag |= 1
        opt.step, opt.max_iter = 0, max_iter
        rst = mwf_rst_t()
        ref.mwf_wfa_exact(None, C.byref(opt), len(ts), ts, len(qs), qs, C.byref(rst))
        if rst.s < 0:
            n_fallback += 1
            opt.step, opt.max_iter = step, -1
            ref.mwf_wfa_chain(None, C.byref(opt), len(ts), ts, len(qs), qs, C.byref(rst))
        want = [rst.cigar[i] for i in range(rst.n_cigar)]
        cap = len(ts) + len(qs) + 8
        buf = (C.c_uint32 * cap)()
        score = C.c_int(0)
        nc = lib.mgb_test_wfa(ts, len(ts), qs, len(qs), max_iter, step, buf, cap, C.byref(score))
        assert nc >= 0, (it, nc)
        got = [buf[i] for i in range(nc)]
        assert got == want and score.value == rst.s, "case %d (tl=%d ql=%d max_iter=%d step=%d): score %d vs %d" % (it, len(ts), len(qs), max_iter, step, score.value, rst.s)
    assert n_fallback >= 3


def check_cigar_invariants(r, qlen):
    """what holds for every mg_gchains_t the reference produces with -c (checked against the reference itself in
    test_hostsim_parity.py): the CIGAR of a chain spans exactly its query and path intervals and sums to its mlen/blen"""
    for g in r["gc"]:
        assert 0 <= g["qs"] < g["qe"] <= qlen and 0 <= g["ps"] < g["pe"] <= g["plen"], g
        if g["cigar"] is None:
            continue
        n_cigar, mlen, blen, aplen, ss, ee = g["cigar_hdr"]
        assert n_cigar == len(g["cigar"]) and all((c & 15) in (1, 2, 7, 8) and (c >> 4) > 0 for c in g["cigar"])
        assert sum(c >> 4 for c in g["cigar"] if (c & 15) in (7, 8, 1)) == g["qe"] - g["qs"]
        assert sum(c >> 4 for c in g["cigar"] if (c & 15) in (7, 8, 2)) == g["pe"] - g["ps"] == aplen
        assert sum(c >> 4 for c in g["cigar"] if (c & 15) == 7) == mlen and sum(c >> 4 for c in g["cigar"]) == blen
        assert all((a & 15) != (b & 15) for a, b in zip(g["cigar"], g["cigar"][1:]))  # adjacent operations are merged


def case_full_size(lib, workdir, n_reads=10000, n_sub=300, n_ref=100, seed=11):
    """BASELINE config 2 at its full size (10 000 x 10 kb ONT-like reads on test/MT.gfa), through properties that do not
    need the reference on every read: (1) reads sampled from the graph map (all but a stray one) and a CIGAR is
    consistent with its intervals; (2) a result does not depend on the batch a read travels in (mg_map_frag is a pure function of the read,
    map-algo.c:340-495): a shuffled sample mapped as its own batch gives the same objects; (3) a smaller sample against
    the reference library itself."""
    import ctypes as C
    import random
    from minigraph_b200 import capi, options
    hap, reads = os.path.join(workdir, "mt.hap.fa"), os.path.join(workdir, "mt.full.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, n_reads, 10000, "ont", seed)
    names, seqs = T.read_fasta(reads)
    n = len(seqs)
    assert n == n_reads
    gfa = os.path.join(T.FIX, "MT.gfa")
    g = lib.mgb_gfa_read(gfa.encode())
    io, mo = options.opt_set("lr", True)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    qlens = (C.c_int * n)(*[len(s) for s in seqs])
    cseqs, cnames = (C.c_char_p * n)(*seqs), (C.c_char_p * n)(*names)
    gcs = (C.POINTER(capi.mg_gchains_t) * n)()
    assert lib.mg_map_batch(gi, n, qlens, cseqs, cnames, gcs, C.byref(mo)) == 0, lib.mgb_last_error()
    n_mapped = sum(1 for i in range(n) if gcs[i] and gcs[i].contents.n_gc > 0)
    assert n_mapped >= 0.999 * n, "%d of %d reads sampled from the graph did not map" % (n - n_mapped, n)
    rng = random.Random(seed)
    sub = rng.sample(range(n), min(n_sub, n))
    full = {i: T.gchains_to_py(gcs[i]) for i in sub}
    lib.mgb_free_batch(n, gcs)
    for i in sub:
        check_cigar_invariants(full[i], len(seqs[i]))
    m = len(sub)
    qlens2 = (C.c_int * m)(*[len(seqs[i]) for i in sub])
    cseqs2, cnames2 = (C.c_char_p * m)(*[seqs[i] for i in sub]), (C.c_char_p * m)(*[names[i] for i in sub])
    gcs2 = (C.POINTER(capi.mg_gchains_t) * m)()
    assert lib.mg_map_batch(gi, m, qlens2, cseqs2, cnames2, gcs2, C.byref(mo)) == 0, lib.mgb_last_error()
    for j, i in enumerate(sub):
        d = T.diff_results(T.gchains_to_py(gcs2[j]), full[i])
        assert d is None, "read %d: alone vs in the full batch: %s" % (i, d)
    lib.mgb_free_batch(m, gcs2)
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
    if T.have_ref() and n_ref > 0:
        pick = sub[:n_ref]
        want, _ = T.map_with_ref(gfa, [names[i] for i in pick], [seqs[i] for i in pick], "lr")
        for i, w in zip(pick, want):
            check_cigar_invariants(w, len(seqs[i]))  # the invariants are the reference's, not ours
            d = T.diff_results(full[i], w)
            assert d is None, "read %d vs reference: %s" % (i, d)


def case_wfa_divergent(lib, n_cases=24, seed=5):
    """unrelated sequences of unequal length: the band reaches the matrix borders, is re-centred and shrinks
    (miniwfa.c:144-171) -- what the tier-3 ring has to get right when slots are reused by narrower wavefronts"""
    import ctypes as C
    import random
    ref = T.load_ref()
    mwf_opt_t, mwf_rst_t = _mwf_types()
    rng = random.Random(seed)
    for it in range(n_cases):
        tl = rng.choice([150, 300, 500, 800])
        ql = max(20, int(tl * rng.choice([0.3, 0.7, 1.0, 1.5])))
        t = "".join(rng.choice("ACGT") for _ in range(tl))
        q = "".join(rng.choice("ACGT") for _ in range(ql))
        if it % 3 == 0:  # a shared core between random flanks
            core = "".join(rng.choice("ACGT") for _ in range(100))
            t, q = t[:tl // 2] + core + t[tl // 2:], q[:ql // 3] + core + q[ql // 3:]
        ts, qs = t.encode(), q.encode()
        opt = mwf_opt_t()
        ref.mwf_opt_init(C.byref(opt))
        opt.flag |= 1
        opt.step, opt.max_iter = 0, 10 ** 8
        rst = mwf_rst_t()
        ref.mwf_wfa_exact(None, C.byref(opt), len(ts), ts, len(qs), qs, C.byref(rst))
        assert rst.s >= 0
        want = [rst.cigar[i] for i in range(rst.n_cigar)]
        cap = len(ts) + len(qs) + 8
        buf = (C.c_uint32 * cap)()
        score = C.c_int(0)
        nc = lib.mgb_test_wfa(ts, len(ts), qs, len(qs), 10 ** 8, 5000, buf, cap, C.byref(score))
        assert nc >= 0 and [buf[i] for i in range(nc)] == want and score.value == rst.s, (it, tl, ql, score.value, rst.s)


def case_wfa_band_shrinks(lib, n_cases=48, seed=99):
    """tier 3 far past score 256: unrelated pairs, noisy copies with a long indel, shared cores between random flanks, low-complexity
    pairs.  The ring keeps 17 H slots but only 3 / 2 slots of E/F; what the band shrink (miniwfa.c:144-171) wants to know about the
    last 17 wavefronts comes from the last-good-score slice.  Same CIGAR and score as the reference's mwf_wfa_exact()."""
    import ctypes as C
    import random
    ref = T.load_ref()
    mwf_opt_t, mwf_rst_t = _mwf_types()
    rng = random.Random(seed)
    n_shrunk = 0
    for it in range(n_cases):
        tl = rng.choice([200, 400, 700, 1200, 2000])
        ql = max(30, int(tl * rng.choice([0.2, 0.5, 0.8, 1.0, 1.3, 2.0])))
        t = "".join(rng.choice("ACGT") for _ in range(tl))
        mode = it % 4
        if mode == 0:
            q = "".join(rng.choice("ACGT") for _ in range(ql))
        elif mode == 1:
            q = "".join(c if rng.random() > 0.25 else rng.choice("ACGT") for c in t)
            cut = rng.randrange(len(q))
            q = q[:cut] + q[cut + rng.choice([50, 150, 400]):]
        elif mode == 2:
            q = "".join(rng.choice("ACGT") for _ in range(ql))
            for _ in range(3):
                core = "".join(rng.choice("ACGT") for _ in range(rng.choice([30, 80])))
                i, j = rng.randrange(len(t)), rng.randrange(len(q))
                t, q = t[:i] + core + t[i:], q[:j] + core + q[j:]
        else:
            q = "".join(rng.choice("AC") for _ in range(ql))
            t = "".join(rng.choice("AC") if rng.random() < 0.7 else rng.choice("GT") for _ in range(tl))
        if not q:
            continue
        ts, qs = t.encode(), q.encode()
        opt = mwf_opt_t()
        ref.mwf_opt_init(C.byref(opt))
        opt.flag |= 1
        opt.step, opt.max_iter = 0, 10 ** 8
        rst = mwf_rst_t()
        ref.mwf_wfa_exact(None, C.byref(opt), len(ts), ts, len(qs), qs, C.byref(rst))
        assert rst.s >= 0
        n_shrunk += rst.s >= 256
        want = [rst.cigar[i] for i in range(rst.n_cigar)]
        cap = len(ts) + len(qs) + 8
        buf = (C.c_uint32 * cap)()
        score = C.c_int(0)
        nc = lib.mgb_test_wfa(ts, len(ts), qs, len(qs), 10 ** 8, 5000, buf, cap, C.byref(score))
        assert nc >= 0 and [buf[i] for i in range(nc)] == want and score.value == rst.s, (it, len(ts), len(qs), score.value, rst.s, nc)
    assert n_shrunk >= n_cases // 2


def case_radix_exact(lib, n_cases=60, seed=17, hot_max=16384):
    """the warp-wide replay of klib's unstable radix sort (mgb_common.cuh radix_sort_exact_w), in place and as a walk over digits, with
    scratch on "chip" and in the arena: the same order as radix_sort_128x() of the reference, ties included (ksort.h:112-162) --
    few distinct keys (long runs of ties), keys that differ in one byte only (one level), bins above 64 elements (recursion), skewed bins.
    Without a build of the reference, its order comes from the plain-C restatement (oracle/mgoracle.c), whose tie order
    tests/test_oracle.py pins against golden vectors of the reference's sort."""
    import ctypes as C
    import random
    from minigraph_b200 import capi
    if T.have_ref():
        ref = T.load_ref()
        ref.radix_sort_128x.restype = None
        ref.radix_sort_128x.argtypes = [C.POINTER(capi.mg128_t), C.POINTER(capi.mg128_t)]

        def ref_sort(a, n):
            ref.radix_sort_128x(a, C.cast(C.byref(a, C.sizeof(a)), C.POINTER(capi.mg128_t)))
    else:
        import subprocess
        subprocess.check_call(["make", "-s", "-C", os.path.join(T.REPO, "oracle"), "liboracle.so"])
        orc = C.CDLL(os.path.join(T.REPO, "oracle", "liboracle.so"))
        orc.orc_radix_sort_128x.restype = None
        orc.orc_radix_sort_128x.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_int64]

        def ref_sort(a, n):
            x, y = (C.c_uint64 * n)(*[a[i].x for i in range(n)]), (C.c_uint64 * n)(*[a[i].y for i in range(n)])
            orc.orc_radix_sort_128x(x, y, n)
            for i in range(n):
                a[i].x, a[i].y = x[i], y[i]
    rng = random.Random(seed)
    for it in range(n_cases):
        n = rng.choice([65, 191, 192, 193, 700, 1100, 3000, 9000])
        nk = rng.choice([2, 7, 300, 5000, 2 ** 40])
        sh = rng.choice([0, 8, 16, 33])
        base = rng.randrange(2 ** 20) << 40
        if it % 5 == 4:  # one heavy bin and a sprinkle of others
            keys = [base + ((rng.randrange(nk) << sh) if rng.random() < 0.1 else (3 << sh)) for _ in range(n)]
        else:
            keys = [base + (rng.randrange(nk) << sh) for _ in range(n)]
        want = (capi.mg128_t * n)()
        for i, x in enumerate(keys):
            want[i].x, want[i].y = x, i
        ref_sort(want, n)
        for walk, hot in ((0, 0), (1, 0), (1, hot_max), (1, n // 4 + 3400), (0, hot_max)):  # (n/4 + 3400: what the callers ask of the on-chip slice; the digits then go to the arena)
            got = (capi.mg128_t * n)()
            for i, x in enumerate(keys):
                got[i].x, got[i].y = x, i
            rc = lib.mgb_test_radix128(got, n, walk, hot)
            assert rc == 0, (it, n, walk, hot, rc)
            bad = next((i for i in range(n) if got[i].y != want[i].y or got[i].x != want[i].x), None)
            assert bad is None, "case %d (n=%d, %d keys << %d, walk=%d, hot=%d): position %d holds element %d, the reference has %d" % (
                it, n, nk, sh, walk, hot, bad, got[bad].y, want[bad].y)


def case_wfa_tiers(lib, workdir, n_struct=60):
    """the gap alignment tiers (mgb_wfa_tiers.cuh: slices that hold -inf outside their range instead of bounds checks).  Same GAF
    for the golden cases (lr and asm presets, both on-chip tiers busy), same mg_gchains_t fields as the reference on an SV graph,
    also with the learned tier routing of a second batch"""
    from minigraph_b200 import capi
    for fn in (case_c2, case_c3, case_c4):
        st = fn(lib, workdir)
        prof = {n: st.prof[i] for i, n in enumerate(capi.PROF_NAMES)}
        assert prof["wfa_fast_n"] > 500, prof
        assert fn is case_c4 or prof["wfa_mid_n"] > 500, prof
    if T.have_ref():
        case_struct_random(lib, workdir, n_reads=n_struct, seed=37)
        case_tier_routing(lib, workdir)
        case_short_reads(lib, workdir, n_pairs=20)  # sr preset: tier 1 only, two-segment fragments
        case_wfa_fallback(lib)  # tier 3 against miniwfa: scores far past 256 (band re-centring), capped runs, a gap beyond the 16-bit ring
        case_wfa_divergent(lib)
        case_wfa_band_shrinks(lib)


def case_gchain_labels(lib, workdir, n_reads=150, graph_len=1000000):
    """graph chaining from the per-source label table (mgb_gclabel.cuh) on a graph dense enough that every read spans a dozen
    segments: every field against the reference with the table on (sources searched once per batch by k_gc_labels), with the
    table off (every read searches its own sources), lr and asm presets (walk bounds of 20 kb and 150 kb)"""
    pre, reads = os.path.join(workdir, "svl"), os.path.join(workdir, "svl.reads.fa")
    T.sim_graph(pre, graph_len, 8, 7)
    T.sim_reads(pre + ".hap.fa", reads, n_reads, 15000, "ont", 5)
    names, seqs = T.read_fasta(reads)
    try:
        for preset, m in (("lr", n_reads), ("asm", n_reads // 3)):
            want, _ = T.map_with_ref(pre + ".gfa", names[:m], seqs[:m], preset)
            for cache in (1, 0):
                assert lib.mgb_set_param(b"lab_cache", cache) == 0
                got, _, st = T.map_with_engine(lib, pre + ".gfa", names[:m], seqs[:m], preset)
                assert (st.n_lab_new > 100) == bool(cache), (preset, cache, st.n_lab_new)
                assert sum(r["n_lc"] for r in got if r) > 5 * m  # the reads do span many segments
                for i, (a, b) in enumerate(zip(want, got)):
                    d = T.diff_results(a, b)
                    assert d is None, "%s lab_cache=%d read %d: %s" % (preset, cache, i, d)
    finally:
        lib.mgb_set_param(b"lab_cache", 1)


def case_tandem_diagonals(lib, workdir, n_reads=48, seed=29):
    """RMQ chaining where two diagonals interleave in target order: a linear reference with tandem duplications (copies 700 bp and
    3 kb apart: narrow and wide blocks of the outer query's summaries, mgb_lchain.cuh chain_rmq_fill_w) and a circular one whose reads
    wrap around; asm preset (RMQ chaining of every read) and lr (the long-join rescue); every field against the reference"""
    import random
    rng = random.Random(seed)

    def rnd(n):
        return "".join(rng.choice("ACGT") for _ in range(n))
    d1, d2 = rnd(700), rnd(3000)
    ref = rnd(6000) + d1 + d1 + d1 + rnd(5000) + d2 + d2 + rnd(7000) + d1 + rnd(4000)
    lin = os.path.join(workdir, "tandem.fa")
    with open(lin, "w") as f:
        f.write(">tandem\n%s\n" % ref)
    for gfa, circular, tag in ((lin, False, "lin"), (os.path.join(T.FIX, "MT-human.fa"), True, "circ")):
        for preset, err, rl in (("asm", "hifi", 18000), ("lr", "ont", 11000)):
            reads = os.path.join(workdir, "tandem.%s.%s.fa" % (tag, preset))
            T.sim_reads(gfa, reads, n_reads, rl, err, seed + len(tag) + len(preset), circular=circular)
            names, seqs = T.read_fasta(reads)
            want, _ = T.map_with_ref(gfa, names, seqs, preset)
            got, _, _ = T.map_with_engine(lib, gfa, names, seqs, preset)
            assert sum(1 for r in want if r and r["n_gc"] > 0) >= n_reads // 2, (tag, preset)
            for i, (a, b) in enumerate(zip(want, got)):
                d = T.diff_results(a, b)
                assert d is None, "%s %s read %d: %s" % (tag, preset, i, d)


def case_chain_skip(lib, workdir, n_reads=40):
    """max_lc_skip far below its default (25): the early stop of the chaining DP and of the RMQ walk -- "too many candidates in
    a row that are already on a better chain" (lchain.c:185-190, 336-343) -- fires all the time instead of almost never;
    every field against the reference, DP chaining (lr) and RMQ chaining (asm)"""
    pre, reads = os.path.join(workdir, "svc"), os.path.join(workdir, "svc.reads.fa")
    T.sim_graph(pre, 300000, 3, 19)
    T.sim_reads(pre + ".hap.fa", reads, n_reads, 12000, "ont", 47)
    names, seqs = T.read_fasta(reads)
    for preset in ("lr", "asm"):
        for skip in (1, 3):
            def tweak(mo, skip=skip):
                mo.max_lc_skip = skip
            want, _ = T.map_with_ref(pre + ".gfa", names, seqs, preset, tweak=tweak)
            got, _, _ = T.map_with_engine(lib, pre + ".gfa", names, seqs, preset, tweak=tweak)
            for i, (a, b) in enumerate(zip(want, got)):
                d = T.diff_results(a, b)
                assert d is None, "%s max_lc_skip=%d read %d: %s" % (preset, skip, i, d)


def case_switches(lib, workdir):
    """the engine's switch lab_cache=0 (graph chaining without the label table) changes the schedule, never the result: the same
    golden GAF; keys the engine does not have are refused"""
    for k in (b"pack2", b"gpu_lock", b"index_dev", b"tier_learn", b"thread_mask", b"block_warps", b"sw8", b"mb8"):
        assert lib.mgb_set_param(k, 1) == -1, k
    try:
        assert lib.mgb_set_param(b"lab_cache", 0) == 0
        case_c3(lib, workdir)
    finally:
        lib.mgb_set_param(b"lab_cache", 1)


def case_concurrent_calls(lib, workdir, n_threads=3, n_reads=90):
    """mg_map_batch() entered by several host threads at once on one index (each call takes a slot of its own; the reference's
    mg_map is re-entrant per thread buffer, minigraph.h:167-170): every thread gets what a single caller gets"""
    import ctypes as C
    import threading
    from minigraph_b200 import capi, options
    pre, reads = os.path.join(workdir, "svt"), os.path.join(workdir, "svt.reads.fa")
    T.sim_graph(pre, 400000, 4, 23)
    T.sim_reads(pre + ".hap.fa", reads, n_reads, 9000, "ont", 61)
    names, seqs = T.read_fasta(reads)
    g = lib.mgb_gfa_read((pre + ".gfa").encode())
    io, mo = options.opt_set("lr", True)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()

    def run(lo, hi, out):
        n = hi - lo
        qlens = (C.c_int * n)(*[len(x) for x in seqs[lo:hi]])
        cs, cn = (C.c_char_p * n)(*seqs[lo:hi]), (C.c_char_p * n)(*names[lo:hi])
        gcs = (C.POINTER(capi.mg_gchains_t) * n)()
        rc = lib.mg_map_batch(gi, n, qlens, cs, cn, gcs, C.byref(mo))
        out.append((lo, rc, [T.gchains_to_py(gcs[i]) for i in range(n)]))
        lib.mgb_free_batch(n, gcs)

    whole = []
    run(0, n_reads, whole)
    assert whole[0][1] == 0
    for rnd in range(2):  # the second round finds the label table warm
        parts, th = [], []
        for t in range(n_threads):
            th.append(threading.Thread(target=run, args=(n_reads * t // n_threads, n_reads * (t + 1) // n_threads, parts)))
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert len(parts) == n_threads
        for lo, rc, res in parts:
            assert rc == 0, lib.mgb_last_error()
            for i, r in enumerate(res):
                d = T.diff_results(whole[0][2][lo + i], r)
                assert d is None, "round %d read %d: %s" % (rnd, lo + i, d)
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)


def case_index_big(lib, workdir, graph_len=50000000, n_probe=40000):
    """the minimizer table of a graph whose index does not fit L2 (built by the passes of mgb_index.cuh, on the device or in the
    simulators) against the reference's (index.c:115-165): the same occurrence list -- content and order -- for tens of thousands
    of probed minimizers and for keys that are not there, and the same quantile-derived mapping options (options.c:120-134)"""
    import ctypes as C
    import random
    from minigraph_b200 import options
    pre = os.path.join(workdir, "big")
    T.sim_graph(pre, graph_len, 3, 17)
    with open(pre + ".gfa") as f:  # repeats: sixty segments once more under another name, so that many minimizers have occurrence lists
        dup = [ln.split("\t") for ln in f if ln.startswith("S\t")][100:160]
    with open(pre + ".gfa", "a") as f:
        for i, t in enumerate(dup):
            f.write("\t".join([t[0], "dup%d" % i] + t[2:]))
    ref = T.load_ref()
    rg = ref.gfa_read((pre + ".gfa").encode())
    io, rmo = options.opt_set("lr")
    rgi = ref.mg_index(rg, C.byref(io), 8, C.byref(rmo))
    assert rgi
    ref.mg_idx_get.restype = C.POINTER(C.c_uint64)
    # probes: the minimizers of random stretches of the graph (through the reference's own sketch), plus random keys
    ref.mg_sketch.restype = None
    ref.mg_sketch.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p]

    class V(C.Structure):
        _fields_ = [("n", C.c_size_t), ("m", C.c_size_t), ("a", C.POINTER(capi_u128))]
    rnd = random.Random(5)
    keys = set()
    n_seg = rg.contents.n_seg
    while len(keys) < n_probe:
        seg = rg.contents.seg[rnd.randrange(n_seg) if len(keys) % 4 else n_seg - 1 - rnd.randrange(60)]
        if seg.len < 200:
            continue
        st = rnd.randrange(seg.len - 199)
        v = V(0, 0, None)
        ref.mg_sketch(None, C.string_at(C.addressof(seg.seq.contents) + st, 200) if False else C.string_at(seg.seq, seg.len)[st:st + 200], 200, io.w, io.k, 0, C.byref(v))
        for i in range(v.n):
            keys.add(v.a[i].x >> 8)
        C.CDLL(None).free(v.a)
    keys = sorted(keys) + [rnd.getrandbits(2 * io.k) for _ in range(2000)]
    n1, n2 = C.c_int(0), C.c_int(0)
    g = lib.mgb_gfa_read((pre + ".gfa").encode())
    io2, mo = options.opt_set("lr")
    gi = lib.mg_index(g, C.byref(io2), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    assert (mo.occ_max1, mo.lc_max_occ, mo.bw_long) == (rmo.occ_max1, rmo.lc_max_occ, rmo.bw_long)
    n_multi = 0
    for k in keys:
        a, b = ref.mg_idx_get(rgi, k, C.byref(n1)), lib.mg_idx_get(gi, k, C.byref(n2))
        assert n1.value == n2.value, (hex(k), n1.value, n2.value)
        assert [a[i] for i in range(n1.value)] == [b[i] for i in range(n2.value)], hex(k)
        n_multi += n1.value > 1
    assert n_multi > 100, n_multi
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
    ref.mg_idx_destroy(rgi)
    ref.gfa_destroy(rg)


def case_multi_device(lib, workdir, devices="0,0,0", n_reads=100):
    """MGB_DEVICES: the index replicated on several devices (here the same one three times, which runs the same code), every
    mg_map_batch() cut into one contiguous part per device: the results, in input order, are what one device gives"""
    pre, reads = os.path.join(workdir, "svm"), os.path.join(workdir, "svm.reads.fa")
    T.sim_graph(pre, 300000, 3, 31)
    T.sim_reads(pre + ".hap.fa", reads, n_reads, 7000, "ont", 71)
    names, seqs = T.read_fasta(reads)
    one, _, _ = T.map_with_engine(lib, pre + ".gfa", names, seqs, "lr")
    os.environ["MGB_DEVICES"] = devices
    try:
        many, _, _ = T.map_with_engine(lib, pre + ".gfa", names, seqs, "lr")
    finally:
        del os.environ["MGB_DEVICES"]
    assert sum(1 for r in one if r and r["n_gc"] > 0) > n_reads // 2
    for i, (a, b) in enumerate(zip(one, many)):
        d = T.diff_results(a, b)
        assert d is None, "read %d: %s" % (i, d)


def case_upload_modes(lib, workdir, n_reads=80):
    """how the reads reach the device does not change what comes back: 2 bits per base (all A/C/G/T), the same with a few reads that
    hold N or lower-case letters (those travel as ASCII beside the packed ones), and the whole batch as ASCII (many such reads); every
    field against the reference, whose alignment compares raw bytes (N matches N, 'a' does not match 'A')"""
    pre, reads = os.path.join(workdir, "svu"), os.path.join(workdir, "svu.reads.fa")
    T.sim_graph(pre, 300000, 3, 29)
    T.sim_reads(pre + ".hap.fa", reads, n_reads, 6000, "ont", 67)
    names, seqs = T.read_fasta(reads)

    def spoil(s, k):
        b = bytearray(s)
        b[1000 + k] = ord("N")
        b[3000:3004] = b[3000:3004].lower()
        return bytes(b)
    few = [spoil(s, i) if i % 29 == 0 else s for i, s in enumerate(seqs)]
    many = [spoil(s, i) for i, s in enumerate(seqs)]
    for tag, ss in (("packed", seqs), ("few", few), ("many", many)):
        want, _ = T.map_with_ref(pre + ".gfa", names, ss, "lr")
        got, _, st = T.map_with_engine(lib, pre + ".gfa", names, ss, "lr")
        bases = sum(len(x) for x in ss)
        assert (st.h2d_bytes < bases // 2) == (tag in ("packed", "few")), (tag, st.h2d_bytes, bases)
        for i, (a, b) in enumerate(zip(want, got)):
            d = T.diff_results(a, b)
            assert d is None, "%s read %d: %s" % (tag, i, d)


def case_tier_routing(lib, workdir, n_reads=120):
    """the WFA tier thresholds learned from one batch route the gaps of the next: same results, and the routing did engage"""
    import ctypes as C
    from minigraph_b200 import capi, options
    hap, reads = os.path.join(workdir, "mt.hap.fa"), os.path.join(workdir, "mt.route.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, n_reads, 10000, "ont", 29)
    names, seqs = T.read_fasta(reads)
    g = lib.mgb_gfa_read(os.path.join(T.FIX, "MT.gfa").encode())
    io, mo = options.opt_set("lr", True)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    n = len(seqs)
    qlens = (C.c_int * n)(*[len(s) for s in seqs])
    cseqs, cnames = (C.c_char_p * n)(*seqs), (C.c_char_p * n)(*names)
    runs, st = [], capi.mgb_stats_t()
    for it in range(2):
        gcs = (C.POINTER(capi.mg_gchains_t) * n)()
        assert lib.mg_map_batch(gi, n, qlens, cseqs, cnames, gcs, C.byref(mo)) == 0, lib.mgb_last_error()
        runs.append([T.gchains_to_py(gcs[i]) for i in range(n)])
        lib.mgb_free_batch(n, gcs)
        lib.mgb_get_stats(gi, C.byref(st))
        if it == 0:
            assert st.skip1_len > 1 << 30  # nothing learned yet: every gap tries every tier
    assert st.skip1_len < 400 and st.skip2_len >= st.skip1_len, (st.skip1_len, st.skip2_len)
    for i, (a, b) in enumerate(zip(*runs)):
        d = T.diff_results(a, b)
        assert d is None, "read %d differs between the unrouted and the routed batch: %s" % (i, d)
    lib.mg_idx_destroy(gi)


def case_multi_segment(lib, workdir, n_frag=40):
    """fragments of 2-3 segments through mg_map_frag (paired reads): one result for the concatenated fragment, no CIGAR, same
    fields as the reference (map-algo.c:34-45,356-360,402,407,464,475)"""
    import ctypes as C
    import random
    from minigraph_b200 import capi, options
    ref = T.load_ref()
    hap, reads = os.path.join(workdir, "mt.hap.fa"), os.path.join(workdir, "mt.seg.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, n_frag, 9000, "ont", 53)
    names, seqs = T.read_fasta(reads)
    rng = random.Random(7)
    gfa = os.path.join(T.FIX, "MT.gfa")
    io, mo = options.opt_set("lr", True)
    g_e = lib.mgb_gfa_read(gfa.encode())
    gi_e = lib.mg_index(g_e, C.byref(io), 1, C.byref(mo))
    assert gi_e, lib.mgb_last_error()
    io_r, mo_r = options.opt_set("lr", True)
    g_r = ref.gfa_read(gfa.encode())
    gi_r = ref.mg_index(g_r, C.byref(io_r), 1, C.byref(mo_r))
    b_r, b_e = ref.mg_tbuf_init(), lib.mg_tbuf_init()
    for f in (lib.mg_map_frag, ref.mg_map_frag):
        f.restype = None
        f.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.POINTER(capi.mg_gchains_t)), C.c_void_p, C.c_void_p, C.c_char_p]
    n_mapped = 0
    for nm, s in zip(names, seqs):
        n_seg = rng.choice([2, 2, 3])
        cut = sorted(rng.sample(range(1500, len(s) - 1500), n_seg - 1))
        parts = [s[a:b] for a, b in zip([0] + cut, cut + [len(s)])]
        if rng.random() < 0.3:
            parts[-1] = parts[-1][:40]  # a segment too short to be sketched in chunks
        ql = (C.c_int * n_seg)(*[len(x) for x in parts])
        sq = (C.c_char_p * n_seg)(*parts)
        res = []
        for lb, gi, mo_x, tb in ((ref, gi_r, mo_r, b_r), (lib, gi_e, mo, b_e)):
            gcs = (C.POINTER(capi.mg_gchains_t) * n_seg)()
            lb.mg_map_frag(C.cast(gi, C.c_void_p), n_seg, ql, sq, gcs, tb, C.cast(C.pointer(mo_x), C.c_void_p), nm)
            assert all(not gcs[i] for i in range(1, n_seg))
            res.append(T.gchains_to_py(gcs[0]))
            lb.mg_gchain_free(gcs[0])
        d = T.diff_results(res[0], res[1])
        assert d is None, (nm, [len(x) for x in parts], d)
        if res[0] and res[0]["n_gc"] > 0:
            n_mapped += 1
    assert n_mapped >= n_frag // 2
    ref.mg_tbuf_destroy(b_r), lib.mg_tbuf_destroy(b_e)
    lib.mg_idx_destroy(gi_e), ref.mg_idx_destroy(gi_r)


def case_short_reads(lib, workdir, n_pairs=60):
    """the `sr` preset: seeds by heap merge instead of the radix sort (map-algo.c:93-150), short-read chaining gaps, read
    pairs as two-segment fragments -- every field against the reference's mg_map_frag"""
    import ctypes as C
    import random
    from minigraph_b200 import capi, options
    ref = T.load_ref()
    hap, reads = os.path.join(workdir, "mt.hap.fa"), os.path.join(workdir, "mt.sr.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, n_pairs, 500, "hifi", 61)
    names, seqs = T.read_fasta(reads)
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    rng = random.Random(3)
    gfa = os.path.join(T.FIX, "MT.gfa")
    io, mo = options.opt_set("sr", False)
    g_e = lib.mgb_gfa_read(gfa.encode())
    gi_e = lib.mg_index(g_e, C.byref(io), 1, C.byref(mo))
    assert gi_e, lib.mgb_last_error()
    io_r, mo_r = options.opt_set("sr", False)
    g_r = ref.gfa_read(gfa.encode())
    gi_r = ref.mg_index(g_r, C.byref(io_r), 1, C.byref(mo_r))
    b_r, b_e = ref.mg_tbuf_init(), lib.mg_tbuf_init()
    for f in (lib.mg_map_frag, ref.mg_map_frag):
        f.restype = None
        f.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.POINTER(capi.mg_gchains_t)), C.c_void_p, C.c_void_p, C.c_char_p]
    n_mapped = 0
    frags, per_frag = [], []
    for nm, s in zip(names, seqs):
        if rng.random() < 0.7:  # a pair: 150 bases from each end, the mate reverse-complemented
            parts = [s[:150], s[-150:].translate(comp)[::-1]]
        else:
            parts = [s[:rng.choice([100, 150, 250])]]
        frags.append((nm, parts))
        n_seg = len(parts)
        ql = (C.c_int * n_seg)(*[len(x) for x in parts])
        sq = (C.c_char_p * n_seg)(*parts)
        res = []
        for lb, gi, mo_x, tb in ((ref, gi_r, mo_r, b_r), (lib, gi_e, mo, b_e)):
            gcs = (C.POINTER(capi.mg_gchains_t) * n_seg)()
            lb.mg_map_frag(C.cast(gi, C.c_void_p), n_seg, ql, sq, gcs, tb, C.cast(C.pointer(mo_x), C.c_void_p), nm)
            res.append(T.gchains_to_py(gcs[0]))
            lb.mg_gchain_free(gcs[0])
        d = T.diff_results(res[0], res[1])
        assert d is None, (nm, [len(x) for x in parts], d)
        per_frag.append(res[0])
        if res[0] and res[0]["n_gc"] > 0:
            n_mapped += 1
    assert n_mapped >= n_pairs // 2, n_mapped
    # the same fragments in one call of the batch entry point
    flat = [x for _, parts in frags for x in parts]
    n_tot = len(flat)
    nseg = (C.c_int * len(frags))(*[len(parts) for _, parts in frags])
    ql = (C.c_int * n_tot)(*[len(x) for x in flat])
    sq = (C.c_char_p * n_tot)(*flat)
    nms = (C.c_char_p * len(frags))(*[nm for nm, _ in frags])
    gcs = (C.POINTER(capi.mg_gchains_t) * n_tot)()
    assert lib.mg_map_batch_frag(gi_e, len(frags), nseg, ql, sq, nms, gcs, C.byref(mo)) == 0, lib.mgb_last_error()
    off = 0
    for f, (nm, parts) in enumerate(frags):
        assert all(not gcs[off + j] for j in range(1, len(parts)))
        d = T.diff_results(per_frag[f], T.gchains_to_py(gcs[off]))
        assert d is None, (nm, d)
        off += len(parts)
    lib.mgb_free_batch(n_tot, gcs)
    ref.mg_tbuf_destroy(b_r), lib.mg_tbuf_destroy(b_e)
    lib.mg_idx_destroy(gi_e), ref.mg_idx_destroy(gi_r)


def case_no_diag(lib, workdir):
    """MG_M_NO_DIAG (-D): a read that carries the name of the sequence it comes from loses the seeds on its own diagonal
    (map-algo.c:167-178): same result fields as the reference, for a full self copy, a prefix, an inner piece and a stranger"""
    fa = os.path.join(T.FIX, "MT-human.fa")
    gname, hs = T.read_fasta(fa)
    full = hs[0]
    names = [gname[0], gname[0], gname[0], b"someone_else", gname[0] + b"x"]
    seqs = [full, full[:6000], full[3000:9000], full[:6000], full[:6000]]
    import minigraph_b200.options as options_mod
    orig = options_mod.opt_set

    def with_flag(preset=None, cigar=True):
        io, mo = orig(preset, cigar)
        mo.flag |= 0x400000  # MG_M_NO_DIAG (minigraph.h:27)
        return io, mo
    options_mod.opt_set = with_flag
    T.options.opt_set = with_flag
    try:
        got, _, _ = T.map_with_engine(lib, fa, names, seqs, "asm")
        want, _ = T.map_with_ref(fa, names, seqs, "asm")
    finally:
        options_mod.opt_set = orig
        T.options.opt_set = orig
    for i, (a, b) in enumerate(zip(want, got)):
        d = T.diff_results(a, b)
        assert d is None, (i, d)
    plain, _ = T.map_with_ref(fa, names[:2], seqs[:2], "asm")
    assert T.diff_results(plain[1], want[1]) is not None  # the flag did change something for the self-named prefix


def _ref_wfa_exact(ts, qs):
    """the reference's exact WFA with traceback and no cap (miniwfa.c:380-435 through mwf_wfa_exact): score, CIGAR, n_iter"""
    import ctypes as C
    ref = T.load_ref()
    mwf_opt_t, mwf_rst_t = _mwf_types()
    opt = mwf_opt_t()
    ref.mwf_opt_init(C.byref(opt))
    opt.flag |= 1
    opt.step, opt.max_iter = 0, 10 ** 8
    rst = mwf_rst_t()
    ref.mwf_wfa_exact(None, C.byref(opt), len(ts), ts, len(qs), qs, C.byref(rst))
    return rst.s, [rst.cigar[i] for i in range(rst.n_cigar)], rst.n_iter


# the two on-chip tiers: (W diagonals in the ring, longest side, traceback bytes in shared memory or 0)
WFA_TIERS = {1: (64, 256, 4096), 2: (256, 1024, 0)}


def wfa_tier_gaps(tier, rng, scale=1):
    """gaps drawn around every limit of an on-chip tier, as (tag, target, query) byte strings"""
    W, maxlen, tbcap = WFA_TIERS[tier]

    def rnd(n, alpha="ACGT"):
        return "".join(rng.choices(alpha, k=n))

    def noisy(s, rate):
        out = []
        for c in s:
            u = rng.random()
            if u < rate * 0.5:
                out.append(rng.choice("ACGT"))
            elif u < rate * 0.75:
                continue
            elif u < rate:
                out += [c, rng.choice("ACGT")]
            else:
                out.append(c)
        return "".join(out) or rng.choice("ACGT")
    gaps = []
    # lengths at the tier's limit and 1 past it, and single bases (jobs never have an empty side)
    for L in sorted({1, 255, 256, 257, maxlen - 1, maxlen, maxlen + 1}):
        t = rnd(L)
        gaps += [("len", t, t), ("len", t, noisy(t, 0.02)), ("len", noisy(t, 0.03), t), ("len", t[:max(1, L - 3)], t),
                 ("len", t, t[2:] or t), ("len", t[:1], t[:1]), ("len", t[:1], rnd(1)), ("len", rnd(3), t[:1])]
    # windows that span the matrix: tl + ql + 1 just below, at and past the W - 2 diagonals the ring can hold
    for span in range(W - 4, W + 1):
        for _ in range(6 * scale):
            tl = rng.randint(max(1, span // 2 - 8), span // 2 + 8)
            ql = span - 1 - tl
            t = rnd(tl)
            gaps.append(("window", t, rnd(ql)))
            gaps.append(("window", t, (noisy(t, rng.choice([0.1, 0.2, 0.35])) + rnd(ql))[:ql]))
    # scores just below and at 255, found by asking the reference (tier 2; tier 1 cannot reach them in a window of 62 diagonals)
    want_s = []
    for _ in range(3000 * scale if tier == 2 else 0):
        if len(want_s) >= 24 * scale:
            break
        n = rng.randint(90, 126)
        t = rnd(n)
        q = rnd(rng.randint(n - 6, min(253 - n, n + 6))) if rng.random() < 0.5 else noisy(t, rng.choice([0.45, 0.6]))[:253 - n]
        s, _, _ = _ref_wfa_exact(t.encode(), q.encode())
        if 236 <= s <= 274:
            want_s.append(("score", t, q))
    gaps += want_s
    # the most traceback bytes a window that fits tier 1 can take: pairs without a single match that span the whole window
    for _ in range(12 * scale if tbcap else 0):
        n = rng.randint(20, 41)
        gaps.append(("tbcap", rnd(n, "AC"), rnd(rng.choice([59, 60, 61]) - n, "GT")))
    # identical pairs (the corner reached at score 0, a hit without extension), prefixes, low-complexity pairs (many ties),
    # and N and lower-case bytes, which the alignment compares as they are
    for n in (1, 2, 5, 40, 200):
        t = rnd(n)
        gaps += [("ident", t, t), ("prefix", t, t + rnd(3)), ("prefix", t + rnd(5), t)]
    for _ in range(8 * scale):
        n = rng.choice([10, 25, 60, 120, 300])
        t = rnd(n, "AC")
        gaps += [("ac", t, noisy(t, 0.1).replace("G", "A").replace("T", "C")), ("ac", t, rnd(max(1, n - 5), "AC"))]
        t = rnd(n)
        b = list(noisy(t, 0.05))
        for j in rng.sample(range(len(b)), min(len(b), 3)):
            b[j] = rng.choice("Nacgtn")
        gaps += [("nlower", t, "".join(b)), ("nlower", t.lower(), t), ("nlower", "N" * n, "N" * (n + 1))]
    return [(tag, t.encode(), q.encode()) for tag, t, q in gaps]


def run_wfa_tier(lib, tier, gaps):
    """all gaps in one call of the tier hook: [(rc, score, n_iter, cigar)] in input order"""
    import ctypes as C
    n = len(gaps)
    ts, qs = b"".join(t for _, t, _ in gaps), b"".join(q for _, _, q in gaps)
    t_off, q_off, tl, ql = (C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int32 * n)(), (C.c_int32 * n)()
    a = b = 0
    for i, (_, t, q) in enumerate(gaps):
        t_off[i], q_off[i], tl[i], ql[i] = a, b, len(t), len(q)
        a, b = a + len(t), b + len(q)
    cap = max(len(t) + len(q) for _, t, q in gaps) + 2
    out, cig = (C.c_int64 * (4 * n))(), (C.c_uint32 * (n * cap))()
    assert lib.mgb_test_wfa_tier(tier, n, ts, t_off, tl, qs, q_off, ql, out, cig, cap) == 0, lib.mgb_last_error()
    return [(out[4 * i], out[4 * i + 1], out[4 * i + 2], list(cig[i * cap:i * cap + out[4 * i + 3]])) for i in range(n)]


def case_wfa_tier_edges(lib, tier, scale=1, seed=None):
    """one on-chip WFA tier (wfa_smem, mgb_wfa_tiers.cuh: no bounds checks, 16-bit cells) on its own, against the reference's
    mwf_wfa_exact, with gaps drawn around each of its limits.  Exact when accepted: a gap the tier aligns has the reference's
    score, CIGAR and n_iter.  Must fit when provably in bounds: the window grows by at most one diagonal per side and score, so
    a gap with both sides within the tier's length, a score below 255, min(2s+1, tl+ql+1) + 2 <= W and (tier 1) no more
    traceback bytes than fit -- the reference's n_iter counts exactly those bytes -- may not be handed on to the next tier.  Must
    give up past a limit that cannot be met: longer sides, score 255 or more, too many traceback bytes.  And every limit is met
    in both directions: some gaps are aligned just inside it and some refused just past it -- except tier 1's traceback bytes,
    which a window of 62 diagonals cannot fill (the gaps that come closest are aligned)."""
    import random
    W, maxlen, tbcap = WFA_TIERS[tier]
    rng = random.Random(seed if seed is not None else 7 + tier)
    gaps = wfa_tier_gaps(tier, rng, scale)
    got = run_wfa_tier(lib, tier, gaps)
    hits = {}
    for i, ((tag, t, q), (rc, s, n_iter, cigar)) in enumerate(zip(gaps, got)):
        tl, ql = len(t), len(q)
        rs, rcig, rn = _ref_wfa_exact(t, q)
        what = "tier %d gap %d (%s, tl=%d ql=%d, reference score %d n_iter %d): " % (tier, i, tag, tl, ql, rs, rn)
        assert rc in (0, 1), what + "rc %d" % rc
        if rc == 0:
            assert (s, cigar, n_iter) == (rs, rcig, rn), what + "score %d n_iter %d, CIGAR %s" % (s, n_iter, "same" if cigar == rcig else "differs")
        len_ok, s_ok = max(tl, ql) <= maxlen, rs <= 254
        w_need = min(2 * rs + 1, tl + ql + 1) + 2
        tb_ok = tbcap == 0 or rn <= tbcap
        if len_ok and s_ok and w_need <= W and tb_ok:
            assert rc == 0, what + "provably fits the tier (window of at most %d of %d columns) but was refused" % (w_need, W)
        if not len_ok or not s_ok or not tb_ok:
            assert rc == 1, what + "cannot fit the tier but was accepted"
        inside, past = [], []
        (inside if max(tl, ql) == maxlen else past if max(tl, ql) == maxlen + 1 else []).append("length")
        if len_ok and s_ok and tb_ok:
            (inside if W - 1 <= w_need <= W else past if W < w_need <= W + 2 else []).append("window")
        if tier == 2 and len_ok and w_need <= W:
            (inside if 240 <= rs <= 254 else past if 255 <= rs <= 270 else []).append("score")
        if tbcap and w_need <= W:
            # (tier 1) the window limit comes first: a gap whose window fits takes fewer than 4000 traceback bytes, so the
            # capacity of 4096 never decides and nothing can be refused just past it; what is checked is that it is enough
            assert rn <= tbcap, what + "fits the window but not the traceback bytes"
            if rn >= tbcap - 300:
                inside.append("traceback bytes")
        for lim in inside:
            hits.setdefault(lim, [0, 0])[0] += rc == 0
        for lim in past:
            hits.setdefault(lim, [0, 0])[1] += rc == 1
    for lim in ["length", "window", "score"] if tier == 2 else ["length", "window", "traceback bytes"]:
        a, r = hits.get(lim, [0, 0])
        both = lim != "traceback bytes"
        assert a > 0 and (r > 0 or not both), "tier %d: the %s limit was not met in both directions (%d gaps aligned just inside it, %d refused just past it)" % (tier, lim, a, r)
    return hits


def case_wfa_tier_rejects_empty(lib):
    """a gap with an empty side is refused before anything runs (real jobs never have one: galign.c:97-99)"""
    import ctypes as C
    for tier in (1, 2):
        for tl, ql in ((0, 5), (5, 0), (0, 0)):
            one = lambda x: (C.c_int64 * 1)(x)  # noqa: E731
            out, cig = (C.c_int64 * 4)(-7, -7, -7, -7), (C.c_uint32 * 16)()
            rc = lib.mgb_test_wfa_tier(tier, 1, b"ACGTA", one(0), (C.c_int32 * 1)(tl), b"ACGTA", one(0), (C.c_int32 * 1)(ql), out, cig, 16)
            assert rc < 0 and list(out) == [-7] * 4, (tier, tl, ql, rc)
    out, cig = (C.c_int64 * 4)(), (C.c_uint32 * 16)()
    assert lib.mgb_test_wfa_tier(3, 1, b"A", (C.c_int64 * 1)(0), (C.c_int32 * 1)(1), b"A", (C.c_int64 * 1)(0), (C.c_int32 * 1)(1), out, cig, 16) < 0


_ged = None


def _gfa_ed_types():
    """ctypes view of gfa-priv.h:73-89 (gfa_edopt_t, gfa_edrst_t) and the prototypes of the reference's graph edit distance"""
    global _ged
    if _ged is None:
        import ctypes as C
        ref = T.load_ref()

        class gfa_edopt_t(C.Structure):
            _fields_ = [("traceback", C.c_int32), ("bw_dyn", C.c_int32), ("max_lag", C.c_int32), ("max_chk", C.c_int32),
                        ("s_term", C.c_int32), ("i_term", C.c_int64)]

        class gfa_edrst_t(C.Structure):
            _fields_ = [("s", C.c_int32), ("end_v", C.c_uint32), ("end_off", C.c_int32), ("wlen", C.c_int32), ("n_end", C.c_int32),
                        ("nv", C.c_int32), ("n_iter", C.c_int64), ("v", C.POINTER(C.c_int32))]
        ref.gfa_edopt_init.restype = None
        ref.gfa_edopt_init.argtypes = [C.POINTER(gfa_edopt_t)]
        ref.gfa_edseq_init.restype = C.c_void_p
        ref.gfa_edseq_init.argtypes = [C.POINTER(capi.gfa_t)]
        ref.gfa_edseq_destroy.restype = None
        ref.gfa_edseq_destroy.argtypes = [C.c_int32, C.c_void_p]
        ref.gfa_ed_init.restype = C.c_void_p
        ref.gfa_ed_init.argtypes = [C.c_void_p, C.POINTER(gfa_edopt_t), C.POINTER(capi.gfa_t), C.c_void_p, C.c_int32, C.c_char_p, C.c_uint32, C.c_int32]
        ref.gfa_ed_step.restype = None
        ref.gfa_ed_step.argtypes = [C.c_void_p, C.c_uint32, C.c_int32, C.c_int32, C.POINTER(gfa_edrst_t)]
        ref.gfa_ed_destroy.restype = None
        ref.gfa_ed_destroy.argtypes = [C.c_void_p]
        _ged = (gfa_edopt_t, gfa_edrst_t)
    return _ged


def _ref_bridge(g, es, q, v0, off0, v1, off1, max_ed, max_lag=None):
    """gchain1.c:349-381 bridge_gwfa: gfa_ed_init + gfa_ed_step of the reference; (s, end_v, end_off, nv, walk, n_iter)"""
    import ctypes as C
    ref = T.load_ref()
    gfa_edopt_t, gfa_edrst_t = _gfa_ed_types()
    opt = gfa_edopt_t()
    ref.gfa_edopt_init(C.byref(opt))
    opt.traceback, opt.max_chk, opt.bw_dyn, opt.max_lag = 1, 1000, 1000, max_ed // 2 if max_lag is None else max_lag
    opt.i_term = 500000000
    r = gfa_edrst_t()
    z = ref.gfa_ed_init(None, C.byref(opt), g, es, len(q), q, v0, off0)
    ref.gfa_ed_step(z, v1, off1, max_ed, C.byref(r))
    ref.gfa_ed_destroy(z)
    walk = [r.v[i] for i in range(r.nv)] if r.s >= 0 else []
    if r.s >= 0:
        C.CDLL(None).free(r.v)
    return r.s, r.end_v, r.end_off, len(walk), walk, r.n_iter


class _Graph:
    """segments and arcs of a GFA as the tests draw walks on it (vertex v = segment << 1 | reverse strand)"""

    def __init__(self, fn):
        self.names, self.seq, self.out = [], [], {}
        ids = {}
        for ln in open(fn):
            t = ln.rstrip("\n").split("\t")
            if t[0] == "S":
                ids[t[1]] = len(self.names)
                self.names.append(t[1])
                self.seq.append(t[2].upper())
        for ln in open(fn):
            t = ln.rstrip("\n").split("\t")
            if t[0] == "L":
                v, w = ids[t[1]] << 1 | (t[2] == "-"), ids[t[3]] << 1 | (t[4] == "-")
                self.out.setdefault(v, []).append(w)
                self.out.setdefault(w ^ 1, []).append(v ^ 1)

    def vseq(self, v):
        s = self.seq[v >> 1]
        return s[::-1].translate(str.maketrans("ACGTN", "TGCAN")) if v & 1 else s

    def walk(self, rng, v, min_len):
        """a random walk from v until it holds min_len bases (or meets a dead end)"""
        w, n = [v], len(self.seq[v >> 1])
        while n < min_len and self.out.get(w[-1]):
            w.append(rng.choice(self.out[w[-1]]))
            n += len(self.seq[w[-1] >> 1])
        return w


def _write_gfa(fn, segs, links):
    with open(fn, "w") as f:
        for name, s in segs:
            f.write("S\t%s\t%s\n" % (name, s))
        for a, sa, b, sb in links:
            f.write("L\t%s\t%s\t%s\t%s\t0M\n" % (a, sa, b, sb))


def _bridge_graphs(workdir, rng):
    """small GFAs for the situations the bridging alignment has to get right: {tag: path}"""
    def rnd(n):
        return "".join(rng.choices("ACGT", k=n))
    out = {}
    segs = [("c%d" % i, rnd(1)) for i in range(80)]  # a chain of 1-bp segments between two longer ones
    segs = [("cL", rnd(30))] + segs + [("cR", rnd(30))]
    out["chain1bp"] = (segs, [(segs[i][0], "+", segs[i + 1][0], "+") for i in range(len(segs) - 1)])
    alle = [rnd(rng.randint(4, 9)) for _ in range(30)]
    alle += [alle[i] for i in range(5)] + [alle[i][:-1] for i in range(5, 10)]  # alleles twice, and alleles one base shorter
    segs = [("fA", rnd(40))] + [("f%d" % i, a) for i, a in enumerate(alle)] + [("fB", rnd(40))]
    out["fanout40"] = (segs, [("fA", "+", "f%d" % i, "+") for i in range(40)] + [("f%d" % i, "+", "fB", "+") for i in range(40)])
    segs, links = [("w0", rnd(20))], []  # eight 40-way bubbles in a row: wavefronts of more than max_chk diagonals (pruning)
    for b in range(8):
        for i in range(40):
            segs.append(("w%d_%d" % (b, i), rnd(rng.randint(3, 12)) if i % 4 else alle[i]))
            links += [("w%d" % b, "+", "w%d_%d" % (b, i), "+"), ("w%d_%d" % (b, i), "+", "w%d" % (b + 1), "+")]
        segs.append(("w%d" % (b + 1), rnd(20)))
    out["wide"] = (segs, links)
    segs = [(n, rnd(rng.randint(5, 40))) for n in "ABCDEFGHIJ"]  # nested bubbles
    out["nested"] = (segs, [("A", "+", "B", "+"), ("A", "+", "F", "+"), ("B", "+", "C", "+"), ("B", "+", "D", "+"), ("C", "+", "E", "+"),
                            ("D", "+", "E", "+"), ("E", "+", "G", "+"), ("F", "+", "G", "+"), ("G", "+", "H", "+"), ("G", "+", "I", "+"),
                            ("H", "+", "J", "+"), ("I", "+", "J", "+"), ("B", "+", "E", "+")])
    segs = [("sA", rnd(25)), ("sL", rnd(6)), ("sB", rnd(9)), ("sC", rnd(7)), ("sD", rnd(30)), ("sZ", rnd(50))]  # loops, strand switches
    out["cycles"] = (segs, [("sA", "+", "sL", "+"), ("sL", "+", "sL", "+"), ("sL", "+", "sB", "+"), ("sB", "+", "sC", "+"), ("sC", "+", "sB", "+"),
                            ("sC", "+", "sD", "-"), ("sD", "-", "sA", "-"), ("sB", "-", "sD", "+")])  # sZ: not connected
    paths = {}
    for tag, (segs, links) in out.items():
        paths[tag] = os.path.join(workdir, "bridge_%s.gfa" % tag)
        _write_gfa(paths[tag], segs, links)
    return paths


def _ont_errors(rng, s, rate):
    out = []
    for c in s:
        u = rng.random()
        if u < rate * 0.4:
            out.append(rng.choice("ACGT"))
        elif u < rate * 0.7:
            continue
        elif u < rate:
            out += [c, rng.choice("ACGT")]
        else:
            out.append(c)
    return "".join(out)


def _draw_bridges(G, rng, n, lens, rates, max_eds):
    """n bridges along random walks of G: (query, v0, off0, v1, off1, max_ed, walk)"""
    out = []
    n_v = 2 * len(G.seq)
    while len(out) < n:
        v = rng.randrange(n_v)
        L = rng.choice(lens)
        w = G.walk(rng, v, L)
        path = "".join(G.vseq(x) for x in w)
        off0 = rng.randrange(len(G.seq[v >> 1])) if rng.random() < 0.7 else len(G.seq[v >> 1]) - 1
        last = len(G.seq[w[-1] >> 1])
        off1 = rng.randrange(last) if len(w) > 1 else rng.randrange(off0, last)
        q = path[off0:len(path) - last + off1 + 1]
        q = _ont_errors(rng, q, rng.choice(rates)) or q
        if q:
            out.append((q.encode(), v, off0, w[-1], off1, rng.choice(max_eds), w))
    return out


def run_gwfa(lib, gi, mode, bridges, walk_cap=4096):
    """all bridges in one call of the bridging hook: [(rc, s, end_v, end_off, nv, walk, n_iter)] in input order"""
    import ctypes as C
    n = len(bridges)
    q = b"".join(b[0] for b in bridges)
    I64, I32, U32 = C.c_int64 * n, C.c_int32 * n, C.c_uint32 * n
    q_off, ql = I64(), I32(*[len(b[0]) for b in bridges])
    a = 0
    for i, b in enumerate(bridges):
        q_off[i], a = a, a + len(b[0])
    v0, off0, v1, off1, med = U32(*[b[1] for b in bridges]), I32(*[b[2] for b in bridges]), U32(*[b[3] for b in bridges]), I32(*[b[4] for b in bridges]), I32(*[b[5] for b in bridges])
    out, walk = (C.c_int64 * (6 * n))(), (C.c_int32 * (n * walk_cap))()
    assert lib.mgb_test_gwfa(gi, mode, n, q, q_off, ql, v0, off0, v1, off1, med, out, walk, walk_cap) == 0, lib.mgb_last_error()
    res = []
    for i in range(n):
        o = out[6 * i:6 * i + 6]
        res.append((o[0], o[1], o[2], o[3], o[4], list(walk[i * walk_cap:i * walk_cap + o[4]]), o[5]))
    return res


def case_gwfa_bridges(lib, workdir, scale=1, seed=13, modes=(0, 1)):
    """the bridging alignment between two linear chains (gchain1.c:349-381: gfa_ed_init + gfa_ed_step with bridge_gwfa's options)
    on its own: the warp-wide gwf_align_w of k_gwfa (mode 0) and the sequential gwf_align of graph chaining (mode 1) against the
    reference's gfa_ed on its own gfa_read of the same file -- score, end vertex and offset, walk and n_iter.  Graphs: a chain of
    1-bp segments, a vertex with 40 out-arcs (more than a warp has lanes) whose alleles repeat (walks of equal cost), eight 40-way
    bubbles in a row (wavefronts past max_chk: pruning with max_lag), nested bubbles, a self-loop, a 2-cycle and arcs that switch
    strand, a segment nothing reaches, and an mgsim SV graph with queries from a few bases to 5 kb with ONT-like errors; plus
    random queries and small max_ed (the s_term stop)."""
    import ctypes as C
    import random
    from minigraph_b200 import options
    ref = T.load_ref()
    rng = random.Random(seed)
    paths = _bridge_graphs(workdir, rng)
    sv = os.path.join(workdir, "bridge_sv")
    T.sim_graph(sv, 200000, 3, seed)
    paths["sv"] = sv + ".gfa"
    plan = {"chain1bp": (30, [40, 120], [0, 0.05, 0.15], [5, 30, 200]), "fanout40": (40, [60, 90], [0, 0.03, 0.1], [4, 30, 200]),
            "wide": (12, [150, 250], [0.1, 0.2], [60, 120]), "nested": (30, [30, 100, 200], [0, 0.05, 0.15], [3, 30, 200]),
            "cycles": (40, [20, 80, 200], [0, 0.05, 0.15], [2, 20, 200]), "sv": (30, [4, 300, 1500, 5000], [0.02, 0.08], [5, 100, 1000, 3000])}
    seen, n_ok, n_all = {}, 0, 0
    for tag, fn in paths.items():
        n, lens, rates, max_eds = plan[tag]
        G = _Graph(fn)
        bridges = _draw_bridges(G, rng, max(4, n * scale // 4), lens, rates, max_eds)
        if tag == "cycles":
            sA, sZ, sL = G.names.index("sA") << 1, G.names.index("sZ") << 1, G.names.index("sL") << 1
            bridges += [(G.seq[sZ >> 1][:20].encode(), sA, 3, sZ, 19, 100, None),  # nothing reaches sZ
                        (G.seq[sA >> 1][5:15].encode(), sA, 5, sA, 14, 50, [sA]),  # the same vertex, off1 after off0
                        ((G.seq[sA >> 1][20:] + G.vseq(sL) * 3 + G.vseq(sL)[:2]).encode(), sA, 20, sL, 1, 60, None),  # round the self-loop
                        (G.vseq(sL)[4:].encode() + G.vseq(sL).encode() + G.vseq(sL)[:2].encode(), sL, 4, sL, 1, 40, None),  # off1 before off0 on one vertex
                        (b"ACGTTGCA" * 3, sA, 24, sA ^ 1, 3, 200, None)]  # from the last base of a segment to its other strand
        if tag == "fanout40":  # through an allele that occurs twice: two walks of the same cost, the reference keeps the first
            fA, fB = G.names.index("fA"), G.names.index("fB")
            for i in range(10):  # the allele as it is, or with its last base changed: one mismatch, or one insertion after the shorter allele
                a = G.seq[i + 1] if i < 5 else G.seq[i + 1][:-1] + "ACGT"["CGTA".index(G.seq[i + 1][-1])]
                bridges.append(((G.seq[fA][-10:] + a + G.seq[fB][:10]).encode(), fA << 1, len(G.seq[fA]) - 10, fB << 1, 9, 30, None))
        bridges += [(bytes(rng.choices(b"ACGT", k=rng.choice([1, 3, 40, 400]))), rng.randrange(2 * len(G.seq)), 0, rng.randrange(2 * len(G.seq)), 0,
                     rng.choice([3, 50, 500]), None) for _ in range(max(2, 6 * scale // 4))]  # random queries
        g = ref.gfa_read(fn.encode())
        es = ref.gfa_edseq_init(g)
        want = [_ref_bridge(g, es, *b[:6]) for b in bridges]
        pruned = [b[5] >= 60 and _ref_bridge(g, es, *b[:6], max_lag=-1) != w for b, w in zip(bridges, want)] if tag == "wide" else [False] * len(bridges)
        ref.gfa_edseq_destroy(g.contents.n_seg, es)
        ref.gfa_destroy(g)
        eg = lib.mgb_gfa_read(fn.encode())
        io, mo = options.opt_set("lr", True)
        gi = lib.mg_index(eg, C.byref(io), 1, C.byref(mo))
        assert gi, lib.mgb_last_error()
        for mode in modes:
            got = run_gwfa(lib, gi, mode, bridges)
            for i, (b, w, r) in enumerate(zip(bridges, want, got)):
                what = "%s bridge %d (mode %d, ql=%d, %d:%d -> %d:%d, max_ed %d)" % (tag, i, mode, len(b[0]), b[1], b[2], b[3], b[4], b[5])
                assert r[0] == 0, what + ": rc %d" % r[0]
                rs, rv, ro, rn, rw, ri = w
                assert (r[1], r[2], r[3], r[6]) == (rs, rv, ro, ri), what + ": s/end_v/end_off/n_iter %r, the reference %r" % ((r[1], r[2], r[3], r[6]), (rs, rv, ro, ri))
                assert (r[4], r[5]) == (rn, rw), what + ": walk %r, the reference %r" % (r[5][:12], rw[:12])
        lib.mg_idx_destroy(gi)
        lib.mgb_gfa_destroy(eg)
        for b, w, p in zip(bridges, want, pruned):
            s, walk = w[0], w[4]
            n_all += 1
            n_ok += s >= 0
            marks = {tag + (" aligned" if s >= 0 else " not aligned")}
            if s >= 0 and len(set(walk)) < len(walk):
                marks.add("walk through a cycle")
            if s >= 0 and len({x & 1 for x in walk}) == 2:
                marks.add("walk switching strand")
            if s >= 0 and any(x == y for x, y in zip(walk, walk[1:])):
                marks.add("self-loop")
            if b[1] == b[3]:
                marks.add("v0 == v1, off1 %s off0" % ("after" if b[4] > b[2] else "before"))
            if b[2] == len(G.seq[b[1] >> 1]) - 1:
                marks.add("off0 on the last base")
            if s < 0 and b[6] is not None:
                marks.add("stopped at max_ed (s_term)")
            if p:
                marks.add("pruned")
            if tag == "fanout40" and s >= 0 and any(G.seq[x >> 1] in G.seq[:x >> 1] + G.seq[(x >> 1) + 1:] or G.seq[x >> 1][:-1] in G.seq for x in walk[1:-1]):
                marks.add("equal-cost walks")
            if s >= 0 and len(b[0]) >= 4000:
                marks.add("query of 4 kb or more")
            if s >= 0 and len(b[0]) <= 5:
                marks.add("query of 5 bases or fewer")
            for m in marks:
                seen[m] = seen.get(m, 0) + 1
    assert n_ok >= n_all // 2, "only %d of %d bridges aligned" % (n_ok, n_all)
    need = ["chain1bp aligned", "fanout40 aligned", "wide aligned", "nested aligned", "cycles aligned", "sv aligned", "cycles not aligned",
            "walk through a cycle", "walk switching strand", "self-loop", "v0 == v1, off1 after off0", "v0 == v1, off1 before off0",
            "off0 on the last base", "stopped at max_ed (s_term)", "pruned", "equal-cost walks", "query of 4 kb or more", "query of 5 bases or fewer"]
    missing = [m for m in need if not seen.get(m)]
    assert not missing, "situations that did not occur: %s (seen: %r)" % (missing, seen)
    return seen


def case_gwfa_rejects_bad_input(lib, workdir):
    """an empty query or an end outside the graph is refused before anything runs"""
    import ctypes as C
    from minigraph_b200 import options
    fn = os.path.join(workdir, "bridge_tiny.gfa")
    _write_gfa(fn, [("a", "ACGTACGTAC"), ("b", "TTGCA")], [("a", "+", "b", "+")])
    g = lib.mgb_gfa_read(fn.encode())
    io, mo = options.opt_set("lr", True)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    for q, v0, off0, v1, off1 in ((b"", 0, 0, 2, 1), (b"ACG", 0, 10, 2, 1), (b"ACG", 0, 0, 2, 5), (b"ACG", 4, 0, 2, 1), (b"ACG", 0, -1, 2, 1)):
        out, walk = (C.c_int64 * 6)(*[-7] * 6), (C.c_int32 * 4)()
        one32, oneu = (lambda x: (C.c_int32 * 1)(x)), (lambda x: (C.c_uint32 * 1)(x))
        rc = lib.mgb_test_gwfa(gi, 0, 1, q, (C.c_int64 * 1)(0), one32(len(q)), oneu(v0), one32(off0), oneu(v1), one32(off1), one32(10), out, walk, 4)
        assert rc < 0 and list(out) == [-7] * 6, (q, v0, off0, v1, off1, rc)
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
