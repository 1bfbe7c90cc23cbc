"""GAF text formatted on the device (mgb_map_batch_gaf): cases shared by the CPU (simulator) and GPU test modules, and the read
pairs of the GAF-option golden files (`python3 tests/gafcases.py pairs reads.fa r1.fa r2.fa`, tests/golden/make_golden_gaf.sh)."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mgtest as T  # noqa: E402
from minigraph_b200 import capi, options  # noqa: E402

# minigraph.h:12-29
FRAG_MERGE, VERTEX_COOR, PRINT_2ND, CAL_COV, INDEPEND_SEG = 0x80, 0x800, 0x2000, 0x4000, 0x20000
SHOW_UNMAP, NO_COMP_PATH, WRITE_LCHAIN, WRITE_MZ = 0x100000, 0x200000, 0x800000, 0x1000000
# --secondary=yes --show-unmap=yes -S --write-mz
X = PRINT_2ND | SHOW_UNMAP | WRITE_LCHAIN | WRITE_MZ

G = os.path.join(T.REPO, "tests", "golden")
EXISTING = [  # (golden, graph, reads, preset)
    ("c1_MT_orangA.lr.gaf", "MT", "orangA", "lr"), ("c1_MT_chimp.lr.gaf", "MT", "chimp", "lr"),
    ("c2_MT_24x10k_ont_s11.lr.gaf", "MT", "c2", "lr"), ("c3_sv300k_h3_s7_24x15k_ont_s5.lr.gaf", "sv", "c3", "lr"),
    ("c4_MThuman_12x20k_hifi_s13.asm.gaf", "MTh", "c4", "asm"), ("L2_MT_240x10k_ont_s111.lr.gaf.gz", "MT", "L2", "lr"),
    ("L3_sv1m_h8_s7_240x15k_ont_s105.lr.gaf.gz", "svL", "L3", "lr"), ("L4_MThuman_200x20k_hifi_s113.asm.gaf.gz", "MTh", "L4", "asm"),
]
FLAGGED = [  # (golden, inputs, cigar, flag bits beyond the preset's)
    ("f1_sv_edge.lr.2nd_unmap_S_mz.gaf.gz", "sv_edge", True, X),
    ("f2_sv_edge.lr.2nd_unmap_S_mz_vc.gaf.gz", "sv_edge", True, X | VERTEX_COOR),
    ("f3_sv_edge.lr.2nd_unmap_S_mz_nocomp.gaf.gz", "sv_edge", True, X | NO_COMP_PATH),
    ("f4_sv_edge.lr_nocigar.2nd_unmap_S_mz.gaf", "sv_edge", False, X),
    ("f6_stable_40x2500_hifi_s17.lr.2nd_unmap_S_mz.gaf", "stable", True, X),
    ("f7_stable_40x2500_hifi_s17.lr.2nd_unmap_S_mz_nocomp.gaf", "stable", True, X | NO_COMP_PATH),
]
PAIRS = "f5_MT_60pairs_hifi_s61.sr.gaf"


def golden(name):
    import gzip
    op = gzip.open if name.endswith(".gz") else open
    with op(os.path.join(G, name), "rb") as f:
        return f.read()


def revcomp(s):
    return s.translate(bytes.maketrans(b"ACGTN", b"TGCAN"))[::-1]


def split_pairs(fa, r1, r2):
    """read pairs from simulated fragments: 150 bases from each end, the second mate reverse-complemented, names /1 and /2"""
    names, seqs = T.read_fasta(fa)
    T.write_fasta(r1, [n + b"/1" for n in names], [s[:150] for s in seqs])
    T.write_fasta(r2, [n + b"/2" for n in names], [revcomp(s[-150:]) for s in seqs])


def inputs(kind, workdir):
    """(graph, read names, read sequences) of the golden files"""
    mt = os.path.join(T.FIX, "MT.gfa")
    if kind in ("orangA", "chimp"):
        return (mt,) + T.read_fasta(os.path.join(T.FIX, "MT-%s.fa" % kind))
    if kind in ("c2", "L2"):
        hap, reads = os.path.join(workdir, "gmt.hap.fa"), os.path.join(workdir, "g%s.fa" % kind)
        T.sim_mt_haps(hap)
        T.sim_reads(hap, reads, 24 if kind == "c2" else 240, 10000, "ont", 11 if kind == "c2" else 111)
        return (mt,) + T.read_fasta(reads)
    if kind in ("c3", "sv_edge", "L3"):
        big = kind == "L3"
        pre, reads = os.path.join(workdir, "gsvL" if big else "gsv"), os.path.join(workdir, "g%s.fa" % kind)
        T.sim_graph(pre, 1000000 if big else 300000, 8 if big else 3, 7)
        T.sim_reads(pre + ".hap.fa", reads, 240 if big else 24, 15000, "ont", 105 if big else 5)
        names, seqs = T.read_fasta(reads)
        if kind == "sv_edge":
            n2, s2 = T.read_fasta(os.path.join(T.FIX, "edge.fa"))
            names, seqs = names + n2, seqs + s2
        return pre + ".gfa", names, seqs
    if kind in ("c4", "L4"):
        reads = os.path.join(workdir, "g%s.fa" % kind)
        T.sim_reads(os.path.join(T.FIX, "MT-human.fa"), reads, 12 if kind == "c4" else 200, 20000, "hifi", 13 if kind == "c4" else 113, circular=True)
        return (os.path.join(T.FIX, "MT-human.fa"),) + T.read_fasta(reads)
    if kind == "stable":
        gfa, hap, reads = os.path.join(T.FIX, "stable.gfa"), os.path.join(workdir, "gst.hap.fa"), os.path.join(workdir, "gst.fa")
        import subprocess
        subprocess.run([T.MGSIM, "walk", "-g", gfa, "-w", ">s1>s2>s3", "-w", ">s1>s4>s3", "-w", ">s1>s5>s3", "-o", hap], check=True)
        T.sim_reads(hap, reads, 40, 2500, "hifi", 17)
        return (gfa,) + T.read_fasta(reads)
    raise ValueError(kind)


def pair_inputs(workdir):
    """fragments of the read-pair golden file: names (of the first mates), n_seg, segment lengths and sequences as
    mg_map_batch_frag() takes them (the second mate reverse-complemented back, gmap.c:38-40 with the sr preset's pe_ori)"""
    hap, reads = os.path.join(workdir, "gmt.hap.fa"), os.path.join(workdir, "gsr.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, 60, 500, "hifi", 61)
    r1, r2 = os.path.join(workdir, "gsr1.fa"), os.path.join(workdir, "gsr2.fa")
    split_pairs(reads, r1, r2)
    (n1, s1), (_, s2) = T.read_fasta(r1), T.read_fasta(r2)
    flat = [x for a, b in zip(s1, s2) for x in (a, revcomp(b))]
    return os.path.join(T.FIX, "MT.gfa"), n1, [2] * len(n1), flat


class Index:
    def __init__(self, lib, gfa, preset, cigar=True, flag_extra=0):
        self.lib = lib
        self.g = lib.mgb_gfa_read(gfa.encode())
        assert self.g, "gfa read failed"
        self.io, self.mo = options.opt_set(preset, cigar)
        self.mo.flag |= flag_extra
        self.gi = lib.mg_index(self.g, C.byref(self.io), 1, C.byref(self.mo))
        assert self.gi, lib.mgb_last_error()

    def close(self):
        self.lib.mg_idx_destroy(self.gi)
        self.lib.mgb_gfa_destroy(self.g)


def map_gaf(lib, ix, names, seqs, n_seg=None, buf=None):
    """mgb_map_batch_gaf(); with buf = (c_void_p, c_size_t) the caller's buffer is reused (and stays the caller's)"""
    n_frag = len(n_seg) if n_seg is not None else len(seqs)
    qlens = (C.c_int * max(1, len(seqs)))(*[len(s) for s in seqs])
    cseqs = (C.c_char_p * max(1, len(seqs)))(*seqs)
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    cnseg = (C.c_int * n_frag)(*n_seg) if n_seg is not None else None
    out, ln = (buf[0], C.c_size_t(0)) if buf else (C.c_void_p(0), C.c_size_t(0))
    rc = lib.mgb_map_batch_gaf(ix.gi, n_frag, cnseg, qlens, cseqs, cnames, C.byref(ix.mo), C.byref(out), C.byref(ln),
                               C.byref(buf[1]) if buf else None)
    text = C.string_at(out, ln.value) if out.value else None
    if rc == 0:
        assert out.value and C.string_at(out.value + ln.value, 1) == b"\0"  # 0-terminated
    if not buf and out.value:
        C.CDLL(None).free(out)
    return rc, text


def gaf_device(lib, gfa, names, seqs, preset="lr", cigar=True, flag_extra=0, n_seg=None):
    ix = Index(lib, gfa, preset, cigar, flag_extra)
    try:
        rc, text = map_gaf(lib, ix, names, seqs, n_seg)
        assert rc == 0, (rc, lib.mgb_last_error())
        st = capi.mgb_stats_t()
        lib.mgb_get_stats(ix.gi, C.byref(st))
        return text, st
    finally:
        ix.close()


def check(got, want):
    import cases
    assert got == want, cases.first_diff(got, want)


def case_existing_goldens(lib, workdir, which=None):
    """every golden file of `-c` runs: byte for byte from the device formatter"""
    for name, _, kind, preset in EXISTING:
        if which is None or name[:2] in which:
            gfa, names, seqs = inputs(kind, workdir)
            check(gaf_device(lib, gfa, names, seqs, preset)[0], golden(name))


def case_flag_goldens(lib, workdir, host_writer=True):
    """the GAF output options: the device text equals the reference's golden file and, on the same batch, the host writer's text
    (mgb_write_gaf_batch over mg_map_batch)"""
    for name, kind, cigar, flag in FLAGGED:
        gfa, names, seqs = inputs(kind, workdir)
        got = gaf_device(lib, gfa, names, seqs, "lr", cigar, flag)[0]
        check(got, golden(name))
        if host_writer:
            check(T.gaf_with_engine(lib, gfa, names, seqs, "lr", cigar, flag)[0], got)


def case_pairs(lib, workdir):
    """read pairs through n_seg: one record per fragment, the first mate's name without "/1", ql:B:i with both lengths"""
    gfa, names, n_seg, flat = pair_inputs(workdir)
    got = gaf_device(lib, gfa, names, flat, "sr", False, SHOW_UNMAP, n_seg=n_seg)[0]
    check(got, golden(PAIRS))
    assert b"\tql:B:i,150,150" in got and b"/1\t" not in got


def case_goldens_reach_the_traps():
    """the fixtures exercise what is easy to get wrong: a compact reverse record followed, in the same read, by a + record whose
    cg:Z / ds:Z are printed reversed (the sticky rev_sign); a -S value that is not 0; a path of a stable sequence with an SO gap,
    one with rank/min != 0 and a segment without a stable name"""
    carry = False
    recs = {}
    for line in golden(FLAGGED[4][0]).split(b"\n"):
        f = line.split(b"\t")
        if len(f) > 12 and f[0] != b"*":
            recs.setdefault(f[0], []).append(f)
    for rs in recs.values():
        for a, b in zip(rs, rs[1:]):
            if a[4] == b"-" and b[4] == b"+" and any(x.startswith(b"cg:Z:") for x in b):
                carry = True
    assert carry
    s_lines = [ln.split(b"\t") for ln in golden(FLAGGED[0][0]).split(b"\n") if ln.startswith(b"*\t")]
    assert any(len(f) > 4 and f[4] not in (b"0",) for f in s_lines)
    paths = [ln.split(b"\t")[5] for ln in golden(FLAGGED[4][0]).split(b"\n") if ln and not ln.startswith(b"*")]
    assert any(b">chr1:" in p and p.count(b">chr1:") >= 2 for p in paths)  # SO gap: two runs of chr1
    assert any(b"alt1:" in p for p in paths)                                # rank 1, min 100: never compact
    assert any(b">s4" in p or b"<s4" in p for p in paths)                     # no SN


def case_api(lib, workdir):
    """n_frag == 0 gives ""; NULL names print "*"; the caller's buffer is reused and grown; --cov and independent segments refused"""
    gfa, names, seqs = inputs("c2", workdir)
    ix = Index(lib, gfa, "lr")
    try:
        rc, text = map_gaf(lib, ix, [], [])
        assert rc == 0 and text == b""
        rc, text = map_gaf(lib, ix, None, seqs[:4])
        assert rc == 0 and text and all(ln.startswith(b"*\t") for ln in text.split(b"\n") if ln)
        want = T.gaf_with_engine(lib, gfa, names, seqs, "lr")[0]
        buf = (C.c_void_p(0), C.c_size_t(0))
        caps = []
        for k in (2, 8, 24):
            rc, text = map_gaf(lib, ix, names[:k], seqs[:k], buf=buf)
            assert rc == 0, lib.mgb_last_error()
            assert want.startswith(text) and text.count(b"\n") >= k // 2
            assert buf[1].value > len(text)
            caps.append(buf[1].value)
        assert caps[0] <= caps[1] <= caps[2] and caps[2] > caps[0]
        rc, text = map_gaf(lib, ix, names[:2], seqs[:2], buf=buf)  # shorter again: the same block, kept
        assert rc == 0 and buf[1].value == caps[2] and want.startswith(text)
        C.CDLL(None).free(buf[0])
        for bit in (CAL_COV, INDEPEND_SEG):
            ix.mo.flag |= bit
            rc, text = map_gaf(lib, ix, names[:2], seqs[:2])
            assert rc < 0 and text is None and b"independent" in lib.mgb_last_error()
            ix.mo.flag &= ~bit
    finally:
        ix.close()


def case_random_vs_reference(lib, workdir, n_graphs=3, n_reads=30):
    """randomised SV graphs and reads (as tools/random_parity.py draws them) against the reference binary under the flag sets"""
    import random
    import subprocess
    rng = random.Random(41)
    opts = [("-c", "--secondary=yes", "--show-unmap=yes", "-S", "--write-mz"), ("-c", "--secondary=yes", "--vc", "-S"),
            ("-c", "--no-comp-path", "--show-unmap=yes"), ("--secondary=yes", "-S", "--write-mz")]
    bits = [(True, X), (True, PRINT_2ND | VERTEX_COOR | WRITE_LCHAIN), (True, NO_COMP_PATH | SHOW_UNMAP), (False, PRINT_2ND | WRITE_LCHAIN | WRITE_MZ)]
    for i in range(n_graphs):
        pre, reads = os.path.join(workdir, "grnd%d" % i), os.path.join(workdir, "grnd%d.fa" % i)
        T.sim_graph(pre, rng.choice([100000, 200000, 300000]), rng.choice([2, 3, 4]), rng.randrange(1, 1000))
        T.sim_reads(pre + ".hap.fa", reads, n_reads, rng.choice([3000, 8000, 15000]), rng.choice(["ont", "hifi"]), rng.randrange(1, 1000))
        names, seqs = T.read_fasta(reads)
        k = i % len(opts)
        want = subprocess.run([T.REF_BIN, "-x", "lr", "-t", "1"] + list(opts[k]) + [pre + ".gfa", reads], check=True,
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
        check(gaf_device(lib, pre + ".gfa", names, seqs, "lr", bits[k][0], bits[k][1])[0], want)


def case_full_c2(lib, workdir, n_reads=10000):
    """config 2 at full size: the device text is what mg_map_batch() + mgb_write_gaf_batch() give, and fewer bytes cross PCIe"""
    hap, reads = os.path.join(workdir, "gmt.hap.fa"), os.path.join(workdir, "gc2full.fa")
    T.sim_mt_haps(hap)
    T.sim_reads(hap, reads, n_reads, 10000, "ont", 11)
    gfa = os.path.join(T.FIX, "MT.gfa")
    names, seqs = T.read_fasta(reads)
    want, st_a = T.gaf_with_engine(lib, gfa, names, seqs, "lr")
    got, st_b = gaf_device(lib, gfa, names, seqs, "lr")
    check(got, want)
    assert 0 < st_b.out_bytes < st_a.out_bytes, (st_b.out_bytes, st_a.out_bytes)
    assert st_b.out_bytes == len(got)


def case_concurrent(lib, workdir, n_threads=3):
    """several host threads in mgb_map_batch_gaf() on one index at once: each gets the text a single caller gets"""
    import threading
    gfa, names, seqs = inputs("sv_edge", workdir)
    ix = Index(lib, gfa, "lr", True, X)
    try:
        rc, whole = map_gaf(lib, ix, names, seqs)
        assert rc == 0, lib.mgb_last_error()
        n = len(seqs)
        for _ in range(2):
            out = [None] * n_threads

            def run(t):
                lo, hi = n * t // n_threads, n * (t + 1) // n_threads
                out[t] = map_gaf(lib, ix, names[lo:hi], seqs[lo:hi])
            th = [threading.Thread(target=run, args=(t,)) for t in range(n_threads)]
            for x in th:
                x.start()
            for x in th:
                x.join()
            assert all(rc == 0 for rc, _ in out), lib.mgb_last_error()
            check(b"".join(text for _, text in out), whole)
    finally:
        ix.close()


def case_multi_device(lib, workdir, devices="0,0,0"):
    """MGB_DEVICES: the batch cut into one part per device, the parts' text joined in input order"""
    gfa, names, seqs = inputs("sv_edge", workdir)
    one = gaf_device(lib, gfa, names, seqs, "lr", True, X)[0]
    os.environ["MGB_DEVICES"] = devices
    try:
        many = gaf_device(lib, gfa, names, seqs, "lr", True, X)[0]
    finally:
        del os.environ["MGB_DEVICES"]
    check(many, one)
    check(one, golden(FLAGGED[0][0]))


def case_no_label_cache(lib, workdir):
    """graph chaining without the label table (lab_cache=0): the same text"""
    lib.mgb_set_param(b"lab_cache", 0)
    try:
        case_flag_goldens(lib, workdir, host_writer=False)
    finally:
        lib.mgb_set_param(b"lab_cache", 1)


if __name__ == "__main__":
    if len(sys.argv) == 5 and sys.argv[1] == "pairs":
        split_pairs(*sys.argv[2:])
    else:
        sys.exit("usage: gafcases.py pairs reads.fa r1.fa r2.fa")
