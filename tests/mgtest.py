"""Shared helpers of the test-suite: oracle bindings, FASTA reader, deep comparison of mg_gchains_t objects."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from minigraph_b200 import capi  # noqa: E402
from minigraph_b200 import options  # noqa: E402

FIX = os.path.join(REPO, "tests", "golden", "fixtures")
REF_SO = os.path.join(REPO, "oracle", "_ref", "libmgref.so")
REF_BIN = os.path.join(REPO, "oracle", "_ref", "minigraph")
HOSTSIM_SO = os.path.join(REPO, "tests", "hostsim", "libmgb_hostsim.so")
MGSIM = os.path.join(REPO, "tools", "mgsim")


def have_ref():
    return os.path.exists(REF_SO) and os.path.exists(REF_BIN)


_ref = None


def load_ref():
    """oracle/_ref/libmgref.so: the unmodified reference compiled as a shared object (test infrastructure)."""
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_SO)
        capi.bind_mapping_api(lib)
        lib.gfa_read.restype = C.POINTER(capi.gfa_t)
        lib.gfa_read.argtypes = [C.c_char_p]
        lib.gfa_destroy.restype = None
        lib.gfa_destroy.argtypes = [C.POINTER(capi.gfa_t)]
        C.c_int.in_dll(lib, "mg_verbose").value = 1
        _ref = lib
    return _ref


_hostsim = None


def load_hostsim():
    global _hostsim
    if _hostsim is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(REPO, "tests", "hostsim")])
        lib = C.CDLL(HOSTSIM_SO)
        _hostsim = capi.apply_env_params(capi.bind_engine_api(capi.bind_mapping_api(lib)))
    return _hostsim


_hostsim32 = None


def load_hostsim32():
    """the CPU build of the device code with a 32-lane warp simulated by fibres (tests/hostsim/Makefile, mgb_simlanes.h)"""
    global _hostsim32
    if _hostsim32 is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(REPO, "tests", "hostsim"), "libmgb_hostsim32.so"])
        lib = C.CDLL(os.path.join(REPO, "tests", "hostsim", "libmgb_hostsim32.so"))
        _hostsim32 = capi.apply_env_params(capi.bind_engine_api(capi.bind_mapping_api(lib)))
    return _hostsim32


def read_fasta(fn, upper=True):
    names, seqs = [], []
    cur = []
    with open(fn, "rb") as f:
        for line in f:
            line = line.rstrip(b"\r\n")
            if line.startswith(b">"):
                if names:
                    seqs.append(b"".join(cur))
                names.append(line[1:].split()[0])
                cur = []
            elif names:
                cur.append(line)
    if names:
        seqs.append(b"".join(cur))
    if upper:
        seqs = [s.upper() for s in seqs]
    return names, seqs


def gchains_to_py(p):
    """Everything mg_write_gaf (format.c:121-291) can see, as plain python data."""
    if not p:
        return None
    gs = p.contents
    out = {"n_gc": gs.n_gc, "n_lc": gs.n_lc, "n_a": gs.n_a, "rep_len": gs.rep_len, "gc": [], "lc": [], "a": []}
    for i in range(gs.n_gc):
        g = gs.gc[i]
        d = {k: getattr(g, k) for k in ("id", "parent", "off", "cnt", "n_anchor", "score", "qs", "qe", "plen", "ps", "pe",
                                         "blen", "mlen", "hash", "subsc", "n_sub", "mapq", "flt")}
        d["div"] = C.c_float(g.div).value
        if g.p:
            c = g.p.contents
            d["cigar_hdr"] = (c.n_cigar, c.mlen, c.blen, c.aplen, c.ss, c.ee)
            arr = C.cast(C.addressof(c) + C.sizeof(capi.mg_cigar_t), C.POINTER(C.c_uint64))
            d["cigar"] = [arr[j] for j in range(c.n_cigar)]
        else:
            d["cigar_hdr"], d["cigar"] = None, None
        if g.ds.ds:
            d["ds"] = C.string_at(g.ds.ds, g.ds.len)
            d["ds_off"] = [g.ds.off[j] for j in range(g.ds.n_off)]
        else:
            d["ds"], d["ds_off"] = None, None
        out["gc"].append(d)
    for i in range(gs.n_lc):
        l = gs.lc[i]
        out["lc"].append((l.off, l.cnt, l.v, l.score, l.ed))
    for i in range(gs.n_a):
        out["a"].append((gs.a[i].x, gs.a[i].y))
    return out


def diff_results(a, b):
    """Return a short description of the first difference, or None."""
    if isinstance(a, RefDigest) or isinstance(b, RefDigest):
        da = a["digest"] if isinstance(a, RefDigest) else None if a is None else result_digest(a)
        db = b["digest"] if isinstance(b, RefDigest) else None if b is None else result_digest(b)
        return None if da == db else "differs from the stored result of the reference (digest %s != %s)" % (db, da)
    if a is None or b is None:
        return None if a is b else "one result is NULL"
    for k in ("n_gc", "n_lc", "n_a", "rep_len"):
        if a[k] != b[k]:
            return "%s: %r != %r" % (k, a[k], b[k])
    for i, (x, y) in enumerate(zip(a["gc"], b["gc"])):
        for k in x:
            if x[k] != y[k]:
                return "gc[%d].%s: %r != %r" % (i, k, str(x[k])[:200], str(y[k])[:200])
    if a["lc"] != b["lc"]:
        return "lc differs: %r vs %r" % (a["lc"][:8], b["lc"][:8])
    if a["a"] != b["a"]:
        for i, (x, y) in enumerate(zip(a["a"], b["a"])):
            if x != y:
                return "a[%d]: %r != %r" % (i, x, y)
    return None


REF_RESULTS = os.path.join(REPO, "tests", "golden", "ref_results.json")


class RefDigest(dict):
    """A result of the reference known only by its digest (stored in REF_RESULTS); compared exactly by diff_results()."""


def result_digest(r):
    return hashlib.sha1(repr(r).encode()).hexdigest()[:16]


def _ref_key(gfa_path, names, seqs, preset, cigar, mo):
    h = hashlib.sha1()
    with open(gfa_path, "rb") as f:
        h.update(f.read())
    h.update(repr((preset, cigar)).encode() + bytes(mo))
    for n, s in zip(names, seqs):
        h.update(n + b"\0" + s + b"\0")
    return h.hexdigest()


def map_with_ref(gfa_path, names, seqs, preset="lr", cigar=True, tweak=None):
    """Run the reference's own mg_index/mg_map on every read (CPU).  tweak(mo) may change mapping options after the preset.
    Without a build of the reference (oracle/_ref), the results are the digests stored in REF_RESULTS for the same inputs;
    MGB_RECORD_REF=1 stores the digests of a run of the reference there."""
    io, mo = options.opt_set(preset, cigar)
    if tweak:
        tweak(mo)
    key = _ref_key(gfa_path, names, seqs, preset, cigar, mo)
    if not have_ref():
        with open(REF_RESULTS) as f:
            rec = json.load(f).get(key)
        assert rec is not None, "no stored reference results for these inputs (%s); run with oracle/_ref and MGB_RECORD_REF=1" % key
        mo.occ_max1, mo.lc_max_occ = rec["mo"]
        return [None if r is None else RefDigest(digest=r[0], n_gc=r[1]) for r in rec["reads"]], mo
    ref = load_ref()
    g = ref.gfa_read(gfa_path.encode())
    assert g, "gfa_read failed"
    gi = ref.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi
    b = ref.mg_tbuf_init()
    res = []
    for nm, s in zip(names, seqs):
        p = ref.mg_map(gi, len(s), s, b, C.byref(mo), nm)
        res.append(gchains_to_py(p))
        ref.mg_gchain_free(p)
    ref.mg_tbuf_destroy(b)
    ref.mg_idx_destroy(gi)
    ref.gfa_destroy(g)
    if os.environ.get("MGB_RECORD_REF"):
        table = {}
        if os.path.exists(REF_RESULTS):
            with open(REF_RESULTS) as f:
                table = json.load(f)
        table[key] = {"mo": [mo.occ_max1, mo.lc_max_occ], "reads": [None if r is None else [result_digest(r), r["n_gc"]] for r in res]}
        with open(REF_RESULTS, "w") as f:
            json.dump(table, f, separators=(",", ":"), sort_keys=True)
            f.write("\n")
    return res, mo


def map_with_engine(lib, gfa_path, names, seqs, preset="lr", cigar=True, gfa_loader=None, tweak=None):
    """Run an engine library (product or hostsim) through mg_index + mg_map_batch."""
    loader = gfa_loader or lib.mgb_gfa_read
    g = loader(gfa_path.encode())
    assert g, "gfa read failed"
    io, mo = options.opt_set(preset, cigar)
    if tweak:
        tweak(mo)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    n = len(seqs)
    qlens = (C.c_int * n)(*[len(s) for s in seqs])
    cseqs = (C.c_char_p * n)(*seqs)
    cnames = (C.c_char_p * n)(*names)
    gcs = (C.POINTER(capi.mg_gchains_t) * n)()
    rc = lib.mg_map_batch(gi, n, qlens, cseqs, cnames, gcs, C.byref(mo))
    assert rc == 0, (rc, lib.mgb_last_error())
    res = []
    for i in range(n):
        res.append(gchains_to_py(gcs[i]))
        lib.mg_gchain_free(gcs[i])
    st = capi.mgb_stats_t()
    lib.mgb_get_stats(gi, C.byref(st))
    lib.mg_idx_destroy(gi)
    return res, mo, st


def gaf_with_engine(lib, gfa_path, names, seqs, preset="lr", cigar=True, flag_extra=0):
    """Map through mg_index + mg_map_batch and format with mgb_write_gaf: the text `minigraph -cx preset` prints."""
    g = lib.mgb_gfa_read(gfa_path.encode())
    assert g, "gfa read failed"
    io, mo = options.opt_set(preset, cigar)
    mo.flag |= flag_extra
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    n = len(seqs)
    qlens = (C.c_int * n)(*[len(s) for s in seqs])
    cseqs = (C.c_char_p * n)(*seqs)
    cnames = (C.c_char_p * n)(*names)
    gcs = (C.POINTER(capi.mg_gchains_t) * n)()
    rc = lib.mg_map_batch(gi, n, qlens, cseqs, cnames, gcs, C.byref(mo))
    assert rc == 0, (rc, lib.mgb_last_error())
    buf, ln = C.c_void_p(0), C.c_size_t(0)
    lib.mgb_write_gaf_batch(g, n, gcs, qlens, cnames, mo.flag, 0, C.byref(buf), C.byref(ln), None)
    for i in range(n):
        lib.mg_gchain_free(gcs[i])
    text = C.string_at(buf, ln.value) if buf else b""
    C.CDLL(None).free(buf)
    st = capi.mgb_stats_t()
    lib.mgb_get_stats(gi, C.byref(st))
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
    return text, st


def gaf_with_ref_binary(gfa_path, fasta_path, preset="lr", threads=1, extra=()):
    """stdout of the unmodified reference CLI (oracle/_ref/minigraph)."""
    cmd = [REF_BIN, "-cx", preset, "-t", str(threads)] + list(extra) + [gfa_path, fasta_path]
    return subprocess.run(cmd, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout


def write_fasta(fn, names, seqs):
    with open(fn, "wb") as f:
        for n, s in zip(names, seqs):
            f.write(b">" + n + b"\n" + s + b"\n")


def sim_reads(hap_fa, out_fa, n, length, err="ont", seed=11, circular=False):
    cmd = [MGSIM, "reads", "-i", hap_fa, "-n", str(n), "-l", str(length), "-e", err, "-s", str(seed), "-o", out_fa]
    if circular:
        cmd.append("-c")
    subprocess.run(cmd, check=True, stderr=subprocess.DEVNULL)


def sim_graph(prefix, length, n_hap, seed=7):
    subprocess.run([MGSIM, "graph", "-l", str(length), "-n", str(n_hap), "-s", str(seed), "-o", prefix], check=True,
                   stderr=subprocess.DEVNULL)


MT_WALKS = [">MTh0>MTh4001>MTh4502>MTh9505>MTh13014>MTh13516", ">MTh0<MTo3426>MTh4502>MTo8961>MTh9505>MTh13516"]


def sim_mt_haps(out_fa):
    cmd = [MGSIM, "walk", "-g", os.path.join(FIX, "MT.gfa"), "-o", out_fa]
    for w in MT_WALKS:
        cmd += ["-w", w]
    subprocess.run(cmd, check=True)
