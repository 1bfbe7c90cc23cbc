"""The stitched CIGAR and the ds:Z string of every chain (k_finish) on reads built to reach the edges of the per-operation scheme
that random reads rarely reach: indels long enough for the whole warp to take them, indels inside homopolymers and tandem
repeats, runs of N in the read, chains with a number of operations around multiples of the warp width, walks over many short
segments on both strands, and reads with several chains.  Field by field against the reference where oracle/_ref is built;
elsewhere against the digests of the reference's results stored in tests/golden/finish_ds_ref.json (MGB_RECORD_FINISH_DS=1
with oracle/_ref records them)."""
import json
import os
import random

import pytest

import mgtest as T
from minigraph_b200 import capi
from minigraph_b200 import options

FIN_REF = os.path.join(T.REPO, "tests", "golden", "finish_ds_ref.json")

_COMP = bytes.maketrans(b"ACGTN", b"TGCAN")


def _revcomp(s):
    return s.translate(_COMP)[::-1]


def _rand_seq(rng, n):
    return bytes(rng.choice(b"ACGT") for _ in range(n))


def _sub(rng, b):
    return rng.choice([c for c in b"ACGT" if c != b])


def _mt_reads(hap):
    """(name, sequence) pairs cut from an MT haplotype, each with the edits one edge of the scheme needs"""
    rng = random.Random(2024)
    out = []
    # long indels: deletions and insertions from 35 bases up to past a kilobase
    for k, n in enumerate((35, 64, 300, 1200)):
        w = hap[1000 + 900 * k:1000 + 900 * k + 7000]
        out.append((b"del%d" % n, w[:3500] + w[3500 + n:]))
        out.append((b"ins%d" % n, w[:3000] + _rand_seq(rng, n) + w[3000:]))
    # indels inside homopolymers and tandem repeats, some a few dozen bases from the ends of the read, so that the repeats
    # in their flanks can run to the ends of the chain
    for k, (unit, copies) in enumerate(((b"C", 6), (b"A", 40), (b"CA", 12), (b"TTG", 25), (b"GATA", 9))):
        w = hap[5000 + 700 * k:5000 + 700 * k + 4000]
        rep = unit * copies
        for at in (2000, 60, len(w) - 60):
            base = w[:at] + rep + w[at:]
            out.append((b"rep_ins_%s_%d_%d" % (unit, copies, at), base[:at] + unit * (copies // 2) + base[at:]))
            out.append((b"rep_del_%s_%d_%d" % (unit, copies, at), w[:at] + rep + w[at:] if at > 100 else base))
    # runs of X with N in the read
    for k, n in enumerate((1, 5, 30, 200)):
        w = bytearray(hap[8000 + 500 * k:8000 + 500 * k + 5000])
        for at in (900, 2500, 4100):
            w[at:at + n] = b"N" * n
        out.append((b"nrun%d" % n, bytes(w)))
    # isolated substitutions every 90 bases: 2 n_sub + 1 operations, one more with an insertion next to one of them
    for n_sub in (15, 16, 31, 32):
        for extra in (False, True):
            w = bytearray(hap[2000 + 37 * n_sub:2000 + 37 * n_sub + 3400])
            for s in range(n_sub):
                at = 150 + 90 * s
                w[at] = _sub(rng, w[at])
            if extra:
                w[150 + 90 * (n_sub // 2) + 1:150 + 90 * (n_sub // 2) + 1] = b"GG"
            out.append((b"sub%d%s" % (n_sub, b"i" if extra else b""), bytes(w)))
    # a chimera: two distant pieces, one chain each
    out.append((b"chimera", hap[500:3500] + _revcomp(hap[9000:12000])))
    return out


def _dup_graph(path, seq):
    """two segments, the second a copy of the first with one difference in 50: reads map to both, one chain a secondary"""
    rng = random.Random(7)
    b = bytearray(seq)
    for at in range(100, len(b), 50):
        b[at] = _sub(rng, b[at])
    with open(path, "wb") as f:
        f.write(b"H\tVN:Z:1.0\n")
        f.write(b"S\ts1\t" + seq + b"\tLN:i:%d\tSN:Z:chrA\tSO:i:0\tSR:i:0\n" % len(seq))
        f.write(b"S\ts2\t" + bytes(b) + b"\tLN:i:%d\tSN:Z:chrB\tSO:i:0\tSR:i:0\n" % len(seq))


def _inputs(workdir):
    """[(gfa, names, seqs)]: the MT graph with the edited reads, an SV graph with reads on both strands, a duplicated region"""
    hap = os.path.join(workdir, "fin.mt.hap.fa")
    T.sim_mt_haps(hap)
    _, haps = T.read_fasta(hap)
    mt = _mt_reads(haps[0]) + [(n + b"_h1", s) for n, s in _mt_reads(haps[1])[:6]]
    pre, sv_fa = os.path.join(workdir, "fin.sv"), os.path.join(workdir, "fin.sv.reads.fa")
    T.sim_graph(pre, 200000, 8, 19)
    T.sim_reads(pre + ".hap.fa", sv_fa, 6, 12000, "ont", 23)
    sn, ss = T.read_fasta(sv_fa)
    sv = list(zip(sn, ss)) + [(n + b"_rc", _revcomp(s)) for n, s in zip(sn, ss)]
    dup_gfa = os.path.join(workdir, "fin.dup.gfa")
    _, human = T.read_fasta(os.path.join(T.FIX, "MT-human.fa"))
    _dup_graph(dup_gfa, human[0][:8000])
    rng = random.Random(11)
    dup = []
    for k in range(4):
        w = bytearray(human[0][700 * k + 300:700 * k + 5300])
        for at in range(40 + 13 * k, len(w), 400):
            w[at] = _sub(rng, w[at])
        dup.append((b"dup%d" % k, bytes(w) if k % 2 == 0 else _revcomp(bytes(w))))
    return [(os.path.join(T.FIX, "MT.gfa"), mt), (pre + ".gfa", sv), (dup_gfa, dup)]


def _want(gfa, names, seqs):
    """the reference's results for these reads: from oracle/_ref, or their digests stored in FIN_REF"""
    key = T._ref_key(gfa, names, seqs, "lr", True, options.opt_set("lr", True)[1])
    if not T.have_ref():
        with open(FIN_REF) as f:
            rec = json.load(f).get(key)
        assert rec is not None, "no stored reference results for these inputs (%s); run with oracle/_ref and MGB_RECORD_FINISH_DS=1" % key
        return [None if r is None else T.RefDigest(digest=r[0], n_gc=r[1]) for r in rec]
    want, _ = T.map_with_ref(gfa, names, seqs, "lr")
    if os.environ.get("MGB_RECORD_FINISH_DS"):
        table = {}
        if os.path.exists(FIN_REF):
            with open(FIN_REF) as f:
                table = json.load(f)
        table[key] = [None if r is None else [T.result_digest(r), r["n_gc"]] for r in want]
        with open(FIN_REF, "w") as f:
            json.dump(table, f, separators=(",", ":"), sort_keys=True)
            f.write("\n")
    return want


def _check(lib, workdir):
    n_cigar, n_sec, n_multi = set(), 0, 0
    for gfa, reads in _inputs(workdir):
        names, seqs = [n for n, _ in reads], [s for _, s in reads]
        want = _want(gfa, names, seqs)
        got, _, _ = T.map_with_engine(lib, gfa, names, seqs, "lr")
        for i, (a, b) in enumerate(zip(want, got)):
            d = T.diff_results(a, b)
            assert d is None, (gfa, names[i], d)
            if b:
                n_cigar.update(len(g["cigar"]) for g in b["gc"] if g["cigar"])
                n_sec += sum(g["id"] != g["parent"] for g in b["gc"])
                n_multi += b["n_gc"] > 1
    assert {31, 32, 33, 64, 65} <= n_cigar, sorted(n_cigar)
    assert n_sec > 0 and n_multi > 0


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")
def test_finish_ds_one_lane(workdir):
    _check(T.load_hostsim(), workdir)


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")
def test_finish_ds_32_lanes(workdir):
    _check(T.load_hostsim32(), workdir)


@pytest.mark.gpu
def test_finish_ds_gpu(workdir):
    _check(capi.load_product(), workdir)
