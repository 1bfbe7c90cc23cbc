"""Graph-chain materialisation and the post filters (K7b: mgb_gchain.cuh gchain_gen, gchain_set_parent, gchain_flt_sub,
gchain_drop_flt, gchain_set_mapq, with the bridging plan of k_gchain and the bridging jobs of k_gwfa), checked on their own through
mgb_test_gchain_gen against map-algo.c:464-474 restated line by line on the reference's own functions (mg_gchain_gen,
mg_gchain_set_parent, mg_gchain_flt_sub, mg_gchain_drop_flt, mg_gchain_set_mapq).  Graph chaining itself is not retested: its
output (u, lc, a) is written by hand (post-filter family) or made by the reference's mg_gchain1_dp (materialisation family).  Every
field of the result, div included, must be the reference's, in the one-lane and the 32-lane simulators and on the GPU; every family
checks that it reached the edges it is there for."""
import collections
import ctypes as C
import os
import random

import numpy as np
import pytest

import mgtest as T
from minigraph_b200 import capi, options

pytestmark = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")

MG_SEED_SEG_SHIFT = 48
ACGT = b"ACGT"
COMP = bytes.maketrans(b"ACGT", b"TGCA")
f32 = np.float32

_libc = C.CDLL(None)
_libc.expf.restype, _libc.expf.argtypes = C.c_float, [C.c_float]
_libc.logf.restype, _libc.logf.argtypes = C.c_float, [C.c_float]
_libc.free.restype, _libc.free.argtypes = None, [C.c_void_p]
_ref = None


def ref():
    global _ref
    if _ref is None:
        r = T.load_ref()
        gp, lcp, ap = C.POINTER(capi.gfa_t), C.POINTER(capi.mg_lchain_t), C.POINTER(capi.mg128_t)
        r.gfa_edseq_init.restype, r.gfa_edseq_init.argtypes = C.c_void_p, [gp]
        r.gfa_edseq_destroy.restype, r.gfa_edseq_destroy.argtypes = None, [C.c_int32, C.c_void_p]
        r.mg_gchain1_dp.restype = C.c_int32
        r.mg_gchain1_dp.argtypes = [C.c_void_p, gp, C.POINTER(C.c_int32), lcp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_float, C.c_float, C.c_float, ap, C.POINTER(C.POINTER(C.c_uint64))]
        r.mg_gchain_gen.restype = C.POINTER(capi.mg_gchains_t)
        r.mg_gchain_gen.argtypes = [C.c_void_p, C.c_void_p, gp, C.c_void_p, C.c_int32, C.POINTER(C.c_uint64), lcp, ap, C.c_uint32, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_char_p]
        r.mg_gchain_set_parent.restype = None
        r.mg_gchain_set_parent.argtypes = [C.c_void_p, C.c_float, C.c_int, C.POINTER(capi.mg_gchain_t), C.c_int, C.c_int]
        r.mg_gchain_flt_sub.restype = C.c_int
        r.mg_gchain_flt_sub.argtypes = [C.c_float, C.c_int, C.c_int, C.c_int, C.POINTER(capi.mg_gchain_t)]
        r.mg_gchain_drop_flt.restype, r.mg_gchain_drop_flt.argtypes = None, [C.c_void_p, C.POINTER(capi.mg_gchains_t)]
        r.mg_gchain_set_mapq.restype = None
        r.mg_gchain_set_mapq.argtypes = [C.c_void_p, C.POINTER(capi.mg_gchains_t), C.c_int, C.c_int, C.c_int]
        _ref = r
    return _ref


def rnd(rng, n):
    return bytes(rng.choices(ACGT, k=n))


def revcomp(s):
    return s.translate(COMP)[::-1]


class Read:
    """a read whose graph chaining is done: segments, hash, rep_len, n_mz, u, lc (tuples of mg_lchain_t's fields) and a"""

    def __init__(self, segs, hash_, rep_len, n_mz, u, lc, a, tag):
        self.segs, self.hash, self.rep_len, self.n_mz, self.u, self.lc, self.a, self.tag = segs, hash_, rep_len, n_mz, u, lc, a, tag
        self.seq = b"".join(segs)


LC_FIELDS = ("off", "cnt", "v", "rs", "re", "qs", "qe", "score", "dist_pre", "hash_pre", "inner_pre")


def lc_array(lc):
    arr = (capi.mg_lchain_t * max(len(lc), 1))()
    for i, t in enumerate(lc):
        for f, x in zip(LC_FIELDS, t):
            setattr(arr[i], f, x)
    return arr


def a_array(a):
    arr = (capi.mg128_t * max(len(a), 1))()
    for i, (x, y) in enumerate(a):
        arr[i].x, arr[i].y = x, y
    return arr


class RefGraph:
    """the reference's gfa_read of a GFA and its gfa_edseq_init, as mg_index keeps them (gi->g, gi->es)"""

    def __init__(self, gfa):
        self.g = ref().gfa_read(gfa.encode())
        assert self.g
        self.es = ref().gfa_edseq_init(self.g)
        self.seg_len = [self.g.contents.seg[i].len for i in range(self.g.contents.n_seg)]

    def close(self):
        ref().gfa_edseq_destroy(self.g.contents.n_seg, self.es)
        ref().gfa_destroy(self.g)


def ref_gen(R, mo, k, rd, snap=None):
    """map-algo.c:464-474: the graph chains of rd and their post filters; snap(gcs) sees them between mg_gchain_gen and the filters"""
    r = ref()
    u = (C.c_uint64 * max(len(rd.u), 1))(*rd.u)
    p = r.mg_gchain_gen(None, None, R.g, R.es, len(rd.u), u, lc_array(rd.lc), a_array(rd.a), rd.hash, mo.min_gc_cnt, mo.min_gc_score,
                        mo.gdp_max_ed, len(rd.segs), rd.seq)
    p.contents.rep_len = rd.rep_len
    if snap:
        snap(T.gchains_to_py(p))
    gs = p.contents
    r.mg_gchain_set_parent(None, mo.mask_level, gs.n_gc, gs.gc, mo.sub_diff, 0)
    r.mg_gchain_flt_sub(mo.pri_ratio, k * 2, mo.best_n, gs.n_gc, gs.gc)
    r.mg_gchain_drop_flt(None, p)
    r.mg_gchain_set_mapq(None, p, len(rd.seq), rd.n_mz, mo.min_gc_score)
    out = T.gchains_to_py(p)
    r.mg_gchain_free(p)
    return out


def run_hook(lib, gi, mo, reads):
    """mgb_test_gchain_gen: per read ((rc, jobs, jobs aligned, pairs bridged again in place), result)"""
    n = len(reads)
    frag = any(len(rd.segs) > 1 for rd in reads)
    seg_off = seg_len = None
    if frag:
        offs, lens = [0], []
        for rd in reads:
            lens += [len(s) for s in rd.segs]
            offs.append(len(lens))
        seg_off, seg_len = (C.c_int32 * (n + 1))(*offs), (C.c_int32 * len(lens))(*lens)
    i32 = lambda xs: (C.c_int32 * max(len(xs), 1))(*xs)  # noqa: E731
    u = [x for rd in reads for x in rd.u]
    lc = [t for rd in reads for t in rd.lc]
    a = [t for rd in reads for t in rd.a]
    out = (C.c_int32 * (4 * n))()
    gcs = (C.POINTER(capi.mg_gchains_t) * n)()
    rc = lib.mgb_test_gchain_gen(gi, C.byref(mo), n, (C.c_int * n)(*[len(rd.seq) for rd in reads]), (C.c_char_p * n)(*[rd.seq for rd in reads]),
                                 seg_off, seg_len, (C.c_uint32 * n)(*[rd.hash for rd in reads]), i32([rd.rep_len for rd in reads]),
                                 i32([rd.n_mz for rd in reads]), i32([len(rd.u) for rd in reads]), (C.c_uint64 * max(len(u), 1))(*u),
                                 i32([len(rd.lc) for rd in reads]), lc_array(lc), i32([len(rd.a) for rd in reads]), a_array(a), out, gcs)
    assert rc == 0, (rc, lib.mgb_last_error())
    res = []
    for i in range(n):
        res.append((tuple(out[4 * i:4 * i + 4]), T.gchains_to_py(gcs[i])))
        lib.mg_gchain_free(gcs[i])
    return res


def engine_index(lib, gfa, k, w=10):
    g = lib.mgb_gfa_read(gfa.encode())
    assert g
    io, mo = options.opt_set("lr")
    io.k, io.w = k, w
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    return g, gi


# ---------------------------------------------------------------------------------------------------------------
# what the filters did: the reference's chains between mg_gchain_gen and the filters, replayed in float32 (events only)
# ---------------------------------------------------------------------------------------------------------------
def filter_events(pre, post, mo, k, rd, ev):
    gc = pre["gc"]
    n = len(gc)
    ml = f32(mo.mask_level)
    ev["chains kept per read > 64"] += n > 64
    keys = collections.Counter((g["score"], g["hash"]) for g in gc)
    ev["sort: chains tied on score and hash"] += sum(c for c in keys.values() if c > 1)
    ev["sort: tied chains in a read of > 64"] += n > 64 and any(c > 1 for c in keys.values())
    ev["sort: tied chains that differ"] += sum(1 for i in range(n - 1) if (gc[i]["score"], gc[i]["hash"]) == (gc[i + 1]["score"], gc[i + 1]["hash"])
                                              and (gc[i]["n_anchor"], gc[i]["qe"]) != (gc[i + 1]["n_anchor"], gc[i + 1]["qe"]))
    parent, w, n_sub = list(range(n)), [0] if n else [], [0] * n
    for i in range(1, n):
        si, ei = gc[i]["qs"], gc[i]["qe"]
        cov = sorted((max(gc[j]["qs"], si), min(gc[j]["qe"], ei)) for j in w if not (gc[j]["qe"] <= si or gc[j]["qs"] >= ei))
        ev["chains that touch"] += sum(1 for j in w if gc[j]["qe"] == si or gc[j]["qs"] == ei)
        found = None
        if cov:
            x, uncov = si, 0
            for s, e in cov:
                if s > x:
                    uncov += s - x
                x = max(x, e)
            uncov += max(0, ei - x)
            ev["covered by several primaries"] += len(cov) > 1
            for j in w:
                sj, ej = gc[j]["qs"], gc[j]["qe"]
                if ej <= si or sj >= ei:
                    continue
                mn, mx = min(ej - sj, ei - si), max(ej - sj, ei - si)
                ol = min(ei, ej) - max(si, sj)
                val = f32(ol) / f32(mn) - f32(uncov) / f32(mx)
                ev["overlap ratio at mask_level"] += val == ml
                ev["overlap ratio just above mask_level"] += ml < val <= ml + f32(0.02)
                ev["overlap ratio just below mask_level"] += ml - f32(0.02) <= val < ml
                ev["uncovered length decides"] += uncov > 0 and (f32(ol) / f32(mn) > ml) != (val > ml)
                ev["nested in a primary"] += sj <= si and ei <= ej
                if val > ml:
                    found = j
                    break
        if found is None:
            w.append(i)
            continue
        parent[i] = parent[found]
        c, cp = gc[i]["cnt"], gc[found]["cnt"]
        ev["child cnt %s parent's" % ("<" if c < cp else "=" if c == cp else ">")] += 1
    if mo.pri_ratio > 0:
        n_2nd = 0
        for i in range(n):
            p = parent[i]
            if p == i:
                continue
            s, sp = gc[i]["score"], gc[p]["score"]
            ev["score at score * pri_ratio"] += f32(s) == f32(sp) * f32(mo.pri_ratio)
            ev["score at score - 2k"] += s + 2 * k == sp
            if f32(s) >= f32(sp) * f32(mo.pri_ratio) or s + 2 * k >= sp:
                if n_2nd >= mo.best_n:
                    ev["secondaries past best_n"] += 1
                    continue
                same = all(gc[i][f] == gc[p][f] for f in ("qs", "qe", "ps", "pe"))
                ev["secondary identical to its parent"] += same
                n_2nd += not same
        ev["eligible secondaries = best_n"] += n_2nd == mo.best_n and mo.best_n > 0
    else:
        ev["pri_ratio = 0"] += 1
    ev["best_n = 0"] += mo.best_n == 0
    # mapq of the kept chains
    if not post or not post["gc"]:
        return
    qlen = len(rd.seq)
    t_sc, t_cnt = min(qlen, 100), max(min(rd.n_mz, 10), 5)
    ev["qlen %s 100" % ("<" if qlen < 100 else ">=")] += qlen in (99, 100)
    if rd.n_mz in (4, 5, 10, 11):
        ev["n_mz = %d" % rd.n_mz] += 1
    ev["rep_len %s" % ("0" if rd.rep_len == 0 else "> 0")] += 1
    sum_sc = sum(g["score"] for g in post["gc"] if g["parent"] == g["id"])
    uniq = f32(sum_sc) / f32(sum_sc + rd.rep_len)
    for g in post["gc"]:
        if g["parent"] != g["id"]:
            continue
        sc = g["score"]
        ev["n_anchor %s t_cnt" % ("<" if g["n_anchor"] < t_cnt else "=" if g["n_anchor"] == t_cnt else ">")] += 1
        pen_s1 = (f32(1.0) if sc > t_sc else f32(sc) * f32(1.0 / t_sc)) * uniq
        pen_cm = f32(1.0) if g["n_anchor"] > t_cnt else f32(g["n_anchor"]) * f32(1.0 / t_cnt)
        pen_cm = min(pen_s1, pen_cm)
        subsc = max(g["subsc"], mo.min_gc_score)
        ev["subsc below min_gc_score"] += g["subsc"] < mo.min_gc_score
        ev["score == subsc"] += sc == subsc
        x = f32(subsc) / f32(sc)
        mq = int(pen_cm * f32(40.0) * (f32(1.0) - x) * f32(_libc.logf(sc)))
        mq -= int(f32(4.343) * f32(_libc.logf(g["n_sub"] + 1)) + f32(.499))
        ev["mapq bumped from 0 to 1"] += mq <= 0 and sc > subsc
        ev["mapq capped at 60"] += mq > 60
        ev["mapq from uniq_ratio < 1"] += rd.rep_len > 0 and 0 < g["mapq"] < 60


def junction_events(rd, mo, ev):
    """the overlap resolution of the kept chains (gchain1.c:409-441) and the merge of consecutive linear chains on one vertex
    (gchain1.c:392-405), replayed on the input: which comparisons were decided at equality"""
    xs = [x & 0xffffffff for x, _ in rd.a]
    ys = [y & 0xffffffff for _, y in rd.a]
    st = 0
    for uu in rd.u:
        n = uu & 0xffffffff
        lcs = [list(rd.lc[st + j][:7]) for j in range(n)]  # off, cnt, v, rs, re, qs, qe
        st += n
        if sum(l[1] for l in lcs) < mo.min_gc_cnt or uu >> 32 < mo.min_gc_score:
            continue
        for j in range(1, n):
            l0, l1 = lcs[j - 1], lcs[j]
            same = l0[2] == l1[2]
            x, y = xs[l1[0]], ys[l1[0]]
            t = l0[1] - 1
            while t >= 0 and not (ys[l0[0] + t] <= y and (not same or xs[l0[0] + t] <= x)):
                t -= 1
            if t >= 0 and ys[l0[0] + t] == y:
                ev["y tie at a junction" + (" on one vertex" if same else " on two vertices")] += 1
            shift0 = l0[1] - 1 - t
            x, y = xs[l0[0] + l0[1] - 1], ys[l0[0] + l0[1] - 1]
            t = 0
            while t < l1[1] and not (ys[l1[0] + t] >= y and (not same or xs[l1[0] + t] >= x)):
                t += 1
            if shift0 > 0:
                l0[1] -= shift0
                if l0[1]:
                    l0[6], l0[4] = ys[l0[0] + l0[1] - 1] + 1, xs[l0[0] + l0[1] - 1] + 1
            if t > 0:
                l1[0] += t
                l1[1] -= t
        j0 = 0
        for j in range(1, n):
            l0, l1 = lcs[j0], lcs[j]
            if l1[1] == 0:
                continue
            if l0[2] == l1[2]:
                an = [(xs[l1[0] + t], ys[l1[0] + t]) for t in range(l1[1])]
                t = next((t for t, (x, y) in enumerate(an) if x > l0[4] and y > l0[6]), len(an))
                ev["one vertex: contained" if t == len(an) else "one vertex: not contained"] += 1
                ev["one vertex: anchor at l0.re"] += any(x == l0[4] and y > l0[6] for x, y in an[:t + 1])
                ev["one vertex: anchor at l0.qe"] += any(y == l0[6] and x > l0[4] for x, y in an[:t + 1])
            j0 = j


def walk_events(pre, ev):
    """the walks of the bridging alignments that were found: the empty linear chains a bridge puts between two with anchors"""
    for g in pre.get("gc", []):
        lcs = pre["lc"][g["off"]:g["off"] + g["cnt"]]
        inner = 0
        for off, cnt, v, score, ed in lcs[1:]:
            if cnt == 0:
                inner += 1
                continue
            if ed >= 0:
                ev["aligned bridge over a walk of %s vertices" % (inner + 2 if inner < 2 else "4+")] += 1
            inner = 0


def check(lib, gi, R, mo, k, reads, seen, what):
    got = run_hook(lib, gi, mo, reads)
    for rd, ((rc, n_jobs, n_ok, n_re), res) in zip(reads, got):
        tag = "%s, read %r (%d bases, %d chains, %d linear chains): " % (what, rd.tag, len(rd.seq), len(rd.u), len(rd.lc))
        pre = {}
        want = ref_gen(R, mo, k, rd, snap=lambda p: pre.update(p))
        assert rc == 0, tag + "rc %d" % rc
        d = T.diff_results(want, res)
        assert d is None, tag + d
        filter_events(pre, want, mo, k, rd, seen)
        # gchain_extra's correction of n_mini for anchors that go back on the query (ql < 0) is not reached, and cannot be from
        # linear chains whose anchors rise on the query, as mg_lchain_dp makes them (lchain.c:119 refuses dq <= 0): resolve_overlap
        # cuts the end of l0 back to anchors at or before l1's first y and the start of l1 to anchors at or after l0's last y, so
        # the anchors of consecutive non-empty linear chains rise on the query; over an emptied one the same holds through it; and
        # the anchors merged from a linear chain on the same vertex lie past l0's qe.
        junction_events(rd, mo, seen)
        walk_events(pre, seen)
        seen["bridging jobs"] += n_jobs
        seen["bridging jobs aligned"] += n_ok
        seen["bridging jobs not aligned"] += n_jobs - n_ok
        seen["pairs bridged again in place"] += n_re
        n_kept = len(pre.get("gc", []))
        seen["reads with chains dropped and kept"] += 0 < n_kept < len(rd.u)
    return got


# ---------------------------------------------------------------------------------------------------------------
# post-filter family: graph chains on one vertex each (one or several linear chains), written by hand
# ---------------------------------------------------------------------------------------------------------------
def write_gfa(fn, segs, links):
    with open(fn, "w") as f:
        for name, s in segs:
            f.write("S\t%s\t%s\tLN:i:%d\n" % (name, s.decode(), len(s)))
        for a, sa, b, sb in links:
            f.write("L\t%s\t%s\t%s\t%s\t0M\n" % (a, sa, b, sb))


def explicit_read(rng, qlen, chains, k, n_mz, rep_len, tag, extra_mini=0):
    """chains: (score, [(v, [(qpos, rpos), ...]), ...]) -> a Read whose graph chains are these linear chains, each scored by its
    share of the chain's score"""
    anchors, lc, u = [], [], []
    for score, lcs in chains:
        for v, an in lcs:
            off = len(anchors)
            anchors += an
            (q0, r0), (q1, r1) = an[0], an[-1]
            lc.append((off, len(an), v, r0 + 1 - k, r1 + 1, q0 + 1 - k, q1 + 1, score // len(lcs), -1, 0, 0))
        u.append(score << 32 | len(lcs))
    pos = sorted(set(q for q, _ in anchors) | set(rng.sample(range(qlen), min(extra_mini, qlen))))
    idx = {p: i for i, p in enumerate(pos)}
    a = [(idx[q] << 32 | r, k << 32 | q) for q, r in anchors]
    return Read([rnd(rng, qlen)], rng.getrandbits(32), rep_len, n_mz, u, lc, a, tag)


def chain_read(rng, qlen, chains, k, n_mz, rep_len, tag, extra_mini=0):
    """chains: (qs, qe, v, rs, score, cnt[, last_dq[, parts]]) -> a Read with one graph chain per chain, cut into `parts` linear
    chains on vertex v (default 1); anchors on the diagonal rs - qs, the last one moved back by last_dq on the query (same re,
    another qe)"""
    out = []
    for ch in chains:
        qs, qe, v, rs, score, cnt = ch[:6]
        dq = ch[6] if len(ch) > 6 else 0
        parts = ch[7] if len(ch) > 7 else 1
        first, last = qs + k - 1, qe - 1
        qp = [first + (last - first) * j // max(cnt - 1, 1) for j in range(cnt)] if cnt > 1 else [last]
        rp = [rs + (q - qs) for q in qp]
        qp[-1] -= dq
        an = list(zip(qp, rp))
        cut = [len(an) * j // parts for j in range(parts + 1)]
        out.append((score, [(v, an[cut[j]:cut[j + 1]]) for j in range(parts)]))
    return explicit_read(rng, qlen, out, k, n_mz, rep_len, tag, extra_mini)


def random_chains(rng, qlen, n, vlen, scores, cnts, grid=50):
    out = []
    for _ in range(n):
        if out and rng.random() < 0.15:  # a copy: an identical secondary, or a tie on (qs, re, v, score) with other anchors
            c = list(rng.choice(out))
            if rng.random() < 0.5:
                c[5] = rng.choice([x for x in cnts if x >= 6])
                c[6] = rng.randint(1, 3)
            out.append(tuple(c))
            continue
        L = grid * rng.randint(2, max(2, min(14, qlen // grid)))
        L = min(L, qlen - qlen % grid)
        qs = grid * rng.randint(0, (qlen - L) // grid)
        cnt = rng.choice(cnts)
        parts = rng.choice([1, 1, 2, 3]) if cnt >= 6 else 1
        out.append((qs, qs + L, rng.randrange(8), grid * rng.randrange((vlen - L) // grid), rng.choice(scores), cnt, 0, parts))
    return out


def postfilter_reads(rng, k, mo, vlen):
    reads = []
    sc = mo.min_gc_score
    scores = [sc - 1, sc, sc + 6, 2 * sc, 2 * sc + 30, 3 * sc, 4 * sc, 5 * sc, 8 * sc, 10 * sc]
    scores += [int(s * 0.8) for s in scores if int(s * 0.8) == s * 0.8] + [s - 2 * k for s in scores if s - 2 * k >= sc]
    cnts = [mo.min_gc_cnt - 1, mo.min_gc_cnt, 6, 9, 10, 11, 12]
    for i in range(40):
        qlen = rng.choice([99, 100, 400, 1000, 3000])
        n = rng.randint(2, 12)
        reads.append(chain_read(rng, qlen, random_chains(rng, qlen, n, vlen, scores, cnts), k, rng.choice([4, 5, 10, 11, 40]),
                                rng.choice([0, 0, 37, 5000]), "random %d" % i, extra_mini=rng.randint(0, 20)))
    # a primary and two halves of it: coverage by several primaries, ratios at, above and below mask_level
    for d in (-1, 0, 1):
        ch = [(0, 400, 0, 1000, 10 * sc, 12), (400, 800, 2, 2000, 9 * sc, 12), (200 + d, 600 + d, 4, 3000, 4 * sc, 10)]
        reads.append(chain_read(rng, 1000, ch, k, 40, 0, "two primaries, child shifted %+d" % d))
    # a parent with exactly best_n and best_n + 1 eligible distinct secondaries, and one identical to it
    for m in (mo.best_n, mo.best_n + 1):
        ch = [(0, 1000, 0, 1000, 10 * sc, 12)] + [(50 * (j % 3), 950 + 50 * (j % 2), 2 + (j % 5), 100 * j, 9 * sc, 10) for j in range(m)]
        ch.append((0, 1000, 0, 1000, 10 * sc, 12))
        reads.append(chain_read(rng, 1200, ch, k, 40, 0, "%d eligible secondaries" % m))
    # well over 64 chains with the same (qs, re, v) and score: the sort's permutation of ties decides the order
    ch = []
    for j in range(150):
        base = (100 * (j % 5), 100 * (j % 5) + 600, 2 * (j % 3), 500, 5 * sc, 12)
        ch.append(base[:5] + (rng.choice([6, 9, 10, 11, 12]), rng.randint(0, 3)))
    reads.append(chain_read(rng, 1000, ch, k, 40, 100, "150 tied chains"))
    ch = [(0, 300, 1, 700, 5 * sc, 12 - (j % 5), j % 4) for j in range(30)]
    reads.append(chain_read(rng, 400, ch, k, 40, 0, "30 tied chains"))
    # mapq edges: short reads, one chain with few anchors, a large repeat length
    for qlen in (99, 100):
        for n_mz in (4, 5, 10, 11):
            for cnt in (4, 5, 6, 10, 11):
                if cnt < mo.min_gc_cnt:
                    continue
                reads.append(chain_read(rng, qlen, [(0, qlen - qlen % 5, 0, 100, sc + 10 * cnt, cnt)], k, n_mz, rng.choice([0, 3000]),
                                        "mapq qlen=%d n_mz=%d cnt=%d" % (qlen, n_mz, cnt)))
    # score == subsc; a product that rounds to 0 above subsc; the cap of 60
    reads.append(chain_read(rng, 1000, [(0, 600, 0, 100, 5 * sc, 12), (0, 600, 2, 300, 5 * sc, 12)], k, 40, 0, "equal scores"))
    reads.append(chain_read(rng, 1000, [(0, 600, 0, 100, 5 * sc, 12), (0, 600, 2, 300, 5 * sc - 1, 12)], k, 40, 0, "one point apart"))
    # two linear chains on one vertex: the next anchor exactly at l0.re or at l0.qe, all of l1 at l0.re (contained), and l1's first
    # anchor at l0's last query position (resolve_overlap at equality on y)
    l0 = [(k - 1 + 20 * j, 1000 + 20 * j) for j in range(8)]
    qe, re = l0[-1][0] + 1, l0[-1][1] + 1
    for what, l1 in (("anchor at l0.re", [(qe + 6, re), (qe + 20, re + 20), (qe + 40, re + 40)]),
                     ("anchor at l0.qe", [(qe, re + 6), (qe + 20, re + 20), (qe + 40, re + 40)]),
                     ("contained", [(qe + 6, re), (qe + 12, re)]),
                     ("tie on y", [(qe - 1, re + 4), (qe + 20, re + 20), (qe + 40, re + 40)])):
        reads.append(explicit_read(rng, 600, [(6 * sc, [(2, l0), (2, l1)])], k, 40, 0, "one vertex, " + what))
    reads.append(chain_read(rng, 3000, [(0, 3000, 0, 100, 3000, 12)], k, 40, 0, "alone"))
    return reads


def case_postfilter(lib, seen, rng, workdir):
    k = 15
    vlen = 30000
    segs = [("s%d" % i, rnd(rng, vlen)) for i in range(4)]
    fn = os.path.join(workdir, "pf.gfa")
    write_gfa(fn, segs, [])
    R = RefGraph(fn)
    g, gi = engine_index(lib, fn, k)
    try:
        for tag, tweak in (("lr", None), ("mask_level 0.25, best_n 1", dict(mask_level=0.25, best_n=1)),
                           ("mask_level 0.75, best_n 0", dict(mask_level=0.75, best_n=0)), ("pri_ratio 0", dict(pri_ratio=0.0)),
                           ("asm gates", dict(min_gc_score=1000, min_gc_cnt=5, pri_ratio=0.5)), ("min_gc_cnt 3", dict(min_gc_cnt=3))):
            _, mo = options.opt_set("lr")
            for key, v in (tweak or {}).items():
                setattr(mo, key, v)
            reads = postfilter_reads(rng, k, mo, vlen)
            check(lib, gi, R, mo, k, reads, seen, "post filters, " + tag)
    finally:
        lib.mg_idx_destroy(gi)
        lib.mgb_gfa_destroy(g)
        R.close()


POSTFILTER_EDGES = ["overlap ratio at mask_level", "overlap ratio just above mask_level", "overlap ratio just below mask_level",
                    "uncovered length decides", "chains that touch", "nested in a primary", "covered by several primaries",
                    "child cnt = parent's", "one vertex: contained",
                    "one vertex: not contained", "one vertex: anchor at l0.re", "one vertex: anchor at l0.qe", "y tie at a junction on one vertex", "score at score * pri_ratio",
                    "score at score - 2k", "secondaries past best_n", "eligible secondaries = best_n", "best_n = 0", "pri_ratio = 0",
                    "secondary identical to its parent", "reads with chains dropped and kept", "chains kept per read > 64",
                    "sort: tied chains in a read of > 64", "sort: tied chains that differ", "qlen < 100", "qlen >= 100",
                    "n_mz = 4", "n_mz = 5", "n_mz = 10", "n_mz = 11", "n_anchor < t_cnt", "n_anchor = t_cnt", "n_anchor > t_cnt",
                    "rep_len 0", "rep_len > 0", "subsc below min_gc_score", "score == subsc", "mapq bumped from 0 to 1",
                    "mapq capped at 60", "mapq from uniq_ratio < 1"]


# ---------------------------------------------------------------------------------------------------------------
# materialisation family: walks through small graphs, linear chains along them, graph chaining by the reference's mg_gchain1_dp
# ---------------------------------------------------------------------------------------------------------------
def make_graph(rng, workdir):
    """bubbles (s1a/s1b, s6a/s6b), a deletion (s2 -> s4 past s3), an inversion (s4 -> s5 reversed -> s7), a tandem duplication
    (s7 -> s7), short segments of 40-60 bases (s8 ... s13) in a row"""
    L = {"s0": 1500, "s1a": 300, "s1b": 320, "s2": 900, "s3": 400, "s4": 800, "s5": 600, "s6a": 250, "s6b": 260, "s7": 700}
    segs = {n: rnd(rng, ln) for n, ln in L.items()}
    for i in range(8, 14):
        segs["s%d" % i] = rnd(rng, rng.randint(40, 60))
    segs["s14"] = rnd(rng, 1500)
    links = [("s0", "+", "s1a", "+"), ("s0", "+", "s1b", "+"), ("s1a", "+", "s2", "+"), ("s1b", "+", "s2", "+"), ("s2", "+", "s3", "+"),
             ("s3", "+", "s4", "+"), ("s2", "+", "s4", "+"), ("s4", "+", "s5", "+"), ("s4", "+", "s5", "-"), ("s5", "+", "s6a", "+"),
             ("s5", "+", "s6b", "+"), ("s5", "-", "s6a", "+"), ("s6a", "+", "s7", "+"), ("s6b", "+", "s7", "+"), ("s7", "+", "s7", "+"),
             ("s7", "+", "s8", "+")] + [("s%d" % i, "+", "s%d" % (i + 1), "+") for i in range(8, 14)]
    fn = os.path.join(workdir, "walks.gfa")
    names = list(segs)
    write_gfa(fn, [(n, segs[n]) for n in names], links)
    ids = {n: i for i, n in enumerate(names)}
    return fn, segs, ids


WALKS = [["s0", "s1a", "s2", "s3", "s4"], ["s0", "s1b", "s2", "s4", "s5"], ["s2", "s4", "-s5", "s6a", "s7"], ["s6b", "s7", "s7", "s8"],
         ["s7", "s8", "s9", "s10", "s11", "s12", "s13", "s14"], ["s1a", "s2", "s3"], ["s4", "s5", "s6a", "s7", "s7", "s8", "s9"]]


def walk_read(rng, segs, ids, walk, k, rand_gap=0, overlap=0, split=0, step=23, n_seg=1):
    """a read along walk (from inside its first vertex to inside its last) and anchors every ~step bases on each vertex, one linear
    chain per vertex piece (split: the longest piece cut in two, as two linear chains on one vertex).  rand_gap: that many bases of
    random sequence at the junctions, with no anchors.  overlap: the first anchors of each piece moved back onto the piece before (query
    overlap at the junction).  Returns a Read with lc in mg_lchain_gen's order and a before mg_update_anchors."""
    pieces = []
    for i, nm in enumerate(walk):
        rev = nm.startswith("-")
        s = segs[nm.lstrip("-")]
        v = ids[nm.lstrip("-")] << 1 | rev
        vs = revcomp(s) if rev else s
        st = len(vs) // 3 if i == 0 else 0
        en = 2 * len(vs) // 3 if i == len(walk) - 1 else len(vs)
        pieces.append((v, vs, st, en))
    read, groups = b"", []
    for i, (v, vs, st, en) in enumerate(pieces):
        q0 = len(read)
        part = vs[st:en]
        if rand_gap and 0 < i:
            g = min(rand_gap, len(part) // 3)
            part = rnd(rng, g) + part[g:]
            first = g + k
        else:
            first = k
        read += part
        an = []
        p = first - 1
        while p < len(part):
            an.append((q0 + p, st + p))
            p += step + rng.randint(-3, 3)
        if overlap and i > 0 and groups and an:
            pv, pan = groups[-1]
            an = [(q - overlap, r - overlap) for q, r in an[:1] if r - overlap >= k - 1] + an  # an extra anchor behind the junction's query position
        groups.append((v, an))
    if split:
        j = max(range(len(groups)), key=lambda t: len(groups[t][1]))
        v, an = groups[j]
        if len(an) >= 4:
            h = len(an) // 2
            groups[j:j + 1] = [(v, an[:h]), (v, an[h:])]
    anchors = []
    lc_raw = []
    for v, an in groups:
        an = [(q, r) for q, r in an if 0 <= q < len(read)]
        if not an:
            continue
        off = len(anchors)
        anchors += [(v << 32 | r, k << 32 | q) for q, r in an]
        lc_raw.append((off, len(an), v))
    if n_seg > 1:
        cut = len(read) // 2
        segs_r = [read[:cut], read[cut:]]
        anchors = [(x, y | (1 << MG_SEED_SEG_SHIFT if (y & 0xffffffff) >= cut else 0)) for x, y in anchors]
    else:
        segs_r = [read]
    return segs_r, anchors, lc_raw


def lchains_of(anchors, lc_raw, k, rng, extra_mini):
    """mg_lchain_gen's linear chains (sorted by qs, then score) and the anchors after mg_update_anchors"""
    z = []
    for off, cnt, v in lc_raw:
        a0, a1 = anchors[off], anchors[off + cnt - 1]
        qs = (a0[1] & 0xffffffff) + 1 - k
        score = 12 * cnt + rng.randint(0, 5)
        rs = max((a0[0] & 0xffffffff) + 1 - k, 0)
        z.append((qs << 32 | score, (off, cnt, v, rs, (a1[0] & 0xffffffff) + 1, qs, (a1[1] & 0xffffffff) + 1, score, 0, 0, 0)))
    z.sort(key=lambda t: t[0])
    lc = [t for _, t in z]
    pos = sorted(set(y & 0xffffffff for _, y in anchors) | set(extra_mini))
    idx = {p: i for i, p in enumerate(pos)}
    a = [(idx[y & 0xffffffff] << 32 | (x & 0xffffffff), y) for x, y in anchors]
    return lc, a


def gchain1_dp(R, mo, k, qlen, lc, a):
    """the reference's mg_gchain1_dp with map-algo.c:461-462's arguments: (u, lc) as it leaves them"""
    n_lc = C.c_int32(len(lc))
    arr = lc_array(lc)
    u = C.POINTER(C.c_uint64)()
    pen = _libc.expf(f32(-mo.div) * f32(k))
    n_u = ref().mg_gchain1_dp(None, R.g, C.byref(n_lc), arr, qlen, mo.bw_long, mo.bw_long, mo.bw_long, mo.max_gc_skip, mo.ref_bonus,
                              f32(mo.chn_pen_gap) * f32(pen), f32(mo.chn_pen_skip) * f32(pen), mo.mask_level, a_array(a), C.byref(u))
    uu = [u[i] for i in range(n_u)]
    if u:
        _libc.free(C.cast(u, C.c_void_p))
    return uu, [tuple(getattr(arr[i], f) for f in LC_FIELDS) for i in range(n_lc.value)]


def walk_reads(rng, segs, ids, R, mo, k):
    reads = []
    for wi, walk in enumerate(WALKS):
        for variant in ("exact", "random gap", "overlap", "split", "two segments", "random gap + overlap"):
            segs_r, anchors, lc_raw = walk_read(rng, segs, ids, walk, k, rand_gap=150 if "random" in variant else 0,
                                                overlap=30 if "overlap" in variant else 0, split="split" in variant,
                                                n_seg=2 if variant == "two segments" else 1)
            qlen = sum(len(s) for s in segs_r)
            lc, a = lchains_of(anchors, lc_raw, k, rng, rng.sample(range(qlen), 10))
            u, lc2 = gchain1_dp(R, mo, k, qlen, lc, a)
            reads.append(Read(segs_r, rng.getrandbits(32), rng.choice([0, 200]), len(set(y & 0xffffffff for _, y in a)) + 10, u, lc2, a,
                              "walk %d %s" % (wi, variant)))
    # anchors on the ends of a walk through the short segments only: the bridge aligns over a walk of eight vertices
    segs_r, anchors, lc_raw = walk_read(rng, segs, ids, ["s7"] + ["s%d" % i for i in range(8, 15)], k)
    lc_raw = [lc_raw[0], lc_raw[-1]]
    lc, a = lchains_of(anchors, lc_raw, k, rng, [])
    u, lc2 = gchain1_dp(R, mo, k, len(segs_r[0]), lc, a)
    reads.append(Read(segs_r, rng.getrandbits(32), 0, len(a) + 5, u, lc2, a, "anchors on the ends of a long walk"))
    # a walk s0 -> s1a -> s2 under one linear chain on s14 with more anchors: a secondary with more linear chains than its primary
    segs_r, anchors, lc_raw = walk_read(rng, segs, ids, ["s0", "s1a", "s2"], k)
    qlen = len(segs_r[0])
    v14 = ids["s14"] << 1
    an = [(q, 14 + (q - 14) * 1400 // qlen) for q in range(14, qlen, 8)]
    lc_raw.append((len(anchors), len(an), v14))
    anchors += [(v14 << 32 | r, k << 32 | q) for q, r in an]
    lc, a = lchains_of(anchors, lc_raw, k, rng, [])
    u, lc2 = gchain1_dp(R, mo, k, qlen, lc, a)
    reads.append(Read(segs_r, rng.getrandbits(32), 0, len(a) + 5, u, lc2, a, "walk under one linear chain"))
    # many kept chains on one read: pieces of several walks side by side, each its own graph chain
    parts, anchors, lc_raw = [], [], []
    for j in range(80):  # on one vertex at falling offsets: no two of them chain
        nm = "s14"
        s = segs[nm]
        st = len(s) - 210 - 16 * j
        q0 = sum(len(p) for p in parts)
        parts.append(s[st:st + 200])
        off = len(anchors)
        an = [(q0 + p, st + p) for p in range(k - 1, 200, 20 if j % 10 else 150)]  # every tenth below the gates
        anchors += [((ids[nm] << 1) << 32 | r, k << 32 | q) for q, r in an]
        lc_raw.append((off, len(an), ids[nm] << 1))
    read = b"".join(parts)
    lc, a = lchains_of(anchors, lc_raw, k, rng, [])
    u, lc2 = gchain1_dp(R, mo, k, len(read), lc, a)
    reads.append(Read([read], rng.getrandbits(32), 0, len(a) + 5, u, lc2, a, "80 pieces"))
    # s2 -> s3 -> s4 on random sequence: the linear chain on s3 overlaps both neighbours on the query, so that resolve_overlap empties
    # it; the bridge from s2 to s4 over it fails (no alignment, and the shortest walk is not the one the DP took), and the pairs are
    # bridged again one by one
    v2, v3, v4 = (ids[x] << 1 for x in ("s2", "s3", "s4"))
    groups = [(v2, [(p, 400 + p) for p in range(k - 1, 395, 20)]), (v3, [(q, q - 330) for q in list(range(344, 393, 4)) + list(range(484, 545, 3))]),
              (v4, [(q, q - 460) for q in range(474, 860, 20)])]
    anchors, lc_raw = [], []
    for v, an in groups:
        lc_raw.append((len(anchors), len(an), v))
        anchors += [(v << 32 | r, k << 32 | q) for q, r in an]
    lc, a = lchains_of(anchors, lc_raw, k, rng, [])
    u, lc2 = gchain1_dp(R, mo, k, 1000, lc, a)
    reads.append(Read([rnd(rng, 1000)], rng.getrandbits(32), 0, len(a), u, lc2, a, "emptied linear chain"))
    # s0 -> s1a with the first anchor on s1a at the query position of the last one on s0 (resolve_overlap at equality on y)
    v0, v1 = ids["s0"] << 1, ids["s1a"] << 1
    read = segs["s0"][1000:] + segs["s1a"]
    groups = [(v0, [(q, 1000 + q) for q in range(k - 1, 495, 20)]), (v1, [(474, 20)] + [(q, q - 480) for q in range(514, 780, 20)])]
    anchors, lc_raw = [], []
    for v, an in groups:
        lc_raw.append((len(anchors), len(an), v))
        anchors += [(v << 32 | r, k << 32 | q) for q, r in an]
    lc, a = lchains_of(anchors, lc_raw, k, rng, [])
    u, lc2 = gchain1_dp(R, mo, k, len(read), lc, a)
    reads.append(Read([read], rng.getrandbits(32), 0, len(a), u, lc2, a, "tie on y across a junction"))
    return reads


def mat_events(R, reads, mo, seen):
    for rd in reads:
        st = 0
        for x in rd.u:
            n = x & 0xffffffff
            vs = [rd.lc[st + j][2] for j in range(n)]
            m = sum(rd.lc[st + j][1] for j in range(n))
            kept = m >= mo.min_gc_cnt and x >> 32 >= mo.min_gc_score
            seen["graph chains below the gates"] += not kept
            if kept:
                seen["graph chains of %s" % (n if n < 3 else "3+")] += 1
                seen["consecutive linear chains on one vertex"] += sum(1 for j in range(1, n) if vs[j] == vs[j - 1])
                seen["reverse-strand vertex in a graph chain"] += any(v & 1 for v in vs) and n > 1
                seen["two-segment read with a graph chain of 2+"] += len(rd.segs) > 1 and n > 1
            st += n


def case_materialise(lib, seen, rng, workdir):
    k = 15
    fn, segs, ids = make_graph(rng, workdir)
    R = RefGraph(fn)
    g, gi = engine_index(lib, fn, k)
    try:
        _, mo = options.opt_set("lr")
        mo.min_gc_cnt, mo.min_gc_score = 3, 30
        for gdp in (10000, 20):  # with 20, a bridge over random sequence fails and mg_shortest_k is tried
            mo.gdp_max_ed = gdp
            reads = walk_reads(rng, segs, ids, R, mo, k)
            mat_events(R, reads, mo, seen)
            check(lib, gi, R, mo, k, reads, seen, "materialisation, gdp_max_ed %d" % gdp)
    finally:
        lib.mg_idx_destroy(gi)
        lib.mgb_gfa_destroy(g)
        R.close()


MATERIALISE_EDGES = ["bridging jobs aligned", "bridging jobs not aligned", "graph chains of 3+", "y tie at a junction on two vertices",
                     "aligned bridge over a walk of 2 vertices", "aligned bridge over a walk of 3 vertices", "aligned bridge over a walk of 4+ vertices",
                     "one vertex: not contained", "child cnt < parent's", "child cnt > parent's",
                     "consecutive linear chains on one vertex", "reverse-strand vertex in a graph chain", "two-segment read with a graph chain of 2+",
                     "graph chains below the gates", "chains kept per read > 64", "pairs bridged again in place"]


def case_all(lib, workdir):
    rng = random.Random(7)
    seen = collections.Counter()
    case_postfilter(lib, seen, rng, workdir)
    missing = [e for e in POSTFILTER_EDGES if not seen[e]]
    assert not missing, (missing, dict(seen))
    seen2 = collections.Counter()
    case_materialise(lib, seen2, rng, workdir)
    missing = [e for e in MATERIALISE_EDGES if not seen2[e]]
    assert not missing, (missing, dict(seen2))
    return seen, seen2


def test_hook_refuses_bad_input(tmp_path):
    lib = T.load_hostsim()
    rng = random.Random(3)
    fn = os.path.join(str(tmp_path), "one.gfa")
    write_gfa(fn, [("s0", rnd(rng, 2000))], [])
    g, gi = engine_index(lib, fn, 15)
    _, mo = options.opt_set("lr")
    good = chain_read(rng, 500, [(0, 300, 0, 100, 200, 8)], 15, 20, 0, "good")
    try:
        assert run_hook(lib, gi, mo, [good])[0][0][0] == 0
        def bad(why, change):
            r = chain_read(rng, 500, [(0, 300, 0, 100, 200, 8)], 15, 20, 0, why)
            change(r)
            with pytest.raises(AssertionError):
                run_hook(lib, gi, mo, [good, r])
            assert why.encode() in lib.mgb_last_error(), (why, lib.mgb_last_error())
        bad("has a negative count", lambda r: setattr(r, "n_mz", -1))
        bad("do not add up to n_lc", lambda r: setattr(r, "u", [200 << 32 | 2]))
        bad("has a chain of no linear chains", lambda r: setattr(r, "u", [200 << 32, 200 << 32 | 1]))
        bad("has a vertex outside the graph", lambda r: setattr(r, "lc", [r.lc[0][:2] + (2,) + r.lc[0][3:]]))
        bad("is empty", lambda r: (setattr(r, "segs", [b""]), setattr(r, "seq", b"")))
        bad("outside its anchors", lambda r: setattr(r, "a", r.a[:3]))
        bad("has linear chains but no anchors", lambda r: setattr(r, "a", []))
    finally:
        lib.mg_idx_destroy(gi)
        lib.mgb_gfa_destroy(g)


@pytest.mark.parametrize("sim", ["one lane", "32 lanes"])
def test_gchain_gen_in_simulator(sim, tmp_path):
    case_all(T.load_hostsim() if sim == "one lane" else T.load_hostsim32(), str(tmp_path))


@pytest.mark.gpu
def test_gchain_gen_on_gpu(tmp_path):
    case_all(capi.load_product(), str(tmp_path))
