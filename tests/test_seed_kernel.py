"""The seeding kernel k_seed (mgb_pipeline.cuh stage_seed, mgb_seed.cuh), the first kernel every read goes through, checked on its
own: the minimizer sketch (mgb_test_sketch) against the reference's mg_sketch, and the whole stage (mgb_test_seed: minimizers,
index lookup with the occurrence filter and the repeat length, seed expansion with its flags, the seed sort or the heap merge of
the sr preset, the self-diagonal filter of MG_M_NO_DIAG, fragments of several segments) against a restatement of map-algo.c:34-192
whose every leaf is the reference's own (mg_sketch, mg_idx_get on the reference's index of the same graph, radix_sort_128x,
ks_heapmake_heap / ks_heapdown_heap).  Seeds, mini_pos, n_mz and rep_len must be the reference's bit for bit, in the one-lane and
the 32-lane simulators and on the GPU (where the minimizer table is built on the device, here also at key widths other than
k = 17's); every family checks that it reached the edge it is there for."""
import collections
import ctypes as C
import os
import random

import numpy as np
import pytest

import mgtest as T
from minigraph_b200 import capi, options

pytestmark = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")

MG_M_HEAP_SORT, MG_M_NO_DIAG = 0x400, 0x400000
SEED_TANDEM, SEED_SEG_SHIFT, SEED_OCC_SHIFT = 1 << 42, 48, 56
MGB_E_POOL = -2
SKETCH_SMEM_W = 12  # widest window whose rings fit the warp's slice (mgb_seed.cuh)
SORT_ON_CHIP_MAX = 10979  # most seeds whose sort scratch fits the 6 KB slice (stage_seed: n_a / 4 + 3400 <= SKETCH_SMEM_BYTES)
ACGT = b"ACGT"
COMP = bytes.maketrans(b"ACGTacgtN", b"TGCAtgcaN")
NT4 = None  # the reference's seq_nt4_table


class _V(C.Structure):  # minigraph.h:42 mg128_v
    _fields_ = [("n", C.c_size_t), ("m", C.c_size_t), ("a", C.POINTER(capi.mg128_t))]


_lib_c = C.CDLL(None)
_lib_c.free.restype, _lib_c.free.argtypes = None, [C.c_void_p]
_ref = None


def ref():
    global _ref, NT4
    if _ref is None:
        r = T.load_ref()
        r.mg_sketch.restype = None
        r.mg_sketch.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.POINTER(_V)]
        r.radix_sort_128x.restype, r.radix_sort_128x.argtypes = None, [C.c_void_p, C.c_void_p]
        r.ks_heapmake_heap.restype, r.ks_heapmake_heap.argtypes = None, [C.c_size_t, C.c_void_p]
        r.ks_heapdown_heap.restype, r.ks_heapdown_heap.argtypes = None, [C.c_size_t, C.c_size_t, C.c_void_p]
        NT4 = bytes((C.c_ubyte * 256).in_dll(r, "seq_nt4_table"))
        _ref = r
    return _ref


def ref_sketch(s, w, k, rid=0):
    """mg_sketch of bytes s: an (n, 2) array of (x, y)"""
    v = _V(0, 0, None)
    ref().mg_sketch(None, s, len(s), w, k, rid, C.byref(v))
    out = np.ctypeslib.as_array(C.cast(v.a, C.POINTER(C.c_uint64)), shape=(2 * v.n,)).reshape(-1, 2).copy() if v.n else np.zeros((0, 2), np.uint64)
    if v.a:
        _lib_c.free(C.cast(v.a, C.c_void_p))
    return out


def rnd(rng, n):
    return bytes(rng.choices(ACGT, k=n))


def revcomp(s):
    return s.translate(COMP)[::-1]


def mutate(rng, s, rate=0.01):
    b = bytearray(s)
    for i in range(len(b)):
        if rng.random() < rate:
            b[i] = rng.choice(ACGT)
    return bytes(b)


# ---------------------------------------------------------------------------------------------------------------
# the sketch
# ---------------------------------------------------------------------------------------------------------------
def run_sketch(lib, k, w, seqs, mode):
    """mgb_test_sketch: per sequence (rc, path, list as an (n, 2) array)"""
    n = len(seqs)
    offs, o = [], 0
    for s in seqs:
        offs.append(o)
        o += len(s)
    mz_off = [0]
    for s in seqs:  # (the reference's lists hold fewer entries than 2 per base)
        mz_off.append(mz_off[-1] + 2 * len(s) + 64)
    out = (C.c_int32 * (3 * n))()
    mz = (capi.mg128_t * (mz_off[-1] + 1))()
    rc = lib.mgb_test_sketch(k, w, n, b"".join(seqs), (C.c_int64 * n)(*offs), (C.c_int32 * n)(*[len(s) for s in seqs]), mode, out, mz,
                             (C.c_int64 * (n + 1))(*mz_off))
    assert rc == 0, lib.mgb_last_error()
    arr = np.frombuffer(mz, dtype=np.uint64).reshape(-1, 2)
    res = []
    for i in range(n):
        r, cnt, path = out[3 * i:3 * i + 3]
        assert cnt <= mz_off[i + 1] - mz_off[i]
        res.append((r, path, arr[mz_off[i]:mz_off[i] + cnt]))
    return res


def chunking(k, w, n):
    """sketch_seq_w's cut of a sequence of n bases: (number of chunks, chunk length, list capacity per chunk)"""
    min_chunk = max(w + 2 * k, 64)
    n_ch = min(n // min_chunk, 32)
    if n_ch < 2:
        return n_ch, 0, 0
    chunk = (n + n_ch - 1) // n_ch
    return n_ch, chunk, chunk + w + 2


def want_path(k, w, s):
    n_ch, _, _ = chunking(k, w, len(s))
    if k % 2 == 0 or n_ch < 2 or any(NT4[c] >= 4 for c in s):
        return capi.SKETCH_PATH_SEQ
    if w > SKETCH_SMEM_W:
        return capi.SKETCH_PATH_ARENA
    return capi.SKETCH_PATH_SMEM_PK if all(c in ACGT for c in s) else capi.SKETCH_PATH_SMEM


def palindrome(rng, n):
    h = rnd(rng, n // 2)
    return h + revcomp(h)


def sketch_seqs(rng, k, w):
    """(tag, sequence) for one (k, w): lengths at the chunk counts 1, 2, 32 and 33 times the least chunk, +-1; packed and ASCII;
    an N in a chunk's warm-up, on a chunk border and last; homopolymers and tandem repeats; k-mer palindromes around chunk borders;
    sequences shorter than k and than a first window"""
    L = max(w + 2 * k, 64)
    out = []
    for m in (1, 2, 32, 33):
        for d in (-1, 0, 1):
            n = m * L + d
            s = rnd(rng, n)
            out.append(("random m=%d%+d" % (m, d), s))
            lo = bytearray(s)
            for i in rng.sample(range(n), max(1, n // 50)):
                lo[i] = lo[i] | 0x20
            out.append(("lower case m=%d%+d" % (m, d), bytes(lo)))
    for m in (2, 5, 33):
        n = m * L
        n_ch, chunk, _ = chunking(k, w, n)
        for where in ("warm-up", "border", "last"):
            b = bytearray(rnd(rng, n))
            if where == "last":
                b[-1] = ord("N")
            elif n_ch >= 2:
                p = chunk * rng.randint(1, n_ch - 1)
                b[p if where == "border" else max(0, p - rng.randint(1, w + k - 1))] = ord("N")
            out.append(("N in %s m=%d" % (where, m), bytes(b)))
    for m in (3, 33):
        n = m * L
        n_ch, chunk, _ = chunking(k, w, n)
        b = bytearray(rnd(rng, n))
        for c in range(1, max(n_ch, 2)):  # palindromes of 2k..2k+3 bases across and in front of the chunk borders
            p = chunk * c if chunk else n // 2
            pl = palindrome(rng, 2 * k + 2 * rng.randint(0, 1))
            at = max(0, min(n - len(pl), p - rng.choice([len(pl) // 2, len(pl) + rng.randint(0, w)])))
            b[at:at + len(pl)] = pl
        out.append(("palindromes m=%d" % m, bytes(b)))
    for m in (2, 32, 33):
        n = m * L
        out.append(("homopolymer m=%d" % m, bytes([rng.choice(ACGT)]) * n))
        for per in (2, 3, 4, 5, 6):
            unit = rnd(rng, per)
            out.append(("period %d m=%d" % (per, m), (unit * (n // per + 1))[:n]))
        out.append(("tandem runs m=%d" % m, b"".join(rnd(rng, rng.randint(1, 6)) * rng.randint(3, 40) for _ in range(n // 20))[:n] or b"A"))
    for n in sorted({1, k - 1, k, w + k - 2, w + k - 1, w + k} - {0}):
        out.append(("short n=%d" % n, rnd(rng, n)))
    return out


def alphabet_seqs(rng):
    """every byte value: raw codes 0-3, U, lower case and everything else nt4 takes for ambiguous"""
    good = list(ACGT) + list(b"acgtUu") + [0, 1, 2, 3]
    out = [("all bytes", bytes(range(256)) * 8)]
    for _ in range(6):
        out.append(("valid codes", bytes(rng.choice(good) for _ in range(rng.randint(300, 3000)))))
        out.append(("mostly valid", bytes(rng.choice(good) if rng.random() < 0.995 else rng.randrange(256) for _ in range(rng.randint(300, 3000)))))
    out.append(("each byte between bases", b"".join(bytes([c]) + rnd(rng, 40) for c in range(256))))
    return out


def case_sketch(lib, seen, rng, kws):
    for k, w in kws:
        seqs = sketch_seqs(rng, k, w) + (alphabet_seqs(rng) if (k, w) in ((15, 11), (16, 100)) else [])
        got0 = run_sketch(lib, k, w, [s for _, s in seqs], 0)
        got1 = run_sketch(lib, k, w, [s for _, s in seqs], 1)
        for i, ((tag, s), (rc0, path, l0), (rc1, path1, l1)) in enumerate(zip(seqs, got0, got1)):
            what = "k=%d w=%d %s (len %d): " % (k, w, tag, len(s))
            want = ref_sketch(s, w, k, i)
            assert rc0 == 0 and rc1 == 0, what + "rc %d / %d" % (rc0, rc1)
            assert np.array_equal(l0, want), what + "chunked list differs (%d vs %d entries)" % (len(l0), len(want))
            assert np.array_equal(l1, want), what + "sequential list differs (%d vs %d entries)" % (len(l1), len(want))
            assert path1 == -1
            wp = want_path(k, w, s)
            if path != wp:  # the chunked sketch may give up only when a chunk's list is full
                assert path == capi.SKETCH_PATH_SEQ, what + "path %d, expected %d" % (path, wp)
                seen["sketch: a chunk's list overflowed"] += 1
            seen["sketch path %d" % path] += 1
            n_ch, chunk, cap = chunking(k, w, len(s))
            seen["sketch n_ch=%d" % min(n_ch, 3 if n_ch < 32 else 32)] += 1
            if wp != capi.SKETCH_PATH_SEQ and len(want):
                per = collections.Counter(int(y & 0xffffffff) >> 1 for y in want[:, 1].tolist())
                dens = max(sum(v for p, v in per.items() if c * chunk <= p < (c + 1) * chunk) for c in range(n_ch)) / cap
                seen["sketch densest chunk list / cap x100"] = max(seen["sketch densest chunk list / cap x100"], int(dens * 100))
            if "all bytes" in tag or "each byte" in tag:
                seen["sketch: all 256 byte values"] += 1


# ---------------------------------------------------------------------------------------------------------------
# the seeding stage
# ---------------------------------------------------------------------------------------------------------------
REP_COPIES, MID_COPIES, FEW_COPIES = 300, 40, 3


def make_graph(rng, workdir):
    """An rGFA (and the same graph with plain segment names): a stable sequence chr1 of about 30 kb with tandem repeats, cut into
    segments, three bubbles on alt sequences, copies of a 600-base unit (300 times, past the 255 of the occurrence byte), a 500-base
    unit (40 times) and a 700-base unit (3 times) under names of their own, two chr1 segments copied as dup, and tiny segments of
    11 to 31 bases (one k-mer or a few).  Returns the paths and the sequences the reads are taken from."""
    parts = [rnd(rng, 3000)]
    for per in (2, 3, 4, 5, 6, 37):
        parts += [rnd(rng, per) * (900 // per), rnd(rng, 1500)]
    parts.append(rnd(rng, 12000))
    chr1 = b"".join(parts)
    cuts = sorted(rng.sample(range(200, len(chr1) - 200), 14))
    segs = []  # (name, seq, sn, so, sr)
    prev = 0
    for c in cuts + [len(chr1)]:
        segs.append(("c%d" % len(segs), chr1[prev:c], "chr1", prev, 0))
        prev = c
    n_chr = len(segs)
    links = [(segs[i][0], segs[i + 1][0]) for i in range(n_chr - 1)]
    for j in (3, 7, 11):  # bubbles: an alt path around chr1 segment j
        alt = mutate(rng, segs[j][1], 0.05)
        segs.append(("alt%d" % j, alt, "alt%d" % j, 0, 1))
        links += [(segs[j - 1][0], "alt%d" % j), ("alt%d" % j, segs[j + 1][0])]
    units = {"rep": (rnd(rng, 600), REP_COPIES), "mid": (rnd(rng, 500), MID_COPIES), "few": (rnd(rng, 700), FEW_COPIES)}
    for u, (s, n) in units.items():
        for i in range(n):
            segs.append(("%s%d" % (u, i), s, "%s%d" % (u, i), 0, 2))
    so = 0
    for j in (5, 9):  # chr1 segments once more, on a stable sequence of their own
        segs.append(("dup%d" % j, segs[j][1], "dupseq", so, 3))
        so += len(segs[j][1])
    tiny = []
    for ln in range(11, 32):
        for _ in range(2):
            t = rnd(rng, ln)
            tiny.append(t)
            segs.append(("tiny%d" % len(tiny), t, "tiny%d" % len(tiny), 0, 4))
    paths = {}
    for kind in ("rgfa", "plain"):
        fn = os.path.join(workdir, "sv.%s.gfa" % kind)
        with open(fn, "w") as f:
            for name, s, sn, off, sr in segs:
                tags = "\tLN:i:%d" % len(s) + ("\tSN:Z:%s\tSO:i:%d\tSR:i:%d" % (sn, off, sr) if kind == "rgfa" else "")
                f.write("S\t%s\t%s%s\n" % (name, s.decode(), tags))
            for a, b in links:
                f.write("L\t%s\t+\t%s\t+\t0M\n" % (a, b))
        paths[kind] = fn
    return paths, dict(chr1=chr1, segs=segs, units={u: s for u, (s, _) in units.items()}, tiny=tiny, tr_at=3000)


class RefIndex:
    """the reference's own gfa_read + mg_index of a graph at (k, w), and what collect_seed_hits reads of the graph"""

    def __init__(self, gfa, k, w):
        r = ref()
        self.k, self.w = k, w
        self.g = r.gfa_read(gfa.encode())
        assert self.g
        io, mo = options.opt_set("lr")
        io.k, io.w = k, w
        self.gi = r.mg_index(self.g, C.byref(io), 1, C.byref(mo))
        assert self.gi
        gs = self.g.contents
        self.seg_len, self.gname, self.soff = [], [], []
        for i in range(gs.n_seg):
            s = gs.seg[i]
            stable = s.snid >= 0 and bool(gs.sseq)
            self.seg_len.append(s.len)
            self.gname.append(gs.sseq[s.snid].name if stable else s.name)  # map-algo.c:168-174
            self.soff.append(s.soff if stable else 0)
        self.cache = {}

    def get(self, key):
        if key not in self.cache:
            t = C.c_int(0)
            p = ref().mg_idx_get(self.gi, key, C.byref(t))
            self.cache[key] = [p[j] for j in range(t.value)]
        return self.cache[key]

    def close(self):
        ref().mg_idx_destroy(self.gi)
        ref().gfa_destroy(self.g)


def ref_seed(ix, name, segs, flag, occ_max1, max_qlen, ev):
    """map-algo.c:34-192 with the reference's leaves: (status, n_mz, rep_len, anchors, mini_pos); counts the edges reached in ev"""
    qlen = sum(len(s) for s in segs)
    if qlen == 0 or (max_qlen > 0 and qlen > max_qlen):  # map-algo.c:350-352: not mapped
        return 1, 0, 0, [], []
    mv, tot = [], 0
    for i, s in enumerate(segs):  # collect_minimizers
        for x, y in ref_sketch(s, ix.w, ix.k, i).tolist():
            mv.append((x, y + (tot << 1)))
        tot += len(s)
    m, mp = [], []  # collect_matches
    rep_len = rep_st = rep_en = 0
    groups = set()
    for i, (x, y) in enumerate(mv):
        q_pos, q_span = y & 0xffffffff, x & 0xff
        cr = ix.get(x >> 8)
        t = len(cr)
        if t >= occ_max1:
            en = (q_pos >> 1) + 1
            st = en - q_span
            if st > rep_en:
                rep_len += rep_en - rep_st
                ev["rep run across 32-minimizer groups"] += len(groups) > 1
                ev["rep runs disjoint"] += rep_en > 0
                rep_st, rep_en, groups = st, en, {i >> 5}
            else:
                rep_en = en
                groups.add(i >> 5)
                ev["rep runs overlap"] += 1
        else:
            tandem = (i > 0 and mv[i - 1][0] >> 8 == x >> 8) or (i < len(mv) - 1 and mv[i + 1][0] >> 8 == x >> 8)
            m.append((t, q_pos, q_span, y >> 32, tandem, cr))
            mp.append(q_pos >> 1)
    rep_len += rep_en - rep_st
    ev["rep run across 32-minimizer groups"] += len(groups) > 1

    def anchor(q, r):
        t, q_pos, q_span, seg_id, tandem, _ = q
        rpos = (r & 0xffffffff) >> 1
        if (r & 1) == (q_pos & 1):
            x = r >> 32 << 33 | rpos
        else:
            x = r >> 32 << 33 | 1 << 32 | ((ix.seg_len[r >> 32] - (rpos + 1 - q_span) - 1) & 0xffffffff)
        y = q_span << 32 | q_pos >> 1 | seg_id << SEED_SEG_SHIFT | (SEED_TANDEM if tandem else 0) | min(t, 255) << SEED_OCC_SHIFT
        return x, y

    n_a = sum(q[0] for q in m)
    if flag & MG_M_HEAP_SORT:  # collect_seed_hits_heap
        words = collections.Counter(r for q in m for r in q[5])
        ev["heap: target words shared by matches"] += sum(c > 1 for c in words.values())
        heap = (capi.mg128_t * max(len(m), 1))()
        hs = 0
        for i, q in enumerate(m):
            if q[0] > 0:
                heap[hs].x, heap[hs].y = q[5][0], i << 32
                hs += 1
        ref().ks_heapmake_heap(hs, heap)
        a = [None] * n_a
        n_for = n_rev = 0
        while hs > 0:
            q = m[heap[0].y >> 32]
            r = heap[0].x
            if (r & 1) == (q[1] & 1):
                a[n_for] = anchor(q, r)
                n_for += 1
            else:
                n_rev += 1
                a[n_a - n_rev] = anchor(q, r)
            if (heap[0].y & 0xffffffff) < q[0] - 1:
                heap[0].y += 1
                heap[0].x = m[heap[0].y >> 32][5][heap[0].y & 0xffffffff]
            else:
                heap[0] = heap[hs - 1]
                hs -= 1
            ref().ks_heapdown_heap(0, hs, heap)
        return 0, len(mv), rep_len, a, mp
    a = []  # collect_seed_hits
    for q in m:
        for r in q[5]:
            if name is not None and flag & MG_M_NO_DIAG:
                g_pos = (ix.soff[r >> 32] + (r & 0xffffffff)) & 0xffffffff
                if g_pos == q[1] and name == ix.gname[r >> 32]:
                    ev["no_diag: seeds dropped"] += 1
                    continue
                ev["no_diag: seeds kept" + (" on the read's own sequence" if name == ix.gname[r >> 32] else "")] += 1
            a.append(anchor(q, r))
    buf = (capi.mg128_t * max(len(a), 1))()
    for j, (x, y) in enumerate(a):
        buf[j].x, buf[j].y = x, y
    ref().radix_sort_128x(C.addressof(buf), C.addressof(buf) + 16 * len(a))
    arr = np.frombuffer(buf, dtype=np.uint64).reshape(-1, 2)[:len(a)]
    return 0, len(mv), rep_len, [tuple(e) for e in arr.tolist()], mp


def run_seed(lib, gi, reads, flag, occ_max1, max_qlen):
    """mgb_test_seed on [(name, [segments])]: per read (status, n_mz, rep_len, anchors, mini_pos)"""
    n = len(reads)
    frag = any(len(segs) > 1 for _, segs in reads)
    qlens = (C.c_int * n)(*[sum(len(s) for s in segs) for _, segs in reads])
    seqs = (C.c_char_p * n)(*[b"".join(segs) for _, segs in reads])
    names = (C.c_char_p * n)(*[nm.encode() if isinstance(nm, str) else nm for nm, _ in reads])
    seg_off = seg_len = None
    if frag:
        offs, lens = [0], []
        for _, segs in reads:
            lens += [len(s) for s in segs]
            offs.append(len(lens))
        seg_off, seg_len = (C.c_int32 * (n + 1))(*offs), (C.c_int32 * len(lens))(*lens)
    out = (C.c_int32 * (5 * n))()
    a_cap, mp_cap = 1 << 16, 1 << 16
    for _ in range(2):
        a, mp = (capi.mg128_t * a_cap)(), (C.c_int32 * mp_cap)()
        rc = lib.mgb_test_seed(gi, n, qlens, seqs, seg_off, seg_len, names, flag, occ_max1, max_qlen, out, a, a_cap, mp, mp_cap)
        if rc != MGB_E_POOL:
            break
        a_cap = sum(out[5 * i + 3] for i in range(n) if out[5 * i] == 0) + 1
        mp_cap = sum(out[5 * i + 4] for i in range(n) if out[5 * i] == 0) + 1
    assert rc == 0, (rc, lib.mgb_last_error())
    arr = np.frombuffer(a, dtype=np.uint64).reshape(-1, 2)
    res, sa, smp = [], 0, 0
    for i in range(n):
        st, n_mz, rep_len, n_a, n_mp = out[5 * i:5 * i + 5]
        if st != 0:
            res.append((st, n_mz, rep_len, [], []))
            continue
        res.append((st, n_mz, rep_len, [tuple(e) for e in arr[sa:sa + n_a].tolist()], list(mp[smp:smp + n_mp])))
        sa, smp = sa + n_a, smp + n_mp
    return res


def check_seeds(lib, gi, ix, reads, flag, occ_max1, max_qlen, seen, what):
    got = run_seed(lib, gi, reads, flag, occ_max1, max_qlen)
    for (name, segs), (st, n_mz, rep_len, a, mp) in zip(reads, got):
        ev = collections.Counter()
        w_st, w_mz, w_rep, w_a, w_mp = ref_seed(ix, name, segs, flag, occ_max1, max_qlen, ev)
        tag = "%s, read %r (%d segments, %d bases): " % (what, name, len(segs), sum(len(s) for s in segs))
        assert st == w_st, tag + "status %d, reference %d" % (st, w_st)
        assert (n_mz, rep_len) == (w_mz, w_rep), tag + "n_mz, rep_len %r, reference %r" % ((n_mz, rep_len), (w_mz, w_rep))
        assert mp == w_mp, tag + "mini_pos differ"
        assert len(a) == len(w_a), tag + "n_a %d, reference %d" % (len(a), len(w_a))
        assert a == w_a, tag + "seeds differ first at %d: %r vs %r" % next((j, a[j], w_a[j]) for j in range(len(a)) if a[j] != w_a[j])
        seen.update({k: v for k, v in ev.items() if v})
        seen["status %d" % st] += 1
        if st != 0:
            continue
        seen["seeds: none but minimizers"] += n_mz > 0 and not a
        if not flag & (MG_M_HEAP_SORT | MG_M_NO_DIAG) and a:
            seen["sort scratch on chip" if len(a) <= SORT_ON_CHIP_MAX else "sort scratch in the arena"] += 1
            if len(a) in (SORT_ON_CHIP_MAX, SORT_ON_CHIP_MAX + 1):
                seen["n_a = %d" % len(a)] += 1
        for x, y in a:
            seen["occurrence byte saturated"] += y >> SEED_OCC_SHIFT == 255  # (only the 300-copy unit has 255 or more)
            seen["tandem flag"] += bool(y & SEED_TANDEM)
            seen["segment id %d" % min(y >> SEED_SEG_SHIFT & 0xff, 2)] += 1
            if x >> 32 & 1:
                span, t = y >> 32 & 0xff, x & 0xffffffff
                ln = ix.seg_len[x >> 33]
                seen["reverse hit: k-mer ends at the segment's last base"] += t == span - 1
                seen["reverse hit: k-mer starts at the segment's first base"] += t == ln - 1
    return got


def seed_reads(rng, G, k, w, max_qlen):
    chr1, u = G["chr1"], G["units"]

    def piece(n):
        p = rng.randrange(len(chr1) - n)
        return chr1[p:p + n]
    reads = []
    for i in range(8):  # unique stretches, both strands, with substitutions
        s = mutate(rng, piece(rng.randint(500, 5000)))
        reads.append(("u%d" % i, [revcomp(s) if i % 2 else s]))
    s = bytearray(piece(3000))
    for j in rng.sample(range(len(s)), 20):
        s[j] = ord("N")
    reads.append(("with N", [bytes(s)]))
    s = bytearray(piece(3000))
    for j in rng.sample(range(len(s)), 300):
        s[j] |= 0x20
    reads.append(("lower case", [bytes(s)]))
    at = G["tr_at"]
    for i in range(4):  # the tandem repeats of chr1 (periods 2-6 and 37) with their flanks
        st = at + 2400 * i
        reads.append(("tandem%d" % i, [mutate(rng, chr1[st - 300:st + 1200], 0.003)]))
    for t in G["tiny"]:  # one k-mer or a few: hits at both ends of a segment, on both strands
        if k <= len(t) <= k + 3:
            reads += [("tiny", [t]), ("tiny rc", [revcomp(t)])]
    rep, mid, few = u["rep"], u["mid"], u["few"]
    reads.append(("rep runs disjoint", [piece(300) + rep[:600] + piece(200) + rep[100:500] + piece(300)]))
    reads.append(("rep runs back to back", [rep + rep[200:] + mid + few + piece(400)]))
    reads.append(("occurrences 3 and 40", [piece(200) + few + piece(200) + mid + piece(200)]))
    reads.append(("stranger", [rnd(rng, 2000)]))
    reads.append(("empty", [b""]))
    reads.append(("at max_qlen", [piece(max_qlen)]))
    reads.append(("over max_qlen", [piece(max_qlen + 1)]))
    return reads


def sort_edge_reads(ix, G, occ_max1):
    """reads whose seeds number just below and just at the sort-scratch switch (n_a = 10979 / 10980 where it can be hit): copies of
    the 300-copy unit and a unique tail grown base by base"""
    chr1, rep = G["chr1"], G["units"]["rep"]

    def n_a(s):  # collect_matches' count
        return sum(t for t in (len(ix.get(x >> 8)) for x in ref_sketch(s, ix.w, ix.k)[:, 0].tolist()) if t < occ_max1)
    base = b""
    for cut in range(20, len(rep) + 1, 10):
        if n_a(rep[:cut]) > SORT_ON_CHIP_MAX - 400:
            break
        base = rep[:cut]
    out, tail0 = [], 5000
    for extra in range(0, 4000, 7):
        s = base + chr1[tail0:tail0 + extra]
        v = n_a(s)
        if v in (SORT_ON_CHIP_MAX, SORT_ON_CHIP_MAX + 1) and v not in [x for x, _ in out]:
            out.append((v, s))
        if v > SORT_ON_CHIP_MAX + 300:
            break
    if len(out) < 2:  # no exact hit: the nearest on both sides
        below = max((x for x in range(0, 4000, 7) if n_a(base + chr1[tail0:tail0 + x]) <= SORT_ON_CHIP_MAX), default=0)
        out = [(0, base + chr1[tail0:tail0 + below]), (0, base + chr1[tail0:tail0 + below + 7]), (0, rep + rep[:200])]
    return [("sort edge", [s]) for _, s in out] + [("sort far", [rep + rep[:300]])]


def with_engine_index(lib, gfa, k, w):
    g = lib.mgb_gfa_read(gfa.encode())
    assert g
    io, mo = options.opt_set("lr")
    io.k, io.w = k, w
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    return g, gi


def case_seeds(lib, seen, rng, paths, G, k, w, full):
    """the seeding stage on one index: occ_max1 below the 300 copies (repeat length), above them (saturated occurrence byte, the
    sort-scratch switch), the heap merge; with full, also MG_M_NO_DIAG on the rGFA and the plain GFA, and fragments"""
    max_qlen = 6000
    ix = RefIndex(paths["rgfa"], k, w)
    g, gi = with_engine_index(lib, paths["rgfa"], k, w)
    try:
        reads = seed_reads(rng, G, k, w, max_qlen)
        what = "k=%d w=%d" % (k, w)
        check_seeds(lib, gi, ix, reads, 0, 50, max_qlen, seen, what + " occ_max1=50")
        high = [r for r in reads if not r[0].startswith("rep runs")] + sort_edge_reads(ix, G, 1000)
        check_seeds(lib, gi, ix, high, 0, 1000, 0, seen, what + " occ_max1=1000")
        heap = [r for r in reads if not r[0].startswith("rep runs")]
        check_seeds(lib, gi, ix, heap, MG_M_HEAP_SORT, 50, max_qlen, seen, what + " heap merge")
        if full:
            chr1, segs = G["chr1"], G["segs"]
            c = [s for s in segs if s[2] == "chr1"]
            nd = []
            for j in (0, 2, 5):  # a piece of chr1 named chr1: from the start, from a segment's offset and from half of it (SO is added to lastPos<<1|strand)
                for st in (c[j][3], c[j][3] // 2):
                    nd.append((b"chr1", [chr1[st:st + 1500]]))
            nd += [(b"chr1", [revcomp(chr1[:1500])]), (b"alt3", [segs[[s[0] for s in segs].index("alt3")][1][:900]]),
                   (b"dupseq", [c[5][1][:800]]), (b"stranger", [chr1[:1500]]), (None, [chr1[:1500]])]
            check_seeds(lib, gi, ix, nd, MG_M_NO_DIAG, 50, 0, seen, what + " NO_DIAG on the rGFA")
            frags = []
            for n_seg in (2, 3, 2, 3):
                parts = []
                for _ in range(n_seg):
                    ln = rng.choice([5, 150, 600, 2000])
                    p = rng.randrange(len(chr1) - ln)
                    s = chr1[p:p + ln]
                    parts.append(revcomp(s) if rng.random() < 0.5 else s)
                frags.append(("frag", parts))
            frags.append(("frag with rep", [G["units"]["mid"], chr1[100:700]]))
            frags.append(("one segment", [chr1[900:2000]]))
            check_seeds(lib, gi, ix, frags, 0, 50, 0, seen, what + " fragments")
            check_seeds(lib, gi, ix, frags, MG_M_HEAP_SORT, 50, 0, seen, what + " fragments, heap merge")
            with_n = []
            for i in range(65):  # more than 64 reads with other letters: the whole batch goes up as ASCII
                p = rng.randrange(len(chr1) - 1000)
                s = bytearray(chr1[p:p + 1000])
                s[rng.randrange(1000)] = ord("N")
                with_n.append(("N %d" % i, [bytes(s)]))
            check_seeds(lib, gi, ix, with_n, 0, 50, 0, seen, what + " a batch uploaded as ASCII")
    finally:
        lib.mg_idx_destroy(gi)
        lib.mgb_gfa_destroy(g)
        ix.close()
    if full:  # the same on the plain GFA: segments go by their own names
        ix = RefIndex(paths["plain"], k, w)
        g, gi = with_engine_index(lib, paths["plain"], k, w)
        try:
            segs = G["segs"]
            nd = []
            for name, s, *_ in segs[:6]:
                nd += [(name.encode(), [s[:1200]]), (name.encode(), [s[100:1300]]), (name.encode(), [revcomp(s[:1200])])]
            nd.append((b"someone", [segs[0][1][:1200]]))
            check_seeds(lib, gi, ix, nd, MG_M_NO_DIAG, 50, 0, seen, "k=%d w=%d NO_DIAG on the plain GFA" % (k, w))
        finally:
            lib.mg_idx_destroy(gi)
            lib.mgb_gfa_destroy(g)
            ix.close()


SKETCH_KW = [(k, w) for k in (11, 15, 16, 27, 28) for w in (1, 2, 11, 12, 13, 100, 255)]
INDEX_KW = [(17, 11), (11, 5), (16, 13), (28, 30)]


def check_sketch_reached(seen):
    need = ["sketch path %d" % p for p in range(4)] + ["sketch n_ch=0", "sketch n_ch=2", "sketch n_ch=32", "sketch: all 256 byte values"]
    missing = [k for k in need if not seen[k]]
    assert not missing, (missing, seen)


def check_seeds_reached(seen):
    need = ["occurrence byte saturated", "rep run across 32-minimizer groups", "rep runs overlap", "rep runs disjoint", "tandem flag",
            "reverse hit: k-mer ends at the segment's last base", "reverse hit: k-mer starts at the segment's first base",
            "sort scratch on chip", "sort scratch in the arena", "seeds: none but minimizers", "status 1",
            "heap: target words shared by matches", "no_diag: seeds dropped", "no_diag: seeds kept on the read's own sequence",
            "segment id 1", "segment id 2"]
    missing = [k for k in need if not seen[k]]
    assert not missing, (missing, seen)
    assert not seen["status -1"] and not seen["status -3"]


def case_all(lib, workdir, sketch_kw=SKETCH_KW, index_kw=INDEX_KW):
    rng = random.Random(11)
    seen = collections.Counter()
    case_sketch(lib, seen, rng, sketch_kw)
    check_sketch_reached(seen)
    paths, G = make_graph(rng, workdir)
    for i, (k, w) in enumerate(index_kw):
        case_seeds(lib, seen, rng, paths, G, k, w, full=i == 0)
    check_seeds_reached(seen)
    return seen


def test_hooks_refuse_bad_input():
    lib = T.load_hostsim()
    out, mz = (C.c_int32 * 3)(), (capi.mg128_t * 4)()
    one64, one32 = (C.c_int64 * 2)(0, 4), (C.c_int32 * 1)(1)
    for k, w, mode, ln in ((0, 5, 0, 1), (29, 5, 0, 1), (15, 0, 0, 1), (15, 256, 0, 1), (15, 5, 2, 1), (15, 5, 0, 0)):
        one32[0] = ln
        assert lib.mgb_test_sketch(k, w, 1, b"ACGT", one64, one32, mode, out, mz, (C.c_int64 * 2)(0, 4)) < 0
    g = lib.mgb_gfa_read(os.path.join(T.FIX, "MT.gfa").encode())
    io, mo = options.opt_set("lr")
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    o5 = (C.c_int32 * 5)()
    a, mp = (capi.mg128_t * 4)(), (C.c_int32 * 4)()
    seqs = (C.c_char_p * 1)(b"ACGTACGTAC")
    for qlen, segs in ((-1, None), (10, ([0, 2], [10, 0])), (10, ([0, 1], [9]))):
        so, sl = ((C.c_int32 * 2)(*segs[0]), (C.c_int32 * 2)(*segs[1])) if segs else (None, None)
        assert lib.mgb_test_seed(gi, 1, (C.c_int * 1)(qlen), seqs, so, sl, None, 0, 50, 0, o5, a, 4, mp, 4) < 0
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)


@pytest.mark.parametrize("sim", ["one lane", "32 lanes"])
def test_seed_kernel_in_simulator(sim, tmp_path):
    case_all(T.load_hostsim() if sim == "one lane" else T.load_hostsim32(), str(tmp_path))


@pytest.mark.gpu
def test_seed_kernel_on_gpu(tmp_path):
    case_all(capi.load_product(), str(tmp_path))
