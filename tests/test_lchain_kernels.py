"""Linear chaining as k_chain and k_chain_rescue run it (mgb_pipeline.cuh chain_staged + chain_run): the DP of the lr preset, the
RMQ chaining of asm and the rescue pass (sort back into target order, RMQ), each checked against the reference's mg_lchain_dp /
mg_lchain_rmq on anchor sets built to sit on the edges of the kernels: the sizes where the seeds and the hot arrays stop fitting
the shared-memory slice, the window borders, the max_iter cut and the skip stop on the lanes of a 32-candidate chunk, score ties,
priority ties (the AVL replay), the cap on the RMQ tree.  The chains (u[]) and the compacted anchors must be the reference's bit
for bit, in the one-lane and the 32-lane simulators and on the GPU; every family checks that it reached its edge."""
import collections
import ctypes as C
import random

import numpy as np
import pytest

import mgtest as T
from minigraph_b200 import capi

pytestmark = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")

F32 = np.float32
# per-set options; the RMQ chaining reads max_dist_x as its max_dist (lr / asm presets: options.py)
LR = dict(max_dist_x=5000, max_dist_y=5000, bw=500, max_skip=25, max_iter=5000, min_cnt=5, min_sc=40, pen_gap=1.0, pen_skip=0.05,
          is_cdna=0, n_seg=1, max_dist_inner=1000, cap_rmq_size=100000)
LOOSE = dict(LR, min_cnt=1, min_sc=1)  # every anchor is an end point: f[] and p[] show through u[] and the anchors
SLICE = {capi.LCHAIN_DP: 16 * 1024, capi.LCHAIN_RMQ: 16 * 1024, capi.LCHAIN_RESCUE: 18 * 1024}  # CHAIN_SMEM_BYTES, CHAIN_RESCUE_SMEM_BYTES
WARPS = {capi.LCHAIN_DP: 7, capi.LCHAIN_RMQ: 7, capi.LCHAIN_RESCUE: 6}  # warps per block of k_chain / k_chain_rescue


def anc(t, q, span=15, tid=0, rev=0, seg=0):
    """an anchor as the seed expansion writes it: x = tid<<33 | rev<<32 | tpos, y = seg<<48 | q_span<<32 | qpos"""
    return (tid << 33 | rev << 32 | t, seg << 48 | span << 32 | q)


def opts(base=LOOSE, **kw):
    return dict(base, **kw)


def chain(rng, n, t0, q0, step=(10, 40), jit=3, span=15, **kw):
    out, t, q = [], t0, q0
    for _ in range(n):
        out.append(anc(t, q, span, **kw))
        d = rng.randint(*step)
        t, q = t + d, q + max(1, d + rng.randint(-jit, jit))
    return out


def by_x(a):
    return sorted(a, key=lambda e: e[0])  # (stable: equal x keep the order they were built in)


def s32(v):
    v &= 0xffffffff
    return v - (1 << 32) if v >> 31 else v


# ---- the reference's scoring and DP loop in Python, to count which edges a set reaches (lchain.c:114-219) ----
def _log2(x):  # mg_log2, float32 throughout
    i = int(np.array([x], dtype=F32).view(np.uint32)[0])
    lg = F32(((i >> 23) & 255) - 128)
    z = np.array([(i & ~(255 << 23)) + (127 << 23)], dtype=np.uint32).view(F32)[0]
    return F32(lg + F32(F32(F32(F32(F32(-0.34484843) * z) + F32(2.02466578)) * z) - F32(0.67487759)))


def score(ai, aj, o, mdx, mdy):
    dq = s32(ai[1]) - s32(aj[1])
    si, sj = ai[1] >> 48 & 0xff, aj[1] >> 48 & 0xff
    if dq <= 0 or dq > mdx:
        return None
    dr = s32(ai[0] - aj[0])
    if si == sj and (dr == 0 or dq > mdy):
        return None
    dd = dr - dq if dr > dq else dq - dr
    if si == sj and dd > o["bw"]:
        return None
    if o["n_seg"] > 1 and not o["is_cdna"] and si == sj and dr > mdy:
        return None
    dg = min(dr, dq)
    qs = aj[1] >> 32 & 0xff
    sc = min(qs, dg)
    if dd or dg > qs:
        lin = F32(F32(F32(o["pen_gap"]) * F32(dd)) + F32(F32(o["pen_skip"]) * F32(dg)))
        lg = _log2(F32(dd + 1)) if dd >= 1 else F32(0)
        half = F32(lin + F32(F32(0.5) * lg))
        if o["is_cdna"] or si != sj:
            if si != sj and dr == 0:
                sc += 1
            elif dr > dq or si != sj:
                sc -= int(lin if lin < lg else lg)
            else:
                sc -= int(half)
        else:
            sc -= int(half)
    return sc


def walk_dp(a, o, ev):
    """mg_lchain_dp's fill loop, counting where the max_iter cut and the skip stop fall in the kernel's chunks of 32 predecessors
    (chunk c holds j = i-1-32c-lane), and the ties the first-maximum rules decide"""
    n, bw = len(a), o["bw"]
    mdx = max(o["max_dist_x"], bw)
    mdy = o["max_dist_y"] if o["max_dist_y"] >= bw or o["is_cdna"] else bw
    f, p, t = [0] * n, [-1] * n, [0] * n
    st, max_ii = 0, -1
    for i in range(n):
        xi, yi = a[i]
        max_j, max_f, n_skip = -1, yi >> 32 & 0xff, 0
        while st < i and (xi >> 32 != a[st][0] >> 32 or xi > a[st][0] + mdx):
            st += 1
        if st > 0 and xi >> 32 == a[st - 1][0] >> 32 and xi - a[st - 1][0] == mdx + 1:
            ev["window: x - x[st-1] = max_dist+1"] += 1
        if st < i:
            ev["window: x - x[st] = max_dist"] += xi - a[st][0] == mdx
        cut = i - st > o["max_iter"]
        if cut:
            st = i - o["max_iter"]
            ev["max_iter cut, %d left in the last chunk" % ((o["max_iter"] - 1) % 32 + 1)] += 1
        j, tops = i - 1, collections.Counter()
        while j >= st:
            sc = score(a[i], a[j], o, mdx, mdy)
            if sc is not None:
                sc += f[j]
                tops[sc] += 1
                if sc > max_f:
                    max_f, max_j = sc, j
                    if n_skip > 0:
                        n_skip -= 1
                elif t[j] == i:
                    n_skip += 1
                    if n_skip > o["max_skip"]:
                        ev["skip stop on lane %d" % ((i - 1 - j) % 32)] += 1
                        break
                if p[j] >= 0:
                    t[p[j]] = i
            j -= 1
        if max_j >= 0 and tops[max_f] > 1:
            ev["best predecessor tied"] += 1
        if cut and max_j == st:
            ev["best predecessor at the cut, %d left in the last chunk" % ((o["max_iter"] - 1) % 32 + 1)] += 1
        end_j = j
        if max_ii < 0 or xi - a[max_ii][0] > mdx:
            if max_ii >= 0:
                ev["max_ii recomputed at max_dist+%d" % min(xi - a[max_ii][0] - mdx, 2)] += 1
            mx, max_ii = -(1 << 31), -1
            for j in range(i - 1, st - 1, -1):
                if mx < f[j]:
                    mx, max_ii = f[j], j
            ev["max_ii tied"] += max_ii >= 0 and sum(f[j] == mx for j in range(st, i)) > 1
        if max_ii >= 0 and max_ii < end_j:
            tmp = score(a[i], a[max_ii], o, mdx, mdy)
            ev["max_ii after a skip stop"] += 1
            if tmp is not None and max_f < tmp + f[max_ii]:
                max_f, max_j = tmp + f[max_ii], max_ii
                ev["max_ii taken"] += 1
        f[i], p[i] = max_f, max_j
        if max_ii < 0 or (xi - a[max_ii][0] <= mdx and f[max_ii] < f[i]):
            max_ii = i
        elif xi - a[max_ii][0] <= mdx and f[max_ii] == f[i]:
            ev["max_ii kept over an equal f"] += 1
    ends = collections.Counter(v for v in f if v >= o["min_sc"])
    ev["end points tied"] += any(c > 1 for c in ends.values())


# ---- the two sides ----
def check_input(mode, a):
    """the preconditions of the pipeline, which the reference asserts"""
    for x, y in a:
        assert 0 <= s32(y) and 1 <= (y >> 32 & 0xff) <= 255, (x, y)
    if mode != capi.LCHAIN_RESCUE:
        assert all(a[k][0] <= a[k + 1][0] for k in range(len(a) - 1)), "anchors not sorted by x"


_libc = None


def ref_lchain(mode, a, o):
    global _libc
    ref = T.load_ref()
    if _libc is None:
        _libc = C.CDLL(None)
        _libc.malloc.restype, _libc.malloc.argtypes = C.c_void_p, [C.c_size_t]
        _libc.free.restype, _libc.free.argtypes = None, [C.c_void_p]
        u64pp = C.POINTER(C.POINTER(C.c_uint64))
        ref.mg_lchain_dp.restype = C.c_void_p
        ref.mg_lchain_dp.argtypes = [C.c_int] * 7 + [C.c_float, C.c_float, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.POINTER(C.c_int), u64pp, C.c_void_p]
        ref.mg_lchain_rmq.restype = C.c_void_p
        ref.mg_lchain_rmq.argtypes = [C.c_int] * 7 + [C.c_float, C.c_float, C.c_int64, C.c_void_p, C.POINTER(C.c_int), u64pp, C.c_void_p]
        ref.radix_sort_128x.restype, ref.radix_sort_128x.argtypes = None, [C.c_void_p, C.c_void_p]
    n = len(a)
    buf = _libc.malloc(16 * max(n, 1))  # km == NULL: the reference free()s its input and returns malloc()ed a[] and u[]
    arr = (capi.mg128_t * max(n, 1)).from_address(buf)
    for k, (x, y) in enumerate(a):
        arr[k].x, arr[k].y = x, y
    if mode == capi.LCHAIN_RESCUE:
        ref.radix_sort_128x(buf, buf + 16 * n)  # map-algo.c:413-414
    n_u, u = C.c_int(0), C.POINTER(C.c_uint64)()
    if mode == capi.LCHAIN_DP:
        res = ref.mg_lchain_dp(o["max_dist_x"], o["max_dist_y"], o["bw"], o["max_skip"], o["max_iter"], o["min_cnt"], o["min_sc"], o["pen_gap"],
                               o["pen_skip"], o["is_cdna"], o["n_seg"], n, buf, C.byref(n_u), C.byref(u), None)
    else:
        res = ref.mg_lchain_rmq(o["max_dist_x"], o["max_dist_inner"], o["bw"], o["max_skip"], o["cap_rmq_size"], o["min_cnt"], o["min_sc"], o["pen_gap"],
                                o["pen_skip"], n, buf, C.byref(n_u), C.byref(u), None)
    us = [u[k] for k in range(n_u.value)]
    n_v = sum(v & 0xffffffff for v in us)
    out = []
    if res:
        ra = (capi.mg128_t * max(n_v, 1)).from_address(res)
        out = [(ra[k].x, ra[k].y) for k in range(n_v)]
    _libc.free(res)
    _libc.free(C.cast(u, C.c_void_p))
    return us, out


def run_lchain(lib, mode, sets):
    """mgb_test_lchain on [(tag, anchors, opts)]: per set (rc, n_u, n_v, staged, path, worker, u[], anchors[])"""
    n = len(sets)
    offs, k = [], 0
    for _, a, _ in sets:
        offs.append(k)
        k += len(a)
    tot = max(k, 1)
    aa, ao = (capi.mg128_t * tot)(), (capi.mg128_t * tot)()
    for (_, a, _), off in zip(sets, offs):
        for j, (x, y) in enumerate(a):
            aa[off + j].x, aa[off + j].y = x, y
    oo = (capi.mgb_lchain_opt_t * max(n, 1))()
    for s, (_, _, o) in enumerate(sets):
        for key, v in o.items():
            setattr(oo[s], key, v)
    out, u = (C.c_int32 * (6 * max(n, 1)))(), (C.c_uint64 * tot)()
    rc = lib.mgb_test_lchain(mode, n, aa, (C.c_int64 * max(n, 1))(*offs), (C.c_int32 * max(n, 1))(*[len(a) for _, a, _ in sets]), oo, out, u, ao)
    assert rc == 0, lib.mgb_last_error()
    res = []
    for s, off in enumerate(offs):
        r = list(out[6 * s:6 * s + 6])
        res.append(r + [list(u[off:off + r[1]]), [(ao[off + j].x, ao[off + j].y) for j in range(r[2] if r[1] > 0 else 0)]])
    return res


# ---- anchor sets ----
def hot_layout(mode, n):
    """which of the arrays the chaining loops re-read are on chip for a set of n anchors: the seeds (staged), then, in the order
    chain_dp_w / chain_rmq_w + chain_rmq_fill_w take them from what is left of the slice (16-byte aligned, MGB_ALLOC_HOT), p f v t
    (DP) or p f t v K blk pri (RMQ)"""
    r16 = lambda b: (max(b, 1) + 15) & ~15
    staged = 16 * n + 16 <= SLICE[mode]
    room = SLICE[mode] - 16 - (16 * n if staged else 0)
    sizes = [4 * n] * 4 if mode == capi.LCHAIN_DP else [4 * n] * 4 + [8 * n, 48 * ((n + 31) >> 5), 8 * n]
    hot = []
    for b in sizes:
        hot.append(r16(b) <= room)
        room -= r16(b) if hot[-1] else 0
    return (staged,) + tuple(hot)


def fam_slice_edges(rng, mode, scale):
    """n on both sides of every size where the seeds or one more hot array stop fitting the slice (for k_chain 511/512: all four of
    f/p/v/t beside the staged seeds, then three; 1023/1024: staged, then not)"""
    edges = sorted({n for n in range(2, 1400) if hot_layout(mode, n) != hot_layout(mode, n - 1)})
    ns = sorted({m for e in edges for m in (e - 2, e - 1, e)})
    out = []
    for n in ns:
        a = chain(rng, n // 2, 1000, 500) + chain(rng, n - n // 2, rng.randint(900, 1100), rng.randint(0, 2000), step=(5, 60), jit=30)
        rng.shuffle(a)
        out.append(("slice n=%d %s" % (n, hot_layout(mode, n)), a if mode == capi.LCHAIN_RESCUE else by_x(a), opts(LOOSE, bw=rng.choice([500, 20000]))))
    return out, edges


def fam_window(rng, mode, scale):
    """anchors whose target distance is max_dist, max_dist + 1 (and the same for max_dist_inner, and the query distance of the RMQ)"""
    out = []
    for md in (300, 1000):
        for mdi in ((0, md // 3, md, md + 100) if mode != capi.LCHAIN_DP else (0,)):
            for _ in range(2 * scale):
                a, t, q = [], 100, 100
                for _ in range(60):
                    a.append(anc(t, q))
                    d = rng.choice([md, md + 1, md, md + 1, mdi or md, (mdi or md) + 1, rng.randint(1, md // 4)])
                    if rng.random() < 0.5:  # a partner exactly d further on, then carry on from near the first one
                        a.append(anc(t + d, q + d + rng.randint(-2, 2)))
                        t, q = t + rng.randint(1, 40), q + rng.randint(1, 40)
                    else:
                        t, q = t + d, q + d + rng.randint(-5, 5)
                out.append(("window md=%d inner=%d" % (md, mdi), by_x(a), opts(LOOSE, max_dist_x=md, max_dist_y=md, bw=50, max_dist_inner=mdi, walk=True)))
    return out


def fam_max_ii(rng, mode, scale):
    """the best anchor of the window (max_ii) recomputed at max_dist + 1 among tied ones, and taken from behind a skip stop"""
    out = []
    for _ in range(2 * scale):
        md, base = rng.choice([600, 1000]), 3000
        a = []
        for dt, dg in ((0, -400), (5, 0), (10, 20)):  # three copies of one chain, ends at x = base, base + 5, base + 10: equal f
            a += [anc(base + dt - 20 * k, base + dt - 20 * k + dg) for k in range(50)]
        for k in range(12):  # a weaker chain on a diagonal too far from the copies to join them; the scan stops in it
            a += [anc(base + 50 + 25 * k, base - 100 + 25 * k), anc(base + 55 + 25 * k, base - 95 + 25 * k)]
        x0 = base + md + 1  # the first copy's end leaves the window: the two others tie, in reach at different distances
        a += [anc(x0, x0 - 50)] + chain(rng, 30, x0 + 30, x0 - 20)  # (long enough for the chain through the copy to outscore the copy)
        out.append(("max_ii", by_x(a), opts(LOOSE, max_dist_x=md, max_dist_y=md, bw=100, max_skip=0, walk=True)))
        # two copies ending at x = base (diagonal 0) and base + 5 (diagonal 30): max_ii stays on the first, which the query anchor on
        # diagonal 60 reaches with a larger gap than the second; a weaker chain on diagonal 150 between them stops the scan
        a = [anc(base + dt - 20 * k, base + dt - 20 * k + dg) for dt, dg in ((0, 0), (5, 30)) for k in range(50)]
        for k in range(12):
            a += [anc(base + 20 + 25 * k, base + 170 + 25 * k), anc(base + 25 + 25 * k, base + 175 + 25 * k)]
        x0 = base + 400
        a += [anc(x0, x0 + 60)] + chain(rng, 30, x0 + 30, x0 + 90)
        out.append(("max_ii kept", by_x(a), opts(LOOSE, max_dist_x=md, max_dist_y=md, bw=100, max_skip=0, walk=True)))
    return out


def tandem(rng, n_x, period, width, t0=1000, q0=1000, span=15, jit=0):
    """a tandem repeat in both sequences: anchors (t0 + k*period, q0 + m*period) for |k - m| <= width"""
    a = []
    for k in range(n_x):
        for m in range(max(0, k - width), k + width + 1):
            a.append(anc(t0 + k * period + rng.randint(0, jit), q0 + m * period + rng.randint(0, jit), span))
    return by_x(a)


def fam_max_iter(rng, mode, scale):
    out = []
    for it in (31, 32, 33, 63, 64, 65):
        out.append(("max_iter=%d" % it, tandem(rng, 40, 7, 3, jit=2), opts(LOOSE, max_iter=it, walk=True)))
    for it in (31, 32, 33, 63, 64, 65):  # chain anchors with k decoys between them: the chain's predecessor sits at i - (k + 1)
        for k in (it - 2, it - 1, it):
            a, t = [], 1000
            for c in range(8):
                a.append(anc(t, t))
                # decoys: query positions far beyond the chain and from each other, so that nothing scores with them
                a += [anc(t + 1 + d, 1_000_000 + 20_000 * (c * 70 + d)) for d in range(k)]
                t += k + 20
            out.append(("max_iter=%d, predecessor at i-%d" % (it, k + 1), a, opts(LOOSE, max_iter=it, walk=True)))
    if scale > 1:  # the default cut: a window of more than 5000 anchors
        out.append(("max_iter=5000", tandem(rng, 700, 3, 4, jit=1), opts(LOOSE, max_iter=5000, max_dist_x=5000, bw=100)))
    return out


def fam_skip(rng, mode, scale):
    """repeats with many predecessors of equal score, so that the skip counter stops the scan; kept where the stop falls on lane 0
    or lane 31 of a chunk, and a few more"""
    out, found = [], collections.Counter()
    for _ in range(400 * scale):
        ms = rng.choice([0, 1, 3, 25])
        a = tandem(rng, rng.randint(8, 30), rng.choice([5, 8, 10, 12]), rng.randint(1, 6), jit=rng.choice([0, 0, 1, 3]))
        o = opts(LOOSE, max_skip=ms, max_iter=rng.choice([5000, 64, 40]), bw=rng.choice([30, 100, 500]))
        ev = collections.Counter()
        walk_dp(a, o, ev)
        lanes = {int(k.split()[-1]) for k in ev if k.startswith("skip stop")}
        want = (0 in lanes and found[0] < 3 * scale) or (31 in lanes and found[31] < 3 * scale) or (lanes and found[ms] < 2 * scale)
        if want:
            found[ms] += 1
            found.update(lanes & {0, 31})
            out.append(("skip max_skip=%d" % ms, a, dict(o, walk=True)))
        if found[0] >= 3 * scale and found[31] >= 3 * scale and all(found[m] >= 2 * scale for m in (0, 1, 3, 25)):
            break
    return out


def fam_ties(rng, mode, scale):
    out = []
    for _ in range(2 * scale):  # a grid: many predecessors at the same distance, equal sc + f
        g = rng.choice([10, 16, 20])
        a = [anc(1000 + g * k, 500 + g * m, 15) for k in range(14) for m in range(14) if abs(k - m) <= 4]
        out.append(("ties grid", by_x(a), opts(LOOSE, bw=rng.choice([50, 500]), walk=True)))
    for _ in range(2 * scale):  # identical copies of one chain on other diagonals and targets: end points with equal f
        base = chain(rng, 12, 0, 0, step=(20, 30), jit=2)
        a = []
        for c in range(6):
            dt, dq = rng.choice([0, 5000 * (c + 1)]), 3000 * c
            a += [anc((x & 0xffffffff) + dt, (y & 0xffffffff) + dq, 15, tid=c % 2) for x, y in base]
        out.append(("ties equal chains", by_x(a), opts(LOOSE, bw=100, walk=True)))
    for _ in range(2 * scale):  # chains that start at the same target position
        t0 = rng.randint(100, 1000)
        a = chain(rng, 10, t0, 100) + chain(rng, 10, t0, 5000) + chain(rng, 8, t0, 9000, step=(5, 9))
        out.append(("ties same start", by_x(a), opts(LOOSE, bw=100, walk=True)))
    return out


def fam_score_args(rng, mode, scale):
    out = []
    for pg in (1.0, 0.2):
        a = []  # dr == 0 and dq == 0 next to scoring pairs
        for k in range(30):
            t, q = 100 + 40 * k, 100 + 40 * k
            a += [anc(t, q), anc(t, q + rng.randint(1, 30)), anc(t + rng.randint(1, 30), q)]
        out.append(("score dr=0 dq=0 pen_gap=%g" % pg, by_x(a), opts(LOOSE, pen_gap=pg, walk=True)))
        for bw in (50, 500):  # dd at bw and bw + 1
            a = []
            for k in range(40):
                t, q = 10000 * k, 10000 * k
                a += [anc(t, q), anc(t + 1000 + bw + rng.randint(0, 1), q + 1000), anc(t + 1000, q + 1000 + bw + rng.randint(0, 1))]
            out.append(("score dd=bw,bw+1", by_x(a), opts(LOOSE, bw=bw, max_dist_x=5000, max_dist_y=5000, pen_gap=pg, walk=True)))
        a = []  # dd swept over 1..10^6: every branch of the log2 approximation
        for k in range(60):
            dd = int(10 ** rng.uniform(0, 6))
            t = 3_000_000 * k
            a += [anc(t, 1000 + k), anc(t + 100 + dd, 1100 + k, span=rng.randint(1, 255))]
        out.append(("score dd 1..1e6", by_x(a), opts(LOOSE, bw=1_100_000, max_dist_x=1_200_000, max_dist_y=1_200_000, pen_gap=pg)))
    for _ in range(scale):  # cDNA: a deletion is charged the smaller of the two penalties
        a = chain(rng, 30, 0, 0, step=(20, 400), jit=200)
        out.append(("score is_cdna", by_x(a), opts(LOOSE, is_cdna=1, max_dist_y=100, walk=True)))
    for _ in range(2 * scale):  # paired segments: segment id in bits 48-55, cross-segment dr == 0 bonus
        a = []
        for seg in range(3):
            t0 = rng.randint(0, 500)
            for x, y in chain(rng, 15, t0, 0, step=(10, 30), jit=5):
                a.append(anc(x & 0xffffffff, (y & 0xffffffff) + 2000 * seg, seg=seg))
        for x, y in list(a[:5]):  # the same target position from another segment
            a.append((x, (y + 2000) & ~(0xff << 48) | 1 << 48))
        out.append(("score n_seg=3", by_x(a), opts(LOOSE, n_seg=3, max_dist_y=rng.choice([30, 5000]), walk=True)))
    return out


def fam_rmq(rng, mode, scale):
    out = []
    for _ in range(2 * scale):  # anchors on one anti-diagonal, f equal: priorities tie, the AVL replay decides
        m, t0, q0 = rng.randint(2, 12), 1000, 2000
        a = [anc(t0 + k, q0 - k) for k in range(m)]
        a += chain(rng, 10, t0 + m + 20, q0 + 30)
        out.append(("rmq tie", by_x(a), opts(LOOSE, pen_gap=rng.choice([1.0, 0.2]))))
    for _ in range(2 * scale):  # cap of n - 1: the sequential fill, with the same meaning as the warp-wide one
        a = chain(rng, 60, 0, 0, jit=20) + chain(rng, 40, 500, 3000, jit=20)
        out.append(("rmq cap n-1", by_x(a), opts(LOOSE, cap_rmq_size=len(a) - 1)))
    for cap in (1, 5, 20):  # a small cap: the reference's tree really loses anchors
        a = chain(rng, 80, 0, 0, jit=10) + chain(rng, 40, 100, 2000, jit=10)
        out.append(("rmq cap %d" % cap, by_x(a), opts(LOOSE, cap_rmq_size=cap)))
    for _ in range(2 * scale):  # two diagonals more than 2048 apart in y, interleaved in x: blocks keep two summaries
        a = chain(rng, 80, 0, 0) + chain(rng, 80, 5, 3000 + rng.randint(0, 500))
        out.append(("rmq interleaved", by_x(a), opts(LOOSE, max_dist_x=5000, max_dist_inner=rng.choice([0, 1000]))))
    for _ in range(2 * scale):  # anchor 0 at y == yi - 1 (the only one the reference's interval lets in on that border), a later one too
        t0, q0 = rng.randint(100, 1000), rng.randint(100, 1000)
        a = [anc(t0, q0, 255), anc(t0 + rng.randint(2, 20), q0 + 1, 15)]
        a += chain(rng, 5, t0 + 40, q0 + 40, span=200)
        x, y = a[-1]
        a += [anc((x & 0xffffffff) + rng.randint(2, 20), (y & 0xffffffff) + 1)]
        a += chain(rng, 6, (x & 0xffffffff) + 60, (y & 0xffffffff) + 60)
        out.append(("rmq y=yi-1", by_x(a), opts(LOOSE, pen_gap=0.2)))
    for _ in range(scale):  # query position 0, and runs of equal x (anchors become available only when x changes)
        a = [anc(50, 0, 1), anc(60, 0, 15)] + chain(rng, 20, 70, 10)
        a += [anc(2000, q) for q in range(0, 400, 37)] + [anc(2001, q) for q in range(5, 400, 41)] + chain(rng, 20, 2100, 450)
        out.append(("rmq y=0, equal x", by_x(a), opts(LOOSE)))
    return out


def rmq_border(a, o):
    """For an x-sorted set of fam_rmq_border: the anchors i whose outer window holds S (the last anchor of q_span 100, the best priority
    by construction) at a query position of exactly yi - max_dist (outside the reference's interval, lchain.c:316) or yi - max_dist + 1
    (inside it), and how chain_rmq_fill_w meets S's block there: 'summary' when the block lies in the window but for S, 'border' when
    its elements are scanned anyway (one summary per block: no block spans more than 2048 query positions)."""
    out, n, md = collections.Counter(), len(a), max(o["max_dist_x"], o["bw"])
    ys = [s32(y) for _, y in a]
    assert all(max(ys[b:b + 32]) - min(ys[b:b + 32]) <= 2048 for b in range(0, n, 32))
    sj = max(k for k in range(n) if a[k][1] >> 32 & 0xff == 100)
    for i in range(n):
        xi, yi = a[i][0], ys[i]
        i0 = next(k for k in range(n) if a[k][0] == xi)  # the anchors before i0 are in the trees
        st = next((k for k in range(i0) if xi >> 32 == a[k][0] >> 32 and xi <= a[k][0] + md), i0)
        off = ys[sj] - (yi - md)
        if not (st <= sj < i0 and off in (0, 1)):
            continue
        b = sj >> 5
        rest = [ys[k] for k in range(b << 5, min((b + 1) << 5, i0)) if k != sj]
        whole = (b << 5) >= st and all(yi - md < y < yi - 1 for y in rest)
        out["rmq best at yi - max_dist + %d, %s" % (off, "summary" if whole else "border")] += 1
    return out


def fam_rmq_border(rng, mode, scale):
    """A chain of q_span 100 ending at S (f of about 1000), and an anchor Q with yQ - yS = max_dist (and max_dist - 1) within bw of S's
    diagonal; the rest of Q's window is a weaker chain on a diagonal more than bw away, so S has the window's best priority.  S starts
    a block whose other anchors all lie in Q's window (the block summary would answer), or shares its block with the chain before it,
    which has left the window (the block's elements are scanned)."""
    out = []
    for _ in range(2 * scale):
        for dq_q in (1000, 999):
            for border in (0, 1):
                md, base = 1000, 20000
                pad = [anc(100 + 37 * k, 13_730 - 10 * k) for k in range(23 - 4 * border)]  # S at index 32 (28 in the border case)
                pre = [anc(base - 100 * (9 - k), base - 5000 - 100 * (9 - k), 100) for k in range(9)]
                s_ = anc(base, base - 5000, 100)
                fill = [anc(base + 3 + 20 * k, base - 5000 + 350 + rng.randint(0, 40) + 20 * k) for k in range(31)]
                q_ = anc(base + 990, base - 5000 + dq_q)
                post = chain(rng, 10, base + 1020, base - 5000 + dq_q + 30)
                a = by_x(pad + pre + [s_] + fill + [q_] + post)
                out.append(("rmq max_dist border dq=%d %s" % (dq_q, "border" if border else "summary"), a,
                            opts(LOOSE, max_dist_x=md, max_dist_inner=0, bw=100, pen_gap=0.2, rmq_border=True)))
    return out


def fam_misc(rng, mode, scale):
    out = [("n=0", [], opts(LR)), ("n=1", [anc(5, 20)], opts(LOOSE))]
    a = []
    for tid in range(3):  # several targets and both strands in one set
        for rev in (0, 1):
            a += chain(rng, 25, rng.randint(0, 100), rng.randint(0, 3000), tid=tid, rev=rev)
    out.append(("targets and strands", by_x(a), opts(LR)))
    out.append(("min_sc too high", by_x(chain(rng, 30, 0, 0)), opts(LR, min_sc=1 << 30)))
    out.append(("lr filters", by_x(chain(rng, 40, 0, 0) + chain(rng, 4, 9000, 100)), opts(LR)))
    return out


def interleave(mode, sets):
    """sets in the order that makes one warp go from staged sets to unstaged ones and back (set i goes to worker i % n_workers)"""
    w = min(len(sets), 2 * WARPS[mode])
    on = [s for s in sets if 16 * len(s[1]) + 16 <= SLICE[mode]]
    off = [s for s in sets if 16 * len(s[1]) + 16 > SLICE[mode]]
    out, r = [], 0
    while on or off:
        src = on if (r % 2 == 0 and on) or not off else off
        out += src[:w]
        del src[:w]
        r += 1
    return out


def case_lchain(lib, scale=1, seed=7):
    rng = random.Random(seed)
    seen = collections.Counter()
    for mode in (capi.LCHAIN_DP, capi.LCHAIN_RMQ, capi.LCHAIN_RESCUE):
        sl, edges = fam_slice_edges(rng, mode, scale)
        fams = [sl, fam_misc(rng, mode, scale), fam_window(rng, mode, scale), fam_ties(rng, mode, scale)]
        if mode == capi.LCHAIN_DP:
            fams += [fam_max_ii(rng, mode, scale), fam_max_iter(rng, mode, scale), fam_skip(rng, mode, scale), fam_score_args(rng, mode, scale)]
        else:
            fams += [fam_rmq(rng, mode, scale), fam_rmq_border(rng, mode, scale)]
        sets = interleave(mode, [(tag, a, {k: v for k, v in o.items() if k not in ("walk", "rmq_border")}) for fam in fams for tag, a, o in fam])
        border = {id(a) for fam in fams for _, a, o in fam if o.get("rmq_border")}
        walk = {id(a) for fam in fams for _, a, o in fam if o.get("walk")}
        got = run_lchain(lib, mode, sets)
        per_worker = collections.defaultdict(list)
        for (tag, a, o), (rc, n_u, n_v, staged, path, worker, u, anchors) in zip(sets, got):
            what = "mode %d, %s (n=%d): " % (mode, tag, len(a))
            check_input(mode, a)
            ru, ra = ref_lchain(mode, a, o)
            assert rc == 0, what + "rc %d" % rc
            assert n_u == len(ru), what + "n_u %d, reference %d" % (n_u, len(ru))
            assert u == ru, what + "u[] differs first at %d" % next(k for k in range(n_u) if u[k] != ru[k])
            assert anchors == ra, what + "anchors differ first at %d" % next((k for k in range(len(ra)) if k >= len(anchors) or anchors[k] != ra[k]), len(ra))
            assert staged == (16 * len(a) + 16 <= SLICE[mode] and len(a) > 0), what + "staged %d" % staged
            want_path = None if not a else capi.LCHAIN_PATH_DP if mode == capi.LCHAIN_DP else capi.LCHAIN_PATH_RMQ_CAP if len(a) > o["cap_rmq_size"] else None
            if want_path is not None:
                assert path == want_path, what + "fill path %d" % path
            if tag.startswith("rmq tie"):
                assert path == capi.LCHAIN_PATH_RMQ_TIE, what + "the priorities tie, but fill path %d" % path
            per_worker[worker].append(staged)
            seen["mode %d path %d" % (mode, path)] += 1
            if mode == capi.LCHAIN_DP and id(a) in walk:
                ev = collections.Counter()
                walk_dp(a, o, ev)
                seen.update({k: v for k, v in ev.items() if v})
            if mode != capi.LCHAIN_DP and a:
                ys = [s32(y) for _, y in by_x(a)]
                seen["rmq two summaries"] += any(max(ys[b:b + 32]) - min(ys[b:b + 32]) > 2048 for b in range(0, len(ys), 32))
                seen["rmq y = y[0] + 1"] += any(ys[k] == ys[0] + 1 and a[k][0] > a[0][0] for k in range(1, len(ys)))
                seen["rmq y = 0"] += 0 in ys
            if id(a) in border:
                assert path == capi.LCHAIN_PATH_RMQ_W, what + "fill path %d" % path
                seen.update(rmq_border(by_x(a), o))
        # sizes just below and at every edge of the slice layout were run (the families' n are edge - 2, edge - 1, edge)
        assert edges and all(any(len(a) == e for _, a, _ in sets) and any(len(a) == e - 1 for _, a, _ in sets) for e in edges), (mode, edges)
        flips = collections.Counter((s[k], s[k + 1]) for s in per_worker.values() for k in range(len(s) - 1))
        assert flips[(1, 0)] and flips[(0, 1)] and flips[(1, 1)], (mode, flips)  # a warp moves between staged and unstaged sets and reuses its slice
    need = ["mode 0 path 0", "mode 1 path 1", "mode 1 path 2", "mode 1 path 3", "mode 2 path 1", "mode 2 path 2", "mode 2 path 3",
            "skip stop on lane 0", "skip stop on lane 31", "best predecessor tied", "max_ii tied", "max_ii taken", "end points tied",
            "max_iter cut, 31 left in the last chunk", "max_iter cut, 32 left in the last chunk", "max_iter cut, 1 left in the last chunk",
            "window: x - x[st] = max_dist", "window: x - x[st-1] = max_dist+1", "max_ii recomputed at max_dist+1",
            "best predecessor at the cut, 31 left in the last chunk", "best predecessor at the cut, 32 left in the last chunk",
            "best predecessor at the cut, 1 left in the last chunk", "max_ii kept over an equal f",
            "rmq best at yi - max_dist + 0, summary", "rmq best at yi - max_dist + 0, border", "rmq best at yi - max_dist + 1, summary",
            "rmq best at yi - max_dist + 1, border", "rmq two summaries", "rmq y = y[0] + 1", "rmq y = 0"]
    missing = [k for k in need if not seen[k]]
    assert not missing, (missing, seen)
    return seen


@pytest.mark.parametrize("sim", ["one lane", "32 lanes"])
def test_lchain_in_simulator(sim):
    case_lchain(T.load_hostsim() if sim == "one lane" else T.load_hostsim32())


@pytest.mark.gpu
def test_lchain_on_gpu():
    case_lchain(capi.load_product(), scale=3)
