"""Batched traceback of the gap alignment (mgb_galign.cuh WfaBatch): a warp of k_wfa_small / k_wfa_mid keeps the traceback rows of
its gaps in its arena and traces up to 32 of them back at once, one per lane.  Batches are cut by the number of gaps and by the
arena budget (a quarter of the arena), a gap handed on to the next tier never enters one, and a gap that runs out of arena
next to a full batch is run again on its own.  Every aligned gap must have the score, CIGAR and n_iter of the reference's
mwf_wfa_exact, in the one-lane and the 32-lane simulators (batches of one and of 32) and on the GPU."""
import random

import pytest

import cases
import mgtest as T
from minigraph_b200 import capi

pytestmark = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")

# warps the hook launches (64 blocks of the kernel's warps): worker w takes gaps w, w + WORKERS, ...
WORKERS = {1: 256, 2: 128, capi.WFA_TIER2_CONT: 128}


def _rnd(rng, n):
    return "".join(rng.choices("ACGT", k=n))


def _noisy(rng, s, rate):
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


def _short(rng, lo, hi):
    t = _rnd(rng, rng.randint(lo, hi))
    q = _noisy(rng, t, rng.uniform(0.0, 0.12))
    if rng.random() < 0.3:  # the last bases differ: the corner is reached without extension (last state from the traceback byte)
        t, q = t + rng.choice("AC"), q + rng.choice("GT")
    return t, q


def _gaps(tier, rng, per_worker, special):
    """per_worker gaps for every worker, short ones, with special(rng) -> (tag, t, q) at a few places in the middle of a
    worker's list; returned in the order the hook deals them out"""
    nw = WORKERS[tier]
    cols = []
    for w in range(nw):
        col = [("short",) + _short(rng, 4, 90) for _ in range(per_worker)]
        if w % 3 == 0:
            for at in rng.sample(range(1, per_worker - 1), 2):
                col[at] = special(rng)
        cols.append(col)
    gaps = [cols[w][k] for k in range(per_worker) for w in range(nw)]
    return [(tag, t.encode(), q.encode()) for tag, t, q in gaps]


def _check(lib, tier, gaps):
    got = cases.run_wfa_tier(lib, tier, gaps)
    seen = {}
    for i, ((tag, t, q), (rc, s, n_iter, cigar)) in enumerate(zip(gaps, got)):
        what = "tier %d gap %d (%s, tl=%d ql=%d): " % (tier, i, tag, len(t), len(q))
        assert rc in (0, 1), what + "rc %d" % rc
        seen[(tag, rc)] = seen.get((tag, rc), 0) + 1
        if rc == 0:
            rs, rcig, rn = cases._ref_wfa_exact(t, q)
            assert (s, cigar, n_iter) == (rs, rcig, rn), what + "score %d/%d n_iter %d/%d, CIGAR %s" % (s, rs, n_iter, rn, "same" if cigar == rcig else "differs")
    return seen


def case_tier1_batches(lib, seed=3):
    """tier 1: 33 gaps per worker (a full batch of 32 and one more), gaps longer than the tier takes handed on in the middle"""
    rng = random.Random(seed)
    gaps = _gaps(1, rng, 33, lambda r: ("long", _rnd(r, 300), _rnd(r, 280)))
    seen = _check(lib, 1, gaps)
    assert seen.get(("short", 0), 0) > 8000 and seen.get(("long", 1), 0) > 100, seen


def case_tier2_batches(lib, seed=5):
    """tier 2 as k_wfa_mid runs it (hand-off to the arena ring), 5 MB arena: 34 gaps per worker, with gaps in the middle that
    are carried on in the ring and whose rows alone pass the budget of a batch (unrelated pairs of about 1000 bases: scores past
    1000, about 2 MB of rows), and gaps longer than tier 2 takes, handed on"""
    rng = random.Random(seed)

    def special(r):
        u = r.random()
        if u < 0.4:
            return ("huge", _rnd(r, r.randint(950, 1024)), _rnd(r, r.randint(950, 1024)))
        if u < 0.8:
            n = r.randint(300, 600)
            t = _rnd(r, n)
            return ("handoff", t, _noisy(r, t, r.uniform(0.08, 0.2)))
        return ("long", _rnd(r, 1100), _rnd(r, 1050))
    gaps = _gaps(capi.WFA_TIER2_CONT, rng, 34, special)
    seen = _check(lib, capi.WFA_TIER2_CONT, gaps)
    assert all(seen.get(k, 0) > 0 for k in (("short", 0), ("huge", 0), ("handoff", 0), ("long", 1))), seen


@pytest.mark.parametrize("sim", ["one lane", "32 lanes"])
def test_tb_batches_in_simulator(sim):
    lib = T.load_hostsim() if sim == "one lane" else T.load_hostsim32()
    case_tier1_batches(lib)
    case_tier2_batches(lib)


@pytest.mark.gpu
def test_tb_batches_on_gpu():
    lib = capi.load_product()
    case_tier1_batches(lib)
    case_tier2_batches(lib)
