"""Tier 2 of the gap alignment as k_wfa_mid runs it: a gap whose window outgrows the 254 diagonals of the shared-memory ring
before score 240 is carried on by the same warp in the arena ring of tier 3 (mgb_wfa_tiers.cuh wfa_smem_continue) instead of
being aligned again from score 0 in tier 3.  Score, CIGAR and n_iter must be the reference's mwf_wfa_exact, in the one-lane and
the 32-lane simulators and on the GPU."""
import random

import pytest

import cases
import mgtest as T
from minigraph_b200 import capi

pytestmark = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")

# An unclipped window widens by one diagonal per side and score from score 16 on, so it outgrows the ring (width + 2 > 256)
# at score 142: tier 2 on its own gives up there, with the hand-off it carries on.
HANDOFF_AT = 142


def _handoff_gaps(rng, scale):
    def rnd(n):
        return "".join(rng.choices("ACGT", k=n))

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
    # final scores just below, at and above the hand-off score (unclipped windows)
    near = []
    for _ in range(4000):
        if len(near) >= 30 * scale:
            break
        n = rng.randint(300, 700)
        t = rnd(n)
        q = noisy(t, rng.uniform(0.7, 1.3) * HANDOFF_AT / (5.0 * n))
        s, _, _ = cases._ref_wfa_exact(t.encode(), q.encode())
        if HANDOFF_AT - 8 <= s <= HANDOFF_AT + 12:
            near.append(("near", t, q))
    gaps += near
    # one side short: the window stops at that side's end and outgrows the ring later, between scores 158 and 220
    for _ in range(6 * scale):
        tl, ql = rng.randint(500, 1024), rng.randint(50, 110)
        t = rnd(tl)
        a = rng.randint(0, tl - ql)
        gaps += [("short", t, noisy(t[a:a + ql], 0.1)), ("short", rnd(ql), t)]
    # noisy copies and unrelated pairs whose scores cross the band shrinks at 256 and 512 after the hand-off
    for _ in range(8 * scale):
        n = rng.randint(400, 1024)
        t = rnd(n)
        gaps.append(("shrink", t, noisy(t, rng.uniform(0.15, 0.5))[:1024]))
    for _ in range(2 * scale):
        gaps.append(("shrink", rnd(rng.randint(600, 1024)), rnd(rng.randint(600, 1024))))
    # sides of 1024 (the longest tier 2 takes), and one past it (tier 3)
    for rate in (0.03, 0.1, 0.3):
        t = rnd(1024)
        gaps.append(("1024", t, (noisy(t, rate) + rnd(64))[:1024]))
    gaps.append(("1024", rnd(1024), rnd(1024)))
    t = rnd(1025)
    gaps += [("1025", t, noisy(t, 0.1)[:1024]), ("1025", rnd(900), t)]
    return [(tag, t.encode(), q.encode()) for tag, t, q in gaps]


def case_tier2_handoff(lib, scale=1, seed=11):
    rng = random.Random(seed)
    gaps = _handoff_gaps(rng, scale)
    plain = cases.run_wfa_tier(lib, 2, gaps)
    cont = cases.run_wfa_tier(lib, capi.WFA_TIER2_CONT, gaps)
    seen = {"below": 0, "at": 0, "above": 0, "short": 0, "past 256": 0, "past 512": 0, "1024": 0}
    for i, ((tag, t, q), p, c) in enumerate(zip(gaps, plain, cont)):
        tl, ql = len(t), len(q)
        rs, rcig, rn = cases._ref_wfa_exact(t, q)
        what = "gap %d (%s, tl=%d ql=%d, reference score %d n_iter %d): " % (i, tag, tl, ql, rs, rn)
        assert c[0] in (0, 1), what + "rc %d" % c[0]
        if c[0] == 0:
            assert (c[1], c[3], c[2]) == (rs, rcig, rn), what + "score %d n_iter %d, CIGAR %s" % (c[1], c[2], "same" if c[3] == rcig else "differs")
        if p[0] == 0:
            assert c == p, what + "aligned by tier 2 alone, but not the same way with the hand-off"
        if max(tl, ql) > 1024:
            assert c[0] == 1, what + "longer than tier 2 takes, but accepted"
            continue
        # every gap here outgrows the ring (if at all) before score 240: none may be handed on to tier 3
        assert c[0] == 0, what + "handed on to tier 3"
        handed = p[0] == 1
        if tag == "near":
            key = "below" if rs < HANDOFF_AT else "at" if rs <= HANDOFF_AT + 3 else "above"
            assert handed == (rs >= HANDOFF_AT), what + ("carried on" if handed else "not carried on")
            seen[key] += 1
        if handed:
            seen["short"] += tag == "short"
            seen["past 256"] += rs > 256
            seen["past 512"] += rs > 512
            seen["1024"] += max(tl, ql) == 1024
    assert all(v > 0 for v in seen.values()), seen
    return seen


@pytest.mark.parametrize("sim", ["one lane", "32 lanes"])
def test_tier2_handoff_in_simulator(sim):
    case_tier2_handoff(T.load_hostsim() if sim == "one lane" else T.load_hostsim32())


@pytest.mark.gpu
def test_tier2_handoff_on_gpu():
    case_tier2_handoff(capi.load_product(), scale=3)
