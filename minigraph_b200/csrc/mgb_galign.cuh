// mgb_galign.cuh -- base-level alignment of graph chains and the per-read result blob.
//   gchain_cigar()  (reference: galign.c:39-145 mg_gchain_cigar)
//   gchain_ds()     (reference: galign.c:182-293 mg_gchain_gen_ds)
//   stage_align()   K6-K8 for one read (reference: map-algo.c:455-479)
#pragma once
#include "mgb_pipeline.cuh"
#include "mgb_gchain.cuh"
#include "mgb_wfa_tiers.cuh"
#if defined(MGB_HOSTSIM)
#include <stdio.h>
#include <stdlib.h>
#endif

namespace mgb {

MG_HD inline int cigar_append1(Arena &A, AVec<uint64_t> &c, int32_t op, int32_t len)
{
	if (c.n > 0 && (int32_t)(c.a[c.n - 1] & 0xf) == op) c.a[c.n - 1] += (uint64_t)(int64_t)len << 4;
	else {
		uint64_t x = (uint64_t)(int64_t)len << 4 | (uint64_t)op;
		MGB_TRY(avec_push(A, c, x));
	}
	return 0;
}

MG_HD inline int cigar_append(Arena &A, AVec<uint64_t> &c, int32_t n_cigar, const uint32_t *cigar)
{
	if (n_cigar == 0) return 0;
	MGB_TRY(cigar_append1(A, c, (int32_t)(cigar[0] & 0xf), (int32_t)(cigar[0] >> 4)));
	MGB_TRY(avec_reserve(A, c, c.n + n_cigar - 1));
	for (int32_t k = 0; k < n_cigar - 1; ++k) c.a[c.n + k] = cigar[1 + k];
	c.n += n_cigar - 1;
	return 0;
}

// One gap between two kept anchors that needs a real alignment.  Produced by the planning pass of K6/K7 (one lane
// per read), consumed by the WFA kernel K8a (one warp per job), stitched back by the finishing pass.
struct WfaJob {
	int32_t rid, gc;
	int32_t l0, l;        // first and last llchain of the gap (indices into the read's LLChain array)
	int32_t t_beg;        // first target base on lc[l0].v  (= q->x + 1)
	int32_t t_last;       // last target base on lc[l].v    (= p->x)
	int32_t tl, ql, q_off;
	int32_t n_cigar, status;
	int64_t lc_off;       // byte offset of the read's LLChain array inside the output pool
	int64_t cig_off;      // byte offset of the job's CIGAR (uint32 len<<4|op) inside the cigar pool
};

static const uint64_t PLAN_JOB = 1ULL << 63;
// The state of a warp's slice {next free byte, end} sits in the 96 bytes between the end of the tier's shared-memory layout and its
// stride (a static array would cost k_wfa_mid its seventh block per SM); tier 3 has no shared memory and few jobs: it asks per gap.
MG_HD inline unsigned long long *wfa_cig_chunk(int32_t *smem, int tier)
{
	static_assert(WfTier1::BYTES % 8 == 0 && WfTier1::BYTES + 16 <= WfTier1::STRIDE && WfTier2::BYTES % 8 == 0 && WfTier2::BYTES + 16 <= WfTier2::STRIDE, "no room for the slice state behind the tier layouts");
	return smem == 0 || tier > 2? (unsigned long long*)0 : (unsigned long long*)((char*)smem + (tier == 1? WfTier1::BYTES : WfTier2::BYTES));
}
static const unsigned long long CIG_CHUNK_BYTES = 2048; // a warp of a WFA kernel takes the CIGAR pool in slices of this size (the host sizes the pool with one slice per worker and kernel to spare)

// Planning pass of mg_gchain_cigar() (reference: galign.c:39-124): walk the kept anchors of every graph chain, emit
// literal CIGAR items for the trivial gaps (galign.c:98-100) and a WfaJob for the others.

// K8a: the wavefronts of one gap.  Warp-uniform (all lanes enter with identical arguments).
// tier 1: small gaps, wavefronts + traceback bytes in shared memory; tier 2: mid-size gaps, wavefronts in shared
// memory, carried on in the worker arena when the window outgrows them (longer sides: in the arena from the start, while
// wf_ring_always_fits); tier 3: anything, wavefronts in the worker arena.
// A job that does not fit a tier is appended to the queue of the next one (jobq[tier-1]); the host launches the next tier
// over that queue.  Returns 1 when the gap is aligned up to its traceback, which waits in *tb (and its rows, CIGAR store and
// stitched target in the arena) for the rest of the warp's batch (WfaBatch); 0 when there is nothing to trace back.
MG_HD inline int wfa_job_run(Arena &A, const PipeCtx &c, int64_t job_idx, int lane, int32_t *smem, int tier, WfTbJob *tb)
{
	WfaJob *J = &c.jobs[job_idx];
	if (J->rid < 0) return 0; // a slot no read wrote (its allocation ran over the end of the pool; the batch is re-run with a larger one)
	const int32_t rid = J->rid, l0 = J->l0, l = J->l, tl = J->tl, ql = J->ql;
	if (c.meta[rid].status < 0) return 0; // the read already failed elsewhere; it will be redone as a whole
	// Routing: a gap that cannot finish in tier 1 costs it up to a full window of cells before it gives up.  Which lengths
	// fail depends on the error rate of the reads, so it is learned: one gap in 64 tries every tier and reports where it
	// finished; the host turns the counts of one batch into the threshold of the next.  (Tier 2 loses nothing when its
	// window overflows, so every gap that fits its lengths stays there.)  The result of a gap does not depend on the tier
	// that computes it.
	const int32_t mlen = tl > ql? tl : ql;
	const int explore = (job_idx & 63) == 0;
	if (!explore && tier == 1 && mlen >= c.skip1_len) {
		if (lane == 0) {
			unsigned int at;
#if MGB_ON_DEVICE
			at = atomicAdd(&c.jobq_n[tier - 1], 1u);
#else
			at = c.jobq_n[tier - 1]++;
#endif
			c.jobq[tier - 1][at] = (int32_t)job_idx;
		}
		return 0;
	}
	const bool t2_long = tl > WfTier2::MAXLEN_ || ql > WfTier2::MAXLEN_; // (tier 2) the sequences do not fit shared memory: the arena ring from score 0
	if ((tier == 1 && (tl > WfTier1::MAXLEN_ || ql > WfTier1::MAXLEN_)) || (tier == 2 && t2_long && !wf_ring_always_fits(tl, ql))) {
		if (lane == 0) {
			unsigned int at;
#if MGB_ON_DEVICE
			at = atomicAdd(&c.jobq_n[tier - 1], 1u);
#else
			at = c.jobq_n[tier - 1]++;
#endif
			c.jobq[tier - 1][at] = (int32_t)job_idx;
		}
		return 0;
	}
	const GraphDev &g = c.g;
	const LLChain *lc = (const LLChain*)(c.out + J->lc_off);
	const char *qs = c.b.seq + c.b.seq_off[rid] + J->q_off;
	const char *tseq;
	if (l == l0) tseq = g_vseq(g, lc[l0].v) + J->t_beg;
	else { // stitch the target across the walk (reference: galign.c:76-93)
		char *seq;
		MGB_ALLOC(A, seq, char, tl + 1);
		int32_t n = g_vlen(g, lc[l0].v) - J->t_beg, at = 0;
		const char *s = g_vseq(g, lc[l0].v) + J->t_beg;
		for (int32_t x = lane; x < n; x += MGB_W) seq[at + x] = s[x];
		at += n;
		for (int32_t k = l0 + 1; k < l; ++k) {
			s = g_vseq(g, lc[k].v), n = g_vlen(g, lc[k].v);
			for (int32_t x = lane; x < n; x += MGB_W) seq[at + x] = s[x];
			at += n;
		}
		s = g_vseq(g, lc[l].v), n = J->t_last + 1;
		for (int32_t x = lane; x < n; x += MGB_W) seq[at + x] = s[x];
		at += n;
		if (at != tl) return MGB_E_INTERNAL;
		warp_sync();
		tseq = seq;
	}
	WfResult rst;
	unsigned long long pt0 = prof_clock();
	int rc;
	int64_t cont_cells = 0;
	if (tier == 1) rc = wfa_smem<WfTier1::W_, WfTier1::MAXLEN_, WfTier1::TBCAP_>(A, smem, tl, tseq, ql, qs, &rst, lane);
	else if (tier == 2 && !t2_long) rc = wfa_smem<WfTier2::W_, WfTier2::MAXLEN_, WfTier2::TBCAP_, true>(A, smem, tl, tseq, ql, qs, &rst, lane, &cont_cells);
	else if (tier == 2) rc = wfa_ring_exact(A, tl, tseq, ql, qs, &rst, lane);
	else rc = wfa_exact(A, tl, tseq, ql, qs, 100000000LL, &rst, lane);
	if (rc < 0) return rc;
	if (lane == 0) {
		unsigned long long dt = prof_clock() - pt0;
		int slot = tier == 1? PROF_WFA_FAST_CYC : tier == 2? PROF_WFA_MID_CYC : PROF_WFA_SLOW_CYC;
		prof_add(c, slot, dt), prof_add(c, slot + 1, 1);
		prof_max(c, PROF_WFA_MAX_CYC, dt << 16 | (unsigned long long)(mlen < 65535? mlen : 65535)); // cycles of the slowest gap, its length in the low 16 bits
		if (rc == 0) prof_add(c, PROF_WFA_CELLS, (unsigned long long)rst.n_iter);
		if (cont_cells > 0) prof_add(c, PROF_WFA_HANDOFF_N, 1), prof_add(c, PROF_WFA_HANDOFF_CELLS, (unsigned long long)cont_cells);
		if (rc == 0 && explore && c.tier_hist) {
			unsigned int *h = &c.tier_hist[(mlen >> 4 < 31? mlen >> 4 : 31) * 4 + tier];
#if MGB_ON_DEVICE
			atomicAdd(h, 1u);
#else
			++*h;
#endif
		}
	}
	if (rc == 1) { // does not fit this tier
		if (lane == 0) {
			unsigned int at;
#if MGB_ON_DEVICE
			at = atomicAdd(&c.jobq_n[tier - 1], 1u);
#else
			at = c.jobq_n[tier - 1]++;
#endif
			c.jobq[tier - 1][at] = (int32_t)job_idx;
		}
		return 0;
	}
	if (rst.s < 0) return MGB_E_INTERNAL;
	wfa_tb_keep(tb, rst, tl, tseq, ql, qs, job_idx, lane);
	return 1;
}

// K8a, after the traceback of the batch: the CIGAR of one gap into the pool.  Warp-uniform.
MG_HD inline int wfa_job_finish(const PipeCtx &c, const WfTbJob &b, int32_t *smem, int tier, int lane)
{
	if (b.rc < 0) return b.rc;
	const int32_t n_cigar = b.n_cigar;
	const uint32_t *cigar = b.cig + b.first;
	int64_t coff = 0;
	if (lane == 0) {
#if MGB_ON_DEVICE
		unsigned long long *ck = wfa_cig_chunk(smem, tier); // the warp's slice of the pool
		const unsigned long long need = ((unsigned long long)n_cigar * 4 + 15) & ~15ULL;
		if (ck == 0) coff = pool_alloc(c.pool_cig, (uint64_t)n_cigar * 4);
		else if (ck[0] + need > ck[1]) {
			const unsigned long long get = need > CIG_CHUNK_BYTES? need : CIG_CHUNK_BYTES;
			const int64_t off = pool_alloc(c.pool_cig, get);
			if (off < 0) ck[0] = ck[1] = 0;
			else ck[0] = (unsigned long long)off, ck[1] = (unsigned long long)off + get;
			coff = off;
		}
		if (ck && coff >= 0) coff = (int64_t)ck[0], ck[0] += need;
#else
		coff = pool_alloc(c.pool_cig, (uint64_t)n_cigar * 4);
#endif
	}
	coff = (int64_t)warp_bcast_u64((uint64_t)coff, 0);
	if (coff < 0) return MGB_E_POOL;
	uint32_t *dst = (uint32_t*)((char*)c.cig + coff);
	for (int32_t x = lane; x < n_cigar; x += MGB_W) dst[x] = cigar[x];
	if (lane == 0) { WfaJob *J = &c.jobs[b.job]; J->n_cigar = n_cigar, J->cig_off = coff; }
	return 0;
}

// The traceback batch of a warp of a WFA kernel.  The warp computes the wavefronts of a gap with all lanes and keeps its traceback
// rows in the arena; after MGB_W gaps, or once what the batch keeps passes a quarter of the arena, lane j traces gap j back
// (wfa_tb_batch) and the warp hands the CIGARs on.  The records sit at the bottom of the arena, the gaps' memory above them.  G is
// what the gaps are to the caller:
//   int run(int item, Arena &, WfTbJob *, int lane)  the wavefronts (wfa_job_run): < 0 failed, 0 nothing to trace back, 1 kept
//   int done(const WfTbJob &, int lane)              the traced CIGAR (wfa_job_finish), < 0 on failure
//   void fail(int item, int rc, int lane)             record the failure of the item
//   void traced(unsigned long long cyc, int lane)     lane 0's clock cycles of the batch's traceback
// A gap that runs out of arena while the batch holds others is run again after the batch is flushed, so that what fails for lack
// of arena is what fails on its own.  Warp-uniform; the state is the same on every lane.
template<typename G>
struct WfaBatch {
	WfTbJob *rec;
	int32_t n;
	MG_HD void open(Arena &A)
	{
		A.top = 0, n = 0;
		rec = (WfTbJob*)arena_alloc(A, (uint64_t)MGB_W * sizeof(WfTbJob)); // (the arena of a WFA kernel is far larger)
	}
	MG_HD void flush(const G &g, Arena &A, int lane)
	{
		if (n > 0) {
			const unsigned long long t0 = prof_clock();
			wfa_tb_batch(rec, n, lane);
			g.traced(prof_clock() - t0, lane);
			for (int32_t j = 0; j < n; ++j) {
				const WfTbJob &b = rec[j];
				const int rc = g.done(b, lane);
				if (rc < 0) g.fail(b.item, rc, lane);
			}
			warp_sync();
		}
		open(A);
	}
	MG_HD void add(const G &g, int item, Arena &A, int lane)
	{
		uint64_t mark = A.top;
		int rc = g.run(item, A, rec + n, lane);
		if (rc == MGB_E_ARENA && n > 0) {
			flush(g, A, lane);
			mark = A.top;
			rc = g.run(item, A, rec + n, lane);
		}
		if (rc < 0) g.fail(item, rc, lane);
		if (rc == 1) {
			if (lane == 0) rec[n].item = item;
			++n;
		} else A.top = mark;
		if (n == MGB_W || A.top > A.cap / 4) flush(g, A, lane);
	}
};

// ---- K8b: the stitched CIGAR and the ds:Z string of every chain, written once, straight into the result blob ----

MG_HD inline int mask_lowest(uint32_t m) // index of the lowest set bit of a non-zero mask
{
#if MGB_ON_DEVICE
	return __ffs(m) - 1;
#else
	return __builtin_ctz(m);
#endif
}

// Finishing pass of mg_gchain_cigar() (reference: galign.c:125-141): the stitched CIGAR of chain i, to *ops (n_cigar of them).
// The reference appends item after item and merges the first operation of an item into the last one written when they are of
// the same kind; nothing else is ever merged.  Here a prefix sum over the plan items gives every item its place in a flat list;
// the warp walks that list MGB_W operations at a time, lane l on operation base+l: it finds its item by a binary search and reads
// the operation (the lanes on one job read neighbouring words of its CIGAR).  An operation starts a run unless it is the first of
// its item and of the same kind as its left neighbour.  The runs are numbered by a ballot and their lengths added up by a
// segmented scan (the inclusive sum less the sum in front of the run's head); a run still open at the end of a group is written
// as it stands and carried into the next group, which writes it again.  Same list as the sequential append, operation for
// operation.  Warp-uniform.
MG_HD inline int gchain_cigar_finish_w(Arena &A, const PipeCtx &c, GcSet &gt, int32_t i, uint64_t **ops, int lane)
{
	GChain *gc = &gt.gc[i];
	const int32_t off_a0 = gt.lc[gc->off].off, n_plan = gc->n_plan;
	const uint64_t *plan = c.plan + gc->plan_off;
	int32_t *ioff;
	MGB_ALLOC(A, ioff, int32_t, n_plan + 1);
	int32_t tot = 0;
	for (int32_t base = 0; base < n_plan; base += MGB_W) {
		const int32_t t = base + lane;
		int32_t cnt = 0;
		if (t < n_plan) cnt = (plan[t] & PLAN_JOB)? c.jobs[plan[t] & ~PLAN_JOB].n_cigar : 1;
		const int32_t incl = warp_incl_scan_i32(cnt, lane);
		if (t < n_plan) ioff[t] = tot + incl - cnt;
		tot += warp_bcast_i32(incl, MGB_W - 1);
	}
	uint64_t *O;
	MGB_ALLOC(A, O, uint64_t, tot);
	warp_sync();
	int32_t n_out = 0, t_lo = 0, carry = 0, prev_op = 0, mlen = 0, blen = 0, aplen = 0, l = 0;
	for (int32_t base = 0; base < tot; base += MGB_W) {
		const int32_t j = base + lane;
		int32_t t = t_lo, op = 0, len = 0, first = 0;
		if (j < tot) {
			for (int32_t hi = n_plan - 1; t < hi; ) { // the last item that starts at or before j (an item without operations starts where the next one does)
				const int32_t mid = (t + hi + 1) >> 1;
				if (ioff[mid] <= j) t = mid;
				else hi = mid - 1;
			}
			uint64_t v = plan[t];
			if (v & PLAN_JOB) {
				const WfaJob *J = &c.jobs[v & ~PLAN_JOB];
				v = ((const uint32_t*)((const char*)c.cig + J->cig_off))[j - ioff[t]];
			}
			op = (int32_t)(v & 0xf), len = (int32_t)(v >> 4), first = j == ioff[t];
			if (op == 7) mlen += len;
			blen += len;
			if (op != 1) aplen += len;
			if (op != 2) l += len;
		}
		const int32_t up = (int32_t)warp_shfl_up1_u64((uint64_t)(uint32_t)op);
		const int32_t left = lane > 0? up : prev_op;
		const int head = j < tot && (j == 0 || !(first && op == left));
		const uint32_t mh = warp_ballot(head);
		const int32_t incl = warp_incl_scan_i32(len, lane);
		const uint64_t hs = warp_incl_scan_max_u64(head? (uint64_t)(incl - len) + 1 : 0, lane); // 1 + the sum in front of the last head up to here
		const int32_t run = hs? incl - (int32_t)(hs - 1) : carry + incl;
		const int32_t o = n_out + mask_rank(mh, lane) + head - 1;
		if (j < tot && (lane == MGB_W - 1 || j == tot - 1 || (mh >> (lane + 1) & 1))) O[o] = (uint64_t)(int64_t)run << 4 | (uint64_t)op;
		carry = warp_bcast_i32(run, MGB_W - 1), prev_op = warp_bcast_i32(op, MGB_W - 1), t_lo = warp_bcast_i32(t, MGB_W - 1);
		n_out += mask_count(mh);
	}
	mlen = warp_sum_i32(mlen), blen = warp_sum_i32(blen), aplen = warp_sum_i32(aplen), l = warp_sum_i32(l);
	if (lane == 0) {
		gc->has_cigar = 1;
		gc->n_cigar = n_out;
		gc->c_ss = (int32_t)gt.a[off_a0].x + 1 - (int32_t)(gt.a[off_a0].y >> 32 & 0xff);
		gc->c_ee = (int32_t)gt.a[off_a0 + gc->n_anchor - 1].x + 1;
		gc->c_mlen = mlen, gc->c_blen = blen, gc->c_aplen = aplen;
	}
	if (!(l == gc->qe - gc->qs && aplen == gc->pe - gc->ps)) return MGB_E_INTERNAL;
	warp_sync();
	*ops = O;
	return 0;
}

// ---- ds:Z difference string (reference: galign.c:182-293 mg_gchain_gen_ds) ----

MG_HD inline char ds_nt(const char *s, int64_t i) { return "acgtn"[nt4((uint8_t)s[i])]; }
MG_HD inline int32_t ds_ndig(uint32_t x) { int32_t n = 1; while (x >= 10) x /= 10, ++n; return n; }
MG_HD inline void ds_put_int(char *w, uint32_t x, int32_t n) { for (int32_t k = n - 1; k >= 0; --k) w[k] = (char)('0' + x % 10), x /= 10; }

// The text of one alignment match of len bases at t[] on the walk and q[] on the read (reference: galign.c:234-254), at w[]
// with its offsets, which count from b0, at off[]; w == 0: only counted.  Returns the bytes, *n_off the offsets.
MG_HD inline int32_t ds_match(char *w, int32_t *off, int32_t b0, int32_t op, int32_t len, const char *t, const char *q, int32_t *n_off)
{
	int32_t nb = 0, no = 0, l = 0, z = 0;
	if (op == 7) l = len, z = len; // '=' runs hold identical characters: nothing to look at
	for (; z < len; ++z) {
		const int cx = nt4((uint8_t)t[z]), cy = nt4((uint8_t)q[z]);
		if (cx != cy) {
			if (l > 0) {
				const int32_t d = ds_ndig((uint32_t)l);
				if (w) off[no] = b0 + nb, w[nb] = ':', ds_put_int(w + nb + 1, (uint32_t)l, d);
				++no, nb += 1 + d;
			}
			if (w) off[no] = b0 + nb, w[nb] = '*', w[nb + 1] = "acgtn"[cx], w[nb + 2] = "acgtn"[cy];
			++no, nb += 3, l = 0;
		} else ++l;
	}
	if (l > 0) {
		const int32_t d = ds_ndig((uint32_t)l);
		if (w) off[no] = b0 + nb, w[nb] = ':', ds_put_int(w + nb + 1, (uint32_t)l, d);
		++no, nb += 1 + d;
	}
	*n_off = no;
	return nb;
}

// How far an indel of len bases at s[p] repeats into its flanks inside [lo, hi): ll bases to its right, lr to its left
// (reference: galign.c:256-264 and 270-278).  One lane, and the same with the whole warp testing MGB_W positions at a time.
MG_HD inline void ds_flanks(const char *s, int32_t p, int32_t len, int32_t lo, int32_t hi, int32_t *ll, int32_t *lr)
{
	int32_t z;
	for (z = 1; z <= len; ++z)
		if (p - z < lo || s[p + len - z] != s[p - z]) break;
	*lr = z - 1;
	for (z = 0; z < len; ++z)
		if (p + len + z >= hi || s[p + len + z] != s[p + z]) break;
	*ll = z;
}
MG_HD inline void ds_flanks_w(const char *s, int32_t p, int32_t len, int32_t lo, int32_t hi, int32_t *ll, int32_t *lr, int lane)
{
	*lr = *ll = len;
	for (int32_t z0 = 1; z0 <= len; z0 += MGB_W) {
		const int32_t z = z0 + lane;
		const uint32_t m = warp_ballot(z <= len && (p - z < lo || s[p + len - z] != s[p - z]));
		if (m) { *lr = z0 + mask_lowest(m) - 1; break; }
	}
	for (int32_t z0 = 0; z0 < len; z0 += MGB_W) {
		const int32_t z = z0 + lane;
		const uint32_t m = warp_ballot(z < len && (p + len + z >= hi || s[p + len + z] != s[p + z]));
		if (m) { *ll = z0 + mask_lowest(m); break; }
	}
}

// The text of an indel (reference: galign.c:153-180 write_indel): its sign, then its bases, those that repeat in the flanks (ll
// on the left, lr on the right) in brackets, all of them when ll + lr >= len.  Its length, and its byte r.
MG_HD inline int32_t ds_indel_bytes(int32_t len, int32_t ll, int32_t lr) { return 1 + (ll + lr >= len? len + 2 : len + (ll > 0? 2 : 0) + (lr > 0? 2 : 0)); }
MG_HD inline char ds_indel_char(int32_t r, int32_t op, int32_t len, const char *s, int32_t ll, int32_t lr)
{
	if (r == 0) return op == 1? '+' : '-';
	r -= 1;
	if (ll + lr >= len) return r == 0? '[' : r == len + 1? ']' : ds_nt(s, r - 1);
	const int32_t a = ll > 0? ll + 2 : 0;
	if (r < a) return r == 0? '[' : r == a - 1? ']' : ds_nt(s, r - 1);
	r -= a;
	if (r < len - ll - lr) return ds_nt(s, ll + r);
	r -= len - ll - lr;
	return r == 0? '[' : r == lr + 1? ']' : ds_nt(s, len - lr + r - 1);
}

static const int32_t DS_LONG_INDEL = 32; // an indel this long or longer is taken by the whole warp: its text and its flank scans grow with its length

// One pass of the ds:Z string of a chain over its n_cigar merged operations ops[], MGB_W at a time, lane l on operation base+l.
// What an operation writes depends only on its kind and length, on where it starts on the walk (x, in seq[0, aplen)) and on
// the read (y, in qseq[qs, qe)) and on the two sequences: a scan of the operations' advances gives every one its x and y, a scan
// of their sizes places their text.  Indels of DS_LONG_INDEL bases or more are taken by the whole warp, one after the other.
//   sizing (WRITE false): at[j] = number of offsets << 32 | bytes in front of operation j; *ds_len and *n_off the totals;
//   writing (WRITE true): the CIGAR to dc[], the text to ds[] and its offsets to dof[], each operation where the sizing pass
//   placed it.
// Warp-uniform.
template<bool WRITE>
MG_HD inline void gchain_ds_pass_w(const uint64_t *ops, int32_t n_cigar, uint64_t *at, const char *seq, int32_t aplen, const char *qseq, int32_t qs, int32_t qe,
                                   uint64_t *dc, char *ds, int32_t *dof, int32_t *ds_len, int32_t *n_off, int lane)
{
	int32_t x0 = 0, y0 = qs, b_tot = 0, o_tot = 0;
	for (int32_t base = 0; base < n_cigar; base += MGB_W) {
		const int32_t j = base + lane;
		int32_t op = -1, len = 0;
		if (j < n_cigar) {
			const uint64_t v = ops[j];
			op = (int32_t)(v & 0xf), len = (int32_t)(v >> 4);
			if (WRITE) dc[j] = v;
		}
		const int match = op == 0 || op == 7 || op == 8, indel = op == 1 || op == 2;
		const int32_t dx = match || op == 2? len : 0, dy = match || op == 1? len : 0;
		const int32_t ix = warp_incl_scan_i32(dx, lane), iy = warp_incl_scan_i32(dy, lane);
		const int32_t x = x0 + ix - dx, y = y0 + iy - dy;
		x0 += warp_bcast_i32(ix, MGB_W - 1), y0 += warp_bcast_i32(iy, MGB_W - 1);
		const char *s = op == 1? qseq : seq;
		const int32_t p = op == 1? y : x, lo = op == 1? qs : 0, hi = op == 1? qe : aplen;
		const int is_long = indel && len >= DS_LONG_INDEL;
		const uint32_t m_long = warp_ballot(is_long);
		int32_t ll = 0, lr = 0;
		for (uint32_t m = m_long; m; m &= m - 1) {
			const int src = mask_lowest(m);
			const int32_t sop = warp_bcast_i32(op, src), slen = warp_bcast_i32(len, src), sp = warp_bcast_i32(p, src);
			int32_t a, b;
			ds_flanks_w(sop == 1? qseq : seq, sp, slen, sop == 1? qs : 0, sop == 1? qe : aplen, &a, &b, lane);
			if (lane == src) ll = a, lr = b;
		}
		if (indel && !is_long) ds_flanks(s, p, len, lo, hi, &ll, &lr);
		int32_t b0, o0;
		if (!WRITE) {
			int32_t nb = 0, no = 0;
			if (indel) nb = ds_indel_bytes(len, ll, lr), no = 1;
			else if (match) nb = ds_match(0, 0, 0, op, len, seq + x, qseq + y, &no);
			const int32_t ib = warp_incl_scan_i32(nb, lane), io = warp_incl_scan_i32(no, lane);
			b0 = b_tot + ib - nb, o0 = o_tot + io - no;
			if (j < n_cigar) at[j] = (uint64_t)(uint32_t)o0 << 32 | (uint32_t)b0;
			b_tot += warp_bcast_i32(ib, MGB_W - 1), o_tot += warp_bcast_i32(io, MGB_W - 1);
			continue;
		}
		b0 = o0 = 0;
		if (j < n_cigar) { const uint64_t v = at[j]; b0 = (int32_t)(uint32_t)v, o0 = (int32_t)(v >> 32); }
		if (indel && !is_long) {
			const int32_t nb = ds_indel_bytes(len, ll, lr);
			dof[o0] = b0;
			for (int32_t r = 0; r < nb; ++r) ds[b0 + r] = ds_indel_char(r, op, len, s + p, ll, lr);
		} else if (match) {
			int32_t no;
			ds_match(ds + b0, dof + o0, b0, op, len, seq + x, qseq + y, &no);
		}
		for (uint32_t m = m_long; m; m &= m - 1) {
			const int src = mask_lowest(m);
			const int32_t sop = warp_bcast_i32(op, src), slen = warp_bcast_i32(len, src), sp = warp_bcast_i32(p, src), sb0 = warp_bcast_i32(b0, src);
			const int32_t sll = warp_bcast_i32(ll, src), slr = warp_bcast_i32(lr, src);
			const char *ss = (sop == 1? qseq : seq) + sp;
			const int32_t nb = ds_indel_bytes(slen, sll, slr);
			for (int32_t r = lane; r < nb; r += MGB_W) ds[sb0 + r] = ds_indel_char(r, sop, slen, ss, sll, slr);
			if (lane == src) dof[o0] = b0;
		}
	}
	*ds_len = b_tot, *n_off = o_tot;
}

// per-read result header, one per read, in an array parallel to ReadMeta
struct ReadOut {
	int32_t status;
	int32_t n_gc, n_lc, n_a, rep_len;
	int32_t n_mz;
	uint32_t blob_size, blob2_size;
	int64_t blob_off;   // output pool: GChain[n_gc] | LLChain[n_lc] | u128 a[n_a]          (written by stage_gchain)
	int64_t blob2_off;  // output pool: per chain CIGAR (u64) | ds text | ds offsets        (written by stage_finish)
};

MG_HD inline uint64_t align8(uint64_t x) { return (x + 7) & ~(uint64_t)7; }

// the three parts of a read's first blob in the output pool (ReadOut::blob_off), each 8-byte aligned
struct ReadBlob { const GChain *gc; const LLChain *lc; const u128 *a; };
MG_HD inline ReadBlob read_blob(const char *pool, const ReadOut &ro)
{
	ReadBlob b;
	const char *blob = pool + ro.blob_off;
	b.gc = (const GChain*)blob;
	b.lc = (const LLChain*)(blob + align8((uint64_t)ro.n_gc * sizeof(GChain)));
	b.a = (const u128*)((const char*)b.lc + align8((uint64_t)ro.n_lc * sizeof(LLChain)));
	return b;
}

// state handed from the graph-chaining DP pass to the materialisation pass
struct GState {
	int32_t n_lc, n_u, n_gc, n_jobs;
	int64_t job_first;
	// followed by LChain lc[n_lc] | uint64 u[n_u] | uint32 gc_hash[n_gc]
};

// K6 for one read: graph chaining DP, overlap resolution, bridging plan (one lane).
// bridging plan of one read and the state K7 picks up again; one lane
MG_HD inline int stage_gchain_plan(const PipeCtx &c, ReadMeta &m, int rid, Arena &A, int32_t n_lc, LChain *lc, int32_t n_u, const uint64_t *u, const u128 *a, uint32_t *gc_hash)
{
	const MapOptDev &o = c.opt;
	int32_t n_gc = 0;
	// a read's jobs must be contiguous in the pool (they are consumed in order): reserve the worst case, one job per
	// linear chain, up front and mark the unused slots
	int64_t job_first;
	{
		int64_t off = pool_alloc(c.pool_gjobs, (uint64_t)(n_lc > 0? n_lc : 1) * sizeof(GwfaJob));
		if (off < 0) return MGB_E_POOL;
		job_first = off / (int64_t)sizeof(GwfaJob);
	}
	struct LocalEmit {
		GwfaJob *dst; int rid; int32_t n, cap;
		MG_HD int operator()(GwfaJob &J) { if (n >= cap) return MGB_E_INTERNAL; J.rid = rid; dst[n++] = J; return 0; }
	} le;
	le.dst = c.gjobs + job_first, le.rid = rid, le.n = 0, le.cap = n_lc > 0? n_lc : 1;
	MGB_TRY(gchain_prep(c.g, n_u, u, lc, a, m.hash, o.min_gc_cnt, o.min_gc_score, o.gdp_max_ed, batch_n_seg(c.b, rid), gc_hash, &n_gc, le));
	for (int32_t i = le.n; i < le.cap; ++i) le.dst[i].rid = -1; // unused reserved slots: skipped by the job kernel
	// persist
	uint64_t sz = sizeof(GState) + align8((uint64_t)n_lc * sizeof(LChain)) + (uint64_t)n_u * 8 + align8((uint64_t)n_gc * 4);
	int64_t goff = pool_alloc(c.pool_gstate, sz);
	if (goff < 0) return MGB_E_POOL;
	GState *gsb = (GState*)(c.gstate + goff);
	gsb->n_lc = n_lc, gsb->n_u = n_u, gsb->n_gc = n_gc, gsb->n_jobs = le.n, gsb->job_first = job_first;
	LChain *dlc = (LChain*)(gsb + 1);
	for (int32_t i = 0; i < n_lc; ++i) dlc[i] = lc[i];
	uint64_t *du = (uint64_t*)((char*)dlc + align8((uint64_t)n_lc * sizeof(LChain)));
	for (int32_t i = 0; i < n_u; ++i) du[i] = u[i];
	uint32_t *dh = (uint32_t*)(du + n_u);
	for (int32_t i = 0; i < n_gc; ++i) dh[i] = gc_hash[i];
	m.gstate_off = goff;
	return 0;
}

// the result header of a read as K6 starts it (lane 0)
MG_HD inline void gchain_out_init(ReadOut &ro, const ReadMeta &m)
{
	ro.status = 0, ro.n_gc = ro.n_lc = ro.n_a = 0, ro.rep_len = m.rep_len, ro.n_mz = m.n_mz, ro.blob_size = ro.blob2_size = 0, ro.blob_off = ro.blob2_off = 0;
}

// the end of K6 after the graph-chaining DP, entered by all lanes: the bridging plan on lane 0, its code on every lane
MG_HD inline int stage_gchain_tail(const PipeCtx &c, ReadMeta &m, int rid, Arena &A, int32_t n_lc, LChain *lc, int32_t n_u, const uint64_t *u, const u128 *a,
								   uint32_t *gc_hash, int lane)
{
	int rc = 0;
	if (lane == 0) {
		Arena B = A;
		rc = stage_gchain_plan(c, m, rid, B, n_lc, lc, n_u, u, a, gc_hash);
		if (B.peak > A.peak) A.peak = B.peak;
	}
	return warp_bcast_i32(rc, 0);
}

// K6 for one read, entered by all lanes of a warp: the graph-chaining DP is warp-wide (gchain_dp_w), the bridging plan and the
// hand-over to K7 (a few dozen words per read) are written by lane 0.
MG_HD inline int stage_gchain(const PipeCtx &c, ReadOut *routs, int rid, Arena &A, int lane)
{
	ReadMeta &m = c.meta[rid];
	ReadOut &ro = routs[rid];
	const MapOptDev &o = c.opt;
	if (lane == 0) gchain_out_init(ro, m);
	if (m.status != 0) { if (lane == 0) ro.status = m.status; return 0; } // status 1: read skipped (empty or too long) -> no result object
	const uint64_t mark = A.top;
	const int32_t qlen = c.b.seq_len[rid];
	const u128 *a = c.anchor + m.a_off;
	int32_t n_lc = m.n_lc, n_u = 0;
	uint64_t *u = 0;
	LChain *lc;
	uint32_t *gc_hash;
	MGB_ALLOC(A, lc, LChain, n_lc);
	MGB_ALLOC(A, gc_hash, uint32_t, n_lc);
	for (int32_t i = lane; i < n_lc; i += MGB_W) lc[i] = c.lchain[m.lc_off + i];
	warp_sync();
	unsigned long long pt0 = prof_clock();
	GcParam gp;
	gp.max_dist_g = gp.max_dist_q = gp.bw = o.bw_long, gp.ref_bonus = o.ref_bonus, gp.chn_pen_gap = o.chn_pen_gap, gp.mask_level = o.mask_level; // reference: map-algo.c:461-462
	MGB_TRY(gchain_dp_w(A, c.g, c.lab, &n_lc, lc, qlen, gp, o.max_gc_skip, a, &u, &n_u, lane));
	if (lane == 0) { unsigned long long dt = prof_clock() - pt0; prof_add(c, PROF_GC_DP_CYC, dt); prof_max(c, PROF_GC_DP_MAX_CYC, dt); }
	const int rc = stage_gchain_tail(c, m, rid, A, n_lc, lc, n_u, u, a, gc_hash, lane);
	A.top = mark;
	return rc;
}

// K7a: one bridging alignment (reference: gchain1.c:349-381), all lanes of the warp on gwf_align_w().  The alignment state
// (GwfShared: the arena header, the wavefront state and the result) sits in the warp's slice of shared memory, where every lane
// sees it; the wavefronts themselves are allocated from the worker's arena in HBM.
static const int GWF_SHARED_BYTES = 1024; // the slice of shared memory per warp of k_gwfa
static_assert(sizeof(GwfShared) <= GWF_SHARED_BYTES, "the alignment state has to fit the warp's slice of shared memory");

MG_HD inline int gwfa_job_run(Arena &A, const PipeCtx &c, int64_t job_idx, int lane, int32_t *smem)
{
	GwfaJob *J = &c.gjobs[job_idx];
	if (J->rid < 0) return 0;
	if (c.meta[J->rid].status < 0) return 0;
	GwfShared *sh = (GwfShared*)smem; // the one copy of the alignment state, seen by all lanes
	GwfOpt opt;
	opt.traceback = 1, opt.max_chk = 1000, opt.bw_dyn = 1000, opt.max_lag = J->max_ed / 2, opt.s_term = -1;
	opt.i_term = 500000000LL;
	const char *qseq = c.b.seq + c.b.seq_off[J->rid];
	unsigned long long t0 = prof_clock();
	if (lane == 0) sh->A = A, sh->A.peak = A.top;
	warp_sync();
	int rc = gwf_align_w(sh, c.g, opt, J->ql, qseq + J->qs, J->v0, J->end0, J->v1, J->end1, J->max_ed, lane);
	if (sh->A.peak > A.peak) A.peak = sh->A.peak;
	if (lane == 0) {
		const GwfResult &r = sh->r;
		{ unsigned long long dt = prof_clock() - t0; prof_add(c, PROF_GC_GWFA_CYC, dt); prof_max(c, PROF_GWFA_MAX_CYC, dt << 16 | (unsigned long long)(J->ql < 65535? J->ql : 65535)); }
		if (rc == 0) {
			J->s = r.s, J->nv = r.s >= 0? r.nv : 0;
			if (r.s >= 0) {
				int64_t woff = pool_alloc(c.pool_walk, (uint64_t)r.nv * 4);
				if (woff < 0) rc = MGB_E_POOL;
				else {
					J->walk_off = woff / 4;
					for (int32_t i = 0; i < r.nv; ++i) c.walk[J->walk_off + i] = r.v[i];
				}
			}
		}
	}
	warp_sync();
	rc = warp_bcast_i32(rc, 0);
	return rc;
}

// What the sequential head of stage_gchain_gen<1>() hands to the warp-wide tail (stage_gchain_gen_w, parameter "gen_v2")
struct GenHand {
	GcSet gs;
	int64_t boff;
	uint64_t off_lc, off_a, sz, mark;
	unsigned long long pt3;
	int32_t want_plan, skip;
};

// gchain_cigar_plan() entered by all lanes of a warp.  Every kept anchor but the first yields exactly one item, which depends on
// the anchor, on the kept anchor in front of it and on the linear chains the two sit on: the kept anchors are listed by an
// ordered compaction, then every lane makes the item of one of them; the jobs of a chunk are allocated with one pool request.
MG_HD inline int gchain_cigar_plan_w(Arena &A, const PipeCtx &c, int rid, const GraphDev &g, GcSet &gt, int64_t lc_off_bytes, int lane)
{
	for (int32_t i = 0; i < gt.n_gc; ++i) {
		GChain *gc = &gt.gc[i];
		const int32_t off_a0 = gt.lc[gc->off].off, n_anchor = gc->n_anchor, l_beg = gc->off, l_end = gc->off + gc->cnt;
		uint64_t mark = A.top;
		int32_t *kj, *kl; // kept anchors (index into the chain's anchors) and the linear chain each sits on; entry 0 is the first anchor
		uint64_t *plan;
		MGB_ALLOC(A, kj, int32_t, n_anchor + 1);
		MGB_ALLOC(A, kl, int32_t, n_anchor + 1);
		MGB_ALLOC(A, plan, uint64_t, n_anchor + 8);
		if (lane == 0) kj[0] = 0, kl[0] = l_beg;
		int32_t nk = 1, bad = 0;
		for (int32_t base = 1; base < n_anchor; base += MGB_W) {
			const int32_t j = base + lane;
			int keep = 0, l = -1;
			if (j < n_anchor) {
				keep = !((gt.a[off_a0 + j].y & SEED_IGNORE) && j != n_anchor - 1);
				if (keep) { // the linear chains of a graph chain own disjoint, ascending runs of its anchors
					for (l = l_beg; l < l_end; ++l)
						if (off_a0 + j >= gt.lc[l].off && off_a0 + j < gt.lc[l].off + gt.lc[l].cnt) break;
					if (l >= l_end) bad = 1;
				}
			}
			const uint32_t mk = warp_ballot(keep);
			if (keep) { const int32_t at = nk + mask_rank(mk, lane); kj[at] = j, kl[at] = l; }
			nk += mask_count(mk);
		}
		if (warp_any(bad)) return MGB_E_INTERNAL;
		warp_sync();
		if (lane == 0) plan[0] = (uint64_t)(gt.a[off_a0].y >> 32 & 0xff) << 4 | 7;
		for (int32_t base = 1; base < nk; base += MGB_W) {
			const int32_t k = base + lane;
			uint64_t item = 0;
			int is_job = 0;
			int32_t l0 = 0, l = 0, l_seq = 0, qlen = 0;
			u128 p, q;
			p.x = p.y = q.x = q.y = 0;
			if (k < nk) {
				p = gt.a[off_a0 + kj[k]], q = gt.a[off_a0 + kj[k - 1]];
				l = kl[k], l0 = kl[k - 1];
				if (l == l0) l_seq = (int32_t)p.x - (int32_t)q.x;
				else {
					l_seq = g.seg_len[gt.lc[l0].v >> 1] - (int32_t)q.x - 1;
					for (int32_t t = l0 + 1; t < l; ++t) l_seq += g_vlen(g, gt.lc[t].v);
					l_seq += (int32_t)p.x + 1;
				}
				qlen = (int32_t)p.y - (int32_t)q.y;
				if (!(l_seq > 0 || qlen > 0)) bad = 1;
				else if (l_seq == 0) item = (uint64_t)(int64_t)qlen << 4 | 1;
				else if (qlen == 0) item = (uint64_t)(int64_t)l_seq << 4 | 2;
				else if (l_seq == qlen && (uint64_t)(int64_t)qlen <= (q.y >> 32 & 0xff)) item = (uint64_t)(int64_t)qlen << 4 | 7;
				else is_job = 1;
			}
			if (warp_any(bad)) return MGB_E_INTERNAL;
			const uint32_t mj = warp_ballot(is_job);
			int64_t jbase = 0;
			if (mj) {
				if (lane == 0) jbase = pool_alloc(c.pool_jobs, (uint64_t)mask_count(mj) * sizeof(WfaJob));
				jbase = (int64_t)warp_bcast_u64((uint64_t)jbase, 0);
				if (jbase < 0) return MGB_E_POOL;
			}
			if (is_job) {
				const int64_t joff = jbase + (int64_t)mask_rank(mj, lane) * (int64_t)sizeof(WfaJob);
				WfaJob *J = (WfaJob*)((char*)c.jobs + joff);
				J->rid = rid, J->gc = i, J->l0 = l0, J->l = l, J->t_beg = (int32_t)q.x + 1, J->t_last = (int32_t)p.x;
				J->tl = l_seq, J->ql = qlen, J->q_off = (int32_t)q.y + 1, J->n_cigar = 0, J->status = 0, J->lc_off = lc_off_bytes, J->cig_off = 0;
				item = PLAN_JOB | (uint64_t)(joff / (int64_t)sizeof(WfaJob));
			}
			if (k < nk) plan[k] = item;
		}
		warp_sync();
		int64_t poff = 0;
		if (lane == 0) poff = pool_alloc(c.pool_plan, (uint64_t)nk * 8);
		poff = (int64_t)warp_bcast_u64((uint64_t)poff, 0);
		if (poff < 0) return MGB_E_POOL;
		uint64_t *dst = c.plan + poff / 8;
		for (int32_t t = lane; t < nk; t += MGB_W) dst[t] = plan[t];
		if (lane == 0) gc->plan_off = poff / 8, gc->n_plan = nk;
		warp_sync();
		A.top = mark;
	}
	return 0;
}

// K7b for one read: materialise graph chains from the DP and the bridging results, post filters, alignment plan.
// n_rebridged: as gchain_gen() has it.
MG_HD inline int stage_gchain_gen_head(const PipeCtx &c, ReadOut *routs, int rid, Arena &A, GenHand *hand, int32_t *n_rebridged = 0)
{
	ReadMeta &m = c.meta[rid];
	ReadOut &ro = routs[rid];
	const MapOptDev &o = c.opt;
	if (m.status != 0) { ro.status = m.status; return 0; }
	uint64_t mark = A.top;
	const char *qseq = c.b.seq + c.b.seq_off[rid];
	const int32_t qlen = c.b.seq_len[rid];
	const u128 *a = c.anchor + m.a_off;
	const GState *gsb = (const GState*)(c.gstate + m.gstate_off);
	const int32_t n_lc = gsb->n_lc, n_u = gsb->n_u;
	LChain *lc;
	MGB_ALLOC(A, lc, LChain, n_lc);
	{
		const LChain *slc = (const LChain*)(gsb + 1);
		for (int32_t i = 0; i < n_lc; ++i) lc[i] = slc[i];
	}
	const uint64_t *u = (const uint64_t*)((const char*)(gsb + 1) + align8((uint64_t)n_lc * sizeof(LChain)));
	const uint32_t *gc_hash = (const uint32_t*)(u + n_u);
	GwfaFeed feed;
	feed.job = c.gjobs + gsb->job_first, feed.walk_pool = c.walk, feed.next = 0, feed.n = gsb->n_jobs;
	GcSet gs;
	unsigned long long pt1 = prof_clock();
	MGB_TRY(gchain_gen(A, c.g, n_u, u, lc, a, m.hash, o.min_gc_cnt, o.min_gc_score, o.gdp_max_ed, batch_n_seg(c.b, rid), qseq, gs, &feed, gc_hash, n_rebridged));
	gs.rep_len = m.rep_len;
	unsigned long long pt2 = prof_clock();
	prof_add(c, PROF_GC_GEN_CYC, pt2 - pt1);
	prof_add(c, PROF_GC_SHORTK_CYC, gs.cyc_shortk), prof_add(c, PROF_GC_EXTRA_CYC, gs.cyc_extra);
	MGB_TRY(gchain_set_parent(A, o.mask_level, gs.n_gc, gs.gc, o.sub_diff));
	gchain_flt_sub(o.pri_ratio, c.ix.k * 2, o.best_n, gs.n_gc, gs.gc);
	MGB_TRY(gchain_drop_flt(A, gs));
	MGB_TRY(gchain_set_mapq(o, gs, qlen, m.n_mz, o.min_gc_score));
	unsigned long long pt3 = prof_clock();
	prof_add(c, PROF_GC_POST_CYC, pt3 - pt2);
	// ---- part 1 of the result ----
	uint64_t off_lc = align8((uint64_t)gs.n_gc * sizeof(GChain));
	uint64_t off_a = off_lc + align8((uint64_t)gs.n_lc * sizeof(LLChain));
	uint64_t sz = off_a + align8((uint64_t)gs.n_a * sizeof(u128));
	int64_t boff = pool_alloc(c.pool_out, sz);
	if (boff < 0) return MGB_E_POOL;
	for (int32_t i = 0; i < gs.n_gc; ++i) {
		GChain *gc = &gs.gc[i];
		gc->has_cigar = 0, gc->n_cigar = 0, gc->cigar_off = gc->ds_off = gc->dsoff_off = 0, gc->ds_len = gc->n_dsoff = 0, gc->plan_off = 0, gc->n_plan = 0;
	}
	hand->gs = gs, hand->boff = boff, hand->off_lc = off_lc, hand->off_a = off_a, hand->sz = sz, hand->mark = mark, hand->pt3 = pt3;
	hand->want_plan = (o.flag & F_CIGAR) && gs.n_gc > 0 && batch_n_seg(c.b, rid) == 1, hand->skip = 0; // reference: map-algo.c:475
	return 0;
}

// stage_gchain_gen() entered by all lanes of a warp (parameter "gen_v2"): lane 0 runs the sequential head, then the plan and
// the copies of the first part of the result are shared by the lanes.
MG_HD inline int stage_gchain_gen(const PipeCtx &c, ReadOut *routs, int rid, Arena &A, int lane, int32_t *n_rebridged = 0)
{
	GenHand h;
	h.gs.n_gc = h.gs.n_lc = h.gs.n_a = h.gs.rep_len = 0, h.gs.gc = 0, h.gs.lc = 0, h.gs.a = 0;
	h.gs.cyc_gwfa = h.gs.cyc_shortk = h.gs.cyc_extra = 0;
	h.boff = 0, h.off_lc = h.off_a = h.sz = 0, h.mark = A.top, h.pt3 = 0, h.want_plan = 0, h.skip = 1;
	int rc = 0;
	Arena B = A;
	if (lane == 0) rc = stage_gchain_gen_head(c, routs, rid, B, &h, n_rebridged);
	rc = warp_bcast_i32(rc, 0);
	A.top = warp_bcast_u64(B.top, 0), A.peak = warp_bcast_u64(B.peak, 0);
	h.skip = warp_bcast_i32(h.skip, 0);
	warp_sync();
	if (rc < 0 || h.skip) { A.top = h.mark; return rc; }
	h.gs.n_gc = warp_bcast_i32(h.gs.n_gc, 0), h.gs.n_lc = warp_bcast_i32(h.gs.n_lc, 0), h.gs.n_a = warp_bcast_i32(h.gs.n_a, 0);
	h.gs.gc = (GChain*)warp_bcast_u64((uint64_t)h.gs.gc, 0), h.gs.lc = (LLChain*)warp_bcast_u64((uint64_t)h.gs.lc, 0), h.gs.a = (u128*)warp_bcast_u64((uint64_t)h.gs.a, 0);
	h.boff = (int64_t)warp_bcast_u64((uint64_t)h.boff, 0), h.off_lc = warp_bcast_u64(h.off_lc, 0), h.off_a = warp_bcast_u64(h.off_a, 0), h.sz = warp_bcast_u64(h.sz, 0);
	h.want_plan = warp_bcast_i32(h.want_plan, 0);
	if (h.want_plan) MGB_TRY(gchain_cigar_plan_w(A, c, rid, c.g, h.gs, h.boff + (int64_t)h.off_lc, lane));
	char *blob = c.out + h.boff;
	{
		GChain *d = (GChain*)blob;
		for (int32_t i = lane; i < h.gs.n_gc; i += MGB_W) d[i] = h.gs.gc[i];
		LLChain *dl = (LLChain*)(blob + h.off_lc);
		for (int32_t i = lane; i < h.gs.n_lc; i += MGB_W) dl[i] = h.gs.lc[i];
		u128 *da = (u128*)(blob + h.off_a);
		for (int32_t i = lane; i < h.gs.n_a; i += MGB_W) da[i] = h.gs.a[i];
	}
	if (lane == 0) {
		ReadOut &ro = routs[rid];
		ro.n_gc = h.gs.n_gc, ro.n_lc = h.gs.n_lc, ro.n_a = h.gs.n_a, ro.blob_size = (uint32_t)h.sz, ro.blob_off = h.boff;
		prof_add(c, PROF_GC_PLAN_CYC, prof_clock() - h.pt3);
	}
	warp_sync();
	A.top = h.mark;
	return 0;
}

// What K8b keeps of a chain between its passes, in the worker's arena: the merged CIGAR, where the ds:Z text of each of its
// operations goes (gchain_ds_pass_w) and the aligned part of the walk.
struct FinChain { uint64_t *ops, *at; char *seq; };

// K8b for one read: stitch the CIGARs, size the ds:Z strings, take part 2 of the result from the pool in one piece and write
// every chain's CIGAR, ds text and ds offsets straight to their place in it.  Warp-uniform: all lanes enter.
MG_HD inline int stage_finish(const PipeCtx &c, ReadOut *routs, int rid, Arena &A, int lane)
{
	ReadMeta &m = c.meta[rid];
	ReadOut &ro = routs[rid];
	if (m.status != 0) { if (lane == 0) ro.status = m.status; return 0; }
	if (!(c.opt.flag & F_CIGAR) || ro.n_gc == 0 || batch_n_seg(c.b, rid) != 1) return 0;
	uint64_t mark = A.top;
	const GraphDev &g = c.g;
	const char *qseq = c.b.seq + c.b.seq_off[rid];
	char *blob = c.out + ro.blob_off;
	GcSet gs;
	gs.n_gc = ro.n_gc, gs.n_lc = ro.n_lc, gs.n_a = ro.n_a, gs.rep_len = ro.rep_len;
	gs.gc = (GChain*)blob;
	gs.lc = (LLChain*)(blob + align8((uint64_t)gs.n_gc * sizeof(GChain)));
	gs.a = (u128*)((char*)gs.lc + align8((uint64_t)gs.n_lc * sizeof(LLChain)));
	FinChain *fc;
	MGB_ALLOC(A, fc, FinChain, gs.n_gc);
	unsigned long long pt0 = prof_clock();
	for (int32_t i = 0; i < gs.n_gc; ++i) {
		uint64_t *ops;
		MGB_TRY(gchain_cigar_finish_w(A, c, gs, i, &ops, lane));
		if (lane == 0) fc[i].ops = ops;
	}
	unsigned long long pt1 = prof_clock();
	uint64_t sz = 0;
	for (int32_t i = 0; i < gs.n_gc; ++i) { // sizing pass
		GChain *gc = &gs.gc[i];
		const int32_t aplen = gc->c_aplen, n_cigar = gc->n_cigar;
		char *seq;
		uint64_t *at;
		MGB_ALLOC(A, seq, char, aplen + 1);
		MGB_ALLOC(A, at, uint64_t, n_cigar);
		int64_t seq_l = 0;
		for (int32_t j = 0; j < gc->cnt; ++j) { // the aligned part of the walk (reference: galign.c:197-207)
			const uint32_t v = gs.lc[gc->off + j].v;
			const int32_t st = j > 0? 0 : gc->c_ss;
			const int32_t en = j < gc->cnt - 1? g_vlen(g, v) : gc->c_ee;
			if (seq_l + (en - st) > aplen) return MGB_E_INTERNAL;
			const char *s = g_vseq(g, v) + st;
			for (int32_t t = lane; t < en - st; t += MGB_W) seq[seq_l + t] = s[t];
			seq_l += en - st;
		}
		if (seq_l != aplen) return MGB_E_INTERNAL;
		warp_sync();
		int32_t ds_len, n_off;
		gchain_ds_pass_w<false>(fc[i].ops, n_cigar, at, seq, aplen, qseq, gc->qs, gc->qe, 0, 0, 0, &ds_len, &n_off, lane);
		sz += align8((uint64_t)n_cigar * 8) + align8((uint64_t)ds_len + 1) + align8((uint64_t)n_off * 4);
		warp_sync();
		if (lane == 0) fc[i].at = at, fc[i].seq = seq, gc->ds_len = ds_len, gc->n_dsoff = n_off;
	}
	int64_t boff = 0;
	if (lane == 0) boff = pool_alloc(c.pool_out, sz);
	boff = (int64_t)warp_bcast_u64((uint64_t)boff, 0);
	if (boff < 0) return MGB_E_POOL;
	warp_sync();
	uint64_t at = (uint64_t)boff;
	for (int32_t i = 0; i < gs.n_gc; ++i) { // writing pass
		GChain *gc = &gs.gc[i];
		const int32_t n_cigar = gc->n_cigar, ds_len = gc->ds_len, n_off = gc->n_dsoff;
		const int64_t cigar_off = (int64_t)at; at += align8((uint64_t)n_cigar * 8);
		const int64_t ds_off = (int64_t)at; at += align8((uint64_t)ds_len + 1);
		const int64_t dsoff_off = (int64_t)at; at += align8((uint64_t)n_off * 4);
		char *dd = c.out + ds_off;
		int32_t wl, wo;
		gchain_ds_pass_w<true>(fc[i].ops, n_cigar, fc[i].at, fc[i].seq, gc->c_aplen, qseq, gc->qs, gc->qe, (uint64_t*)(c.out + cigar_off), dd, (int32_t*)(c.out + dsoff_off), &wl, &wo, lane);
		warp_sync();
		if (lane == 0) gc->cigar_off = cigar_off, gc->ds_off = ds_off, gc->dsoff_off = dsoff_off, dd[ds_len] = 0;
	}
	if (lane == 0) prof_add(c, PROF_FIN_CIGAR_CYC, pt1 - pt0), prof_add(c, PROF_FIN_DS_CYC, prof_clock() - pt1);
	if (lane == 0) ro.blob2_off = boff, ro.blob2_size = (uint32_t)sz;
	A.top = mark;
	return 0;
}

} // namespace mgb
