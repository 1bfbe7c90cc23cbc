// mgb_gchain.cuh -- graph chaining over linear chains and materialisation of graph chains.
//   gchain1_dp()   (reference: gchain1.c:62-240 mg_gchain1_dp, :38-60 cal_sc)
//   gchain_gen()   (reference: gchain1.c:443-520 mg_gchain_gen with resolve_overlap / bridge_* helpers)
//   gchain_extra() (reference: gchain1.c:242-297 mg_gchain_extra; the log() for `div` is left to the host)
//   post-filters   (reference: gcmisc.c:56-223)
#pragma once
#include "mgb_model.cuh"
#include "mgb_lchain.cuh"
#include "mgb_shortk.cuh"
#include "mgb_gclabel.cuh"
#include "mgb_gwfa.cuh"

namespace mgb {

// reference: minigraph.h:108-113 mg_llchain_t
struct LLChain {
	int32_t off, cnt;
	uint32_t v;
	int32_t score, ed;
};

// device-side graph chain: mg_gchain_t (minigraph.h:125-138) without host pointers, plus what the host needs to
// finish it (n_mini/q_span for `div`, CIGAR and ds locations inside the result blob)
struct GChain {
	int32_t id, parent;
	int32_t off, cnt;
	int32_t n_anchor, score;
	int32_t qs, qe;
	int32_t plen, ps, pe;
	int32_t blen, mlen;
	uint32_t hash;
	int32_t subsc, n_sub;
	int32_t mapq, flt;
	int32_t n_mini, q_span;
	// base alignment
	int32_t has_cigar, n_cigar, c_mlen, c_blen, c_aplen, c_ss, c_ee;
	int32_t ds_len, n_dsoff;
	int64_t cigar_off, ds_off, dsoff_off; // byte offsets into the output pool
	int64_t plan_off;                     // element offset into the plan pool (alignment plan of this chain)
	int32_t n_plan, pad_;
};

struct GcFrag { uint32_t srt; int32_t i; };
struct KeyGcFrag { MG_HD uint64_t operator()(const GcFrag &p) const { return p.srt; } };

// ---- graph chaining DP (reference: gchain1.c:62-240 mg_gchain1_dp, :38-60 cal_sc) ----
// The reference walks, for every linear chain i in query-end order, back over the chains j in front of it, collects those that
// could precede i, asks mg_shortest_k() for the graph distance to each, and scores them.  Here:
//   * what mg_shortest_k() would answer comes from the per-source label table (mgb_gclabel.cuh) -- a binary search;
//   * whether j can precede i, the graph distance and everything of the score but f[j] depend on the two chains alone, so that
//     part is evaluated for ALL pairs (i, j) at once, one pair per lane;
//   * only the order-dependent part is replayed row by row, 32 predecessors per step: the walk stops at the first pair whose
//     query gap is too long, and after max_skip predecessors that are already the chosen predecessor of a chain visited before
//     them in the same walk (the t[] marks of the reference; p[j] < j, so a mark only ever lands on a lane further along and one
//     ballot per step replays the counter), then the best score in walk order wins.

// a linear chain as the DP sees it, in DP order (non-isolated chains by ascending query end)
struct GcNode {
	int32_t qs, qe, rs, re, score, vlen;
	uint32_t v;
	int32_t seg_f, seg_l; // read segment of the first / last anchor (paired reads; 0 otherwise)
	int32_t lci;          // index into lc[]
};

enum { GCP_SKIP = 0, GCP_CAND = 1, GCP_STOP = 2 };
struct GcPair {
	int32_t sc;     // score of chaining i after j without f[j]; SC_NONE: j is not reachable from i or out of band
	int32_t dist;
	uint32_t hash;
	int32_t st;     // GCP_* | inner << 4
};

// where the walk of row i starts: the reference's find_max() (gchain1.c:16-30) over the i chains in front, with its quirk --
// when some but not all of them end before x it returns the first one that does NOT
MG_HD inline int32_t gc_walk_start(int32_t i, const GcNode *N, int32_t x)
{
	int32_t lo = 0, hi = i; // number of chains with qe < x (they are sorted by qe)
	while (lo < hi) { const int32_t mid = (lo + hi) >> 1; if (N[mid].qe < x) lo = mid + 1; else hi = mid; }
	if (lo == i) return i - 1;
	return lo == 0? -1 : lo;
}

struct GcParam { int32_t max_dist_g, max_dist_q, bw, ref_bonus; float chn_pen_gap, mask_level; };

MG_HD inline bool gc_overlap_too_big(int32_t o, int32_t len_j, int32_t len_i, float mask_level)
{
	return (float)o > (float)len_j * mask_level || (float)o > (float)len_i * mask_level;
}

// One pair: can chain j (ending first on the query) precede chain i, and at what score?  `rec` holds the labels of i's source.
MG_HD inline GcPair gc_eval_pair(const GcNode &I, const GcNode &J, const GcParam &P, const char *rec)
{
	GcPair r;
	r.sc = SC_NONE, r.dist = -1, r.hash = 0, r.st = GCP_SKIP;
	if (J.qs >= I.qs) return r;                                    // j inside i on the query
	const int32_t dq = I.qs - J.qe;
	if (dq < 0 && gc_overlap_too_big(-dq, J.qe - J.qs, I.qe - I.qs, P.mask_level)) return r;
	const bool same_seg = I.seg_f == J.seg_l;
	if (same_seg? dq > P.max_dist_q : (dq > P.max_dist_g && dq > P.max_dist_q)) { r.st = GCP_STOP; return r; } // every chain further back is further away
	const int32_t tail_j = J.vlen - J.re, head_i = I.rs;            // bases behind j / in front of i on their segments
	const bool inner = I.v == J.v;
	if (!inner) {
		const int32_t min_dist = head_i + tail_j;
		if (min_dist > P.max_dist_g) return r;
		if (same_seg && min_dist - P.bw > dq) return r;
	} else {
		if (J.rs >= I.rs || J.re >= I.re) return r;                // not colinear on the segment
		const int32_t dr = I.rs - J.re, w = dr > dq? dr - dq : dq - dr;
		if (same_seg && w > P.bw) return r;
		if (dr > P.max_dist_g || dr < -P.max_dist_g) return r;
		if (dr < 0 && gc_overlap_too_big(-dr, J.re - J.rs, I.re - I.rs, P.mask_level)) return r;
	}
	const int32_t target = dq - tail_j + (I.vlen - I.rs);          // mg_target_dist(): graph distance that would match the query gap
	if (!inner && target < 0) return r;
	r.st = GCP_CAND | (inner? 16 : 0);
	int32_t dist = 0, is_0 = 0;
	uint32_t hash = 0;
	if (!inner && !lab_query(rec, J.v ^ 1, P.max_dist_g + (I.vlen - I.rs), target, &dist, &hash, &is_0)) return r; // not reachable
	r.dist = dist, r.hash = hash;
	int32_t gap = dist - target;
	if (gap < 0) gap = -gap;
	if (same_seg && gap > P.bw) return r;
	int32_t sc = I.score;
	if (J.qe > I.qs) sc = (int32_t)((double)(I.qe - J.qe) / (double)(I.qe - I.qs) * (double)I.score + .499); // i's share beyond the query overlap
	if (is_0) sc += P.ref_bonus;
	const float lin_pen = P.chn_pen_gap * (float)gap, log_pen = gap >= 2? fast_log2((float)gap) : 0.0f;
	r.sc = sc - (int32_t)(lin_pen + log_pen);
	return r;
}

// Entered by all lanes of a warp.  lc[] (in the arena) is permuted into chain order; u[] (score<<32|#lchains) sits at the caller's mark.
MG_HD inline int gchain_dp_w(Arena &A, const GraphDev &g, const LabTab &T, int32_t *n_lc_, LChain *lc, int32_t qlen, const GcParam &P, int32_t max_skip,
							 const u128 *an, uint64_t **u_, int32_t *n_u_, int lane)
{
	const int32_t n_lc = *n_lc_;
	*u_ = 0, *n_u_ = 0;
	if (n_lc == 0) return 0;
	uint64_t *u_store;
	MGB_ALLOC(A, u_store, uint64_t, n_lc);
	const uint64_t mark = A.top;
	GcFrag *a;
	MGB_ALLOC(A, a, GcFrag, n_lc);
	int32_t n_ext = 0;
	for (int32_t i0 = 0; i0 < n_lc; i0 += MGB_W) { // chains far from both segment ends (or small against that distance) do not take part
		const int32_t i = i0 + lane;
		int ext = 0;
		if (i < n_lc) {
			LChain *r = &lc[i];
			const uint32_t isolated = gc_isolated(g, *r, P.max_dist_g);
			r->dist_pre = -1;
			a[i].srt = isolated << 31 | (uint32_t)r->qe, a[i].i = i;
			ext = !isolated;
		}
		n_ext += mask_count(warp_ballot(ext));
	}
	warp_sync();
	if (n_ext < 2) {
		for (int32_t i = lane; i < n_lc; i += MGB_W) u_store[i] = (uint64_t)(int64_t)lc[i].score << 32 | 1;
		warp_sync();
		A.top = mark;
		*u_ = u_store, *n_u_ = n_lc;
		return 0;
	}
	MGB_TRY(radix_sort_exact_w(A, a, n_lc, 4, KeyGcFrag(), lane)); // klib's unstable sort: its tie order is the DP order
	GcNode *N;
	int32_t *v, *f, *p, *t, *x0, *roff;
	const char **rec;
	MGB_ALLOC(A, N, GcNode, n_ext);
	MGB_ALLOC(A, v, int32_t, n_lc);
	MGB_ALLOC(A, f, int32_t, n_ext);
	MGB_ALLOC(A, p, int32_t, n_ext);
	MGB_ALLOC(A, t, int32_t, n_ext);
	MGB_ALLOC(A, x0, int32_t, n_ext);
	MGB_ALLOC(A, roff, int32_t, n_ext + 1);
	MGB_ALLOC(A, rec, const char*, n_ext);
	for (int32_t i = lane; i < n_ext; i += MGB_W) {
		const LChain &r = lc[a[i].i];
		GcNode n;
		n.qs = r.qs, n.qe = r.qe, n.rs = r.rs, n.re = r.re, n.score = r.score, n.v = r.v, n.vlen = g.seg_len[r.v >> 1], n.lci = a[i].i;
		n.seg_f = (int32_t)((an[r.off].y & SEED_SEG_MASK) >> SEED_SEG_SHIFT);
		n.seg_l = (int32_t)((an[r.off + r.cnt - 1].y & SEED_SEG_MASK) >> SEED_SEG_SHIFT);
		N[i] = n, t[i] = 0;
	}
	warp_sync();
	for (int32_t i = lane; i < n_ext; i += MGB_W) {
		int32_t x = N[i].qs + P.bw;
		if (x > qlen) x = qlen;
		x0[i] = gc_walk_start(i, N, x);
		const long long off = T.src_off && x0[i] >= 0? T.src_off[N[i].v ^ 1] : LAB_NONE;
		rec[i] = off >= 0? T.pool + off : 0;
	}
	warp_sync();
	{ // row offsets into the pair buffer; sources the table does not have (yet) are searched here
		Arena B = A;
		int rc = 0;
		if (lane == 0) {
			roff[0] = 0;
			for (int32_t i = 0; i < n_ext; ++i) roff[i + 1] = roff[i] + (x0[i] + 1);
			for (int32_t i = 1; i < n_ext && rc == 0; ++i) {
				if (rec[i] || x0[i] < 0) continue;
				for (int32_t k = 1; k < i; ++k) if (N[k].v == N[i].v && rec[k]) { rec[i] = rec[k]; break; }
				if (rec[i]) continue;
				const uint64_t m2 = B.top;
				char *r0;
				uint64_t bytes;
				rc = label_search(B, g, N[i].v ^ 1, P.max_dist_g + N[i].vlen, &r0, &bytes);
				if (rc < 0) break;
				uint64_t *d = (uint64_t*)(B.base + m2); // the record moves down over the search's scratch
				const uint64_t *s = (const uint64_t*)r0;
				for (uint64_t q = 0; q < bytes / 8; ++q) d[q] = s[q];
				B.top = m2 + ((bytes + 15) & ~(uint64_t)15);
				rec[i] = (const char*)d;
			}
		}
		rc = warp_bcast_i32(rc, 0);
		A.top = warp_bcast_u64(B.top, 0);
		const uint64_t pk = warp_bcast_u64(B.peak, 0);
		if (pk > A.peak) A.peak = pk;
		warp_sync();
		if (rc < 0) return rc;
	}
	if (lane == 0) { // row 0 has nobody in front of it
		LChain *l0 = &lc[N[0].lci];
		f[0] = N[0].score, p[0] = -1, v[0] = N[0].score, l0->dist_pre = -1, l0->hash_pre = 0, l0->inner_pre = 0;
	}
	warp_sync();
	const int32_t n_pairs = roff[n_ext];
	int32_t max_row = 0;
	for (int32_t i = lane; i < n_ext; i += MGB_W) max_row = x0[i] + 1 > max_row? x0[i] + 1 : max_row;
	max_row = warp_max_i32(max_row);
	const int32_t budget = n_pairs < 16384? n_pairs : (max_row > 16384? max_row : 16384); // pairs evaluated per block of rows
	GcPair *Q;
	MGB_ALLOC(A, Q, GcPair, budget);
	for (int32_t i0 = 1; i0 < n_ext;) {
		int32_t i1 = i0 + 1;
		while (i1 < n_ext && roff[i1 + 1] - roff[i0] <= budget) ++i1;
		const int32_t base = roff[i0], n_blk = roff[i1] - base;
		// (1) all pairs of rows [i0, i1), one per lane, stored in walk order (descending j)
		for (int32_t q = lane; q < n_blk; q += MGB_W) {
			int32_t lo = i0, hi = i1; // the row whose range holds q
			while (hi - lo > 1) { const int32_t mid = (lo + hi) >> 1; if (roff[mid] - base <= q) lo = mid; else hi = mid; }
			const int32_t i = lo, j = x0[i] - (q - (roff[i] - base));
			Q[q] = gc_eval_pair(N[i], N[j], P, rec[i]);
		}
		warp_sync();
		// (2) the walks, row by row
		for (int32_t i = i0; i < i1; ++i) {
			const GcNode &I = N[i];
			const GcPair *row = Q + (roff[i] - base);
			const int32_t cnt = x0[i] + 1;
			int32_t max_f = I.score, max_j = -1, max_d = -1, max_inner = 0, n_skip = 0;
			uint32_t max_hash = 0;
			for (int32_t k0 = 0; k0 < cnt; k0 += MGB_W) {
				const int32_t k = k0 + lane, j = x0[i] - k;
				GcPair e;
				e.sc = SC_NONE, e.dist = -1, e.hash = 0, e.st = GCP_SKIP;
				if (k < cnt) e = row[k];
				const uint32_t stop_m = warp_ballot((e.st & 15) == GCP_STOP);
				const int first_stop = stop_m? ctz32(stop_m) : MGB_W;
				const int cand = (e.st & 15) == GCP_CAND && lane < first_stop;
				const int32_t pj = cand? p[j] : -1;
				if (pj >= 0) t[pj] = i; // marks of lanes past the cut below are never looked at
				warp_sync();
				const int marked = cand && t[j] == i;
				const uint32_t mark_m = warp_ballot(marked);
				const int over = marked && n_skip + mask_rank(mark_m, lane) + 1 > max_skip;
				const uint32_t over_m = warp_ballot(over);
				const int cut = over_m? ctz32(over_m) : MGB_W; // the walk ends with this lane's chain (it is still a candidate)
				const int live = cand && lane <= cut;
				int32_t sc = SC_NONE;
				if (live && e.sc != SC_NONE) { sc = e.sc + f[j]; if (sc + I.score < 0) sc = SC_NONE; }
				const int32_t best = warp_max_i32(sc);
				if (best != SC_NONE && best > max_f) { // the first chain of the walk that reaches the best score
					const int w = ctz32(warp_ballot(sc == best));
					max_f = best, max_j = warp_bcast_i32(j, w), max_d = warp_bcast_i32(e.dist, w);
					max_hash = (uint32_t)warp_bcast_i32((int32_t)e.hash, w), max_inner = warp_bcast_i32(e.st >> 4, w);
				}
				n_skip += mask_count(mark_m);
				warp_sync();
				if (stop_m || over_m) break;
			}
			if (lane == 0) {
				LChain *li = &lc[I.lci];
				f[i] = max_f, p[i] = max_j;
				li->dist_pre = max_d, li->hash_pre = max_hash, li->inner_pre = max_inner;
				v[i] = max_j >= 0 && v[max_j] > max_f? v[max_j] : max_f;
			}
			warp_sync();
		}
		i0 = i1;
	}
	// ---- peel the chains (lchain.c:27-77, shared with linear chaining), isolated chains behind them, lc[] into chain order ----
	uint64_t *u = 0;
	int32_t n_u = 0, n_v = 0;
	{
		Arena B = A;
		int rc = 0;
		if (lane == 0) rc = chain_backtrack(B, n_ext, f, p, v, t, 0, 0, INT32_MAX, n_lc - n_ext, &u, &n_u, &n_v);
		rc = warp_bcast_i32(rc, 0);
		if (rc < 0) return rc;
		A.top = warp_bcast_u64(B.top, 0);
		const uint64_t pk = warp_bcast_u64(B.peak, 0);
		if (pk > A.peak) A.peak = pk;
		u = (uint64_t*)warp_bcast_u64((uint64_t)u, 0), n_u = warp_bcast_i32(n_u, 0), n_v = warp_bcast_i32(n_v, 0);
	}
	if (u == 0) { MGB_ALLOC(A, u, uint64_t, n_lc); n_u = n_v = 0; } // every f >= 0 = min_sc, so this does not happen
	LChain *ordered;
	int32_t *first;
	MGB_ALLOC(A, ordered, LChain, n_v + (n_lc - n_ext));
	MGB_ALLOC(A, first, int32_t, n_u + 1);
	if (lane == 0) { first[0] = 0; for (int32_t c = 0; c < n_u; ++c) first[c + 1] = first[c] + (int32_t)u[c]; }
	warp_sync();
	if (first[n_u] != n_v) return MGB_E_INTERNAL;
	for (int32_t c = lane; c < n_u; c += MGB_W) { // v[] lists a chain from its end: turn every chain around
		const int32_t k0 = first[c], n = (int32_t)u[c];
		for (int32_t s = 0; s < n; ++s) ordered[k0 + s] = lc[a[v[k0 + n - 1 - s]].i];
	}
	for (int32_t s = lane; s < n_lc - n_ext; s += MGB_W) {
		const LChain &r = lc[a[n_ext + s].i];
		u[n_u + s] = (uint64_t)(int64_t)r.score << 32 | 1;
		ordered[n_v + s] = r;
	}
	n_u += n_lc - n_ext, n_v += n_lc - n_ext;
	warp_sync();
	for (int32_t s = lane; s < n_v; s += MGB_W) lc[s] = ordered[s];
	for (int32_t s = lane; s < n_u; s += MGB_W) u_store[s] = u[s];
	warp_sync();
	*n_lc_ = n_v;
	A.top = mark;
	*u_ = u_store, *n_u_ = n_u;
	return 0;
}


// ---- materialise graph chains ----

struct GcSet { // device analogue of mg_gchains_t
	int32_t n_gc, n_lc, n_a, rep_len;
	GChain *gc;
	LLChain *lc;
	u128 *a;
	unsigned long long cyc_gwfa, cyc_shortk, cyc_extra; // instrumentation
};

// One bridging alignment between two linear chains on different vertices (reference: gchain1.c:349-381 bridge_gwfa).
// Independent of every other bridge of the read, so the planning pass (gchain_prep) emits them as jobs for the
// warp-cooperative K7a kernel and gchain_gen() consumes the results in the same order.
struct GwfaJob {
	int32_t rid;
	uint32_t v0, v1;
	int32_t end0, end1;
	int32_t qs, ql;
	int32_t max_ed;
	int32_t s, nv, status;  // results: edit distance (-1: none within max_ed), walk length
	int64_t walk_off;       // element offset of the walk (int32 vertices) in the walk pool
};

struct GwfaFeed { // precomputed bridge results of one read, consumed in order
	const GwfaJob *job;
	const int32_t *walk_pool;
	int32_t next, n;
};

struct BridgeAux {
	const GraphDev *g;
	GwfaFeed *feed;
	const char *qseq;
	AVec<LLChain> llc;
	int32_t n_a;
	u128 *a_new;
	unsigned long long cyc_gwfa, cyc_shortk;
};

MG_HD inline void gc_copy_lchain(LLChain *q, const LChain *p, int32_t *n_a, u128 *a_new, const u128 *a_old, int32_t ed)
{
	q->cnt = p->cnt, q->v = p->v, q->score = p->score, q->ed = ed;
	for (int32_t i = 0; i < p->cnt; ++i) a_new[*n_a + i] = a_old[p->off + i];
	q->off = *n_a;
	(*n_a) += q->cnt;
}

MG_HD inline int gc_push_empty(Arena &A, BridgeAux &aux, uint32_t v)
{
	LLChain q;
	q.off = q.cnt = q.score = 0, q.v = v, q.ed = -1;
	return avec_push(A, aux.llc, q);
}

// reference: gchain1.c:319-347 bridge_shortk; returns 0, or 1 when no consistent walk exists (the reference's -1)
MG_HD inline int gc_bridge_shortk(Arena &A, BridgeAux &aux, const LChain *l0, const LChain *l1, int *failed)
{
	uint64_t mark = A.top;
	int32_t n_pathv;
	PathDst dst;
	PathV *p;
	*failed = 0;
	memset(&dst, 0, sizeof(dst));
	dst.v = l0->v ^ 1;
	if (l1->dist_pre < 0) return MGB_E_INTERNAL;
	dst.target_dist = l1->dist_pre;
	dst.target_hash = l1->hash_pre;
	dst.check_hash = 1;
	MGB_TRY(shortest_k(A, *aux.g, l1->v ^ 1, 1, &dst, dst.target_dist, MAX_SHORT_K, &p, &n_pathv));
	if (n_pathv == 0 || dst.target_hash != dst.hash) {
		A.top = mark;
		*failed = 1;
		return 0;
	}
	// the path was found backwards: reverse it and flip orientations.  llc may grow above p, p stays valid.
	for (int32_t s = n_pathv - 2; s >= 1; --s) MGB_TRY(gc_push_empty(A, aux, p[s].v ^ 1));
	return 0; // NB: p[] is not released here when llc grew above it; the caller's mark reclaims it
}

// reference: gchain1.c:349-381 bridge_gwfa; *ok = 1 when an alignment within gdp_max_ed was found
MG_HD inline int gc_bridge_gwfa(Arena &A, BridgeAux &aux, int32_t kmer_size, int32_t gdp_max_ed, const LChain *l0, const LChain *l1, int32_t *ed, int *ok)
{
	uint32_t v0 = l0->v, v1 = l1->v;
	int32_t qs = l0->qe - kmer_size, qe = l1->qs + kmer_size, end0, end1;
	GwfOpt opt;
	GwfResult r;
	*ed = -1, *ok = 0;
	end0 = l0->re - kmer_size;
	end1 = l1->rs + kmer_size - 1;
	opt.traceback = 1, opt.max_chk = 1000, opt.bw_dyn = 1000, opt.max_lag = gdp_max_ed / 2, opt.s_term = -1;
	opt.i_term = 500000000LL;
	if (aux.feed) { // the alignment was done by the job kernel
		if (aux.feed->next >= aux.feed->n) return MGB_E_INTERNAL;
		const GwfaJob *J = &aux.feed->job[aux.feed->next++];
		if (J->v0 != v0 || J->v1 != v1 || J->end0 != end0 || J->end1 != end1 || J->qs != qs || J->ql != qe - qs) return MGB_E_INTERNAL;
		if (J->s < 0) return 0;
		const int32_t *w = aux.feed->walk_pool + J->walk_off;
		for (int32_t j = 1; j < J->nv - 1; ++j) MGB_TRY(gc_push_empty(A, aux, (uint32_t)w[j]));
		*ed = J->s, *ok = 1;
		return 0;
	}
	uint64_t mark = A.top;
	// walk vertices are copied out before llc can grow over them
	MGB_TRY(gwf_align(A, *aux.g, opt, qe - qs, &aux.qseq[qs], v0, end0, v1, end1, gdp_max_ed, &r));
	if (r.s < 0) { A.top = mark; return 0; }
	// r.v sits at `mark`; pushing to llc may allocate above it, which is fine
	for (int32_t j = 1; j < r.nv - 1; ++j) MGB_TRY(gc_push_empty(A, aux, (uint32_t)r.v[j]));
	*ed = r.s, *ok = 1;
	return 0;
}

// reference: gchain1.c:383-407 bridge_lchains; *failed mirrors the reference's negative return
MG_HD inline int gc_bridge_lchains(Arena &A, BridgeAux &aux, int32_t n_seg, int32_t kmer_size, int32_t gdp_max_ed, const LChain *l0, const LChain *l1,
								   const u128 *a, int *failed)
{
	*failed = 0;
	if (l1->v != l0->v) {
		int32_t ed = -1;
		int ok = 0, sk_failed = 0;
		unsigned long long t0 = prof_clock();
		if (n_seg <= 1) MGB_TRY(gc_bridge_gwfa(A, aux, kmer_size, gdp_max_ed, l0, l1, &ed, &ok));
		unsigned long long t1 = prof_clock();
		aux.cyc_gwfa += t1 - t0;
		if (!ok) MGB_TRY(gc_bridge_shortk(A, aux, l0, l1, &sk_failed));
		aux.cyc_shortk += prof_clock() - t1;
		if (sk_failed) { *failed = 1; return 0; }
		LLChain q;
		gc_copy_lchain(&q, l1, &aux.n_a, aux.a_new, a, ed);
		MGB_TRY(avec_push(A, aux.llc, q));
	} else {
		int32_t k;
		LLChain *t = &aux.llc.a[aux.llc.n - 1];
		for (k = 0; k < l1->cnt; ++k) {
			const u128 *ak = &a[l1->off + k];
			if ((int32_t)ak->x > l0->re && (int32_t)ak->y > l0->qe) break;
		}
		if (k < l1->cnt) {
			t->cnt += l1->cnt - k, t->score += l1->score;
			for (int32_t i = 0; i < l1->cnt - k; ++i) aux.a_new[aux.n_a + i] = a[l1->off + k + i];
			aux.n_a += l1->cnt - k;
		}
	}
	return 0;
}

// reference: gchain1.c:409-441 resolve_overlap
MG_HD inline int gc_resolve_overlap(LChain *l0, LChain *l1, const u128 *a)
{
	int32_t j, x, y, shift0, shift1;
	x = (int32_t)a[l1->off].x;
	y = (int32_t)a[l1->off].y;
	for (j = l0->cnt - 1; j >= 0; --j)
		if ((int32_t)a[l0->off + j].y <= y && (l0->v != l1->v || (int32_t)a[l0->off + j].x <= x)) break;
	shift0 = l0->cnt - 1 - j;
	x = (int32_t)a[l0->off + l0->cnt - 1].x;
	y = (int32_t)a[l0->off + l0->cnt - 1].y;
	for (j = 0; j < l1->cnt; ++j)
		if ((int32_t)a[l1->off + j].y >= y && (l0->v != l1->v || (int32_t)a[l1->off + j].x >= x)) break;
	shift1 = j;
	if (shift1 >= l1->cnt) return MGB_E_INTERNAL;
	if (shift0 > 0) {
		l0->cnt -= shift0;
		if (l0->cnt) {
			l0->qe = (int32_t)a[l0->off + l0->cnt - 1].y + 1;
			l0->re = (int32_t)a[l0->off + l0->cnt - 1].x + 1;
		}
	}
	if (shift1 > 0) {
		l1->off += shift1, l1->cnt -= shift1;
		l1->qs = (int32_t)a[l1->off].y + 1 - (int32_t)(a[l1->off].y >> 32 & 0xff);
		l1->rs = (int32_t)a[l1->off].x + 1 - (int32_t)(a[l1->off].y >> 32 & 0xff);
	}
	if (l0->cnt == 0) l0->qs = l0->qe = l1->qs, l0->rs = l0->re = l1->rs;
	return 0;
}

// reference: gchain1.c:242-297 mg_gchain_extra (integer part; div = f(n_mini, n_anchor, q_span) is finished on the host)
MG_HD inline int gchain_extra(const GraphDev &g, GcSet &gs)
{
	for (int32_t i = 0; i < gs.n_gc; ++i) {
		GChain *p = &gs.gc[i];
		const LLChain *q;
		const u128 *last_a;
		int32_t q_span, rest_pl, tmp, n_mini;
		p->qs = p->qe = p->ps = p->pe = -1, p->plen = p->blen = p->mlen = 0, p->n_mini = 0, p->q_span = 0;
		if (p->cnt == 0) continue;
		if (!(gs.lc[p->off].cnt > 0 && gs.lc[p->off + p->cnt - 1].cnt > 0)) return MGB_E_INTERNAL;
		q = &gs.lc[p->off];
		q_span = (int32_t)(gs.a[q->off].y >> 32 & 0xff);
		p->qs = (int32_t)gs.a[q->off].y + 1 - q_span;
		p->ps = (int32_t)gs.a[q->off].x + 1 - q_span;
		tmp = (int32_t)(gs.a[q->off].x >> 32);
		q = &gs.lc[p->off + p->cnt - 1];
		p->qe = (int32_t)gs.a[q->off + q->cnt - 1].y + 1;
		p->pe = g.seg_len[q->v >> 1] - (int32_t)gs.a[q->off + q->cnt - 1].x - 1;
		n_mini = (int32_t)(gs.a[q->off + q->cnt - 1].x >> 32) - tmp + 1;
		rest_pl = 0;
		last_a = &gs.a[gs.lc[p->off].off];
		for (int32_t j = 0; j < p->cnt; ++j) {
			const LLChain *qq = &gs.lc[p->off + j];
			int32_t vlen = g.seg_len[qq->v >> 1];
			p->plen += vlen;
			for (int32_t k = 0; k < qq->cnt; ++k) {
				const u128 *r = &gs.a[qq->off + k];
				int32_t pl, ql = (int32_t)r->y - (int32_t)last_a->y;
				int32_t span = (int32_t)(r->y >> 32 & 0xff);
				if (j == 0 && k == 0) pl = ql = span;
				else if (j > 0 && k == 0) pl = (int32_t)r->x + 1 + rest_pl;
				else pl = (int32_t)r->x - (int32_t)last_a->x;
				if (ql < 0) ql = -ql, n_mini += (int32_t)(last_a->x >> 32) - (int32_t)(r->x >> 32);
				p->blen += pl > ql? pl : ql;
				p->mlen += pl > span && ql > span? span : pl < ql? pl : ql;
				last_a = r;
			}
			if (qq->cnt == 0) rest_pl += vlen;
			else rest_pl = vlen - (int32_t)gs.a[qq->off + qq->cnt - 1].x - 1;
		}
		p->pe = p->plen - p->pe;
		if (p->pe < p->ps) return MGB_E_INTERNAL;
		p->n_mini = n_mini, p->q_span = q_span;
	}
	return 0;
}

// reference: gcmisc.c:8-33 mg_gchain_restore_order
MG_HD inline int gchain_restore_order(Arena &A, GcSet &gs)
{
	uint64_t mark = A.top;
	int32_t i, n_a, n_lc;
	LLChain *lc;
	u128 *a;
	MGB_ALLOC(A, lc, LLChain, gs.n_lc);
	MGB_ALLOC(A, a, u128, gs.n_a);
	for (i = 0, n_a = n_lc = 0; i < gs.n_gc; ++i) {
		GChain *gc = &gs.gc[i];
		if (gc->cnt <= 0) return MGB_E_INTERNAL;
		for (int32_t k = 0; k < gc->cnt; ++k) lc[n_lc + k] = gs.lc[gc->off + k];
		const u128 *src = &gs.a[gs.lc[gc->off].off];
		for (int32_t k = 0; k < gc->n_anchor; ++k) a[n_a + k] = src[k];
		n_lc += gc->cnt, n_a += gc->n_anchor;
	}
	for (i = 0; i < gs.n_lc; ++i) gs.lc[i] = lc[i];
	for (i = 0; i < gs.n_a; ++i) gs.a[i] = a[i];
	for (i = 0, n_lc = 0; i < gs.n_gc; ++i) {
		gs.gc[i].off = n_lc;
		n_lc += gs.gc[i].cnt;
	}
	for (i = 0, n_a = 0; i < gs.n_lc; ++i) {
		gs.lc[i].off = n_a;
		n_a += gs.lc[i].cnt;
	}
	A.top = mark;
	return 0;
}

// reference: gcmisc.c:56-71 mg_gchain_sort_by_score
MG_HD inline int gchain_sort_by_score(Arena &A, GcSet &gs)
{
	uint64_t mark = A.top;
	u128 *z;
	GChain *gc;
	MGB_ALLOC(A, z, u128, gs.n_gc);
	MGB_ALLOC(A, gc, GChain, gs.n_gc);
	for (int32_t i = 0; i < gs.n_gc; ++i)
		z[i].x = (uint64_t)(int64_t)gs.gc[i].score << 32 | gs.gc[i].hash, z[i].y = (uint64_t)i;
	MGB_TRY(radix_sort_128x(A, z, gs.n_gc));
	for (int32_t i = gs.n_gc - 1; i >= 0; --i) gc[gs.n_gc - 1 - i] = gs.gc[z[i].y];
	for (int32_t i = 0; i < gs.n_gc; ++i) gs.gc[i] = gc[i];
	A.top = mark;
	return gchain_restore_order(A, gs);
}

// Build graph chains from the DP result.  Output arrays are allocated at the caller's mark (gs.gc, gs.a, gs.lc).
// Planning pass of gchain_gen(): hash the chains that will be kept, resolve their overlaps (lc[] is modified) and
// emit one GwfaJob per bridge between different vertices (same pair enumeration as the loop in gchain_gen()).
template<typename Emit>
MG_HD inline int gchain_prep(const GraphDev &g, int32_t n_u, const uint64_t *u, LChain *lc, const u128 *a, uint32_t hash, int32_t min_gc_cnt,
							 int32_t min_gc_score, int32_t gdp_max_ed, int32_t n_seg, uint32_t *gc_hash, int32_t *n_gc_, Emit &emit)
{
	int32_t i, j, k, st, kmer_size = 0;
	*n_gc_ = 0;
	for (i = k = 0, st = 0; i < n_u; ++i) {
		int32_t m = 0, nui = (int32_t)u[i];
		for (j = 0; j < nui; ++j) m += lc[st + j].cnt;
		if (m >= min_gc_cnt && (int64_t)(u[i] >> 32) >= (int64_t)min_gc_score) {
			uint32_t h = hash;
			int32_t j0;
			if (k == 0) kmer_size = (int32_t)(a[0].y >> 32 & 0xff);
			for (j = 0; j < nui; ++j) {
				const LChain *p = &lc[st + j];
				h += hash32((uint32_t)p->qs) + hash32((uint32_t)p->re) + hash32(p->v);
			}
			gc_hash[k] = hash32(h);
			for (j = 1; j < nui; ++j) MGB_TRY(gc_resolve_overlap(&lc[st + j - 1], &lc[st + j], a));
			for (j0 = 0, j = 1; j < nui; ++j) {
				const LChain *l0 = &lc[st + j0], *l1 = &lc[st + j];
				if (l1->cnt > 0) {
					if (l1->v != l0->v && n_seg <= 1) { // multi-segment fragments are bridged by shortest walks only (gchain1.c:387)
						GwfaJob J;
						J.rid = 0, J.v0 = l0->v, J.v1 = l1->v;
						J.qs = l0->qe - kmer_size, J.ql = (l1->qs + kmer_size) - J.qs;
						J.end0 = l0->re - kmer_size, J.end1 = l1->rs + kmer_size - 1;
						J.max_ed = gdp_max_ed, J.s = -1, J.nv = 0, J.status = 0, J.walk_off = 0;
						MGB_TRY(emit(J));
					}
					j0 = j;
				}
			}
			++k;
		}
		st += nui;
	}
	*n_gc_ = k;
	return 0;
}

// With `feed`, gchain_prep() has already hashed the chains (gc_hash) and resolved overlaps, and the bridging
// alignments come from the job kernel.  n_rebridged (NULL in the pipeline) counts the pairs bridged again in place.
MG_HD inline int gchain_gen(Arena &A, const GraphDev &g, int32_t n_u, const uint64_t *u, LChain *lc, const u128 *a, uint32_t hash,
							int32_t min_gc_cnt, int32_t min_gc_score, int32_t gdp_max_ed, int32_t n_seg, const char *qseq, GcSet &gs,
							GwfaFeed *feed, const uint32_t *gc_hash, int32_t *n_rebridged = 0)
{
	int32_t i, j, k, st, kmer_size;
	gs.n_gc = gs.n_lc = gs.n_a = 0, gs.rep_len = 0, gs.gc = 0, gs.lc = 0, gs.a = 0, gs.cyc_gwfa = gs.cyc_shortk = gs.cyc_extra = 0;
	int32_t n_lc_in = 0;
	for (i = 0, st = 0; i < n_u; ++i) {
		int32_t m = 0, nui = (int32_t)u[i];
		for (j = 0; j < nui; ++j) m += lc[st + j].cnt;
		if (m >= min_gc_cnt && (int64_t)(u[i] >> 32) >= (int64_t)min_gc_score) gs.n_gc++, gs.n_a += m;
		st += nui;
	}
	n_lc_in = st;
	if (gs.n_gc == 0) return 0;
	MGB_ALLOC(A, gs.gc, GChain, gs.n_gc);
	memset(gs.gc, 0, sizeof(GChain) * (size_t)gs.n_gc);
	MGB_ALLOC(A, gs.a, u128, gs.n_a);
	// llc can hold at most one entry per input lchain plus the bridging vertices: give it head room below the scratch
	BridgeAux aux;
	aux.g = &g, aux.feed = feed, aux.qseq = qseq, aux.n_a = 0, aux.a_new = gs.a, aux.cyc_gwfa = aux.cyc_shortk = 0;
	avec_init(aux.llc);
	MGB_TRY(avec_reserve(A, aux.llc, n_lc_in + 64));
	kmer_size = (int32_t)(a[0].y >> 32 & 0xff);
	for (i = k = 0, st = 0; i < n_u; ++i) {
		int32_t n_a0 = aux.n_a, n_llc0 = (int32_t)aux.llc.n, m = 0, nui = (int32_t)u[i];
		for (j = 0; j < nui; ++j) m += lc[st + j].cnt;
		if (m >= min_gc_cnt && (int64_t)(u[i] >> 32) >= (int64_t)min_gc_score) {
			uint32_t h = hash;
			int32_t j0;
			gs.gc[k].score = (int32_t)(u[i] >> 32);
			gs.gc[k].off = n_llc0;
			if (feed) gs.gc[k].hash = gc_hash[k];
			else {
				for (j = 0; j < nui; ++j) {
					const LChain *p = &lc[st + j];
					h += hash32((uint32_t)p->qs) + hash32((uint32_t)p->re) + hash32(p->v);
				}
				gs.gc[k].hash = hash32(h);
				for (j = 1; j < nui; ++j) MGB_TRY(gc_resolve_overlap(&lc[st + j - 1], &lc[st + j], a));
			}
			{
				LLChain q;
				gc_copy_lchain(&q, &lc[st], &aux.n_a, gs.a, a, -1);
				MGB_TRY(avec_push(A, aux.llc, q));
			}
			for (j0 = 0, j = 1; j < nui; ++j) {
				const LChain *l0 = &lc[st + j0], *l1 = &lc[st + j];
				if (l1->cnt > 0) {
					int failed;
					MGB_TRY(gc_bridge_lchains(A, aux, n_seg, kmer_size, gdp_max_ed, l0, l1, a, &failed));
					if (failed) {
						aux.feed = 0; // the rare re-bridging of consecutive pairs is not planned: align in place
						for (int32_t t = j0; t < j; ++t) {
							if (n_rebridged) ++*n_rebridged;
							MGB_TRY(gc_bridge_lchains(A, aux, n_seg, kmer_size, gdp_max_ed, &lc[st + t], &lc[st + t + 1], a, &failed));
							if (failed) return MGB_E_INTERNAL;
						}
						aux.feed = feed;
					}
					j0 = j;
				}
			}
			gs.gc[k].cnt = (int32_t)aux.llc.n - n_llc0;
			gs.gc[k].n_anchor = aux.n_a - n_a0;
			++k;
		}
		st += nui;
	}
	if (aux.n_a > gs.n_a) return MGB_E_INTERNAL;
	gs.n_a = aux.n_a;
	gs.n_lc = (int32_t)aux.llc.n;
	gs.lc = aux.llc.a;
	gs.cyc_gwfa = aux.cyc_gwfa, gs.cyc_shortk = aux.cyc_shortk;
	unsigned long long t0 = prof_clock();
	MGB_TRY(gchain_extra(g, gs));
	MGB_TRY(gchain_sort_by_score(A, gs));
	gs.cyc_extra = prof_clock() - t0;
	return 0;
}

// ---- primary/secondary bookkeeping (reference: gcmisc.c:74-223) ----

MG_HD inline int gchain_set_parent(Arena &A, float mask_level, int n, GChain *r, int sub_diff)
{
	uint64_t mark = A.top;
	int i, j, k, *w;
	uint64_t *cov;
	if (n <= 0) return 0;
	for (i = 0; i < n; ++i) r[i].id = i;
	MGB_ALLOC(A, cov, uint64_t, n);
	MGB_ALLOC(A, w, int, n);
	w[0] = 0, r[0].parent = 0;
	for (i = 1, k = 1; i < n; ++i) {
		GChain *ri = &r[i];
		int si = ri->qs, ei = ri->qe, n_cov = 0, uncov_len = 0;
		for (j = 0; j < k; ++j) {
			GChain *rp = &r[w[j]];
			int sj = rp->qs, ej = rp->qe;
			if (ej <= si || sj >= ei) continue;
			if (sj < si) sj = si;
			if (ej > ei) ej = ei;
			cov[n_cov++] = (uint64_t)(int64_t)sj << 32 | (uint64_t)(int64_t)ej;
		}
		if (n_cov > 0) {
			int x = si;
			MGB_TRY(radix_sort_64(A, cov, n_cov));
			for (j = 0; j < n_cov; ++j) {
				if ((int)(cov[j] >> 32) > x) uncov_len += (int)((cov[j] >> 32) - (uint64_t)(int64_t)x);
				x = (int32_t)cov[j] > x? (int32_t)cov[j] : x;
			}
			if (ei > x) uncov_len += ei - x;
			for (j = 0; j < k; ++j) {
				GChain *rp = &r[w[j]];
				int sj = rp->qs, ej = rp->qe, mn, mx, ol;
				if (ej <= si || sj >= ei) continue;
				mn = ej - sj < ei - si? ej - sj : ei - si;
				mx = ej - sj > ei - si? ej - sj : ei - si;
				ol = si < sj? (ei < sj? 0 : ei < ej? ei - sj : ej - sj) : (ej < si? 0 : ej < ei? ej - si : ei - si);
				if ((float)ol / (float)mn - (float)uncov_len / (float)mx > mask_level) {
					int cnt_sub = 0;
					ri->parent = rp->parent;
					rp->subsc = rp->subsc > ri->score? rp->subsc : ri->score;
					if (ri->cnt >= rp->cnt) cnt_sub = 1;
					if (cnt_sub) ++rp->n_sub;
					break;
				}
			}
		} else j = k;
		if (j == k) w[k++] = i, ri->parent = i, ri->n_sub = 0;
	}
	(void)sub_diff;
	A.top = mark;
	return 0;
}

MG_HD inline void gchain_flt_sub(float pri_ratio, int min_diff, int best_n, int n, GChain *r)
{
	if (pri_ratio > 0.0f && n > 0) {
		int i, n_2nd = 0;
		for (i = 0; i < n; ++i) {
			int p = r[i].parent;
			if (p == i) r[i].flt = 0;
			else if (((float)r[i].score >= (float)r[p].score * pri_ratio || r[i].score + min_diff >= r[p].score) && n_2nd < best_n) {
				if (!(r[i].qs == r[p].qs && r[i].qe == r[p].qe && r[i].ps == r[p].ps && r[i].pe == r[p].pe)) r[i].flt = 0, ++n_2nd;
				else r[i].flt = 1;
			} else r[i].flt = 1;
		}
	}
}

// reference: gcmisc.c:151-188 mg_gchain_drop_flt (+ restore_offset)
MG_HD inline int gchain_drop_flt(Arena &A, GcSet &gs)
{
	uint64_t mark = A.top;
	int32_t i, j, n_gc, n_lc, n_a, n_lc0, n_a0, *o2n;
	if (gs.n_gc == 0) return 0;
	MGB_ALLOC(A, o2n, int32_t, gs.n_gc);
	for (i = 0, n_gc = 0; i < gs.n_gc; ++i) {
		GChain *r = &gs.gc[i];
		o2n[i] = -1;
		if (r->flt || r->cnt == 0) continue;
		o2n[i] = n_gc++;
	}
	n_gc = n_lc = n_a = 0;
	n_lc0 = n_a0 = 0;
	for (i = 0; i < gs.n_gc; ++i) {
		GChain *r = &gs.gc[i];
		if (o2n[i] >= 0) {
			int32_t r_cnt = r->cnt, r_na = r->n_anchor;
			for (j = 0; j < r_na; ++j) gs.a[n_a + j] = gs.a[n_a0 + j];
			for (j = 0; j < r_cnt; ++j) gs.lc[n_lc + j] = gs.lc[n_lc0 + j];
			gs.gc[n_gc] = *r;
			gs.gc[n_gc].id = n_gc;
			gs.gc[n_gc].parent = o2n[gs.gc[n_gc].parent];
			++n_gc, n_lc += r_cnt, n_a += r_na;
			n_lc0 += r_cnt, n_a0 += r_na;
		} else n_lc0 += r->cnt, n_a0 += r->n_anchor;
	}
	if (n_lc0 != gs.n_lc || n_a0 != gs.n_a) return MGB_E_INTERNAL;
	gs.n_gc = n_gc, gs.n_lc = n_lc, gs.n_a = n_a;
	for (i = 0, n_a = n_lc = 0; i < gs.n_gc; ++i) { // restore_offset
		GChain *gc = &gs.gc[i];
		gc->off = n_lc;
		for (j = 0, gc->n_anchor = 0; j < gc->cnt; ++j) {
			LLChain *lc = &gs.lc[n_lc + j];
			lc->off = n_a;
			n_a += lc->cnt;
			gc->n_anchor += lc->cnt;
		}
		n_lc += gc->cnt;
	}
	if (n_lc != gs.n_lc || n_a != gs.n_a) return MGB_E_INTERNAL;
	A.top = mark;
	return 0;
}

// reference: gcmisc.c:191-223 mg_gchain_set_mapq; logf() comes from the host-tabulated glibc values
MG_HD inline int gchain_set_mapq(const MapOptDev &o, GcSet &gs, int qlen, int max_mini, int min_gc_score)
{
	const float q_coef = 40.0f;
	int64_t sum_sc = 0;
	float uniq_ratio, r_sc, r_cnt;
	int i, t_sc, t_cnt;
	if (gs.n_gc == 0) return 0;
	t_sc = qlen < 100? qlen : 100;
	t_cnt = max_mini < 10? max_mini : 10;
	if (t_cnt < 5) t_cnt = 5;
	r_sc = (float)(1.0 / (double)t_sc);
	r_cnt = (float)(1.0 / (double)t_cnt);
	for (i = 0; i < gs.n_gc; ++i)
		if (gs.gc[i].parent == gs.gc[i].id) sum_sc += gs.gc[i].score;
	uniq_ratio = (float)sum_sc / (float)(sum_sc + gs.rep_len);
	for (i = 0; i < gs.n_gc; ++i) {
		GChain *r = &gs.gc[i];
		if (r->parent == r->id) {
			int mapq, subsc;
			float pen_s1 = (r->score > t_sc? 1.0f : (float)r->score * r_sc) * uniq_ratio;
			float x, pen_cm = r->n_anchor > t_cnt? 1.0f : (float)r->n_anchor * r_cnt;
			pen_cm = pen_s1 < pen_cm? pen_s1 : pen_cm;
			subsc = r->subsc > min_gc_score? r->subsc : min_gc_score;
			x = (float)subsc / (float)r->score;
			if (r->score < 0 || r->score >= o.n_logf_tab || r->n_sub + 1 >= o.n_logf_tab) return MGB_E_UNSUPPORTED;
			mapq = (int)(pen_cm * q_coef * (1.0f - x) * o.logf_tab[r->score]);
			mapq -= (int)(4.343f * o.logf_tab[r->n_sub + 1] + .499f);
			mapq = mapq > 0? mapq : 0;
			if (r->score > subsc && mapq == 0) mapq = 1;
			r->mapq = mapq < 60? mapq : 60;
		} else r->mapq = 0;
	}
	return 0;
}

} // namespace mgb
