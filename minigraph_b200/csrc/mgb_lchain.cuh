// mgb_lchain.cuh -- stage B: linear chaining of one read's seeds.
//   chain_dp()      banded DP with skip heuristics          (reference: lchain.c:149-219 mg_lchain_dp)
//   chain_rmq()     RMQ-tree DP for long gaps               (reference: lchain.c:252-372 mg_lchain_rmq)
//   chain_backtrack / chain_compact                          (reference: lchain.c:9-112)
//   lchain_gen, end trimming and bad-seed filters            (reference: lchain.c:374-441, map-algo.c:194-330)
#pragma once
#include "mgb_model.cuh"
#include "mgb_rmq.cuh"

namespace mgb {

static const int32_t SC_NONE = INT32_MIN;

// The chaining loops re-read a handful of small per-anchor arrays for every anchor.  They are taken from the "hot" arena -- the
// warp's slice of shared memory when the kernel has one -- and fall back to the worker's HBM arena (the "cold" one, which holds
// everything that is touched once: end-point lists, sort scratch, tree nodes) when the slice is full.  Hot == cold is fine.
#define MGB_ALLOC_HOT(H, C, ptr, type, n) do { \
		(ptr) = (type*)mgb::arena_alloc((H), (uint64_t)sizeof(type) * (uint64_t)((n) > 0? (n) : 1)); \
		if ((ptr) == 0) (ptr) = (type*)mgb::arena_alloc((C), (uint64_t)sizeof(type) * (uint64_t)((n) > 0? (n) : 1)); \
		if ((ptr) == 0) return mgb::MGB_E_ARENA; \
	} while (0)

// chaining score between anchors i (later) and j (earlier)  (reference: lchain.c:114-139 comput_sc)
MG_HD inline int32_t chain_score(const u128 &ai, const u128 &aj, int32_t max_dist_x, int32_t max_dist_y, int32_t bw,
								 float pen_gap, float pen_skip, int is_cdna, int n_seg)
{
	int32_t dq = (int32_t)ai.y - (int32_t)aj.y, dr, dd, dg, q_span, sc;
	int32_t sidi = (int32_t)((ai.y & SEED_SEG_MASK) >> SEED_SEG_SHIFT);
	int32_t sidj = (int32_t)((aj.y & SEED_SEG_MASK) >> SEED_SEG_SHIFT);
	if (dq <= 0 || dq > max_dist_x) return SC_NONE;
	dr = (int32_t)(ai.x - aj.x);
	if (sidi == sidj && (dr == 0 || dq > max_dist_y)) return SC_NONE;
	dd = dr > dq? dr - dq : dq - dr;
	if (sidi == sidj && dd > bw) return SC_NONE;
	if (n_seg > 1 && !is_cdna && sidi == sidj && dr > max_dist_y) return SC_NONE;
	dg = dr < dq? dr : dq;
	q_span = (int32_t)(aj.y >> 32 & 0xff);
	sc = q_span < dg? q_span : dg;
	if (dd || dg > q_span) {
		float lin_pen = pen_gap * (float)dd + pen_skip * (float)dg;
		float log_pen = dd >= 1? fast_log2((float)(dd + 1)) : 0.0f;
		if (is_cdna || sidi != sidj) {
			if (sidi != sidj && dr == 0) ++sc;
			else if (dr > dq || sidi != sidj) sc -= (int)(lin_pen < log_pen? lin_pen : log_pen);
			else sc -= (int)(lin_pen + .5f * log_pen);
		} else sc -= (int)(lin_pen + .5f * log_pen);
	}
	return sc;
}

// follow one chain backwards from z[k] until the score drops too far (reference: lchain.c:9-25)
MG_HD inline int64_t chain_bk_end(int32_t max_drop, const u128 *z, const int32_t *f, const int32_t *p, int32_t *t, int64_t k)
{
	int64_t i = (int64_t)z[k].y, end_i = -1, max_i = i;
	int32_t max_s = 0;
	if (i < 0 || t[i] != 0) return i;
	do {
		int32_t s;
		t[i] = 2;
		end_i = i = p[i];
		s = i < 0? (int32_t)z[k].x : (int32_t)z[k].x - f[i];
		if (s > max_s) max_s = s, max_i = i;
		else if (max_s - s > max_drop) break;
	} while (i >= 0 && t[i] == 0);
	for (i = (int64_t)z[k].y; i >= 0 && i != end_i; i = p[i]) t[i] = 0;
	return max_i;
}

// peel chains best-score-first (reference: lchain.c:27-77 mg_chain_backtrack). u[] gets extra_u spare entries.
MG_HD inline int chain_backtrack(Arena &A, int64_t n, const int32_t *f, const int32_t *p, int32_t *v, int32_t *t, int32_t min_cnt, int32_t min_sc,
								 int32_t max_drop, int32_t extra_u, uint64_t **u_, int32_t *n_u_, int32_t *n_v_)
{
	u128 *z;
	uint64_t *u;
	int64_t i, k, n_z = 0, n_v;
	int32_t n_u;
	*n_u_ = *n_v_ = 0, *u_ = 0;
	for (i = 0; i < n; ++i) if (f[i] >= min_sc) ++n_z;
	if (n_z == 0) return 0;
	// u[] must outlive z[]: reserve the worst case first (one chain per end point), then z on top
	MGB_ALLOC(A, u, uint64_t, n_z + extra_u);
	uint64_t mark = A.top;
	MGB_ALLOC(A, z, u128, n_z);
	for (i = 0, k = 0; i < n; ++i)
		if (f[i] >= min_sc) z[k].x = (uint64_t)(int64_t)f[i], z[k++].y = (uint64_t)i;
	MGB_TRY(radix_sort_128x(A, z, n_z));
	for (i = 0; i < n; ++i) t[i] = 0;
	for (k = n_z - 1, n_v = n_u = 0; k >= 0; --k) {
		if (t[z[k].y] == 0) {
			int64_t n_v0 = n_v, end_i;
			int32_t sc;
			end_i = chain_bk_end(max_drop, z, f, p, t, k);
			for (i = (int64_t)z[k].y; i != end_i; i = p[i])
				v[n_v++] = (int32_t)i, t[i] = 1;
			sc = i < 0? (int32_t)z[k].x : (int32_t)z[k].x - f[i];
			if (sc >= min_sc && n_v > n_v0 && n_v - n_v0 >= min_cnt)
				u[n_u++] = (uint64_t)sc << 32 | (uint64_t)(n_v - n_v0);
			else n_v = n_v0;
		}
	}
	A.top = mark;
	*u_ = u, *n_u_ = n_u, *n_v_ = (int32_t)n_v;
	return 0;
}

// The end-point list of chain_finish_w(): score and anchor index in one word.  The sort key is the score widened exactly as the
// reference's 128-bit records hold it ((uint64_t)(int64_t)f), so klib's radix sort makes the same moves on these 8-byte records.
struct KeyHi32 { MG_HD uint64_t operator()(const uint64_t &p) const { return (uint64_t)(int64_t)(int32_t)(p >> 32); } };
MG_HD inline int64_t chain_bk_end_p(int32_t max_drop, const uint64_t *z, const int32_t *f, const int32_t *p, int32_t *t, int64_t k)
{ // chain_bk_end() on the packed list (reference: lchain.c:9-25)
	const int32_t zf = (int32_t)(z[k] >> 32);
	int64_t i = (int64_t)(uint32_t)z[k], end_i = -1, max_i = i;
	int32_t max_s = 0;
	if (t[i] != 0) return i;
	do {
		int32_t s;
		t[i] = 2;
		end_i = i = p[i];
		s = i < 0? zf : zf - f[i];
		if (s > max_s) max_s = s, max_i = i;
		else if (max_s - s > max_drop) break;
	} while (i >= 0 && t[i] == 0);
	for (i = (int64_t)(uint32_t)z[k]; i >= 0 && i != end_i; i = p[i]) t[i] = 0;
	return max_i;
}

// chain_backtrack() + chain_compact() entered by all lanes of a warp: the end-point list, the sorts and the copies are
// spread over the lanes, the peeling itself (a walk over p[] with the visit marks) stays on lane 0.  u_store receives
// the chain descriptors; a[0..n_v) the chained anchors.
MG_HD inline int chain_finish_w(Arena &H, Arena &A, int64_t n, const int32_t *f, const int32_t *p, int32_t *v, int32_t *t, int32_t min_cnt, int32_t min_sc,
								int32_t max_drop, u128 *a, uint64_t *u_store, int32_t *n_u_, int32_t *n_v_, int lane)
{
	const uint64_t mark = A.top;
	*n_u_ = *n_v_ = 0;
	int32_t n_z = 0;
	for (int64_t i = lane; i < n; i += MGB_W) n_z += f[i] >= min_sc;
	n_z = warp_sum_i32(n_z);
	if (n_z == 0) return 0;
	const uint64_t hmark = H.top;
	uint64_t *u, *z;
	MGB_ALLOC(A, u, uint64_t, n_z);
	MGB_ALLOC_HOT(H, A, z, uint64_t, n_z); // the peeling below walks this list on one lane: it wants to be on chip, and so do the sort's bin tables
	{
		int32_t k = 0;
		for (int64_t base = 0; base < n; base += MGB_W) {
			const int64_t i = base + lane;
			const int keep = i < n && f[i] >= min_sc;
			const uint32_t m = warp_ballot(keep);
			if (keep) z[k + mask_rank(m, lane)] = (uint64_t)(uint32_t)f[i] << 32 | (uint64_t)(uint32_t)i;
			k += mask_count(m);
		}
	}
	for (int64_t i = lane; i < n; i += MGB_W) t[i] = 0;
	warp_sync();
	{
		Arena &S = H.cap - H.top >= (uint64_t)n_z / 4 + 3400? H : A; // range stack + three 1 KB bin tables
		MGB_TRY(radix_sort_exact_w(S, z, n_z, 8, KeyHi32(), lane)); // (in place: the list is on chip)
	}
	int32_t n_u = 0, n_v = 0;
	if (lane == 0) { // reference: lchain.c:27-77
		for (int64_t k = n_z - 1; k >= 0; --k) {
			if (t[(uint32_t)z[k]] == 0) {
				int64_t n_v0 = n_v, end_i, i;
				int32_t sc;
				const int32_t zf = (int32_t)(z[k] >> 32);
				end_i = chain_bk_end_p(max_drop, z, f, p, t, k);
				for (i = (int64_t)(uint32_t)z[k]; i != end_i; i = p[i])
					v[n_v++] = (int32_t)i, t[i] = 1;
				sc = i < 0? zf : zf - f[i];
				if (sc >= min_sc && n_v > n_v0 && n_v - n_v0 >= min_cnt)
					u[n_u++] = (uint64_t)sc << 32 | (uint64_t)(n_v - n_v0);
				else n_v = (int32_t)n_v0;
			}
		}
	}
	n_u = warp_bcast_i32(n_u, 0), n_v = warp_bcast_i32(n_v, 0);
	warp_sync();
	if (n_u > 0) { // reference: lchain.c:79-112 compact_a
		u128 *b, *w;
		int32_t *koff;
		MGB_ALLOC(A, b, u128, n_v);
		MGB_ALLOC(A, w, u128, n_u);
		MGB_ALLOC(A, koff, int32_t, n_u + 1);
		if (lane == 0) { int32_t k = 0; for (int32_t i = 0; i < n_u; ++i) koff[i] = k, k += (int32_t)u[i]; koff[n_u] = k; }
		warp_sync();
		for (int32_t i = 0; i < n_u; ++i) {
			const int32_t k0 = koff[i], ni = (int32_t)u[i];
			for (int32_t j = lane; j < ni; j += MGB_W) b[k0 + j] = a[v[k0 + (ni - j - 1)]];
		}
		warp_sync();
		for (int32_t i = lane; i < n_u; i += MGB_W) w[i].x = b[koff[i]].x, w[i].y = (uint64_t)koff[i] << 32 | (uint64_t)i;
		warp_sync();
		MGB_TRY(radix_sort_128x_w(A, w, n_u, lane));
		int32_t k = 0;
		for (int32_t i = 0; i < n_u; ++i) {
			const int32_t j2 = (int32_t)w[i].y, cnt = (int32_t)u[j2];
			const u128 *src = &b[w[i].y >> 32];
			for (int32_t x = lane; x < cnt; x += MGB_W) a[k + x] = src[x];
			if (lane == 0) u_store[i] = u[j2];
			k += cnt;
		}
		warp_sync();
	}
	A.top = mark;
	if (&H != &A) H.top = hmark;
	*n_u_ = n_u, *n_v_ = n_v;
	return 0;
}

// chain_dp() entered by all lanes of a warp.  The predecessors of anchor i are scored 32 at a time; the sequential
// rules (strict improvement keeps the first maximum, the skip counter with its early exit, the t[] marks left by
// visited predecessors) are then replayed on the ballots of the chunk, in visiting order.
MG_HD inline int chain_dp_w(Arena &H, Arena &A, int max_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc,
							float pen_gap, float pen_skip, int is_cdna, int n_seg, int64_t n, u128 *a,
							int32_t *n_u_, uint64_t **u_, int32_t *n_a_, int lane)
{
	int32_t *f, *t, *v, *p, max_drop = bw;
	int64_t i, max_ii, st = 0;
	*u_ = 0, *n_u_ = 0, *n_a_ = 0;
	if (n == 0) return 0;
	if (max_dist_x < bw) max_dist_x = bw;
	if (max_dist_y < bw && !is_cdna) max_dist_y = bw;
	if (is_cdna) max_drop = INT32_MAX;
	uint64_t *u_store;
	MGB_ALLOC(A, u_store, uint64_t, n);
	const uint64_t mark = A.top, hmark = H.top;
	MGB_ALLOC_HOT(H, A, p, int32_t, n);
	MGB_ALLOC_HOT(H, A, f, int32_t, n);
	MGB_ALLOC_HOT(H, A, v, int32_t, n);
	MGB_ALLOC_HOT(H, A, t, int32_t, n);
	for (i = lane; i < n; i += MGB_W) t[i] = 0;
	warp_sync();
	for (i = 0, max_ii = -1; i < n; ++i) {
		const u128 ai = a[i];
		int64_t max_j = -1, end_j;
		int32_t max_f = (int32_t)(ai.y >> 32 & 0xff), n_skip = 0;
		while (st < i && (ai.x >> 32 != a[st].x >> 32 || ai.x > a[st].x + (uint64_t)max_dist_x)) ++st;
		if (i - st > max_iter) st = i - max_iter;
		end_j = st - 1;
		for (int64_t base = i - 1; base >= st; base -= MGB_W) {
			const int64_t j = base - lane;
			int32_t sc = SC_NONE, pj = -1;
			if (j >= st) {
				sc = chain_score(ai, a[j], max_dist_x, max_dist_y, bw, pen_gap, pen_skip, is_cdna, n_seg);
				if (sc != SC_NONE) sc += f[j], pj = p[j];
			}
			const int active = sc != SC_NONE;
			if (pj >= 0) t[pj] = (int32_t)i; // marks of lanes past an early exit only touch anchors that are not visited either
			warp_sync();
			const int marked = active && t[j] == (int32_t)i;
			const int32_t before = warp_excl_prefix_max_i32(sc, lane);
			const int improves = active && sc > (before > max_f? before : max_f);
			const uint32_t m_imp = warp_ballot(improves), m_mk = warp_ballot(marked && !improves);
			const int brk = replay_skips(m_imp, m_mk, max_skip, &n_skip);
			const int eligible = active && (brk < 0 || lane < brk);
			const int32_t best = warp_max_i32(eligible? sc : SC_NONE);
			if (best > max_f) {
				max_f = best;
				max_j = base - ctz32(warp_ballot(eligible && sc == best));
			}
			if (brk >= 0) { end_j = base - brk; break; }
		}
		if (max_ii < 0 || (int64_t)(ai.x - a[max_ii].x) > (int64_t)max_dist_x) {
			int32_t mx = INT32_MIN, bj = -1;
			for (int64_t j = i - 1 - lane; j >= st; j -= MGB_W)
				if (mx < f[j]) mx = f[j], bj = (int32_t)j;
			const int32_t m = warp_max_i32(mx);
			max_ii = warp_max_i32(bj >= 0 && mx == m? bj : -1); // first in visiting order = the largest index among equals
		}
		if (max_ii >= 0 && max_ii < end_j) {
			int32_t tmp = chain_score(ai, a[max_ii], max_dist_x, max_dist_y, bw, pen_gap, pen_skip, is_cdna, n_seg);
			if (tmp != SC_NONE && max_f < tmp + f[max_ii])
				max_f = tmp + f[max_ii], max_j = max_ii;
		}
		const int32_t vi = max_j >= 0 && v[max_j] > max_f? v[max_j] : max_f;
		if (max_ii < 0 || ((int64_t)(ai.x - a[max_ii].x) <= (int64_t)max_dist_x && f[max_ii] < max_f))
			max_ii = i;
		if (lane == 0) f[i] = max_f, p[i] = (int32_t)max_j, v[i] = vi;
		warp_sync();
	}
	int32_t n_u = 0, n_v = 0;
	MGB_TRY(chain_finish_w(H, A, n, f, p, v, t, min_cnt, min_sc, max_drop, a, u_store, &n_u, &n_v, lane));
	A.top = mark;
	if (&H != &A) H.top = hmark;
	*u_ = u_store, *n_u_ = n_u, *n_a_ = n_u > 0? n_v : 0;
	return 0;
}

// gap-only score used by the RMQ DP (reference: lchain.c:234-250 comput_sc_simple)
MG_HD inline int32_t chain_score_simple(const u128 &ai, const u128 &aj, float pen_gap, float pen_skip, int32_t *exact, int32_t *width)
{
	int32_t dq = (int32_t)ai.y - (int32_t)aj.y, dr, dd, dg, q_span, sc;
	dr = (int32_t)(ai.x - aj.x);
	*width = dd = dr > dq? dr - dq : dq - dr;
	dg = dr < dq? dr : dq;
	q_span = (int32_t)(aj.y >> 32 & 0xff);
	sc = q_span < dg? q_span : dg;
	if (exact) *exact = (dd == 0 && dg <= q_span);
	if (dd || dq > q_span) {
		float lin_pen = pen_gap * (float)dd + pen_skip * (float)dg;
		float log_pen = dd >= 1? fast_log2((float)(dd + 1)) : 0.0f;
		sc -= (int)(lin_pen + .5f * log_pen);
	}
	return sc;
}

// RMQ chaining, DP fill with the reference's two AVL trees replayed node for node (reference: lchain.c:271-359).
// Computes f, p, v for all anchors; t is scratch.  Sequential (one lane).
MG_HD inline int chain_rmq_fill_seq(Arena &A, int max_dist, int max_dist_inner, int bw, int max_chn_skip, int cap_rmq_size,
									float pen_gap, float pen_skip, int64_t n, const u128 *a, int32_t *f, int32_t *p, int32_t *t, int32_t *v)
{
	int64_t i, i0, st = 0, st_inner = 0;
	RmqTree root, root_inner;
	for (i = 0; i < n; ++i) t[i] = 0;
	uint64_t mark_tree = A.top;
	MGB_TRY(rmq_init(A, root, (int32_t)n));
	root_inner.nd = 0, root_inner.root = RMQ_NIL, root_inner.n_nd = root_inner.m_nd = 0;
	if (max_dist_inner > 0) MGB_TRY(rmq_init(A, root_inner, (int32_t)n));

	for (i = i0 = 0; i < n; ++i) {
		int64_t max_j = -1;
		int32_t q_span = (int32_t)(a[i].y >> 32 & 0xff), max_f = q_span;
		int32_t q;
		// add in-range anchors
		if (i0 < i && a[i0].x != a[i].x) {
			for (int64_t j = i0; j < i; ++j) {
				double pri = -(f[j] + 0.5 * pen_gap * ((int32_t)a[j].x + (int32_t)a[j].y));
				if (rmq_insert(root, (int32_t)a[j].y, (int32_t)j, pri) < 0) return MGB_E_INTERNAL;
				if (max_dist_inner > 0)
					if (rmq_insert(root_inner, (int32_t)a[j].y, (int32_t)j, pri) < 0) return MGB_E_INTERNAL;
			}
			i0 = i;
		}
		// drop anchors out of range
		while (st < i && (a[i].x >> 32 != a[st].x >> 32 || a[i].x > a[st].x + (uint64_t)max_dist || rmq_size(root) > (uint32_t)cap_rmq_size)) {
			rmq_erase(root, (int32_t)a[st].y, (int32_t)st);
			++st;
		}
		if (max_dist_inner > 0) {
			while (st_inner < i && (a[i].x >> 32 != a[st_inner].x >> 32 || a[i].x > a[st_inner].x + (uint64_t)max_dist_inner || rmq_size(root_inner) > (uint32_t)cap_rmq_size)) {
				rmq_erase(root_inner, (int32_t)a[st_inner].y, (int32_t)st_inner);
				++st_inner;
			}
		}
		// RMQ
		q = rmq_query(root, (int32_t)a[i].y - max_dist, INT32_MAX, (int32_t)a[i].y - 1, 0);
		if (q != RMQ_NIL) {
			int32_t sc, exact, width, n_skip = 0;
			int64_t j = root.nd[q].i;
			sc = f[j] + chain_score_simple(a[i], a[j], pen_gap, pen_skip, &exact, &width);
			if (width <= bw && sc > max_f) max_f = sc, max_j = j;
			if (!exact && root_inner.root != RMQ_NIL && (int32_t)a[i].y > 0) {
				int32_t lo = rmq_lower(root_inner, (int32_t)a[i].y - 1, (int32_t)n);
				if (lo != RMQ_NIL) {
					RmqItr itr;
					int32_t qi;
					rmq_itr_find(root_inner, lo, itr);
					while ((qi = rmq_itr_at(itr)) != RMQ_NIL) {
						if (root_inner.nd[qi].y < (int32_t)a[i].y - max_dist_inner) break;
						j = root_inner.nd[qi].i;
						sc = f[j] + chain_score_simple(a[i], a[j], pen_gap, pen_skip, 0, &width);
						if (width <= bw) {
							if (sc > max_f) {
								max_f = sc, max_j = j;
								if (n_skip > 0) --n_skip;
							} else if (t[j] == (int32_t)i) {
								if (++n_skip > max_chn_skip) break;
							}
							if (p[j] >= 0) t[p[j]] = (int32_t)i;
						}
						if (!rmq_itr_prev(root_inner, itr)) break;
					}
				}
			}
		}
		f[i] = max_f, p[i] = (int32_t)max_j;
		v[i] = max_j >= 0 && v[max_j] > max_f? v[max_j] : max_f;
	}
	A.top = mark_tree;
	return 0;
}

// ---- warp-cooperative RMQ fill ----
// The two trees of the reference only ever hold index windows of the x-sorted anchor array: outer = [st, i0),
// inner = [st_inner, i0).  Hence
//   * the range-minimum query is a lane-parallel scan of the outer window with the (y,idx) interval test of
//     krmq_rmq() and a min-reduction on pri; the answer is independent of the tree shape unless two candidates tie
//     on pri, in which case the fill gives up (returns 1) and the caller replays the AVL version (SURVEY H2);
//   * the in-order walk over the inner tree is a walk over an array kept sorted by (y,idx); candidates are scored 32
//     at a time and the order-dependent (max_f, n_skip) state machine is replayed from registers.  The marks
//     "t[j] == i" only ever come from successors of j inside the same candidate set (p[j'] = j implies y_j < y_j'),
//     so they are scattered for the whole set first and read afterwards.
// Exact only while the outer tree never exceeds cap_rmq_size (the caller checks n <= cap).
MG_HD inline int32_t warp_sum_i32_all(int32_t x) { return warp_sum_i32(x); }

MG_HD inline double warp_min_f64(double x)
{
#if MGB_ON_DEVICE
	for (int o = 16; o > 0; o >>= 1) { double y = __shfl_xor_sync(0xffffffffu, x, o); x = y < x? y : x; }
#elif defined(MGB_SIM_LANES)
	{ uint64_t o[32], b; memcpy(&b, &x, 8); sim::exchange(b, o, 15); for (int i = 0; i < MGB_W; ++i) { double y; memcpy(&y, &o[i], 8); if (y < x) x = y; } }
#endif
	return x;
}

struct RmqBlock { double best; int32_t cnt, j, ymin, ymax; };

MG_HD inline int chain_rmq_fill_w(Arena &H, Arena &A, int max_dist, int max_dist_inner, int bw, int max_chn_skip, float pen_gap, float pen_skip,
								  int64_t n, const u128 *a, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int lane)
{
	const uint64_t mark = A.top, hmark = H.top;
	double *pri;
	uint64_t *K; // inner window, keys y<<32|idx ascending
	MGB_ALLOC_HOT(H, A, K, uint64_t, n); // (the window is re-read for every anchor, the priorities only where a block straddles a border: hot space goes to the window first)
	// Summaries of the available anchors in blocks of 32 consecutive indices: the smallest priority, how many hold it and one of
	// them, and the span of query positions.  The outer query then looks at one summary per block and at the elements of the
	// few blocks that straddle a border of the window, instead of at every anchor of the window.
	// Where it pays (below), a block keeps TWO summaries, one for its anchors at or below the middle of the block's span of query positions and one for those
	// above it (blk[2b], blk[2b+1]; ysplit[b] is that middle, known up front because the positions are).  Where two diagonals
	// interleave in target order -- a read that wraps around a circular genome, a tandem duplication -- a block spans both, would
	// straddle the border of nearly every query and be scanned element by element; its halves are narrow and answer from the summary.
	RmqBlock *blk;
	const int64_t n_blk = (n + 31) >> 5;
	MGB_ALLOC_HOT(H, A, blk, RmqBlock, 2 * n_blk);
	MGB_ALLOC_HOT(H, A, pri, double, n);
	int32_t *ys, *ysplit; // query positions by themselves (the border scan below reads one 128-byte line per block instead of four)
	MGB_ALLOC(A, ys, int32_t, n);
	MGB_ALLOC(A, ysplit, int32_t, n_blk);
	for (int64_t j = lane; j < n; j += MGB_W) ys[j] = (int32_t)a[j].y;
	for (int64_t b = lane; b < 2 * n_blk; b += MGB_W) { RmqBlock e; e.best = 1e300, e.cnt = 0, e.j = -1, e.ymin = INT32_MAX, e.ymax = INT32_MIN; blk[b] = e; }
	warp_sync();
	int wide = 0; // does any block span more query positions than 32 anchors of one diagonal do?  If none does, one summary per block is enough
	for (int64_t b = lane; b < n_blk; b += MGB_W) {
		int32_t mn = INT32_MAX, mx = INT32_MIN;
		for (int64_t j = b << 5; j < n && j < (b + 1) << 5; ++j) { const int32_t y = ys[j]; mn = y < mn? y : mn, mx = y > mx? y : mx; }
		ysplit[b] = (int32_t)(((int64_t)mn + mx) >> 1);
		wide |= (int64_t)mx - mn > 2048;
	}
	const int hs = warp_any(wide)? 1 : 0; // summaries per block: 1 << hs; half-block hb belongs to block hb >> hs
	int32_t nK = 0;
	int64_t i, i0 = 0, st = 0, st_inner = 0;
	for (i = lane; i < n; i += MGB_W) t[i] = 0;
	warp_sync();
	for (i = 0; i < n; ++i) {
		const uint64_t xi = a[i].x, yi64 = a[i].y;
		const int32_t yi = (int32_t)yi64;
		int64_t max_j = -1;
		int32_t max_f = (int32_t)(yi64 >> 32 & 0xff);
		// (1) anchors with a smaller target position become available
		if (i0 < i && a[i0].x != xi) {
			for (int64_t j = i0; j < i; ++j) {
				const uint64_t xj = a[j].x, yj = a[j].y;
				if (lane == 0) {
					const double pj = -(f[j] + 0.5 * pen_gap * ((int32_t)xj + (int32_t)yj));
					RmqBlock &B = blk[((j >> 5) << hs) + (hs & (int)((int32_t)yj > ysplit[j >> 5]))];
					pri[j] = pj;
					if (pj < B.best) B.best = pj, B.cnt = 1, B.j = (int32_t)j;
					else if (pj == B.best) ++B.cnt;
					if ((int32_t)yj < B.ymin) B.ymin = (int32_t)yj;
					if ((int32_t)yj > B.ymax) B.ymax = (int32_t)yj;
				}
				if (max_dist_inner > 0) { // insert (y,idx) into the sorted inner window
					const uint64_t key = (uint64_t)(uint32_t)(int32_t)yj << 32 | (uint64_t)(uint32_t)j;
					if (nK == 0 || K[nK - 1] < key) { // colinear anchors arrive in ascending query order: the new key goes on top
						if (lane == 0) K[nK] = key;
						++nK;
						warp_sync();
						continue;
					}
					int32_t cnt = 0;
					for (int32_t x = lane; x < nK; x += MGB_W) cnt += K[x] < key;
					const int32_t pos = warp_sum_i32(cnt);
					for (int32_t e = nK; e > pos; e -= MGB_W) { // shift [pos, nK) up by one, top chunk first
						int32_t idx = e - 1 - lane;
						uint64_t val = 0;
						if (idx >= pos) val = K[idx];
						warp_sync();
						if (idx >= pos) K[idx + 1] = val;
						warp_sync();
					}
					if (lane == 0) K[pos] = key;
					++nK;
					warp_sync();
				}
			}
			i0 = i;
			warp_sync();
		}
		// (2) retire anchors that fell out of range
		while (st < i && (xi >> 32 != a[st].x >> 32 || xi > a[st].x + (uint64_t)max_dist)) ++st;
		if (max_dist_inner > 0) {
			while (st_inner < i && (xi >> 32 != a[st_inner].x >> 32 || xi > a[st_inner].x + (uint64_t)max_dist_inner)) {
				if (st_inner < i0) { // it is in the window: remove its key
					const uint64_t key = (uint64_t)(uint32_t)(int32_t)a[st_inner].y << 32 | (uint64_t)(uint32_t)st_inner;
					if (K[0] == key) { ++K, --nK, ++st_inner; continue; } // ... and leave from the bottom: the window is a queue, its array slides
					int32_t cnt = 0;
					for (int32_t x = lane; x < nK; x += MGB_W) cnt += K[x] < key;
					const int32_t pos = warp_sum_i32(cnt);
					for (int32_t b = pos; b + 1 < nK; b += MGB_W) { // shift (pos, nK) down by one, bottom chunk first
						int32_t idx = b + lane;
						uint64_t val = 0;
						if (idx + 1 < nK) val = K[idx + 1];
						warp_sync();
						if (idx + 1 < nK) K[idx] = val;
						warp_sync();
					}
					--nK;
				}
				++st_inner;
			}
		}
		// (3) range-minimum query on the outer window (reference: lchain.c:317-325, interval of krmq_rmq)
		{
			const int64_t hi_j = st < i0? i0 : st; // window [st, i0)
			double best = 1e300;
			int32_t best_j = -1, n_best = 0;
			for (int64_t b0 = (st >> 5) << hs; ((b0 >> hs) << 5) < hi_j; b0 += MGB_W) { // one (half-)block per lane
				const int64_t hb = b0 + lane, b = hb >> hs;
				int kind = 0; // 0: nothing of this half-block qualifies, 1: all of it does (the summary answers), 2: look at its elements
				if ((b << 5) < hi_j) {
					const RmqBlock B = blk[hb];
					if (B.cnt > 0 && B.ymax > yi - max_dist && B.ymin <= yi - 1 && !(B.ymin == yi - 1 && b != 0))
						kind = (b << 5) >= st && B.ymin > yi - max_dist && B.ymax < yi - 1? 1 : 2;
					if (kind == 1) {
						if (B.best < best) best = B.best, best_j = B.j, n_best = B.cnt;
						else if (B.best == best) n_best += B.cnt;
					}
				}
				uint32_t scan = warp_ballot(kind == 2);
				while (scan) { // half-blocks on a border of the window: their elements, one per lane, four at a time (eight loads in flight per lane)
					int32_t j0s[4];
					int nb = 0;
					int32_t halves = 0; // bit u: the upper half of block u is the one to look at
					while (scan && nb < 4) { const int64_t h = b0 + ctz32(scan); halves |= (int32_t)(h & hs) << nb, j0s[nb++] = (int32_t)((h >> hs) << 5); scan &= scan - 1; }
					for (int32_t off = lane; off < 32; off += MGB_W) {
						int32_t yv[4];
						double pv[4];
						uint32_t okm = 0;
#if MGB_ON_DEVICE
#pragma unroll
#endif
						for (int u = 0; u < 4; ++u) {
							const int32_t j = (u < nb? j0s[u] : j0s[0]) + off;
							const int ok = u < nb && j >= st && j < hi_j;
							okm |= (uint32_t)ok << u;
							yv[u] = ok? ys[j] : 0, pv[u] = ok? pri[j] : 1e300;
						}
#if MGB_ON_DEVICE
#pragma unroll
#endif
						for (int u = 0; u < 4; ++u) {
							if (!(okm >> u & 1)) continue;
							const int32_t j = j0s[u] + off;
							const int32_t yj = yv[u];
							if (hs && (yj > ysplit[j >> 5]) != (halves >> u & 1)) continue; // an anchor of the block's other half
							if (!(yj > yi - max_dist)) continue;
							if (!(yj < yi - 1 || (yj == yi - 1 && j == 0))) continue;
							if (pv[u] < best) best = pv[u], best_j = j, n_best = 1;
							else if (pv[u] == best) ++n_best;
						}
					}
				}
			}
			const double gbest = warp_min_f64(best);
			const int32_t n_at_min = warp_sum_i32(best_j >= 0 && best == gbest? n_best : 0);
			if (n_at_min > 1) { A.top = mark; if (&H != &A) H.top = hmark; return 1; } // pri tie: the winner depends on the AVL shape
			if (n_at_min == 1) {
				const int32_t j = warp_max_i32(best_j >= 0 && best == gbest? best_j : -1);
				int32_t exact, width, n_skip = 0;
				int32_t sc = f[j] + chain_score_simple(a[i], a[j], pen_gap, pen_skip, &exact, &width);
				if (width <= bw && sc > max_f) max_f = sc, max_j = j;
				if (!exact && nK > 0 && yi > 0) { // (4) walk the inner window downwards from (yi-1, n)
					const uint64_t hi_key = (uint64_t)(uint32_t)(yi - 1) << 32 | 0xffffffffULL;
					const int32_t ylo = yi - max_dist_inner;
					const uint64_t lo_key = ylo > 0? (uint64_t)(uint32_t)ylo << 32 : 0;
					int32_t c_hi = 0, c_lo = 0;
					for (int32_t x = lane; x < nK; x += MGB_W) c_hi += K[x] <= hi_key, c_lo += K[x] < lo_key;
					const int32_t ub = warp_sum_i32(c_hi), lb = warp_sum_i32(c_lo); // candidates K[lb, ub)
					// marks: t[p[j]] = i for every in-band candidate
					for (int32_t x = lb + lane; x < ub; x += MGB_W) {
						const int32_t jj = (int32_t)(uint32_t)K[x];
						int32_t w2;
						chain_score_simple(a[i], a[jj], pen_gap, pen_skip, 0, &w2);
						if (w2 <= bw && p[jj] >= 0) t[p[jj]] = (int32_t)i;
					}
					warp_sync();
					int stop = 0;
					for (int32_t top = ub; top > lb && !stop; top -= MGB_W) {
						const int32_t x = top - 1 - lane;
						int32_t c_ok = 0, c_sc = 0, c_mk = 0, c_j = -1;
						if (x >= lb) {
							int32_t w2;
							c_j = (int32_t)(uint32_t)K[x];
							c_sc = f[c_j] + chain_score_simple(a[i], a[c_j], pen_gap, pen_skip, 0, &w2);
							c_ok = w2 <= bw;
							c_mk = t[c_j] == (int32_t)i;
						}
						{ // lane c holds candidate c of this chunk; the rules below are the sequential ones, evaluated for all lanes at once
							const int32_t sc_eff = c_ok? c_sc : SC_NONE;
							const int32_t before = warp_excl_prefix_max_i32(sc_eff, lane);
							const int improves = c_ok && c_sc > (before > max_f? before : max_f); // strictly above everything in front of it
							const uint32_t m_imp = warp_ballot(improves), m_mk = warp_ballot(c_ok && !improves && c_mk);
							const int brk = replay_skips(m_imp, m_mk, max_chn_skip, &n_skip);
							const int eligible = improves && (brk < 0 || lane < brk);
							const int32_t best = warp_max_i32(eligible? c_sc : SC_NONE);
							if (best > max_f) { // improvements rise strictly: the last one before the stop holds the maximum
								max_f = best;
								max_j = warp_max_i32(eligible && c_sc == best? c_j : -1);
							}
							if (brk >= 0) stop = 1;
						}
					}
				}
			}
		}
		if (lane == 0) {
			f[i] = max_f, p[i] = (int32_t)max_j;
			v[i] = max_j >= 0 && v[max_j] > max_f? v[max_j] : max_f;
		}
		warp_sync();
	}
	A.top = mark;
	if (&H != &A) H.top = hmark;
	return 0;
}

// How chain_rmq_w() filled f/p/v (reported to the tests through its `path` argument)
enum { CHAIN_PATH_DP = 0, CHAIN_PATH_RMQ_W = 1, CHAIN_PATH_RMQ_TIE = 2, CHAIN_PATH_RMQ_CAP = 3 };

// Warp-uniform RMQ chaining: same contract as chain_rmq(); all lanes enter with identical arguments and leave with
// identical results (outputs are broadcast from lane 0, which runs the sequential backtrack/compaction).  path (may be NULL):
// CHAIN_PATH_RMQ_W when the cooperative fill ran, _TIE when it gave up on a priority tie, _CAP when n > cap_rmq_size.
MG_HD inline int chain_rmq_w(Arena &H, Arena &A, int max_dist, int max_dist_inner, int bw, int max_chn_skip, int cap_rmq_size, int min_cnt, int min_sc,
							 float pen_gap, float pen_skip, int64_t n, u128 *a, int32_t *n_u_, uint64_t **u_, int32_t *n_a_, int lane, int *path = 0)
{
	int32_t *f, *t, *v, *p;
	*u_ = 0, *n_u_ = 0, *n_a_ = 0;
	if (n == 0) return 0;
	const int max_drop = bw;
	if (max_dist < bw) max_dist = bw;
	if (max_dist_inner <= 0 || max_dist_inner >= max_dist) max_dist_inner = 0;
	uint64_t *u_store;
	MGB_ALLOC(A, u_store, uint64_t, n);
	const uint64_t mark = A.top, hmark = H.top;
	MGB_ALLOC_HOT(H, A, p, int32_t, n);
	MGB_ALLOC_HOT(H, A, f, int32_t, n);
	MGB_ALLOC_HOT(H, A, t, int32_t, n);
	MGB_ALLOC_HOT(H, A, v, int32_t, n);
	int rc = n <= cap_rmq_size? chain_rmq_fill_w(H, A, max_dist, max_dist_inner, bw, max_chn_skip, pen_gap, pen_skip, n, a, f, p, t, v, lane) : 1;
	if (rc < 0) return rc;
	if (path) *path = n > cap_rmq_size? CHAIN_PATH_RMQ_CAP : rc == 1? CHAIN_PATH_RMQ_TIE : CHAIN_PATH_RMQ_W;
	int32_t n_u = 0, n_v = 0;
	if (rc == 1) { // too many anchors for the cooperative fill: sequential replay on one lane
		int rc2 = 0;
		if (lane == 0) {
			Arena B = A;
			rc2 = chain_rmq_fill_seq(B, max_dist, max_dist_inner, bw, max_chn_skip, cap_rmq_size, pen_gap, pen_skip, n, a, f, p, t, v);
			if (B.peak > A.peak) A.peak = B.peak;
		}
		rc2 = warp_bcast_i32(rc2, 0);
		warp_sync();
		if (rc2 < 0) return rc2;
	}
	MGB_TRY(chain_finish_w(H, A, n, f, p, v, t, min_cnt, min_sc, max_drop, a, u_store, &n_u, &n_v, lane));
	A.top = mark;
	if (&H != &A) H.top = hmark;
	*u_ = u_store, *n_u_ = n_u, *n_a_ = n_u > 0? n_v : 0;
	return 0;
}

// chain descriptors ordered by query start (reference: lchain.c:374-408 mg_lchain_gen)
MG_HD inline int lchain_gen(Arena &A, int n_u, const uint64_t *u, const u128 *a, LChain *r)
{
	uint64_t mark = A.top;
	u128 *z;
	int i, k;
	if (n_u == 0) return 0;
	MGB_ALLOC(A, z, u128, n_u);
	for (i = k = 0; i < n_u; ++i) {
		int32_t qs = (int32_t)a[k].y + 1 - (int32_t)(a[k].y >> 32 & 0xff);
		z[i].x = (uint64_t)(uint32_t)qs << 32 | u[i] >> 32;
		z[i].y = (uint64_t)k << 32 | (uint64_t)(uint32_t)(int32_t)u[i];
		k += (int32_t)u[i];
	}
	MGB_TRY(radix_sort_128x(A, z, n_u));
	for (i = 0; i < n_u; ++i) {
		LChain *ri = &r[i];
		int32_t k2 = (int32_t)(z[i].y >> 32), q_span = (int32_t)(a[k2].y >> 32 & 0xff);
		ri->off = k2;
		ri->cnt = (int32_t)z[i].y;
		ri->score = (int32_t)(uint32_t)z[i].x;
		ri->v = (uint32_t)(a[k2].x >> 32);
		ri->rs = (int32_t)a[k2].x + 1 > q_span? (int32_t)a[k2].x + 1 - q_span : 0;
		ri->qs = (int32_t)(z[i].x >> 32);
		ri->re = (int32_t)a[k2 + ri->cnt - 1].x + 1;
		ri->qe = (int32_t)a[k2 + ri->cnt - 1].y + 1;
		ri->dist_pre = 0, ri->hash_pre = 0, ri->inner_pre = 0;
	}
	A.top = mark;
	return 0;
}

// trim chain ends made of high-occurrence seeds (reference: map-algo.c:194-206 mm_fix_bad_ends)
MG_HD inline void fix_bad_ends(const u128 *a, int32_t lc_max_occ, int32_t lc_max_trim, int32_t *as, int32_t *cnt)
{
	int32_t i, k, as0 = *as, cnt0 = *cnt;
	for (i = as0 + cnt0 - 1, k = 0; k < lc_max_trim && k < cnt0; ++k, --i)
		if ((int64_t)(a[i].y >> SEED_OCC_SHIFT) <= (int64_t)lc_max_occ) break;
	*cnt -= k;
	for (i = as0, k = 0; k < *cnt && k < lc_max_trim; ++i, ++k)
		if ((int64_t)(a[i].y >> SEED_OCC_SHIFT) <= (int64_t)lc_max_occ) break;
	*as += k, *cnt -= k;
}

// trim ends that hang off through a large indel (reference: map-algo.c:208-242 mm_fix_bad_ends_alt)
MG_HD inline void fix_bad_ends_alt(const u128 *a, int32_t score, int bw, int min_match, int32_t *as, int32_t *cnt)
{
	int32_t i, l, m, as0 = *as, cnt0 = *cnt;
	if (cnt0 < 3) return;
	m = l = (int32_t)(a[as0].y >> 32 & 0xff);
	for (i = as0 + 1; i < as0 + cnt0 - 1; ++i) {
		int32_t lq, lr, mn, mx;
		int32_t q_span = (int32_t)(a[i].y >> 32 & 0xff);
		lr = (int32_t)a[i].x - (int32_t)a[i-1].x;
		lq = (int32_t)a[i].y - (int32_t)a[i-1].y;
		mn = lr < lq? lr : lq;
		mx = lr > lq? lr : lq;
		if (mx - mn > l >> 1) *as = i;
		l += mn;
		m += mn < q_span? mn : q_span;
		if (l >= bw << 1 || (m >= min_match && m >= bw) || m >= score >> 1) break;
	}
	*cnt = as0 + cnt0 - *as;
	m = l = (int32_t)(a[as0 + cnt0 - 1].y >> 32 & 0xff);
	for (i = as0 + cnt0 - 2; i > *as; --i) {
		int32_t lq, lr, mn, mx;
		int32_t q_span = (int32_t)(a[i+1].y >> 32 & 0xff);
		lr = (int32_t)a[i+1].x - (int32_t)a[i].x;
		lq = (int32_t)a[i+1].y - (int32_t)a[i].y;
		mn = lr < lq? lr : lq;
		mx = lr > lq? lr : lq;
		if (mx - mn > l >> 1) *cnt = i + 1 - *as;
		l += mn;
		m += mn < q_span? mn : q_span;
		if (l >= bw << 1 || (m >= min_match && m >= bw) || m >= score >> 1) break;
	}
}

MG_HD inline int32_t anchor_gap(const u128 *a, int32_t i) // query advance minus target advance between a[i-1] and a[i]
{
	return ((int32_t)a[i].y - (int32_t)a[i-1].y) - ((int32_t)a[i].x - (int32_t)a[i-1].x);
}

// positions of long gaps inside a chain (reference: map-algo.c:244-263 collect_long_gaps); K=0 when fewer than two
MG_HD inline int collect_long_gaps(Arena &A, int as1, int cnt1, const u128 *a, int min_gap, int **K_, int *n_)
{
	int i, n, *K;
	*n_ = 0, *K_ = 0;
	for (i = 1, n = 0; i < cnt1; ++i) {
		// NB: the reference mixes int32 and uint64 here; the result truncated to int is the same
		int gap = (int)(((int64_t)(int32_t)a[as1 + i].y - (int64_t)a[as1 + i - 1].y) - ((int64_t)(int32_t)a[as1 + i].x - (int64_t)a[as1 + i - 1].x));
		if (gap < -min_gap || gap > min_gap) ++n;
	}
	if (n <= 1) return 0;
	MGB_ALLOC(A, K, int, n);
	for (i = 1, n = 0; i < cnt1; ++i) {
		int gap = (int)(((int64_t)(int32_t)a[as1 + i].y - (int64_t)a[as1 + i - 1].y) - ((int64_t)(int32_t)a[as1 + i].x - (int64_t)a[as1 + i - 1].x));
		if (gap < -min_gap || gap > min_gap) K[n++] = i;
	}
	*n_ = n, *K_ = K;
	return 0;
}

// flag seeds inside clusters of opposite indels (reference: map-algo.c:265-300 mm_filter_bad_seeds)
MG_HD inline int filter_bad_seeds(Arena &A, int as1, int cnt1, u128 *a, int min_gap, int diff_thres, int max_ext_len, int max_ext_cnt)
{
	uint64_t mark = A.top;
	int max_st, max_en, n, i, k, mx, *K;
	MGB_TRY(collect_long_gaps(A, as1, cnt1, a, min_gap, &K, &n));
	if (K == 0) return 0;
	mx = 0, max_st = max_en = -1;
	for (k = 0;; ++k) {
		int gap, l, n_ins = 0, n_del = 0, qs, rs, max_diff = 0, max_diff_l = -1;
		if (k == n || k >= max_en) {
			if (max_en > 0)
				for (i = K[max_st]; i < K[max_en]; ++i)
					a[as1 + i].y |= SEED_IGNORE;
			mx = 0, max_st = max_en = -1;
			if (k == n) break;
		}
		i = K[k];
		gap = ((int32_t)a[as1 + i].y - (int32_t)a[as1 + i - 1].y) - (int32_t)(a[as1 + i].x - a[as1 + i - 1].x);
		if (gap > 0) n_ins += gap;
		else n_del += -gap;
		qs = (int32_t)a[as1 + i - 1].y;
		rs = (int32_t)a[as1 + i - 1].x;
		for (l = k + 1; l < n && l <= k + max_ext_cnt; ++l) {
			int j = K[l], diff;
			if ((int32_t)a[as1 + j].y - qs > max_ext_len || (int32_t)a[as1 + j].x - rs > max_ext_len) break;
			gap = ((int32_t)a[as1 + j].y - (int32_t)a[as1 + j - 1].y) - (int32_t)(a[as1 + j].x - a[as1 + j - 1].x);
			if (gap > 0) n_ins += gap;
			else n_del += -gap;
			diff = n_ins + n_del - (n_ins > n_del? n_ins - n_del : n_del - n_ins);
			if (max_diff < diff) max_diff = diff, max_diff_l = l;
		}
		if (max_diff > diff_thres && max_diff > mx)
			mx = max_diff, max_st = k, max_en = max_diff_l;
	}
	A.top = mark;
	return 0;
}

// flag seeds between compensating long gaps (reference: map-algo.c:302-338 mm_filter_bad_seeds_alt)
MG_HD inline int filter_bad_seeds_alt(Arena &A, int as1, int cnt1, u128 *a, int min_gap, int max_ext)
{
	uint64_t mark = A.top;
	int n, k, *K;
	MGB_TRY(collect_long_gaps(A, as1, cnt1, a, min_gap, &K, &n));
	if (K == 0) return 0;
	for (k = 0; k < n;) {
		int i = K[k], l;
		int gap1 = ((int32_t)a[as1 + i].y - (int32_t)a[as1 + i - 1].y) - ((int32_t)a[as1 + i].x - (int32_t)a[as1 + i - 1].x);
		int re1 = (int32_t)a[as1 + i].x;
		int qe1 = (int32_t)a[as1 + i].y;
		gap1 = gap1 > 0? gap1 : -gap1;
		for (l = k + 1; l < n; ++l) {
			int j = K[l], gap2, q_span_pre, rs2, qs2, m;
			if ((int32_t)a[as1 + j].y - qe1 > max_ext || (int32_t)a[as1 + j].x - re1 > max_ext) break;
			gap2 = ((int32_t)a[as1 + j].y - (int32_t)a[as1 + j - 1].y) - (int32_t)(a[as1 + j].x - a[as1 + j - 1].x);
			q_span_pre = (int)(a[as1 + j - 1].y >> 32 & 0xff);
			rs2 = (int32_t)a[as1 + j - 1].x + q_span_pre;
			qs2 = (int32_t)a[as1 + j - 1].y + q_span_pre;
			m = rs2 - re1 < qs2 - qe1? rs2 - re1 : qs2 - qe1;
			gap2 = gap2 > 0? gap2 : -gap2;
			if (m > gap1 + gap2) break;
			re1 = (int32_t)a[as1 + j].x;
			qe1 = (int32_t)a[as1 + j].y;
			gap1 = gap2;
		}
		if (l > k + 1) {
			int j, end = K[l - 1];
			for (j = K[k]; j < end; ++j) a[as1 + j].y |= SEED_IGNORE;
			a[as1 + end].y |= SEED_FIXED;
		}
		k = l;
	}
	A.top = mark;
	return 0;
}

// replace the high half of a[].x by the index of the minimizer on the query (reference: lchain.c:410-441)
MG_HD inline int update_anchors(int32_t n_a, u128 *a, int32_t n, const int32_t *mini_pos)
{
	int32_t st = -1, j, k, L = 0, R = n - 1, x;
	if (n_a <= 0) return 0;
	x = (int32_t)a[0].y;
	while (L <= R) {
		int32_t m = (int32_t)(((uint64_t)L + (uint64_t)R) >> 1);
		int32_t y = mini_pos[m];
		if (y < x) L = m + 1;
		else if (y > x) R = m - 1;
		else { st = m; break; }
	}
	if (st < 0) return MGB_E_INTERNAL;
	for (k = 0, j = st; j < n && k < n_a; ++j)
		if ((int32_t)a[k].y == mini_pos[j])
			a[k].x = (uint64_t)j << 32 | (a[k].x & 0xffffffffULL), ++k;
	return k == n_a? 0 : MGB_E_INTERNAL;
}

// update_anchors() entered by all lanes of a warp: one anchor per lane.  mini_pos[] (query positions of the kept minimizers) is
// strictly ascending and so are the query positions along a chain, hence the sequential merge above pairs anchor k with THE entry
// that equals its position: a binary search per anchor finds the same index.
MG_HD inline int update_anchors_w(int32_t n_a, u128 *a, int32_t n, const int32_t *mini_pos, int lane)
{
	int bad = 0;
	for (int32_t k = lane; k < n_a; k += MGB_W) {
		const int32_t x = (int32_t)a[k].y;
		int32_t lo = 0, hi = n;
		while (lo < hi) { const int32_t m = (int32_t)(((uint32_t)lo + (uint32_t)hi) >> 1); if (mini_pos[m] < x) lo = m + 1; else hi = m; }
		if (lo < n && mini_pos[lo] == x) a[k].x = (uint64_t)lo << 32 | (a[k].x & 0xffffffffULL);
		else bad = 1;
	}
	bad = warp_any(bad);
	warp_sync();
	return bad? MGB_E_INTERNAL : 0;
}

} // namespace mgb
