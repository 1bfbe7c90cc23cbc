// mgb_pipeline.cuh -- per-read stage functions glued to the global pools.
//   stage_seed()  : K1 sketch + K2 lookup/expand + K3 seed sort      (reference: map-algo.c:366-368)
//   stage_chain() : K4/K5 linear chaining, rescue, chain post-filters (reference: map-algo.c:377-449)
//   stage_align() : K6-K8 graph chaining, bridging, base alignment    (mgb_galign.cuh)
#pragma once
#include "mgb_model.cuh"
#include "mgb_seed.cuh"
#include "mgb_lchain.cuh"
#include "mgb_gclabel.cuh"
#include "mgb_tma.cuh"

namespace mgb {

struct PipeCtx {
	GraphDev g;
	IndexDev ix;
	MapOptDev opt;
	BatchDev b;
	ReadMeta *meta;        // [n_reads]
	// global pools (element arrays + bump allocators)
	Pool *pool_anchor;     u128 *anchor;
	Pool *pool_minipos;    int32_t *minipos;
	Pool *pool_lchain;     LChain *lchain;
	Pool *pool_out;        char *out;
	Pool *pool_plan;       uint64_t *plan;       // alignment plans (literal CIGAR items and job references)
	Pool *pool_jobs;       struct WfaJob *jobs;  // gap alignment jobs
	Pool *pool_cig;        uint32_t *cig;        // per-job CIGARs
	int32_t *jobq[2];      unsigned int *jobq_n;   // jobs handed to WFA tier 2 / tier 3
	Pool *pool_gstate;     char *gstate;         // per-read state between the two graph-chaining passes
	Pool *pool_gjobs;      struct GwfaJob *gjobs; // bridging alignment jobs (K7a)
	Pool *pool_walk;       int32_t *walk;        // walks found by the bridging jobs
	int32_t *rescue_list;  unsigned int *rescue_n; // reads handed from k_chain to k_chain_rescue
	LabTab lab;            // reachability labels of the graph (mgb_gclabel.cuh); persistent across batches
	// work queue
	unsigned int *next_read;
	// instrumentation: 32 counters, see PROF_* below
	unsigned long long *prof;
	// tier routing of the gap alignments, learned from the batches before (see wfa_job_run)
	int32_t skip1_len;            // gaps with max(tl,ql) at or above this go past tier 1 without trying it
	unsigned int *tier_hist;      // [32 length buckets of 16 bases][4]: final tier of the gaps that tried every tier
};

enum { PROF_WFA_FAST_CYC = 0, PROF_WFA_FAST_N, PROF_WFA_SLOW_CYC, PROF_WFA_SLOW_N, PROF_WFA_MAX_CYC, PROF_WFA_CELLS, PROF_WFA_TB_CYC,
	   PROF_GC_DP_CYC, PROF_GC_GEN_CYC, PROF_GC_POST_CYC, PROF_GC_PLAN_CYC, PROF_FIN_CIGAR_CYC, PROF_FIN_DS_CYC, PROF_SEED_SKETCH_CYC,
	   PROF_SEED_MATCH_CYC, PROF_SEED_SORT_CYC, PROF_CHAIN_DP_CYC, PROF_CHAIN_BT_CYC, PROF_CHAIN_RMQ_CYC, PROF_CHAIN_POST_CYC, PROF_WFA_MID_CYC, PROF_WFA_MID_N, PROF_GC_GWFA_CYC, PROF_GC_SHORTK_CYC, PROF_GC_EXTRA_CYC, PROF_GWFA_MAX_CYC, PROF_GC_DP_MAX_CYC, PROF_WFA_HANDOFF_CELLS, PROF_WFA_HANDOFF_N, PROF_LAB_CYC, PROF_LAB_N, PROF_N = 32 };

MG_HD inline unsigned long long prof_clock()
{
#if MGB_ON_DEVICE
	return (unsigned long long)clock64();
#else
	return 0;
#endif
}
// The counters of a launch are summed per block in shared memory and reach the global ones once, when the block ends
// (stage_loop): a gap alignment job bumps four of them, and 17 million jobs per step doing that with global atomics is
// 70 million reductions on one 32-byte sector of L2, which serialises them.
#if defined(__CUDACC__)
MG_D inline unsigned long long *prof_block() { __shared__ unsigned long long s_prof[PROF_N]; return s_prof; }
MG_D inline bool prof_is_max(int slot) { return slot == PROF_WFA_MAX_CYC || slot == PROF_GWFA_MAX_CYC || slot == PROF_GC_DP_MAX_CYC; }
MG_D inline void prof_block_begin() { if (threadIdx.x < PROF_N) prof_block()[threadIdx.x] = 0; __syncthreads(); }
MG_D inline void prof_block_end(unsigned long long *prof)
{
	__syncthreads();
	if (prof && threadIdx.x < PROF_N) {
		const unsigned long long v = prof_block()[threadIdx.x];
		if (v) { if (prof_is_max((int)threadIdx.x)) atomicMax(&prof[threadIdx.x], v); else atomicAdd(&prof[threadIdx.x], v); }
	}
}
#endif
MG_HD inline void prof_add(const PipeCtx &c, int slot, unsigned long long v)
{
#if MGB_ON_DEVICE
	if (c.prof) atomicAdd(&prof_block()[slot], v);
#else
	if (c.prof) c.prof[slot] += v;
#endif
}
MG_HD inline void prof_max(const PipeCtx &c, int slot, unsigned long long v)
{
#if MGB_ON_DEVICE
	if (c.prof) atomicMax(&prof_block()[slot], v);
#else
	if (c.prof && c.prof[slot] < v) c.prof[slot] = v;
#endif
}

// K1-K3 for one read.  Writes sorted seeds to the anchor pool and the query positions of kept minimizers to the
// mini_pos pool.
// Warp-uniform: all lanes enter; the sketch is cut into chunks over the lanes, the index probes and the seed expansion
// are spread over the lanes, the (order-sensitive, unstable) seed sort runs on lane 0.
MG_HD inline int stage_seed(const PipeCtx &c, int rid, Arena &A, int lane, int32_t *smem = 0)
{
	ReadMeta &m = c.meta[rid];
	const char *seq = c.b.seq + c.b.seq_off[rid];
	const int32_t qlen = c.b.seq_len[rid];
	const uint64_t mark = A.top;
	const int skip = qlen <= 0 || (c.opt.max_qlen > 0 && qlen > c.opt.max_qlen);
	if (lane == 0) {
		m.status = 0, m.n_mz = 0, m.rep_len = 0, m.n_a = 0, m.a_off = 0, m.n_mp = 0, m.mp_off = 0, m.n_lc = 0, m.lc_off = 0;
		m.n_seed0 = 0, m.n_u0 = 0;
		{ // reference: map-algo.c:362-364
			uint32_t h = c.b.name_hash[rid];
			h ^= hash32((uint32_t)qlen) + hash32((uint32_t)c.opt.seed);
			m.hash = hash32(h);
		}
		if (skip) m.status = 1; // unmapped by definition
	}
	if (skip) return 0;
	AVec<u128> mv;
	avec_init(mv);
	unsigned long long t0 = prof_clock();
	const int32_t n_seg = batch_n_seg(c.b, rid);
	if (n_seg == 1) {
		MGB_TRY(sketch_seq_w(A, seq, qlen, c.ix.w, c.ix.k, 0, mv, lane, (u128*)smem, c.b.pk && c.b.pk_off[rid] != ~0ULL? c.b.pk + c.b.pk_off[rid] : 0)); // (a read with letters other than A/C/G/T came up as ASCII)
	} else { // reference: map-algo.c:34-45 collect_minimizers: every segment on its own, positions shifted by the lengths before it
		const int32_t *sl = c.b.seg_len + c.b.seg_off[rid];
		MGB_ALLOC(A, mv.a, u128, (int64_t)qlen + 16 * (int64_t)n_seg);
		mv.m = (int64_t)qlen + 16 * (int64_t)n_seg;
		const uint64_t keep = A.top;
		int32_t sum = 0;
		for (int32_t i = 0; i < n_seg; ++i) {
			AVec<u128> one;
			avec_init(one);
			if (sl[i] > 0) MGB_TRY(sketch_seq_w(A, seq + sum, sl[i], c.ix.w, c.ix.k, (uint32_t)i, one, lane, (u128*)smem));
			if (mv.n + one.n > mv.m) return MGB_E_INTERNAL;
			for (int64_t j = lane; j < one.n; j += MGB_W) { u128 e = one.a[j]; e.y += (uint64_t)sum << 1; mv.a[mv.n + j] = e; }
			warp_sync();
			mv.n += one.n, sum += sl[i];
			A.top = keep;
		}
	}
	unsigned long long t1 = prof_clock();
	SeedMatch *sm;
	int n_m, n_mp, rep_len;
	int64_t n_a;
	int32_t *mp_tmp, *a_off;
	MGB_ALLOC(A, mp_tmp, int32_t, mv.n);
	MGB_TRY(collect_matches_w(A, c.ix, c.opt.occ_max1, mv, &sm, &n_m, &n_a, &rep_len, mp_tmp, &n_mp, &a_off, lane));
	int64_t off_a = 0, off_mp = 0;
	if (lane == 0) {
		off_a = pool_alloc(c.pool_anchor, (uint64_t)n_a * sizeof(u128));
		off_mp = pool_alloc(c.pool_minipos, (uint64_t)n_mp * sizeof(int32_t));
	}
	off_a = (int64_t)warp_bcast_u64((uint64_t)off_a, 0), off_mp = (int64_t)warp_bcast_u64((uint64_t)off_mp, 0);
	if (off_a < 0 || off_mp < 0) return MGB_E_POOL;
	u128 *a = c.anchor + off_a / (int64_t)sizeof(u128);
	int32_t *mp = c.minipos + off_mp / (int64_t)sizeof(int32_t);
	if (lane == 0) {
		m.n_mz = (int32_t)mv.n, m.rep_len = rep_len;
		m.a_off = off_a / (int64_t)sizeof(u128), m.mp_off = off_mp / (int64_t)sizeof(int32_t);
		m.n_a = (int32_t)n_a, m.n_mp = n_mp, m.n_seed0 = (int32_t)n_a;
	}
	for (int i = lane; i < n_mp; i += MGB_W) mp[i] = mp_tmp[i];
	unsigned long long t2;
	if (c.opt.flag & F_HEAP_SORT) { // reference: map-algo.c:367
		int rc = 0;
		if (lane == 0) { Arena B = A; rc = expand_seeds_heap(B, c.g, n_m, sm, n_a, a); if (B.peak > A.peak) A.peak = B.peak; }
		rc = warp_bcast_i32(rc, 0);
		warp_sync();
		if (rc < 0) return rc;
		t2 = prof_clock();
	} else {
		if ((c.opt.flag & F_NO_DIAG) && c.b.self_id) { // reference: map-algo.c:167 (the heap variant above has no such filter)
			int32_t kept = 0;
			if (lane == 0) kept = (int32_t)expand_seeds_nodiag(c.g, n_m, sm, c.b.self_id[rid], a);
			n_a = warp_bcast_i32(kept, 0);
			if (lane == 0) m.n_a = (int32_t)n_a, m.n_seed0 = (int32_t)n_a;
		} else expand_seeds_w(c.g, n_m, sm, a_off, a, lane);
		warp_sync();
		t2 = prof_clock();
		{ // the sort's range stack and bin tables in the shared-memory slice the sketch's rings no longer need
			Arena R;
			arena_init(R, smem, smem? (uint64_t)SKETCH_SMEM_BYTES : 0);
			Arena &S = smem && R.cap >= (uint64_t)n_a / 4 + 3400? R : A;
			MGB_TRY(radix_sort_128x_w(S, a, n_a, lane, &A, true)); // digit walk: the seeds are in HBM
		}
	}
	if (lane == 0) prof_add(c, PROF_SEED_SKETCH_CYC, t1 - t0), prof_add(c, PROF_SEED_MATCH_CYC, t2 - t1), prof_add(c, PROF_SEED_SORT_CYC, prof_clock() - t2);
	A.top = mark;
	return 0;
}

// chain records, end trimming, bad-seed filters, anchor update, pool write (reference: map-algo.c:419-449); one lane
// part 1 (one lane): chain records, end trimming, bad-seed filters; leaves the kept chains in lc_[0..*n_lc_) (in the arena)
MG_HD inline int stage_chain_tail(const PipeCtx &c, ReadMeta &m, Arena &A, u128 *a, const uint64_t *u, int32_t n_lc, int32_t n_a_new, LChain **lc_, int32_t *n_lc_)
{
	const MapOptDev &o = c.opt;
	m.n_a = n_lc > 0? n_a_new : 0;
	m.n_lc = 0;
	*lc_ = 0, *n_lc_ = 0;
	if (n_lc > 0) {
		LChain *lc;
		MGB_ALLOC(A, lc, LChain, n_lc);
		MGB_TRY(lchain_gen(A, n_lc, u, a, lc));
		if (n_lc > 1) { // reference: map-algo.c:425-444
			int32_t n_new = 0;
			for (int32_t i = 0; i < n_lc; ++i) {
				LChain *p = &lc[i];
				int32_t cnt = p->cnt, off = p->off;
				fix_bad_ends(a, o.lc_max_occ, o.lc_max_trim, &off, &cnt);
				fix_bad_ends_alt(a, p->score, o.bw, 100, &off, &cnt);
				MGB_TRY(filter_bad_seeds(A, off, cnt, a, 10, 40, o.max_gap >> 1, 10));
				MGB_TRY(filter_bad_seeds_alt(A, off, cnt, a, 30, o.max_gap >> 1));
				p->off = off, p->cnt = cnt;
				if (cnt >= o.min_lc_cnt) {
					int32_t q_span = (int32_t)(a[p->off].y >> 32 & 0xff);
					p->rs = (int32_t)a[p->off].x + 1 - q_span;
					p->qs = (int32_t)a[p->off].y + 1 - q_span;
					p->re = (int32_t)a[p->off + p->cnt - 1].x + 1;
					p->qe = (int32_t)a[p->off + p->cnt - 1].y + 1;
					lc[n_new++] = *p;
				}
			}
			n_lc = n_new;
		}
		*lc_ = lc, *n_lc_ = n_lc;
	}
	return 0;
}
// part 2 (one lane, after the warp-wide anchor update): sources for graph chaining, chain records into the pool
MG_HD inline int stage_chain_tail2(const PipeCtx &c, ReadMeta &m, const LChain *lc, int32_t n_lc)
{
	const MapOptDev &o = c.opt;
	{
		if (n_lc > 1 && c.lab.src_off) { // graph chaining will ask for walks out of these chains' vertices (gchain_dp_w applies the same test)
			int32_t n_ext = 0;
			for (int32_t i = 0; i < n_lc; ++i) n_ext += !gc_isolated(c.g, lc[i], o.bw_long);
			if (n_ext >= 2)
				for (int32_t i = 0; i < n_lc; ++i)
					if (!gc_isolated(c.g, lc[i], o.bw_long)) lab_want(c.lab, lc[i].v ^ 1);
		}
		int64_t lc_off = pool_alloc(c.pool_lchain, (uint64_t)n_lc * sizeof(LChain));
		if (lc_off < 0) return MGB_E_POOL;
		m.lc_off = lc_off / (int64_t)sizeof(LChain);
		LChain *dst = c.lchain + m.lc_off;
		for (int32_t i = 0; i < n_lc; ++i) dst[i] = lc[i];
		m.n_lc = n_lc;
	}
	return 0;
}

// K4/K5 for one read: seeds -> linear chains, in two kernels.
//   k_chain         (pass 0): chaining DP (lr) or RMQ chaining (asm), backtracking, compaction; then either the chain records
//                   (stage_chain_tail) or, for a read whose best chain leaves much of it uncovered (map-algo.c:407-417: in practice
//                   every read that spans several segments), a place on the rescue list with its compacted anchors;
//   k_chain_rescue  (pass 1): the listed reads: anchors sorted back into target order, RMQ chaining with the long bandwidth, tail.
// ON CHIP: the read's seeds are bulk-copied (cp.async.bulk + mbarrier, mgb_tma.cuh) into the warp's slice of shared memory, and the
// arrays the chaining loops re-read for every anchor (f/p/v/t, the RMQ priorities and window) are taken from the rest of the slice
// (MGB_ALLOC_HOT); only the surviving anchors go back to HBM, as one bulk store.  What is touched once (end-point list, sort
// scratch, chain records) stays in the worker's HBM arena, so that a slice is small and many warps are resident: the loops are
// bound by the latency of their warp-wide votes, and what hides that is warps (everything in a 36 KB slice, 6 warps per SM, was
// faster per warp but slower per kernel than many more warps per SM working in HBM).
// A read whose seeds do not fit the slice works on the HBM copy, with whatever fits of the hot arrays still on chip.
static const int CHAIN_SMEM_BYTES = 16 * 1024;        // per warp, k_chain: anchors + f/p/v/t of a read of up to ~500 seeds
static const int CHAIN_RESCUE_SMEM_BYTES = 18 * 1024; // per warp, k_chain_rescue: + window and block summaries of the RMQ pass (the priorities if they fit)

struct ChainRun { // what one pass leaves behind
	int32_t n_keep;   // anchors of a[] to write back
	int32_t rescue;   // pass 0: the read goes on the rescue list
};

// The arguments of one chaining call (reference: mg_lchain_dp / mg_lchain_rmq); the RMQ chaining takes max_dist_x as its max_dist
// and ignores max_dist_y, max_iter, is_cdna and n_seg, the DP ignores max_dist_inner and cap_rmq_size.
struct LChainOpt {
	int32_t max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc;
	float pen_gap, pen_skip;
	int32_t is_cdna, n_seg, max_dist_inner, cap_rmq_size;
};

// The chaining of one pass on a read's anchors a[0..n_a) (reference: map-algo.c:386-392, 413-415): pass 0 chains them in target
// order by DP (lr) or by RMQ (asm, rmq != 0); pass 1 sorts the anchors it was handed back into target order and chains them by RMQ.
// The n_u chains go to u (score<<32 | anchors), their anchors to a[0..n_v).  path (may be NULL): which fill ran, CHAIN_PATH_*.
template<int PASS>
MG_HD inline int chain_run(Arena &H, Arena &A, int rmq, const LChainOpt &co, int64_t n_a, u128 *a, int32_t *n_u, uint64_t **u, int32_t *n_v, int lane,
						   int *path = 0)
{
	if (PASS == 1) { // back into target order; the sort's range stack and bin tables on chip when the slice has the room (it is empty but for the anchors)
		Arena &S = H.cap - H.top >= (uint64_t)n_a / 4 + 3400? H : A;
		MGB_TRY(radix_sort_128x_w(S, a, n_a, lane, 0, false)); // (in place: the list is on chip, where the digit walk was slower)
	}
	if (PASS == 1 || rmq)
		return chain_rmq_w(H, A, co.max_dist_x, co.max_dist_inner, co.bw, co.max_skip, co.cap_rmq_size, co.min_cnt, co.min_sc, co.pen_gap, co.pen_skip,
						   n_a, a, n_u, u, n_v, lane, path);
	if (path && n_a > 0) *path = CHAIN_PATH_DP;
	return chain_dp_w(H, A, co.max_dist_x, co.max_dist_y, co.bw, co.max_skip, co.max_iter, co.min_cnt, co.min_sc, co.pen_gap, co.pen_skip, co.is_cdna,
					  co.n_seg, n_a, a, n_u, u, n_v, lane);
}

template<int PASS>
MG_HD inline int chain_pass(const PipeCtx &c, int rid, Arena &H, Arena &A, u128 *a, int64_t n_a, int lane, ChainRun *run)
{
	ReadMeta &m = c.meta[rid];
	const MapOptDev &o = c.opt;
	const uint64_t mark = A.top;
	const int32_t qlen = c.b.seq_len[rid];
	int32_t n_lc = 0, n_a_new = 0;
	uint64_t *u = 0;
	run->n_keep = 0, run->rescue = 0;
	unsigned long long t0 = prof_clock();
	if (PASS == 0) {
		const int is_splice = !!(o.flag & F_SPLICE), is_sr = !!(o.flag & F_SR);
		int max_gap_qry, max_gap_ref;
		// reference: map-algo.c:377-386
		if (is_sr) max_gap_qry = qlen > o.max_gap? qlen : o.max_gap;
		else max_gap_qry = o.max_gap;
		if (o.max_gap_ref > 0) max_gap_ref = o.max_gap_ref;
		else if (o.max_frag_len > 0) {
			max_gap_ref = o.max_frag_len - qlen;
			if (max_gap_ref < o.max_gap) max_gap_ref = o.max_gap;
		} else max_gap_ref = o.max_gap;
		if (n_a > 0) {
			const int rmq = !!(o.flag & F_RMQ);
			LChainOpt co;
			co.max_dist_x = rmq? o.max_gap : max_gap_ref, co.max_dist_y = max_gap_qry, co.bw = o.bw, co.max_skip = o.max_lc_skip, co.max_iter = o.max_lc_iter;
			co.min_cnt = o.min_lc_cnt, co.min_sc = o.min_lc_score, co.pen_gap = o.chn_pen_gap, co.pen_skip = o.chn_pen_skip;
			co.is_cdna = is_splice, co.n_seg = batch_n_seg(c.b, rid), co.max_dist_inner = o.max_gap_pre, co.cap_rmq_size = o.rmq_size_cap;
			MGB_TRY(chain_run<0>(H, A, rmq, co, n_a, a, &n_lc, &u, &n_a_new, lane));
		}
		if (lane == 0) m.n_u0 = n_lc, prof_add(c, PROF_CHAIN_DP_CYC, prof_clock() - t0);
		// long-join rescue (reference: map-algo.c:407-417)
		if (o.bw_long > o.bw && (o.flag & (F_SPLICE | F_SR)) == 0 && batch_n_seg(c.b, rid) == 1 && n_lc > 1) {
			int32_t st = (int32_t)a[0].y, en = (int32_t)a[(int32_t)u[0] - 1].y;
			if (qlen - (en - st) > o.rmq_rescue_size || (float)(qlen - (en - st)) > (float)qlen * o.rmq_rescue_ratio) {
				int32_t n2 = 0;
				for (int32_t i = 0; i < n_lc; ++i) n2 += (int32_t)u[i];
				warp_sync();
				if (lane == 0) {
					m.n_a = n2; // the chained anchors are what the second pass starts from
#if MGB_ON_DEVICE
					c.rescue_list[atomicAdd(c.rescue_n, 1u)] = rid;
#else
					c.rescue_list[(*c.rescue_n)++] = rid;
#endif
				}
				run->n_keep = n2, run->rescue = 1;
				A.top = mark;
				return 0;
			}
		}
	} else {
		LChainOpt co;
		co.max_dist_x = o.max_gap, co.max_dist_y = 0, co.bw = o.bw_long, co.max_skip = o.max_lc_skip, co.max_iter = 0;
		co.min_cnt = o.min_lc_cnt, co.min_sc = o.min_lc_score, co.pen_gap = o.chn_pen_gap, co.pen_skip = o.chn_pen_skip;
		co.is_cdna = 0, co.n_seg = 1, co.max_dist_inner = o.max_gap_pre, co.cap_rmq_size = o.rmq_size_cap;
		MGB_TRY(chain_run<1>(H, A, 1, co, n_a, a, &n_lc, &u, &n_a_new, lane));
		if (lane == 0) prof_add(c, PROF_CHAIN_RMQ_CYC, prof_clock() - t0);
	}
	unsigned long long t2 = prof_clock();
	int rc = 0;
	LChain *lc = 0;
	int32_t n_keep_lc = 0;
	{
		Arena B = A;
		if (lane == 0) rc = stage_chain_tail(c, m, B, a, u, n_lc, n_a_new, &lc, &n_keep_lc);
		rc = warp_bcast_i32(rc, 0);
		lc = (LChain*)warp_bcast_u64((uint64_t)lc, 0), n_keep_lc = warp_bcast_i32(n_keep_lc, 0);
		A.top = warp_bcast_u64(B.top, 0);
		const uint64_t pk = warp_bcast_u64(B.peak, 0);
		if (pk > A.peak) A.peak = pk;
		warp_sync();
	}
	if (rc == 0) { // minimizer indices into the anchors (reference: lchain.c:424-441), one anchor per lane
		const int32_t *mp = c.minipos + m.mp_off;
		for (int32_t i = 0; i < n_keep_lc && rc == 0; ++i) rc = update_anchors_w(lc[i].cnt, &a[lc[i].off], m.n_mp, mp, lane);
	}
	if (rc == 0) {
		if (lane == 0 && lc) rc = stage_chain_tail2(c, m, lc, n_keep_lc);
		rc = warp_bcast_i32(rc, 0);
	}
	if (lane == 0) prof_add(c, PROF_CHAIN_POST_CYC, prof_clock() - t2);
	warp_sync();
	run->n_keep = n_lc > 0? n_a_new : 0;
	A.top = mark;
	return rc;
}

// smem: the warp's slice of CHAIN_SMEM_BYTES, or NULL.  Its first 16 bytes hold the transaction barrier of the bulk loads and the
// parity the next wait has to use (chain_smem_init() once per kernel).
MG_HD inline void chain_smem_init(int32_t *smem, int lane)
{
	if (lane == 0) { mbar_init((uint64_t*)smem, 1); smem[2] = 0; }
	warp_sync();
}

// A read's anchors a[0..n_a) in HBM, worked on in the warp's slice of `slice` bytes (NULL: no slice): staged there by one bulk copy
// when they fit, the rest of the slice as the hot arena.  run(H, aw, &n_keep) chains the anchors aw[] (the staged copy or a[] itself)
// and returns its code; the first n_keep of them are stored back to a[] by one bulk copy.  *staged: whether the anchors went on chip.
template<typename Run>
MG_HD inline int chain_staged(int32_t *smem, uint64_t slice, Arena &A, u128 *a, int64_t n_a, int lane, int *staged_, Run &&run)
{
	int32_t n_keep = 0;
	*staged_ = 0;
	if (smem == 0 || n_a == 0) return run(A, a, &n_keep);
	const uint64_t a_bytes = (uint64_t)n_a * sizeof(u128);
	const int staged = a_bytes + 16 <= slice;
	uint64_t *bar = (uint64_t*)smem;
	u128 *as = (u128*)((char*)smem + 16);
	if (staged) { // the read's seeds: one bulk copy, completion on the slice's barrier
		const uint32_t parity = (uint32_t)smem[2];
		if (lane == 0) bulk_load(as, a, (uint32_t)a_bytes, bar);
		mbar_wait(bar, parity);
		warp_sync();
		if (lane == 0) smem[2] = (int32_t)(parity ^ 1);
	}
	Arena S; // what is left of the slice
	arena_init(S, (char*)as + (staged? a_bytes : 0), slice - 16 - (staged? a_bytes : 0));
	const int rc = run(S, staged? as : a, &n_keep);
	if (staged && rc == 0 && n_keep > 0) {
		warp_sync();
		if (lane == 0) { bulk_store(a, as, (uint32_t)n_keep * (uint32_t)sizeof(u128)); bulk_store_wait(); }
		warp_sync();
	}
	*staged_ = staged;
	return rc;
}

template<int PASS>
MG_HD inline int stage_chain(const PipeCtx &c, int rid, Arena &A, int lane, int32_t *smem)
{
	ReadMeta &m = c.meta[rid];
	if (m.status != 0) return 0;
	u128 *a = c.anchor + m.a_off;
	const int64_t n_a = m.n_a;
	int staged;
	const int rc = chain_staged(smem, PASS == 0? CHAIN_SMEM_BYTES : CHAIN_RESCUE_SMEM_BYTES, A, a, n_a, lane, &staged,
								[&](Arena &H, u128 *aw, int32_t *n_keep) {
									ChainRun run;
									const int r = chain_pass<PASS>(c, rid, H, A, aw, n_a, lane, &run);
									*n_keep = run.n_keep;
									return r;
								});
	if (staged && lane == 0 && c.prof) prof_add(c, PROF_CHAIN_BT_CYC, 1); // reads whose anchors were chained on chip
	return rc;
}

} // namespace mgb
