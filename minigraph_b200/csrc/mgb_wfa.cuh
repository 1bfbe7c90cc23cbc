// mgb_wfa.cuh -- global alignment of one inter-anchor gap with the 2-piece affine wavefront algorithm (K8a).
// (reference: miniwfa.c:380-435 mwf_wfa_core, :281-308 wf_next_tb, :329-377 wf_traceback, :144-171 wf_stripe_shrink)
// Penalties: mismatch 4, gap1 4+2l, gap2 15+1l.  CIGAR bytes depend on the tie preferences of the recurrence
// (>= everywhere, E before F, mismatch before gap) and on the traceback state machine (SURVEY H7); both are kept.
//
// One warp aligns one gap.  Lanes own diagonals in the three data-parallel phases of a score step (exact-match
// extension, recurrence, traceback-byte store); the scalar bookkeeping ([lo,hi] tracking, iteration counting) is
// replicated on all lanes; the traceback walk is sequential, so the job tiers keep the traceback rows of up to MGB_W gaps and walk
// them back one gap per lane (wfa_tb_batch).  Two storage schemes share that skeleton:
//   wfa_smem<W,..>  wavefront ring in shared memory for windows of at most W diagonals and scores below 255
//   wfa_exact       ring in the worker arena (global memory), any size, incl. the band re-centring every 256 scores
// Only one diagonal (d = ql - tl) can reach the end of both sequences, so "the first diagonal that finishes" of the
// sequential reference needs no ordering between lanes.
#pragma once
#include "mgb_common.cuh"

namespace mgb {

static const int32_t WF_NEG_INF = -0x40000000;
static const int WF_X = 4, WF_O1 = 4, WF_E1 = 2, WF_O2 = 15, WF_E2 = 1;
static const int WF_MAX_PEN = 16;           // max(x, o1+e1, o2+e2)
static const int WF_NSLICE = WF_MAX_PEN + 1;
static const int WF_PAD = WF_MAX_PEN + 1;   // m1 in the reference
static const int WF_SEQ_PAD = 16;           // sentinel bytes after each staged sequence

#define MGB_WF_MAX(a, b) ((a) >= (b)? (a) : (b))

struct WfTbRow;
struct WfResult {
	int32_t s;        // score, -1 if the iteration cap was hit
	int32_t n_cigar;
	int64_t n_iter;
	uint32_t *cigar;  // len<<4|op  (op: 7 '=', 8 'X', 1 'I', 2 'D'), allocated at the caller's mark
	// The job tiers stop after the score loop: rows != 0 means that the traceback is still to run (wfa_tb_batch), from these rows,
	// into cigar[0 .. tl + ql + 2); the rows stay in the arena above the caller's mark.  rows == 0: cigar[0 .. n_cigar) is final.
	const WfTbRow *rows;
	int32_t n_rows, last_state;
};

// ---- sequence staging: 4-byte aligned copies followed by sentinel bytes that match nothing ----
// (the reference pads both strings with two distinct unused characters for the same purpose, miniwfa.c:182-209)

MG_HD inline void wf_stage_seq(char *dst, const char *src, int32_t len, uint8_t sentinel, int lane)
{
	for (int32_t i = lane; i < len; i += MGB_W) dst[i] = src[i];
	for (int32_t i = len + lane; i < len + WF_SEQ_PAD; i += MGB_W) dst[i] = (char)sentinel;
}

MG_HD inline uint32_t wf_ld32u(const char *base, int32_t pos) // unaligned 32-bit read from an aligned, padded buffer
{
	const uint32_t *w = (const uint32_t*)base;
	uint32_t lo = w[pos >> 2], hi = w[(pos >> 2) + 1];
	int sh = (pos & 3) << 3;
#if MGB_ON_DEVICE
	return __funnelshift_r(lo, hi, sh);
#else
	return sh? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}

// furthest k on diagonal d reachable by exact matches from k (reference: miniwfa.c:212-226 wf_extend1_padded)
MG_HD inline int32_t wf_extend(const char *ts, const char *qs, int32_t k, int32_t d)
{
	for (;;) {
		uint32_t x = wf_ld32u(ts, k + 1) ^ wf_ld32u(qs, d + k + 1);
		if (x) {
#if MGB_ON_DEVICE
			return k + ((__ffs((int)x) - 1) >> 3);
#else
			return k + (__builtin_ctz(x) >> 3);
#endif
		}
		k += 4;
	}
}

// ---- traceback (reference: miniwfa.c:329-377 wf_traceback), one lane per gap ----
// TB::get(s, d) returns the traceback byte of (score s, diagonal d) or -1 if out of range.  Operations are
// accumulated in registers and written from the back of cig_store, so no reversal pass is needed.
template<typename TB>
MG_HD inline int wf_traceback(const TB &tb, int32_t n_scores, int32_t tl, const char *ts, int32_t ql, const char *qs, int32_t last_state,
							  uint32_t *cig_store, int64_t max_cigar, int32_t *n_cigar, int64_t *first)
{
	int32_t i = ql - 1, k = tl - 1, s = n_scores - 1, last = last_state;
	int64_t w = max_cigar; // next write position is w-1
	int32_t cur_op = -1, cur_len = 0;
#define MGB_CIG_PUSH(op_, len_) do { \
		if (cur_op == (op_)) cur_len += (len_); \
		else { \
			if (cur_op >= 0) { if (w <= 0) return MGB_E_INTERNAL; cig_store[--w] = (uint32_t)cur_len << 4 | (uint32_t)cur_op; } \
			cur_op = (op_), cur_len = (len_); \
		} \
	} while (0)
	while (i >= 0 && k >= 0) {
		int32_t k0 = k, x, state, ext;
		if (last == 0) {
			while (i >= 0 && k >= 0 && qs[i] == ts[k]) --i, --k;
			if (k0 - k > 0) MGB_CIG_PUSH(7, k0 - k);
			if (i < 0 || k < 0) break;
		}
		if (s < 0) return MGB_E_INTERNAL;
		x = tb.get(s, i - k);
		if (x < 0) return MGB_E_INTERNAL;
		state = last == 0? x & 7 : last;
		ext = state > 0? x >> (state + 2) & 1 : 0;
		if (state == 0) { MGB_CIG_PUSH(8, 1); --i, --k, s -= WF_X; }
		else if (state == 1) { MGB_CIG_PUSH(1, 1); --i, s -= ext? WF_E1 : WF_O1 + WF_E1; }
		else if (state == 3) { MGB_CIG_PUSH(1, 1); --i, s -= ext? WF_E2 : WF_O2 + WF_E2; }
		else if (state == 2) { MGB_CIG_PUSH(2, 1); --k, s -= ext? WF_E1 : WF_O1 + WF_E1; }
		else if (state == 4) { MGB_CIG_PUSH(2, 1); --k, s -= ext? WF_E2 : WF_O2 + WF_E2; }
		else return MGB_E_INTERNAL;
		last = state > 0 && ext? state : 0;
	}
	if (i >= 0) MGB_CIG_PUSH(1, i + 1);
	else if (k >= 0) MGB_CIG_PUSH(2, k + 1);
	if (cur_op >= 0) { if (w <= 0) return MGB_E_INTERNAL; cig_store[--w] = (uint32_t)cur_len << 4 | (uint32_t)cur_op; }
#undef MGB_CIG_PUSH
	*n_cigar = (int32_t)(max_cigar - w), *first = w;
	return 0;
}

// =================================================================================================================
// shared-memory scheme
// =================================================================================================================
// * H keeps 17 scores, E1/F1 keep 3, E2/F2 keep 2 (the deepest look-backs are o2+e2 = 16, e1 = 2, e2 = 1);
// * instead of padding every slice with -inf cells, reads are bounds-checked against the per-score [lo,hi]
//   (warp-uniform, the last 16 of them held in registers), which returns exactly what the reference's padding holds;
// * a new cell is extended along its exact matches right after it is computed (the reference extends the whole
//   wavefront at the top of the next iteration: same cells, same values, one pass over shared memory less);
// * diagonals map to columns modulo W, so any window of at most W diagonals fits;
// * both sequences are staged in shared memory; with TBCAP > 0 the traceback bytes live there too.
// The scheme gives up (returns 1, nothing written) when the window would exceed W diagonals, the traceback bytes
// would exceed TBCAP, or the score reaches 255 -- the reference re-centres its band every 256 scores by inspecting
// all 17 E/F slices (wf_stripe_shrink), which only wfa_exact() keeps -- and the job moves to the next tier.

// HS = number of H slices kept in shared memory (17 = all).  With HS = 7 the slices older than 6 scores -- only read
// once more, as H[s-16] -- live in a ring in the worker arena (coalesced global loads), which halves the footprint.
// Cells are 16-bit: a valid offset is in [-1, MAXLEN], an invalid one is the sentinel plus the at most 255 increments the
// recurrence can add, so every comparison and maximum orders the cells exactly as the reference's 32-bit ones do.
typedef int16_t wf_cell_t;
static const int32_t WF_NEG_INF16 = -30000;

template<int W, int MAXLEN, int TBCAP, int HS = 17>
struct WfSmemLayout {
	static const int W_ = W, MAXLEN_ = MAXLEN, TBCAP_ = TBCAP, HS_ = HS;
	static const int N_CELLS = (HS + 3 + 3 + 2 + 2) * W;
	static const int N_INTS = N_CELLS / 2;
	static const int SEQ_BYTES = (MAXLEN + WF_SEQ_PAD + 3) / 4 * 4;
	static const int TB_ROW_BYTES = TBCAP > 0? 256 * 8 : 0; // per score: int32 lo, int32 off
	static const int BYTES = N_INTS * 4 + 2 * SEQ_BYTES + TB_ROW_BYTES + TBCAP;
	static const int STRIDE = (BYTES + 127) / 128 * 128;
};

template<int W>
MG_HD inline int32_t wfs_col(int32_t d) { return (d + (1 << 20)) & (W - 1); }

struct WfTbRow { int32_t lo, hi; uint8_t *x; };
struct WfTbArena { // traceback rows bump-allocated in the worker arena (reference: miniwfa.c:31-44 wf_tb_add)
	const WfTbRow *row;
	MG_HD int32_t get(int32_t s, int32_t d) const
	{
		int32_t j = d - row[s].lo;
		return (j < 0 || j > row[s].hi - row[s].lo)? -1 : (int32_t)row[s].x[j];
	}
};

// A gap whose wavefronts are done and whose traceback waits for the other gaps of its batch.  Its rows, its CIGAR store and a
// stitched target stay in the worker arena until then; the read and the graph sequences are read where they live in global memory
// (the staged copies in shared memory belong to the next gap by then).
struct WfTbJob {
	const WfTbRow *rows;      // 0: nothing to trace back, the CIGAR is cig[0 .. n_cigar) already
	const char *ts, *qs;
	uint32_t *cig;            // tl + ql + 2 entries, written from the back by the traceback
	int64_t n_iter, first;    // first: where the CIGAR starts in cig
	int64_t job;              // the caller's: which job this is
	int32_t n_rows, last_state, tl, ql, s, item, rc, n_cigar;
};

MG_HD inline void wfa_tb_keep(WfTbJob *b, const WfResult &r, int32_t tl, const char *ts, int32_t ql, const char *qs, int64_t job, int lane)
{
	if (lane == 0) {
		b->rows = r.rows, b->ts = ts, b->qs = qs, b->cig = r.cigar, b->n_iter = r.n_iter, b->first = 0, b->job = job;
		b->n_rows = r.n_rows, b->last_state = r.last_state, b->tl = tl, b->ql = ql, b->s = r.s, b->item = 0, b->rc = 0, b->n_cigar = r.n_cigar;
	}
}

// The tracebacks of a batch of n <= MGB_W gaps, lane j on gap j; rc, n_cigar and first of every record are set on return.
// Warp-uniform.
MG_HD inline void wfa_tb_batch(WfTbJob *rec, int32_t n, int lane)
{
	warp_sync(); // the records are complete
	for (int32_t j = lane; j < n; j += MGB_W) {
		WfTbJob &b = rec[j];
		if (b.rows == 0) continue;
		WfTbArena t;
		t.row = b.rows;
		int32_t n_cig = 0;
		int64_t first = 0;
		b.rc = wf_traceback(t, b.n_rows, b.tl, b.ts, b.ql, b.qs, b.last_state, b.cig, (int64_t)b.tl + b.ql + 2, &n_cig, &first);
		b.n_cigar = n_cig, b.first = first;
	}
	warp_sync();
}


// =================================================================================================================
// general scheme: ring in the worker arena, mirrors the reference's memory layout
// =================================================================================================================
// The last max_pen+1 = 17 wavefronts live in fixed slots of the arena, five int32 lanes each (H,E1,F1,E2,F2) padded
// by 17 cells of -inf on both sides.  `nl` is the number of cooperating lanes: 32 when a whole warp enters, 1 when a
// single lane runs the function (the chaining fallback below is sequential).

#define MGB_NL_SYNC(nl) do { if ((nl) > 1) warp_sync(); } while (0)

struct WfSlice {
	int32_t lo, hi;
	int32_t *H, *E1, *F1, *E2, *F2; // indexable by diagonal d in [lo-PAD, hi+PAD]
};

struct WfState {
	WfSlice sl[WF_NSLICE];
	int32_t *mem;        // WF_NSLICE slots
	int64_t slot_stride; // int32 elements per slot
	int64_t lane_stride; // int32 elements per lane inside a slot
	int32_t s, top, lo, hi;
};

MG_HD inline int wf_state_alloc(Arena &A, WfState &wf, int32_t tl, int32_t ql)
{
	int64_t maxw = (int64_t)tl + ql + 1;
	wf.lane_stride = maxw + 2 * WF_PAD;
	wf.slot_stride = 5 * wf.lane_stride;
	MGB_ALLOC(A, wf.mem, int32_t, wf.slot_stride * WF_NSLICE);
	return 0;
}

MG_HD inline void wf_slice_bind(WfState &wf, int slot, int32_t lo, int32_t hi, int lane, int nl)
{
	WfSlice &f = wf.sl[slot];
	int32_t n = hi - lo + 1;
	int32_t *base = wf.mem + (int64_t)slot * wf.slot_stride;
	f.lo = lo, f.hi = hi;
	f.H = base + WF_PAD;
	f.E1 = f.H + wf.lane_stride;
	f.F1 = f.E1 + wf.lane_stride;
	f.E2 = f.F1 + wf.lane_stride;
	f.F2 = f.E2 + wf.lane_stride;
	for (int32_t i = -WF_PAD + lane; i < 0; i += nl) f.H[i] = f.E1[i] = f.E2[i] = f.F1[i] = f.F2[i] = WF_NEG_INF;
	for (int32_t i = n + lane; i < n + WF_PAD; i += nl) f.H[i] = f.E1[i] = f.E2[i] = f.F1[i] = f.F2[i] = WF_NEG_INF;
	f.H -= lo, f.E1 -= lo, f.E2 -= lo, f.F1 -= lo, f.F2 -= lo;
}

// reference: miniwfa.c:80-101 wf_stripe_add
MG_HD inline WfSlice &wf_stripe_add(WfState &wf, int32_t lo, int32_t hi, int lane, int nl)
{
	++wf.s;
	++wf.top;
	if (wf.top == WF_NSLICE) wf.top = 0;
	wf_slice_bind(wf, wf.top, lo, hi, lane, nl);
	return wf.sl[wf.top];
}

// reference: miniwfa.c:103-121 wf_stripe_init
MG_HD inline void wf_stripe_init(WfState &wf, int lane, int nl)
{
	wf.s = 0, wf.top = 0, wf.lo = wf.hi = 0;
	for (int i = 0; i < WF_NSLICE; ++i) {
		WfSlice &f = wf_stripe_add(wf, 0, 0, lane, nl);
		if (lane == 0) f.H[0] = f.E1[0] = f.E2[0] = f.F1[0] = f.F2[0] = WF_NEG_INF;
	}
	wf.s = 0;
	if (lane == 0) wf.sl[wf.top].H[0] = -1;
	MGB_NL_SYNC(nl);
}

MG_HD inline const WfSlice &wf_stripe_get(const WfState &wf, int32_t x)
{
	int32_t y = wf.top - x;
	if (y < 0) y += WF_NSLICE;
	return wf.sl[y];
}

MG_HD inline int wf_good_diag(int32_t d, int32_t k, int32_t tl, int32_t ql)
{
	return ((k >= -1 && k < tl) && (d + k >= -1 && d + k < ql));
}

// narrow [lo,hi] to diagonals that still hold a cell inside the DP matrix (reference: miniwfa.c:144-171)
MG_HD inline int wf_stripe_shrink(WfState &wf, int32_t tl, int32_t ql)
{
	int32_t j, d;
	for (d = wf.lo; d <= wf.hi; ++d) {
		for (j = 0; j < WF_NSLICE; ++j) {
			const WfSlice *p = &wf.sl[(wf.top + 1 + j) % WF_NSLICE];
			if (d < p->lo || d > p->hi) continue;
			if (wf_good_diag(d, p->H[d], tl, ql)) break;
			if (wf_good_diag(d, p->E1[d], tl, ql) || wf_good_diag(d, p->F1[d], tl, ql)) break;
			if (wf_good_diag(d, p->E2[d], tl, ql) || wf_good_diag(d, p->F2[d], tl, ql)) break;
		}
		if (j < WF_NSLICE) break;
	}
	if (d > wf.hi) return MGB_E_INTERNAL;
	wf.lo = d;
	for (d = wf.hi; d >= wf.lo; --d) {
		for (j = 0; j < WF_NSLICE; ++j) {
			const WfSlice *p = &wf.sl[(wf.top + 1 + j) % WF_NSLICE];
			if (d < p->lo || d > p->hi) continue;
			if (wf_good_diag(d, p->H[d], tl, ql)) break;
			if (wf_good_diag(d, p->E1[d], tl, ql) || wf_good_diag(d, p->F1[d], tl, ql)) break;
			if (wf_good_diag(d, p->E2[d], tl, ql) || wf_good_diag(d, p->F2[d], tl, ql)) break;
		}
		if (j < WF_NSLICE) break;
	}
	if (d < wf.lo) return MGB_E_INTERNAL;
	wf.hi = d;
	return 0;
}

// one cell of the recurrence with its traceback byte (reference: miniwfa.c:281-308 wf_next_tb)
MG_HD inline uint8_t wf_cell(int32_t d, int32_t *H, int32_t *E1, int32_t *F1, int32_t *E2, int32_t *F2,
							 const int32_t *pHx, const int32_t *pHo1, const int32_t *pHo2,
							 const int32_t *pE1, const int32_t *pF1, const int32_t *pE2, const int32_t *pF2)
{
	int32_t h, f, e, e1, e2, f1, f2;
	uint8_t x = 0, ze, zf, z;
	x |= pHo1[d-1] >= pE1[d-1]? 0 : 0x08;
	e1 = MGB_WF_MAX(pHo1[d-1], pE1[d-1]);
	x |= pHo2[d-1] >= pE2[d-1]? 0 : 0x20;
	e2 = MGB_WF_MAX(pHo2[d-1], pE2[d-1]);
	ze = e1 >= e2? 1 : 3;
	e = MGB_WF_MAX(e1, e2);
	x |= pHo1[d+1] >= pF1[d+1]? 0 : 0x10;
	f1 = MGB_WF_MAX(pHo1[d+1], pF1[d+1]) + 1;
	x |= pHo2[d+1] >= pF2[d+1]? 0 : 0x40;
	f2 = MGB_WF_MAX(pHo2[d+1], pF2[d+1]) + 1;
	zf = f1 >= f2? 2 : 4;
	f = MGB_WF_MAX(f1, f2);
	z = e >= f? ze : zf;
	h = MGB_WF_MAX(e, f);
	z = pHx[d] + 1 >= h? 0 : z;
	E1[d] = e1, E2[d] = e2, F1[d] = f1, F2[d] = f2;
	H[d] = MGB_WF_MAX(pHx[d] + 1, h);
	return x | z;
}

struct WfChkpt { int32_t s, d; }; // reference: miniwfa.c:173-175 wf_chkpt_t

// Exact WFA with traceback for any size (reference: miniwfa.c:380-435 mwf_wfa_core).  ts/qs are STAGED copies
// (4-byte aligned, sentinel padded).  seg (may be null): checkpoints that pin the wavefront to one diagonal at given
// scores (low-memory mode).  max_iter <= 0: unbounded.
MG_HD inline int wfa_core(Arena &A, int32_t tl, const char *ts, int32_t ql, const char *qs, int64_t max_iter, int32_t n_seg, const WfChkpt *seg,
						  WfResult *r, uint32_t *cig_store, int64_t max_cigar, int lane, int nl)
{
	uint64_t mark = A.top;
	WfState wf;
	int32_t last_state = 0, stopped = 0, sid = 0;
	MGB_TRY(wf_state_alloc(A, wf, tl, ql));
	AVec<WfTbRow> rows;
	avec_init(rows);
	if (nl > 1) MGB_TRY(avec_reserve_w(A, rows, 1024, lane));
	else MGB_TRY(avec_reserve(A, rows, 1024));
	wf_stripe_init(wf, lane, nl);
	for (;;) {
		WfSlice *p = &wf.sl[wf.top];
		int32_t lo, hi, *H = p->H;
		int hit = 0, hit_noext = 0;
		for (int32_t d = p->lo + lane; d <= p->hi; d += nl) { // extension along exact matches
			int32_t k0 = H[d];
			if (k0 < -1 || d + k0 < -1 || k0 >= tl || d + k0 >= ql) continue;
			int32_t k = wf_extend(ts, qs, k0, d);
			if (k == tl - 1 && d + k == ql - 1) { hit = 1, hit_noext = (k == k0); if (nl == 1) break; }
			else H[d] = k;
		}
		MGB_NL_SYNC(nl);
		if (nl > 1? warp_any(hit) : hit) {
			if (nl > 1? warp_any(hit && hit_noext) : hit_noext) {
				WfTbArena t; t.row = rows.a;
				last_state = t.get((int32_t)rows.n - 1, ql - tl) & 7;
			}
			break;
		}
		if (seg && sid < n_seg && seg[sid].s == wf.s) {
			if (!(seg[sid].d >= wf.lo && seg[sid].d <= wf.hi)) { A.top = mark; return MGB_E_INTERNAL; }
			wf.lo = wf.hi = seg[sid++].d;
		}
		lo = wf.lo > -tl? wf.lo - 1 : -tl;
		hi = wf.hi < ql? wf.hi + 1 : ql;
		{ // reference: miniwfa.c:313-327 wf_next_basic (traceback variant)
			const WfSlice &ft = wf_stripe_add(wf, lo, hi, lane, nl);
			const WfSlice &fx = wf_stripe_get(wf, WF_X);
			const WfSlice &fo1 = wf_stripe_get(wf, WF_O1 + WF_E1);
			const WfSlice &fo2 = wf_stripe_get(wf, WF_O2 + WF_E2);
			const WfSlice &fe1 = wf_stripe_get(wf, WF_E1);
			const WfSlice &fe2 = wf_stripe_get(wf, WF_E2);
			if (nl > 1) MGB_TRY(avec_reserve_w(A, rows, rows.n + 1, lane));
			else MGB_TRY(avec_reserve(A, rows, rows.n + 1));
			uint8_t *x;
			MGB_ALLOC(A, x, uint8_t, hi - lo + 1);
			if (lane == 0) rows.a[rows.n].lo = lo, rows.a[rows.n].hi = hi, rows.a[rows.n].x = x;
			++rows.n;
			uint8_t *ax = x - lo;
			for (int32_t dd = lo + lane; dd <= hi; dd += nl)
				ax[dd] = wf_cell(dd, ft.H, ft.E1, ft.F1, ft.E2, ft.F2, fx.H, fo1.H, fo2.H, fe1.E1, fe1.F1, fe2.E2, fe2.F2);
			MGB_NL_SYNC(nl);
			if (ft.H[lo] >= -1 || ft.E1[lo] >= -1 || ft.F1[lo] >= -1 || ft.E2[lo] >= -1 || ft.F2[lo] >= -1) wf.lo = lo;
			if (ft.H[hi] >= -1 || ft.E1[hi] >= -1 || ft.F1[hi] >= -1 || ft.E2[hi] >= -1 || ft.F2[hi] >= -1) wf.hi = hi;
		}
		if ((wf.s & 0xff) == 0) MGB_TRY(wf_stripe_shrink(wf, tl, ql));
		r->n_iter += hi - lo + 1;
		if (max_iter > 0 && r->n_iter > max_iter) { stopped = 1; break; }
	}
	r->s = stopped? -1 : wf.s;
	if (!stopped) {
		int rc = 0;
		int32_t n_cig = 0;
		int64_t first = 0;
		if (lane == 0) {
			WfTbArena t; t.row = rows.a;
			rc = wf_traceback(t, (int32_t)rows.n, tl, ts, ql, qs, last_state, cig_store, max_cigar, &n_cig, &first);
		}
		if (nl > 1) {
			rc = warp_bcast_i32(rc, 0), n_cig = warp_bcast_i32(n_cig, 0), first = (int64_t)warp_bcast_u64((uint64_t)first, 0);
			warp_sync();
		}
		if (rc < 0) { A.top = mark; return rc; }
		r->n_cigar = n_cig, r->cigar = cig_store + first;
	}
	A.top = mark;
	return 0;
}

// ---- low-memory mode (reference: miniwfa.c:437-601): find the checkpoints the optimal path passes through ----
// A second stripe `sf` carries, for every cell, the index of the cell of the previous snapshot it descends from.
// Sequential (one lane); only reached from the chaining fallback.

struct WfSnap { int32_t n, n_intv, max_s; int32_t *x; uint64_t *intv; };

MG_HD inline int wf_snapshot(Arena &A, AVec<WfSnap> &sss, WfState &sf) // reference: miniwfa.c:452-489
{
	WfSnap ss;
	int32_t j, k, t;
	ss.n = 0, ss.max_s = sf.s;
	for (j = 0; j < WF_NSLICE; ++j) ss.n += 5 * (sf.sl[j].hi - sf.sl[j].lo + 1);
	MGB_ALLOC(A, ss.x, int32_t, ss.n);
	ss.n_intv = WF_NSLICE;
	MGB_ALLOC(A, ss.intv, uint64_t, ss.n_intv);
	for (j = 0, t = 0; j < WF_NSLICE; ++j) {
		WfSlice *p = &sf.sl[(sf.top + 1 + j) % WF_NSLICE];
		ss.intv[j] = (uint64_t)(int64_t)p->lo << 32 | (uint64_t)(uint32_t)((p->hi - p->lo + 1) * 5);
		for (k = p->lo; k <= p->hi; ++k) {
			ss.x[t] = p->H[k],  p->H[k]  = t++;
			ss.x[t] = p->E1[k], p->E1[k] = t++;
			ss.x[t] = p->F1[k], p->F1[k] = t++;
			ss.x[t] = p->E2[k], p->E2[k] = t++;
			ss.x[t] = p->F2[k], p->F2[k] = t++;
		}
	}
	if (t != ss.n) return MGB_E_INTERNAL;
	return avec_push(A, sss, ss);
}

// checkpoints of the optimal alignment, one per snapshot (reference: miniwfa.c:551-601 mwf_wfa_seg); seg is allocated at
// the caller's mark
MG_HD inline int wfa_seg(Arena &A, int32_t step, int32_t tl, const char *ts, int32_t ql, const char *qs, WfChkpt **seg_, int32_t *n_seg_)
{
	uint64_t mark = A.top;
	WfState wf, sf;
	AVec<WfSnap> sss;
	uint8_t *xbuf;
	int32_t last = -1;
	avec_init(sss);
	*seg_ = 0, *n_seg_ = 0;
	MGB_ALLOC(A, xbuf, uint8_t, (int64_t)tl + ql + 1);
	MGB_TRY(wf_state_alloc(A, wf, tl, ql));
	MGB_TRY(wf_state_alloc(A, sf, tl, ql));
	wf_stripe_init(wf, 0, 1);
	wf_stripe_init(sf, 0, 1);
	for (;;) {
		WfSlice *p = &wf.sl[wf.top];
		int32_t d, lo, hi, *H = p->H;
		for (d = p->lo; d <= p->hi; ++d) {
			int32_t k0 = H[d];
			if (k0 < -1 || d + k0 < -1 || k0 >= tl || d + k0 >= ql) continue;
			int32_t k = wf_extend(ts, qs, k0, d);
			if (k == tl - 1 && d + k == ql - 1) { last = sf.sl[sf.top].H[d]; break; }
			H[d] = k;
		}
		if (d <= p->hi) break;
		lo = wf.lo > -tl? wf.lo - 1 : -tl;
		hi = wf.hi < ql? wf.hi + 1 : ql;
		if ((wf.s + 1) % step == 0) MGB_TRY(wf_snapshot(A, sss, sf));
		{ // reference: miniwfa.c:491-530 wf_next_seg
			uint8_t *ax = xbuf - lo;
			{
				const WfSlice &ft = wf_stripe_add(wf, lo, hi, 0, 1);
				const WfSlice &fx = wf_stripe_get(wf, WF_X), &fo1 = wf_stripe_get(wf, WF_O1 + WF_E1), &fo2 = wf_stripe_get(wf, WF_O2 + WF_E2);
				const WfSlice &fe1 = wf_stripe_get(wf, WF_E1), &fe2 = wf_stripe_get(wf, WF_E2);
				for (int32_t dd = lo; dd <= hi; ++dd)
					ax[dd] = wf_cell(dd, ft.H, ft.E1, ft.F1, ft.E2, ft.F2, fx.H, fo1.H, fo2.H, fe1.E1, fe1.F1, fe2.E2, fe2.F2);
			}
			const WfSlice &gt = wf_stripe_add(sf, lo, hi, 0, 1);
			const WfSlice &gx = wf_stripe_get(sf, WF_X), &go1 = wf_stripe_get(sf, WF_O1 + WF_E1), &go2 = wf_stripe_get(sf, WF_O2 + WF_E2);
			const WfSlice &ge1 = wf_stripe_get(sf, WF_E1), &ge2 = wf_stripe_get(sf, WF_E2);
			for (int32_t dd = lo; dd <= hi; ++dd) {
				uint8_t x = ax[dd];
				int32_t e1, f1, e2, f2, h;
				e1 = gt.E1[dd] = (x & 0x08) == 0? go1.H[dd-1] : ge1.E1[dd-1];
				f1 = gt.F1[dd] = (x & 0x10) == 0? go1.H[dd+1] : ge1.F1[dd+1];
				e2 = gt.E2[dd] = (x & 0x20) == 0? go2.H[dd-1] : ge2.E2[dd-1];
				f2 = gt.F2[dd] = (x & 0x40) == 0? go2.H[dd+1] : ge2.F2[dd+1];
				x &= 7;
				h = gx.H[dd];
				h = x == 1? e1 : h;
				h = x == 2? f1 : h;
				h = x == 3? e2 : h;
				h = x == 4? f2 : h;
				gt.H[dd] = h;
			}
			// NB: the reference tests the *snapshot* stripe here (its H..F2 variables were rebound), kept as is
			if (gt.H[lo] >= -1 || gt.E1[lo] >= -1 || gt.F1[lo] >= -1 || gt.E2[lo] >= -1 || gt.F2[lo] >= -1) wf.lo = lo;
			if (gt.H[hi] >= -1 || gt.E1[hi] >= -1 || gt.F1[hi] >= -1 || gt.E2[hi] >= -1 || gt.F2[hi] >= -1) wf.hi = hi;
		}
		if ((wf.s & 0xff) == 0) MGB_TRY(wf_stripe_shrink(wf, tl, ql));
	}
	// reference: miniwfa.c:532-549 wf_traceback_seg
	const int32_t n_seg = (int32_t)sss.n;
	WfChkpt *tmp;
	MGB_ALLOC(A, tmp, WfChkpt, n_seg);
	for (int32_t j = n_seg - 1; j >= 0; --j) {
		const WfSnap *p = &sss.a[j];
		int32_t k, m;
		for (k = 0, m = 0; k < p->n_intv; ++k) {
			if (last >= m && last < m + (int32_t)p->intv[k]) break;
			m += (int32_t)p->intv[k];
		}
		if (k >= p->n_intv) { A.top = mark; return MGB_E_INTERNAL; }
		tmp[j].s = p->max_s - (p->n_intv - k - 1);
		tmp[j].d = (int32_t)(p->intv[k] >> 32) + (last - m) / 5;
		last = p->x[last];
	}
	if (last != -1) { A.top = mark; return MGB_E_INTERNAL; }
	WfChkpt *seg = (WfChkpt*)(A.base + mark);
	for (int32_t j = 0; j < n_seg; ++j) { WfChkpt x = tmp[j]; seg[j] = x; } // destination lies below the source
	A.top = mark + (((uint64_t)n_seg * sizeof(WfChkpt) + 15) & ~(uint64_t)15);
	if (A.top > A.peak) A.peak = A.top;
	*seg_ = seg, *n_seg_ = n_seg;
	return 0;
}

// exact alignment of raw (unstaged) sequences; step > 0 selects the low-memory mode (reference: miniwfa.c:603-615)
MG_HD inline int wfa_exact_seq(Arena &A, int32_t step, int32_t tl, const char *ts_g, int32_t ql, const char *qs_g, int64_t max_iter, WfResult *r,
							   uint32_t *cig_store, int64_t max_cigar)
{
	uint64_t mark = A.top;
	char *ts, *qs;
	WfChkpt *seg = 0;
	int32_t n_seg = 0;
	MGB_ALLOC(A, ts, char, tl + WF_SEQ_PAD + 4);
	MGB_ALLOC(A, qs, char, ql + WF_SEQ_PAD + 4);
	wf_stage_seq(ts, ts_g, tl, 0xfe, 0);
	wf_stage_seq(qs, qs_g, ql, 0xff, 0);
	for (int32_t i = 1; i < MGB_W; ++i) { wf_stage_seq(ts, ts_g, tl, 0xfe, i); wf_stage_seq(qs, qs_g, ql, 0xff, i); } // single lane covers all strides
	if (step > 0) MGB_TRY(wfa_seg(A, step, tl, ts, ql, qs, &seg, &n_seg));
	r->s = -1, r->n_cigar = 0, r->n_iter = 0, r->cigar = 0;
	MGB_TRY(wfa_core(A, tl, ts, ql, qs, max_iter, n_seg, seg, r, cig_store, max_cigar, 0, 1));
	A.top = mark;
	return 0;
}

// ---- chaining heuristic for gaps whose exact alignment exceeds the iteration cap (reference: miniwfa.c:617-822) ----

// longest strictly increasing subsequence (reference: miniwfa.c:620-639 mg_lis_64); b receives the indices
MG_HD inline int wf_lis_64(Arena &A, int32_t n, const uint64_t *a, int32_t *b, int32_t *L_)
{
	uint64_t mark = A.top;
	int32_t i, k, L = 0, *M, *P = b;
	MGB_ALLOC(A, M, int32_t, n + 1);
	for (i = 0; i < n; ++i) {
		int32_t lo = 1, hi = L, newL;
		while (lo <= hi) {
			int32_t mid = (lo + hi + 1) >> 1;
			if (a[M[mid]] < a[i]) lo = mid + 1;
			else hi = mid - 1;
		}
		newL = lo, P[i] = M[newL - 1], M[newL] = i;
		if (newL > L) L = newL;
	}
	if (n > 0) {
		k = M[L];
		for (i = 0; i < n; ++i) M[i] = P[i];
		for (i = L - 1; i >= 0; --i) b[i] = k, k = M[k];
	}
	A.top = mark;
	*L_ = L;
	return 0;
}

MG_HD inline int32_t wf_fc_kmer(int32_t len, const char *seq, int32_t rid, int32_t k, uint64_t *a) // reference: miniwfa.c:644-656
{
	int32_t i, l, n;
	uint64_t x, mask = (1ULL << k * 2) - 1;
	for (i = l = 0, x = 0, n = 0; i < len; ++i) {
		int32_t c = nt4((uint8_t)seq[i]);
		if (c < 4) {
			x = (x << 2 | (uint64_t)c) & mask;
			if (++l >= k) a[n++] = (x << 1 | (uint64_t)rid) << 32 | (uint64_t)(uint32_t)i;
		} else l = 0, x = 0;
	}
	return n;
}

// co-linear k-mer matches (reference: miniwfa.c:658-710 mg_chain); result (pos1<<32|pos2) allocated at the caller's mark
MG_HD inline int wf_kmer_chain(Arena &A, int32_t l1, const char *s1, int32_t l2, const char *s2, int32_t k, int32_t max_occ, uint64_t **out_, int32_t *n_out_)
{
	uint64_t mark = A.top;
	*out_ = 0, *n_out_ = 0;
	if (l1 < k || l2 < k) return 0;
	uint64_t *a;
	MGB_ALLOC(A, a, uint64_t, (int64_t)l1 + l2);
	int32_t n_a = wf_fc_kmer(l1, s1, 0, k, a);
	n_a += wf_fc_kmer(l2, s2, 1, k, &a[n_a]);
	MGB_TRY(radix_sort_64(A, a, n_a));
	AVec<uint64_t> b;
	avec_init(b);
	for (int32_t i0 = 0, i = 1; i <= n_a; ++i) {
		if (i == n_a || a[i0] >> 33 != a[i] >> 33) {
			if (i - i0 >= 2) {
				int32_t j, s, t;
				for (j = i0; j < i && (a[j] >> 32 & 1) == 0; ++j) {}
				if (j > i0 && j < i && j - i0 <= max_occ && i - j <= max_occ)
					for (s = i0; s < j; ++s)
						for (t = j; t < i; ++t) {
							uint64_t v = a[s] << 32 | (uint64_t)(uint32_t)a[t];
							MGB_TRY(avec_push(A, b, v));
						}
			}
			i0 = i;
		}
	}
	int32_t n_b = (int32_t)b.n;
	MGB_TRY(radix_sort_64(A, b.a, n_b));
	for (int32_t i = 0; i < n_b; ++i) b.a[i] = b.a[i] >> 32 | b.a[i] << 32;
	int32_t *lis, n_lis;
	MGB_ALLOC(A, lis, int32_t, n_b);
	MGB_TRY(wf_lis_64(A, n_b, b.a, lis, &n_lis));
	uint64_t *tmp;
	MGB_ALLOC(A, tmp, uint64_t, n_lis);
	for (int32_t i = 0; i < n_lis; ++i) { uint64_t v = b.a[lis[i]]; tmp[i] = v >> 32 | v << 32; }
	uint64_t *out = (uint64_t*)(A.base + mark);
	for (int32_t i = 0; i < n_lis; ++i) { uint64_t v = tmp[i]; out[i] = v; }
	A.top = mark + (((uint64_t)n_lis * 8 + 15) & ~(uint64_t)15);
	if (A.top > A.peak) A.peak = A.top;
	*out_ = out, *n_out_ = n_lis;
	return 0;
}

MG_HD inline int wf_ksim(Arena &A, int32_t l1, const char *s1, int32_t l2, const char *s2, int32_t k, double *sim) // reference: miniwfa.c:712-738
{
	uint64_t mark = A.top;
	int32_t i, i0, j, n_a, n1 = 0, n2 = 0, t1 = 0, t2 = 0;
	*sim = 0;
	if (l1 < k || l2 < k) return 0;
	uint64_t *a;
	MGB_ALLOC(A, a, uint64_t, (int64_t)l1 + l2);
	n_a = wf_fc_kmer(l1, s1, 0, k, a);
	n_a += wf_fc_kmer(l2, s2, 1, k, &a[n_a]);
	MGB_TRY(radix_sort_64(A, a, n_a));
	for (i0 = 0, i = 1; i <= n_a; ++i) {
		if (i == n_a || a[i0] >> 33 != a[i] >> 33) {
			int32_t m1, m2, mn;
			for (j = i0; j < i && (a[j] >> 32 & 1) == 0; ++j) {}
			m1 = j - i0, m2 = i - j;
			mn = m1 < m2? m1 : m2;
			n1 += m1, n2 += m2;
			if (m1 > 0 && m2 > 0) t1 += mn, t2 += mn;
			i0 = i;
		}
	}
	A.top = mark;
	double p1 = (double)t1 / n1, p2 = (double)t2 / n2;
	*sim = p1 > p2? p1 : p2;
	return 0;
}

MG_HD inline int32_t wf_anchor_filter(int32_t n, uint64_t *a, int32_t tl, int32_t ql, int32_t k, int32_t min_l) // reference: miniwfa.c:755-774
{
	int32_t i, st, x0, y0, x1, y1, j, l, m;
	for (i = 0, x0 = y0 = x1 = y1 = 0, st = -1, l = 0; i <= n; ++i) {
		int32_t x, y;
		if (i == n) x = tl, y = ql;
		else x = (int32_t)(a[i] >> 32) + 1, y = (int32_t)a[i] + 1;
		if (x - x0 != y - y0) {
			if (l < min_l)
				for (j = st > 0? st : 0; j < i; ++j) a[j] = 0;
			x0 = x, y0 = y, st = i, l = k;
		} else l += x - x1;
		x1 = x, y1 = y;
	}
	for (i = 0, m = 0; i < n; ++i)
		if (a[i] != 0) a[m++] = a[i];
	return m;
}

MG_HD inline int wf_cig_push1(uint32_t *c, int64_t *n, int64_t cap, int32_t op, int32_t len)
{
	if (*n && (uint32_t)op == (c[*n - 1] & 0xf)) c[*n - 1] += (uint32_t)len << 4;
	else { if (*n >= cap) return MGB_E_INTERNAL; c[(*n)++] = (uint32_t)len << 4 | (uint32_t)op; }
	return 0;
}

// reference: miniwfa.c:776-822 mwf_wfa_chain with opt.step = 5000, opt.max_iter = -1 (as set by mwf_wfa_auto :824-834).
// Sequential (one lane).  The CIGAR is written to cig_store[0..n).
MG_HD inline int wfa_chain(Arena &A, int32_t tl, const char *ts, int32_t ql, const char *qs, WfResult *r, uint32_t *cig_store, int64_t max_cigar, int32_t step)
{
	const int32_t kmer = 13, max_occ = 2, min_len = 30;
	uint64_t mark = A.top;
	uint64_t *a;
	int32_t n_a, i, x0, y0;
	int64_t nc = 0;
	MGB_TRY(wf_kmer_chain(A, tl, ts, ql, qs, kmer, max_occ, &a, &n_a));
	n_a = wf_anchor_filter(n_a, a, tl, ql, kmer, min_len);
	r->s = 0, r->n_iter = 0;
	for (i = 0, x0 = y0 = 0; i <= n_a; ++i) {
		int32_t x1, y1;
		if (i == n_a) x1 = tl, y1 = ql;
		else x1 = (int32_t)(a[i] >> 32) + 1, y1 = (int32_t)a[i] + 1;
		if (i < n_a && x1 - x0 == y1 - y0 && x1 - x0 <= kmer) {
			MGB_TRY(wf_cig_push1(cig_store, &nc, max_cigar, 7, x1 - x0));
		} else if (x0 < x1 && y0 < y1) {
			double sim = 1.0;
			if (x1 - x0 >= 10000 && y1 - y0 >= 10000) MGB_TRY(wf_ksim(A, x1 - x0, &ts[x0], y1 - y0, &qs[y0], kmer, &sim));
			if (x1 - x0 >= 10000 && y1 - y0 >= 10000 && sim < 0.02) {
				MGB_TRY(wf_cig_push1(cig_store, &nc, max_cigar, 2, x1 - x0));
				MGB_TRY(wf_cig_push1(cig_store, &nc, max_cigar, 1, y1 - y0));
				r->s += WF_O2 * 2 + WF_E2 * ((x1 - x0) + (y1 - y0));
			} else {
				uint64_t m2 = A.top;
				WfResult q;
				uint32_t *cs;
				const int64_t mc = (int64_t)(x1 - x0) + (y1 - y0) + 2;
				MGB_ALLOC(A, cs, uint32_t, mc);
				MGB_TRY(wfa_exact_seq(A, step, x1 - x0, &ts[x0], y1 - y0, &qs[y0], -1, &q, cs, mc));
				if (q.n_cigar > 0) { // reference: miniwfa.c:742-753 wf_cigar_push
					MGB_TRY(wf_cig_push1(cig_store, &nc, max_cigar, (int32_t)(q.cigar[0] & 0xf), (int32_t)(q.cigar[0] >> 4)));
					if (nc + q.n_cigar - 1 > max_cigar) return MGB_E_INTERNAL;
					for (int32_t t = 1; t < q.n_cigar; ++t) cig_store[nc++] = q.cigar[t];
				}
				r->s += q.s;
				A.top = m2;
			}
		} else if (x0 < x1) {
			MGB_TRY(wf_cig_push1(cig_store, &nc, max_cigar, 2, x1 - x0));
			r->s += WF_O2 + (x1 - x0) * WF_E2 < WF_O1 + (x1 - x0) * WF_E1? WF_O2 + (x1 - x0) * WF_E2 : WF_O1 + (x1 - x0) * WF_E1;
		} else if (y0 < y1) {
			MGB_TRY(wf_cig_push1(cig_store, &nc, max_cigar, 1, y1 - y0));
			r->s += WF_O2 + (y1 - y0) * WF_E2 < WF_O1 + (y1 - y0) * WF_E1? WF_O2 + (y1 - y0) * WF_E2 : WF_O1 + (y1 - y0) * WF_E1;
		}
		x0 = x1, y0 = y1;
	}
	A.top = mark;
	r->n_cigar = (int32_t)nc, r->cigar = cig_store;
	return 0;
}

// =================================================================================================================
// compact ring in the worker arena (tier 3 on the device)
// =================================================================================================================
// The scheme of wfa_smem() without its limits: 16-bit cells, diagonals mapped to columns modulo W (a power of two covering
// every diagonal of the matrix), the ring in the arena, and all five arrays keeping 17 scores so that the band can be
// re-centred every 256 scores exactly as the reference does (miniwfa.c:144-171 inspects all of them).  Against the layout
// that mirrors the reference (wfa_core: 32-bit cells, every slice padded) it halves the bytes a cell moves.
// 16 bits are enough while tl + ql <= 16000: the score never exceeds o2 + e2*tl + o2 + e2*ql <= tl + ql + 30, so an
// invalid cell (sentinel plus at most one increment per score) stays far below -1 and orders like the 32-bit one.
// Returns 1 when it does not apply (the caller then uses wfa_core), 0 otherwise; r->s = -1 when max_iter cells were exceeded.

// Tier 3 entry (reference: miniwfa.c:824-834 mwf_wfa_auto): exact alignment capped at max_iter cells by the whole warp;
// beyond the cap the chaining heuristic takes over on lane 0.
MG_HD inline int wfa_ring_g(Arena &A, int32_t tl, const char *ts, int32_t ql, const char *qs, int64_t max_iter, WfResult *r, int lane); // mgb_wfa_tiers.cuh
// the two rare continuations of tier 3, out of line: they are most of the kernel's code and would set its register count
MG_HD MG_NOINLINE inline int wfa_core_cold(Arena &A, int32_t tl, const char *ts, int32_t ql, const char *qs, int64_t max_iter, WfResult *r, uint32_t *cig_store, int64_t max_cigar, int lane)
{
	return wfa_core(A, tl, ts, ql, qs, max_iter, 0, 0, r, cig_store, max_cigar, lane, MGB_W);
}
MG_HD MG_NOINLINE inline int wfa_chain_cold(Arena &A, int32_t tl, const char *ts_g, int32_t ql, const char *qs_g, WfResult *r, uint32_t *cig_store, int64_t max_cigar, int32_t step)
{
	return wfa_chain(A, tl, ts_g, ql, qs_g, r, cig_store, max_cigar, step);
}

// With the 16-bit ring the traceback is left to the caller (WfResult::rows); the 32-bit ring and the chaining heuristic, both rare,
// trace back on their own (the heuristic piece by piece) and return the CIGAR.
MG_HD inline int wfa_exact(Arena &A, int32_t tl, const char *ts_g, int32_t ql, const char *qs_g, int64_t max_iter, WfResult *r, int lane, int32_t step = 5000)
{
	uint64_t mark = A.top;
	r->s = -1, r->n_cigar = 0, r->n_iter = 0, r->cigar = 0, r->rows = 0, r->n_rows = 0, r->last_state = 0;
	uint32_t *cig_store;
	const int64_t max_cigar = (int64_t)tl + ql + 2;
	MGB_ALLOC(A, cig_store, uint32_t, max_cigar);
	uint64_t mark_keep = A.top;
	char *ts, *qs;
	MGB_ALLOC(A, ts, char, tl + WF_SEQ_PAD + 4);
	MGB_ALLOC(A, qs, char, ql + WF_SEQ_PAD + 4);
	wf_stage_seq(ts, ts_g, tl, 0xfe, lane);
	wf_stage_seq(qs, qs_g, ql, 0xff, lane);
	warp_sync();
	{
		int rc = wfa_ring_g(A, tl, ts, ql, qs, max_iter, r, lane);
		if (rc < 0) return rc;
		if (rc == 0 && r->s >= 0) { r->cigar = cig_store; return 0; } // the rows stay above mark_keep
		if (rc == 1) { // (through a copy: an arena header whose address is taken would live in local memory for the whole kernel)
			Arena B = A;
			rc = wfa_core_cold(B, tl, ts, ql, qs, max_iter, r, cig_store, max_cigar, lane);
			A.top = B.top, A.peak = B.peak;
			if (rc < 0) return rc;
		}
	}
	if (r->s < 0) { // iteration cap hit
		int rc = 0;
		int32_t n_cig = 0, sc = 0;
		if (lane == 0) {
			Arena B = A;
			rc = wfa_chain_cold(B, tl, ts_g, ql, qs_g, r, cig_store, max_cigar, step);
			n_cig = r->n_cigar, sc = r->s;
			if (B.peak > A.peak) A.peak = B.peak;
		}
		rc = warp_bcast_i32(rc, 0), n_cig = warp_bcast_i32(n_cig, 0), sc = warp_bcast_i32(sc, 0);
		warp_sync();
		if (rc < 0) { A.top = mark; return rc; }
		r->s = sc, r->n_cigar = n_cig, r->cigar = cig_store;
	}
	A.top = mark_keep;
	return 0;
}

// the tiers of the job kernels (K8a)
typedef WfSmemLayout<64, 256, 4096, 17> WfTier1;  // small gaps: 4 warps per block, traceback bytes in shared memory
typedef WfSmemLayout<256, 1024, 0, 17> WfTier2;   // mid-size gaps: 2 warps per block, traceback rows in the arena

} // namespace mgb
