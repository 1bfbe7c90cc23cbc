// mgb_wfa_tiers.cuh -- the gap alignment of the job kernels (K8a): wfa_smem() for tiers 1/2 (wavefront ring in shared memory) and
// wfa_ring_g() for tier 3 (ring in the worker arena).  Same recurrence and results as miniwfa.c:177-327; the layout is chosen so that
// a cell costs as few instructions as possible:
// * no bounds checks.  In tiers 1/2 the window never shrinks (lo only falls, hi only rises; the reference's band
//   re-centring needs score 256, which is tier 3), and a slot of the ring is reused by a later score, whose range contains
//   the old one.  So when all slices start filled with -inf, every cell outside the range a slice was last written with
//   still holds -inf: exactly what the reference's padding holds (miniwfa.c:182-209).  The nine neighbour reads are plain
//   shared-memory loads at columns (d-1, d, d+1) mod W.  The window may hold W - 2 diagonals (column lo-1 must not alias hi+1);
// * the four votes of a wavefront are one OR-reduction of four bits; the corner test runs on the one diagonal that can
//   reach the corner; the "does the window still grow" test runs on the two edge cells only.
// The layout compiles to about two thirds of the SASS instructions per 32 cells of the bounds-checked layout it replaced.
#pragma once
#include "mgb_wfa.cuh"

namespace mgb {

#if MGB_ON_DEVICE
MG_D inline uint32_t warp_or_u32(uint32_t x) { return __reduce_or_sync(0xffffffffu, x); }
#elif defined(MGB_SIM_LANES)
inline uint32_t warp_or_u32(uint32_t x) { uint64_t o[32]; sim::exchange(x, o, 15); uint32_t r = 0; for (int i = 0; i < MGB_W; ++i) r |= (uint32_t)o[i]; return r; }
#else
inline uint32_t warp_or_u32(uint32_t x) { return x; }
#endif

// keeps a value in a register: the compiler may not look through it (no code is generated)
#define MGB_OPAQUE(x) asm("" : "+r"(x))

// one cell as a 32-bit value (opaque, so that the arithmetic on it stays 32-bit: left alone, the compiler narrows the maxima to
// packed 16-bit operations and spends more on moving halves around than it saves)
MG_HD inline int32_t wf2_ld(const void *base, int32_t off)
{
	int32_t v = *(const wf_cell_t*)((const char*)base + off);
	MGB_OPAQUE(v);
	return v;
}

// ---- one cell of a wavefront, in two halves so that two cells can be in flight per lane ----
// LOAD: the nine neighbour reads and the recurrence (reference: miniwfa.c:281-308 wf_next_tb); FINISH: traceback byte, window
// votes, extension along exact matches (miniwfa.c:212-226) and the five stores.  The slots of score ns are not read while a
// wavefront is computed, so the FINISH of one cell may follow the LOAD of the next.  Expected in scope: H E1 F1 E2 F2 (arrays),
// bHx bHo1 bHo2 bE1 bE2 bnH bn3 bn2 (byte offsets of the slices), colmask2 (2W-1), ax, lo, hi, tl, ql, ts, qs, d_corner, vote.
// Tiers 1/2 (ring in shared memory) walk a wavefront one cell per lane at a time -- two cells in flight were slower, and so was a
// packed walk of two adjacent diagonals per lane (word loads, VIMNMX.S16x2 maxima whose predicates are the traceback bits; per pair
// it executes as many instructions as two cells, on half the lanes); tier 3 (ring in L2) keeps two cells in flight: eighteen loads
// before the first use, at 16 warps per SM (more warps cost registers and spills; more cells in flight did not help: the kernel
// is bound by what L2 delivers, not by the latency one warp sees).
#define MGB_WF_CELL_LOAD(S, d_) \
	int32_t h##S, e1##S, e2##S, f1##S, f2##S; \
	uint8_t xz##S; \
	const int32_t c##S = (((d_) + (1 << 20)) * 2) & colmask2; /* byte column */ \
	{ \
		const int32_t cm_ = (c##S - 2) & colmask2, cp_ = (c##S + 2) & colmask2; \
		int32_t a0_, b0_, e_, f_; \
		uint8_t x_ = 0, ze_, zf_, z_; \
		a0_ = wf2_ld(H, bHo1 + cm_), b0_ = wf2_ld(E1, bE1 + cm_); \
		x_ |= a0_ >= b0_? 0 : 0x08; e1##S = MGB_WF_MAX(a0_, b0_); \
		a0_ = wf2_ld(H, bHo2 + cm_), b0_ = wf2_ld(E2, bE2 + cm_); \
		x_ |= a0_ >= b0_? 0 : 0x20; e2##S = MGB_WF_MAX(a0_, b0_); \
		ze_ = e1##S >= e2##S? 1 : 3; \
		e_ = MGB_WF_MAX(e1##S, e2##S); \
		a0_ = wf2_ld(H, bHo1 + cp_), b0_ = wf2_ld(F1, bE1 + cp_); \
		x_ |= a0_ >= b0_? 0 : 0x10; f1##S = MGB_WF_MAX(a0_, b0_) + 1; \
		a0_ = wf2_ld(H, bHo2 + cp_), b0_ = wf2_ld(F2, bE2 + cp_); \
		x_ |= a0_ >= b0_? 0 : 0x40; f2##S = MGB_WF_MAX(a0_, b0_) + 1; \
		zf_ = f1##S >= f2##S? 2 : 4; \
		f_ = MGB_WF_MAX(f1##S, f2##S); \
		z_ = e_ >= f_? ze_ : zf_; \
		h##S = MGB_WF_MAX(e_, f_); \
		a0_ = wf2_ld(H, bHx + c##S) + 1; \
		z_ = a0_ >= h##S? 0 : z_; \
		h##S = MGB_WF_MAX(a0_, h##S); \
		xz##S = x_ | z_; \
	}
#define MGB_WF_CELL_FINISH(S, d_) \
	{ \
		const int32_t dd_ = (d_); \
		ax[dd_] = xz##S; \
		if (dd_ == lo || dd_ == hi) { /* does the window still grow on this side? */ \
			if (h##S >= -1 || e1##S >= -1 || f1##S >= -1 || e2##S >= -1 || f2##S >= -1) vote |= (dd_ == lo? 1u : 0u) | (dd_ == hi? 2u : 0u); \
		} \
		if (!(h##S < -1 || dd_ + h##S < -1 || h##S >= tl || dd_ + h##S >= ql)) { /* extend the new cell right away */ \
			const int32_t k_ = wf_extend(ts, qs, h##S, dd_); \
			if (dd_ == d_corner && k_ == tl - 1) vote |= 4u | (k_ == h##S? 8u : 0u); \
			else h##S = k_; \
		} \
		*(wf_cell_t*)((char*)E1 + bn3 + c##S) = (wf_cell_t)e1##S, *(wf_cell_t*)((char*)F1 + bn3 + c##S) = (wf_cell_t)f1##S; \
		*(wf_cell_t*)((char*)E2 + bn2 + c##S) = (wf_cell_t)e2##S, *(wf_cell_t*)((char*)F2 + bn2 + c##S) = (wf_cell_t)f2##S; \
		*(wf_cell_t*)((char*)H + bnH + c##S) = (wf_cell_t)h##S; \
	}

template<int W, int MAXLEN, int TBCAP>
MG_HD inline int wfa_smem(Arena &A, int32_t *smem, int32_t tl, const char *ts_g, int32_t ql, const char *qs_g, WfResult *r, int lane)
{
	typedef WfSmemLayout<W, MAXLEN, TBCAP, 17> LY;
	const int HS = 17;
	if (tl > MAXLEN || ql > MAXLEN) return 1;
	if (MAXLEN > 16000) return 1; // cells are 16-bit
	uint64_t mark = A.top;
	wf_cell_t *H = (wf_cell_t*)smem, *E1 = H + HS * W, *F1 = E1 + 3 * W, *E2 = F1 + 3 * W, *F2 = E2 + 2 * W;
	char *ts = (char*)(smem + LY::N_INTS), *qs = ts + LY::SEQ_BYTES;
	int32_t *tb_row = (int32_t*)(qs + LY::SEQ_BYTES); // TBCAP > 0 only
	uint8_t *tb_x = (uint8_t*)tb_row + LY::TB_ROW_BYTES;
	{ // every slice starts as -inf
		const uint32_t two = (uint32_t)(uint16_t)(wf_cell_t)WF_NEG_INF16 * 0x10001u;
		uint32_t *cells = (uint32_t*)smem;
		for (int32_t i = lane; i < LY::N_INTS; i += MGB_W) cells[i] = two;
	}
	wf_stage_seq(ts, ts_g, tl, 0xfe, lane);
	wf_stage_seq(qs, qs_g, ql, 0xff, lane);
	r->s = -1, r->n_cigar = 0, r->n_iter = 0, r->cigar = 0;
	uint32_t *cig_store;
	const int64_t max_cigar = (int64_t)tl + ql + 2;
	MGB_ALLOC(A, cig_store, uint32_t, max_cigar);
	uint64_t mark_keep = A.top;
	AVec<WfTbRow> rows; // TBCAP == 0 only
	avec_init(rows);
	if (TBCAP == 0) MGB_TRY(avec_reserve_w(A, rows, 256, lane)); // a row per score, and the score stays below 255
	int32_t n_rows = 0, tb_used = 0;
	int32_t wlo = 0, whi = 0, last_state = 0, s = 0;
	int64_t n_iter = 0;
	int hs = 0, m3 = 0, m2 = 0; // s % 17, s % 3, s % 2, kept incrementally
	const int32_t d_corner = ql - tl; // the diagonal of the last cell of the matrix
	int hit = 0, hit_noext = 0;
	warp_sync(); // the staged sequences and the cleared slices are complete
	if (lane == 0) { // score 0: the main diagonal, extended from the corner (E/F of score 0 stay -inf)
		int32_t k0 = -1, k = -1;
		if (!(k0 >= tl || k0 >= ql)) {
			k = wf_extend(ts, qs, k0, 0);
			if (k == tl - 1 && k == ql - 1) hit = 1, hit_noext = (k == k0), k = k0;
		}
		H[wfs_col<W>(0)] = (wf_cell_t)k;
	}
	{
		const uint32_t vb = warp_or_u32((hit? 1u : 0u) | (hit_noext? 2u : 0u));
		hit = vb & 1, hit_noext = vb >> 1 & 1;
	}
	warp_sync();
	for (;;) {
		// invariant: the wavefront of score s is computed, extended along exact matches and visible to all lanes;
		// a slice holds -inf everywhere outside the range it was last written with
		if (hit) {
			if (hit_noext) { // no extension on the last diagonal: the state comes from the traceback byte
				int32_t x;
				if (TBCAP > 0) { WfTbSmem t; t.row = tb_row, t.x = tb_x, t.n_rows = n_rows, t.used = tb_used; x = t.get(n_rows - 1, ql - tl); }
				else { WfTbArena t; t.row = rows.a; x = t.get(n_rows - 1, ql - tl); }
				last_state = x & 7;
			}
			break;
		}
		const int32_t lo = wlo > -tl? wlo - 1 : -tl;
		const int32_t hi = whi < ql? whi + 1 : ql;
		const int32_t width = hi - lo + 1;
		if (width + 2 > W || s + 1 >= 255 || (TBCAP > 0 && tb_used + width > TBCAP)) { A.top = mark; return 1; }
		const int32_t ns = s + 1;
		const int nhs = hs + 1 == 17? 0 : hs + 1, n3 = m3 + 1 == 3? 0 : m3 + 1, n2 = m2 ^ 1;
		uint8_t *ax;
		if (TBCAP > 0) {
			if (lane == 0) tb_row[2 * n_rows] = lo, tb_row[2 * n_rows + 1] = tb_used;
			ax = tb_x + tb_used - lo;
			tb_used += width;
		} else {
			uint8_t *x;
			MGB_ALLOC(A, x, uint8_t, width);
			if (lane == 0) rows.a[n_rows].lo = lo, rows.a[n_rows].hi = hi, rows.a[n_rows].x = x;
			rows.n = n_rows + 1;
			ax = x - lo;
		}
		++n_rows;
		// source slices: score ns-4 (mismatch), ns-6 and ns-16 (gap opens), ns-2 and ns-1 (gap extensions)
		const int r4 = nhs >= WF_X? nhs - WF_X : nhs - WF_X + 17, r6 = nhs >= WF_O1 + WF_E1? nhs - (WF_O1 + WF_E1) : nhs - (WF_O1 + WF_E1) + 17;
		const int r16 = nhs >= WF_O2 + WF_E2? nhs - (WF_O2 + WF_E2) : nhs - (WF_O2 + WF_E2) + 17;
		const int e1slot = n3 >= 2? n3 - 2 : n3 + 1; // (ns-2) % 3
		// byte offsets of the slices inside their arrays, held in registers through the cell loop (MGB_OPAQUE: the compiler would
		// otherwise re-derive each of them from the slot numbers for every cell)
		int32_t bHx = r4 * W * 2, bHo1 = r6 * W * 2, bHo2 = r16 * W * 2, bE1 = e1slot * W * 2, bE2 = m2 * W * 2, bnH = nhs * W * 2, bn3 = n3 * W * 2, bn2 = n2 * W * 2;
		MGB_OPAQUE(bHx); MGB_OPAQUE(bHo1); MGB_OPAQUE(bHo2); MGB_OPAQUE(bE1); MGB_OPAQUE(bE2); MGB_OPAQUE(bnH); MGB_OPAQUE(bn3); MGB_OPAQUE(bn2);
		const int32_t colmask2 = 2 * W - 1;
		uint32_t vote = 0; // 1: window grows on the low side, 2: on the high side, 4: corner reached, 8: ... without extension
		for (int32_t d = lo + lane; d <= hi; d += MGB_W) {
			MGB_WF_CELL_LOAD(A, d)
			MGB_WF_CELL_FINISH(A, d)
		}
		vote = warp_or_u32(vote);
		if (vote & 1) wlo = lo;
		if (vote & 2) whi = hi;
		hit = vote >> 2 & 1, hit_noext = vote >> 3 & 1;
		s = ns, hs = nhs, m3 = n3, m2 = n2;
		n_iter += width;
		warp_sync();
	}
	r->n_iter = n_iter;
	r->s = s;
	{
		int rc = 0;
		int32_t n_cig = 0;
		int64_t first = 0;
		if (lane == 0) {
			if (TBCAP > 0) { WfTbSmem t; t.row = tb_row, t.x = tb_x, t.n_rows = n_rows, t.used = tb_used; rc = wf_traceback(t, n_rows, tl, ts, ql, qs, last_state, cig_store, max_cigar, &n_cig, &first); }
			else { WfTbArena t; t.row = rows.a; rc = wf_traceback(t, n_rows, tl, ts, ql, qs, last_state, cig_store, max_cigar, &n_cig, &first); }
		}
		rc = warp_bcast_i32(rc, 0), n_cig = warp_bcast_i32(n_cig, 0), first = (int64_t)warp_bcast_u64((uint64_t)first, 0);
		warp_sync();
		if (rc < 0) { A.top = mark; return rc; }
		r->n_cigar = n_cig, r->cigar = cig_store + first;
	}
	A.top = mark_keep;
	return 0;
}

// =================================================================================================================
// tier 3: the same scheme with the ring in the worker arena and clean slices
// =================================================================================================================
// Same idea as above, with three additions the long runs need.  (1) The ring covers every diagonal of the matrix, far more
// than a gap ever touches, so the slices are initialised lazily: [flo,fhi] is the span of columns on which all slices hold
// -inf or real cells, and it is extended ahead of the window, 128 columns at a time.  (2) Every 256 scores the band is
// re-centred and can shrink (miniwfa.c:144-171); a slot then still holds cells of a wider, older wavefront outside the new
// range, which the bounds checks of the first version hide.  Here the part of the old range that sticks out is set back to
// -inf when the slot is rewritten, which keeps the invariant "a slice holds -inf outside the range it was last written with"
// and with it every value the recurrence reads.  (3) The band shrink asks, per diagonal, whether one of the last 17 wavefronts
// has a cell inside the matrix in any of its five components -- the one reader of E/F values older than two scores.  Instead of
// keeping 17 slots of all five arrays for it (85 slices), the 17 wavefronts in front of a shrink note, per diagonal, the last
// score with such a cell in one extra slice G; the ring is then H x 17, E1/F1 x 3, E2/F2 x 2 as in the on-chip tiers: 28 slices.
// An 85-slice ring of the resident warps does not fit L2: every wavefront is evicted before its slot is reused, and each cell
// costs about 11 bytes of DRAM writes.
static const int WF3_NSL = 17 + 3 + 3 + 2 + 2 + 1;
#define MGB_WF2_FILL(need_lo_, need_hi_) do { \
		const int32_t nl_ = (need_lo_), nh_ = (need_hi_); \
		if (fhi < flo || nl_ < flo || nh_ > fhi) { \
			int32_t tlo_ = nl_ - 128 > -tl - 1? nl_ - 128 : -tl - 1, thi_ = nh_ + 128 < ql + 1? nh_ + 128 : ql + 1; \
			if (fhi >= flo) { if (nl_ >= flo) tlo_ = flo; if (nh_ <= fhi) thi_ = fhi; } \
			const int32_t a0_ = tlo_, a1_ = fhi >= flo? flo - 1 : thi_, b0_ = fhi >= flo? fhi + 1 : thi_ + 1, b1_ = thi_; \
			for (int sl_ = 0; sl_ < WF3_NSL; ++sl_) { \
				wf_cell_t *p_ = cells + (int64_t)sl_ * W; \
				for (int32_t d_ = a0_ + lane; d_ <= a1_; d_ += MGB_W) p_[(d_ + (1 << 20)) & mask] = (wf_cell_t)WF_NEG_INF16; \
				for (int32_t d_ = b0_ + lane; d_ <= b1_; d_ += MGB_W) p_[(d_ + (1 << 20)) & mask] = (wf_cell_t)WF_NEG_INF16; \
			} \
			flo = tlo_, fhi = thi_; \
			warp_sync(); \
		} \
	} while (0)
// the slot about to be rewritten held the wavefront with range g_: what of it sticks out of [lo,hi] becomes -inf again
#define MGB_WF2_CLEAN(p_, g_) do { \
		const int32_t olo_ = (int32_t)((g_) & 0xffffu) - 0x8000, ohi_ = (int32_t)((g_) >> 16) - 0x8000; \
		if (olo_ < lo || ohi_ > hi) { \
			wf_cell_t *q_ = (p_); \
			for (int32_t d_ = olo_ + lane; d_ <= ohi_ && d_ < lo; d_ += MGB_W) q_[(d_ + (1 << 20)) & mask] = (wf_cell_t)WF_NEG_INF16; \
			for (int32_t d_ = (hi + 1 > olo_? hi + 1 : olo_) + lane; d_ <= ohi_; d_ += MGB_W) q_[(d_ + (1 << 20)) & mask] = (wf_cell_t)WF_NEG_INF16; \
		} \
	} while (0)

MG_HD inline int wfa_ring_g(Arena &A, int32_t tl, const char *ts, int32_t ql, const char *qs, int64_t max_iter, WfResult *r,
							uint32_t *cig_store, int64_t max_cigar, int lane)
{
	if (tl + ql > 16000 || tl <= 0 || ql <= 0) return 1; // (scores stay below 2^15 too: deleting one sequence and inserting the other costs tl + ql + 30)
	uint64_t mark = A.top;
	int32_t W = 64;
	while (W < tl + ql + 2) W <<= 1;
	const int32_t mask = W - 1;
	wf_cell_t *cells;
	MGB_ALLOC(A, cells, wf_cell_t, (int64_t)WF3_NSL * W);
	wf_cell_t *H = cells, *E1 = H + 17 * W, *F1 = E1 + 3 * W, *E2 = F1 + 3 * W, *F2 = E2 + 2 * W, *G = F2 + 2 * W;
	int32_t flo = 0, fhi = -1; // columns on which all slices have been initialised with -inf (empty so far)
	const int32_t d_corner = ql - tl;
	AVec<WfTbRow> rows;
	avec_init(rows);
	MGB_TRY(avec_reserve_w(A, rows, 1024, lane));
	int32_t n_rows = 0;
	int32_t wlo = 0, whi = 0, last_state = 0, s = 0, stopped = 0;
	int64_t n_iter = 0;
	int hs = 0, m3 = 0, m2 = 0; // s % 17, s % 3, s % 2, kept incrementally
#define MGB_WF_RG(lo_, hi_) ((uint32_t)((hi_) + 0x8000) << 16 | (uint32_t)((lo_) + 0x8000))
	// [lo,hi] of the last 17 wavefronts, by score modulo 17 (empty ranges before score 0).  On the device lane j keeps entry j in a
	// register (three shuffles per score instead of a 17-register shift chain); a simulator with fewer lanes keeps the array.
#if MGB_W >= 32
	uint32_t g_mine = lane == 0? MGB_WF_RG(0, 0) : MGB_WF_RG(1, 0);
#define MGB_WF_GGET(slot_) ((uint32_t)warp_bcast_i32((int32_t)g_mine, (slot_)))
#define MGB_WF_GSET(slot_, v_) do { if (lane == (slot_)) g_mine = (v_); } while (0)
#else
	uint32_t g_all[17];
	for (int j = 0; j < 17; ++j) g_all[j] = j == 0? MGB_WF_RG(0, 0) : MGB_WF_RG(1, 0);
#define MGB_WF_GGET(slot_) (g_all[(slot_)])
#define MGB_WF_GSET(slot_, v_) (g_all[(slot_)] = (v_))
#endif
	int hit = 0, hit_noext = 0;
	MGB_WF2_FILL(-1, 1);
	if (lane == 0) { // score 0: the main diagonal, extended from the corner
		const int32_t c0 = (1 << 20) & mask;
		int32_t k0 = -1, k = -1;
		k = wf_extend(ts, qs, k0, 0);
		if (k == tl - 1 && k == ql - 1) hit = 1, hit_noext = (k == k0), k = k0;
		H[c0] = (wf_cell_t)k;
	}
	{
		const uint32_t vb = warp_or_u32((hit? 1u : 0u) | (hit_noext? 2u : 0u));
		hit = vb & 1, hit_noext = vb >> 1 & 1;
	}
	warp_sync();
	for (;;) {
		if (hit) {
			if (hit_noext) { WfTbArena t; t.row = rows.a; last_state = t.get(n_rows - 1, ql - tl) & 7; }
			break;
		}
		const int32_t lo = wlo > -tl? wlo - 1 : -tl;
		const int32_t hi = whi < ql? whi + 1 : ql;
		const int32_t width = hi - lo + 1;
		const int32_t ns = s + 1;
		const int nhs = hs + 1 == 17? 0 : hs + 1, n3 = m3 + 1 == 3? 0 : m3 + 1, n2 = m2 ^ 1;
		MGB_TRY(avec_reserve_w(A, rows, n_rows + 1, lane));
		uint8_t *x;
		MGB_ALLOC(A, x, uint8_t, width);
		if (lane == 0) rows.a[n_rows].lo = lo, rows.a[n_rows].hi = hi, rows.a[n_rows].x = x;
		rows.n = ++n_rows;
		uint8_t *ax = x - lo;
		const int r4 = nhs >= WF_X? nhs - WF_X : nhs - WF_X + 17, r6 = nhs >= WF_O1 + WF_E1? nhs - (WF_O1 + WF_E1) : nhs - (WF_O1 + WF_E1) + 17;
		const int r16 = nhs >= WF_O2 + WF_E2? nhs - (WF_O2 + WF_E2) : nhs - (WF_O2 + WF_E2) + 17;
		const int e1slot = n3 >= 2? n3 - 2 : n3 + 1; // (ns-2) % 3
		MGB_WF2_FILL(lo - 1, hi + 1);
		// the slots of score ns held scores ns-17 (H), ns-3 (E1/F1) and ns-2 (E2/F2): after a band shrink those ranges can reach beyond [lo,hi]
		const uint32_t g16 = MGB_WF_GGET(nhs), g2 = MGB_WF_GGET(nhs >= 3? nhs - 3 : nhs + 14), g1 = MGB_WF_GGET(nhs >= 2? nhs - 2 : nhs + 15);
		MGB_WF2_CLEAN(H + (int64_t)nhs * W, g16);
		MGB_WF2_CLEAN(E1 + (int64_t)n3 * W, g2);
		MGB_WF2_CLEAN(F1 + (int64_t)n3 * W, g2);
		MGB_WF2_CLEAN(E2 + (int64_t)n2 * W, g1);
		MGB_WF2_CLEAN(F2 + (int64_t)n2 * W, g1);
		// byte offsets of the source and destination slices inside their arrays (kept in registers, see wfa_smem)
		int32_t bHx = r4 * W * 2, bHo1 = r6 * W * 2, bHo2 = r16 * W * 2, bE1 = e1slot * W * 2, bE2 = m2 * W * 2, bnH = nhs * W * 2, bn3 = n3 * W * 2, bn2 = n2 * W * 2;
		MGB_OPAQUE(bHx); MGB_OPAQUE(bHo1); MGB_OPAQUE(bHo2); MGB_OPAQUE(bE1); MGB_OPAQUE(bE2); MGB_OPAQUE(bnH); MGB_OPAQUE(bn3); MGB_OPAQUE(bn2);
		const int track = ((ns + 16) & 0xff) <= 16; // one of the 17 wavefronts the next band shrink (at a multiple of 256) looks at
		uint32_t vote = 0; // 1: window grows on the low side, 2: on the high side, 4: corner reached, 8: ... without extension
		const int32_t colmask2 = 2 * W - 1;
		// what wf_stripe_shrink() will ask of a cell (the values as stored)
#define MGB_WF_TRACK(S, d_) do { if (track && (wf_good_diag((d_), h##S, tl, ql) || wf_good_diag((d_), e1##S, tl, ql) || wf_good_diag((d_), f1##S, tl, ql) || wf_good_diag((d_), e2##S, tl, ql) || wf_good_diag((d_), f2##S, tl, ql))) \
				*(wf_cell_t*)((char*)G + c##S) = (wf_cell_t)ns; } while (0)
		for (int32_t d = lo + lane; d <= hi; d += 2 * MGB_W) { // two cells per lane in flight
			const int32_t dB = d + MGB_W <= hi? d + MGB_W : d;
			MGB_WF_CELL_LOAD(A, d)
			MGB_WF_CELL_LOAD(B, dB)
			MGB_WF_CELL_FINISH(A, d)
			MGB_WF_TRACK(A, d);
			if (dB != d) { MGB_WF_CELL_FINISH(B, dB) MGB_WF_TRACK(B, dB); }
		}
#undef MGB_WF_TRACK
		vote = warp_or_u32(vote);
		if (vote & 1) wlo = lo;
		if (vote & 2) whi = hi;
		hit = vote >> 2 & 1, hit_noext = vote >> 3 & 1;
		MGB_WF_GSET(nhs, MGB_WF_RG(lo, hi));
		s = ns, hs = nhs, m3 = n3, m2 = n2;
		warp_sync();
		if ((s & 0xff) == 0) { // reference: miniwfa.c:144-171 wf_stripe_shrink: keep the diagonals on which one of the 17 wavefronts still has a cell inside the matrix
			int32_t nlo = 0, nhi = 0, found = 0;
			for (int pass = 0; pass < 2; ++pass) {
				found = 0;
				for (int32_t base = pass == 0? wlo : whi; pass == 0? base <= whi : base >= wlo; base += pass == 0? MGB_W : -MGB_W) {
					const int32_t d = pass == 0? base + lane : base - lane;
					int good = 0;
					if (d >= wlo && d <= whi) good = G[(d + (1 << 20)) & mask] >= s - 16; // noted by one of the wavefronts s-16 .. s
					const uint32_t m = warp_ballot(good);
					if (m) { found = 1; if (pass == 0) nlo = base + ctz32(m); else nhi = base - ctz32(m); break; }
				}
				if (!found) break;
			}
			if (!found) { A.top = mark; return MGB_E_INTERNAL; }
			wlo = nlo, whi = nhi;
		}
		n_iter += width;
		if (max_iter > 0 && n_iter > max_iter) { stopped = 1; break; }
	}
#undef MGB_WF_RG
#undef MGB_WF_GGET
#undef MGB_WF_GSET
	r->n_iter = n_iter;
	r->s = stopped? -1 : s;
	if (!stopped) {
		int rc = 0;
		int32_t n_cig = 0;
		int64_t first = 0;
		if (lane == 0) {
			WfTbArena t; t.row = rows.a;
			rc = wf_traceback(t, n_rows, tl, ts, ql, qs, last_state, cig_store, max_cigar, &n_cig, &first);
		}
		rc = warp_bcast_i32(rc, 0), n_cig = warp_bcast_i32(n_cig, 0), first = (int64_t)warp_bcast_u64((uint64_t)first, 0);
		warp_sync();
		if (rc < 0) { A.top = mark; return rc; }
		r->n_cigar = n_cig, r->cigar = cig_store + first;
	}
	A.top = mark;
	return 0;
}
#undef MGB_WF2_CLEAN
#undef MGB_WF2_FILL


} // namespace mgb
