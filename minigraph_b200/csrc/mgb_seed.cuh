// mgb_seed.cuh -- stage A: minimizer sketch, index lookup, seed expansion and seed sort for one read.
#pragma once
#include "mgb_model.cuh"

namespace mgb {

// Symmetric (w,k)-minimizers of one sequence (reference: sketch.c:56-109 mg_sketch()).
//   out[i].x = hash<<8 | span ;  out[i].y = rid<<32 | lastPos<<1 | strand
// Quirks kept on purpose (SURVEY H6): a symmetric k-mer does not advance the window slot, an
// ambiguous base resets the run but still occupies a slot, ties pick the rightmost, equal-hash
// duplicates inside one window are all reported, and the last minimum is flushed at the end.
MG_HD inline int sketch_seq(Arena &A, const char *str, int len, int w, int k, uint32_t rid, AVec<u128> &out)
{
	const uint64_t shift1 = 2 * (k - 1), mask = (1ULL << 2 * k) - 1;
	uint64_t kmer[2] = {0, 0};
	int l = 0, buf_pos = 0, min_pos = 0, kmer_span = 0;
	const u128 none = { ~0ULL, ~0ULL };
	u128 mn = none, *buf;
	if (!(len > 0 && w > 0 && w < 256 && k > 0 && k <= 28)) return MGB_E_INTERNAL;
	MGB_TRY(avec_reserve(A, out, out.n + len / w + 16));
	MGB_ALLOC(A, buf, u128, w);
	for (int j = 0; j < w; ++j) buf[j] = none;
	for (int i = 0; i < len; ++i) {
		int c = nt4((uint8_t)str[i]);
		u128 info = none;
		if (c < 4) {
			kmer_span = l + 1 < k? l + 1 : k;
			kmer[0] = (kmer[0] << 2 | (uint64_t)c) & mask;
			kmer[1] = (kmer[1] >> 2) | (3ULL ^ (uint64_t)c) << shift1;
			if (kmer[0] == kmer[1]) continue; // strand unknown
			int z = kmer[0] < kmer[1]? 0 : 1;
			++l;
			if (l >= k && kmer_span < 256) {
				info.x = hash64_mask(z? kmer[1] : kmer[0], mask) << 8 | (uint64_t)kmer_span; // a select: indexing kmer[] by z would put it in local memory
				info.y = (uint64_t)rid << 32 | (uint64_t)((uint32_t)i << 1) | (uint64_t)z;
			}
		} else l = 0, kmer_span = 0;
		buf[buf_pos] = info;
		if (l == w + k - 1 && mn.x != ~0ULL) { // first full window: report earlier copies of the minimum
			for (int j = buf_pos + 1; j < w; ++j)
				if (mn.x == buf[j].x && buf[j].y != mn.y) MGB_TRY(avec_push(A, out, buf[j]));
			for (int j = 0; j < buf_pos; ++j)
				if (mn.x == buf[j].x && buf[j].y != mn.y) MGB_TRY(avec_push(A, out, buf[j]));
		}
		if (info.x <= mn.x) { // new minimum (rightmost on ties)
			if (l >= w + k && mn.x != ~0ULL) MGB_TRY(avec_push(A, out, mn));
			mn = info, min_pos = buf_pos;
		} else if (buf_pos == min_pos) { // the old minimum slides out
			if (l >= w + k - 1 && mn.x != ~0ULL) MGB_TRY(avec_push(A, out, mn));
			mn.x = ~0ULL;
			for (int j = buf_pos + 1; j < w; ++j)
				if (mn.x >= buf[j].x) mn = buf[j], min_pos = j;
			for (int j = 0; j <= buf_pos; ++j)
				if (mn.x >= buf[j].x) mn = buf[j], min_pos = j;
			if (l >= w + k - 1 && mn.x != ~0ULL) {
				for (int j = buf_pos + 1; j < w; ++j)
					if (mn.x == buf[j].x && mn.y != buf[j].y) MGB_TRY(avec_push(A, out, buf[j]));
				for (int j = 0; j <= buf_pos; ++j)
					if (mn.x == buf[j].x && mn.y != buf[j].y) MGB_TRY(avec_push(A, out, buf[j]));
			}
		}
		if (++buf_pos == w) buf_pos = 0;
	}
	if (mn.x != ~0ULL) MGB_TRY(avec_push(A, out, mn));
	return 0;
}

// ---- the same sketch, cut into chunks that are independent of each other ----
// A chunk that does not start the sequence replays w slots of warm-up before its first position: with k odd and no
// ambiguous base every position fills a slot, the window before position p holds exactly the k-mers ending at
// p-w..p-1, the minimum is a function of the window, and the run length l only matters below w+k (it is beyond that
// once p >= w+2k-1, whatever happened in the first k-1 bases).  Whatever a chunk reports while processing positions
// [p, end) is therefore what the sequential scan reports there; the lists are concatenated in chunk order.
// Returns 1 when the chunk cannot be done this way (ambiguous base in its span, list full): the caller then runs
// sketch_seq() on the whole sequence.
static const int SKETCH_CHUNKS = 32;

// BS: distance between two slots of the window ring (1: a private ring in the arena; 32: the rings of the 32 lanes interleaved in
// shared memory, slot j of lane l at [j * 32 + l], so that the lanes of a warp touch consecutive 16-byte words)
// PK: the bases come 2 bits each from `pk` (32 per 64-bit word, base i in bits 2*(i%32).. of word i/32; no ambiguous base by
// construction), one 8-byte load per 32 bases, instead of one byte each from `str`
template<int BS = 1, int PK = 0>
MG_HD inline int sketch_chunk(const char *str, const uint64_t *pk, int w, int k, uint32_t rid, int p, int end, int is_first, int is_last, u128 *buf, u128 *outp, int cap, int *n_out)
{
	const uint64_t shift1 = 2 * (k - 1), mask = (1ULL << 2 * k) - 1;
	uint64_t kmer[2] = {0, 0};
	int l = 0, buf_pos = 0, min_pos = 0, kmer_span = 0, n = 0, i0 = 0;
	const u128 none = { ~0ULL, ~0ULL };
	u128 mn = none;
	for (int j = 0; j < w; ++j) buf[(j) * BS] = none;
	if (!is_first) {
		i0 = p - w;
		for (int i = i0 - k + 1; i < i0; ++i) { // the k-1 bases in front of the first warm-up slot
			int c = PK? (int)(pk[i >> 5] >> ((i & 31) << 1) & 3) : nt4((uint8_t)str[i]);
			if (c >= 4) return 1;
			kmer[0] = (kmer[0] << 2 | (uint64_t)c) & mask;
			kmer[1] = (kmer[1] >> 2) | (3ULL ^ (uint64_t)c) << shift1;
		}
		l = w + k + 1; // any value the thresholds below cannot tell from the true one
	}
#define MGB_SK_PUSH(v) do { if (i >= p) { if (n >= cap) return 1; outp[n++] = (v); } } while (0)
	uint64_t word = 0;
	if (PK && i0 < end) word = pk[i0 >> 5] >> ((i0 & 31) << 1);
	for (int i = i0; i < end; ++i) {
		int c;
		if (PK) {
			if ((i & 31) == 0) word = pk[i >> 5];
			c = (int)(word & 3), word >>= 2;
		} else c = nt4((uint8_t)str[i]);
		u128 info = none;
		if (c >= 4) return 1;
		kmer_span = l + 1 < k? l + 1 : k;
		kmer[0] = (kmer[0] << 2 | (uint64_t)c) & mask;
		kmer[1] = (kmer[1] >> 2) | (3ULL ^ (uint64_t)c) << shift1;
		if (kmer[0] == kmer[1]) { if (is_first) continue; return 1; }
		int z = kmer[0] < kmer[1]? 0 : 1;
		if (l < w + k + 1) ++l;
		if (l >= k && kmer_span < 256) {
			info.x = hash64_mask(z? kmer[1] : kmer[0], mask) << 8 | (uint64_t)kmer_span; // a select: indexing kmer[] by z would put it in local memory
			info.y = (uint64_t)rid << 32 | (uint64_t)((uint32_t)i << 1) | (uint64_t)z;
		}
		buf[(buf_pos) * BS] = info;
		if (l == w + k - 1 && mn.x != ~0ULL) {
			for (int j = buf_pos + 1; j < w; ++j)
				if (mn.x == buf[(j) * BS].x && buf[(j) * BS].y != mn.y) MGB_SK_PUSH(buf[(j) * BS]);
			for (int j = 0; j < buf_pos; ++j)
				if (mn.x == buf[(j) * BS].x && buf[(j) * BS].y != mn.y) MGB_SK_PUSH(buf[(j) * BS]);
		}
		if (info.x <= mn.x) {
			if (l >= w + k && mn.x != ~0ULL) MGB_SK_PUSH(mn);
			mn = info, min_pos = buf_pos;
		} else if (buf_pos == min_pos) {
			if (l >= w + k - 1 && mn.x != ~0ULL) MGB_SK_PUSH(mn);
			mn.x = ~0ULL;
			for (int j = buf_pos + 1; j < w; ++j)
				if (mn.x >= buf[(j) * BS].x) mn = buf[(j) * BS], min_pos = j;
			for (int j = 0; j <= buf_pos; ++j)
				if (mn.x >= buf[(j) * BS].x) mn = buf[(j) * BS], min_pos = j;
			if (l >= w + k - 1 && mn.x != ~0ULL) {
				for (int j = buf_pos + 1; j < w; ++j)
					if (mn.x == buf[(j) * BS].x && mn.y != buf[(j) * BS].y) MGB_SK_PUSH(buf[(j) * BS]);
				for (int j = 0; j <= buf_pos; ++j)
					if (mn.x == buf[(j) * BS].x && mn.y != buf[(j) * BS].y) MGB_SK_PUSH(buf[(j) * BS]);
			}
		}
		if (++buf_pos == w) buf_pos = 0;
	}
	if (is_last && mn.x != ~0ULL) { const int i = end; MGB_SK_PUSH(mn); }
#undef MGB_SK_PUSH
	*n_out = n;
	return 0;
}

// sketch_seq() entered by all lanes of a warp; `out` (replicated on every lane) must be empty.
static const int SKETCH_SMEM_W = 12; // widest window whose rings fit the shared-memory variant ("seed_v2")
static const int SKETCH_SMEM_BYTES = SKETCH_SMEM_W * 32 * 16; // per warp

// The ways sketch_seq_w() makes the list: chunks with the rings in shared memory reading the 2-bit words or ASCII, chunks with the
// rings in the arena (w > SKETCH_SMEM_W or no slice), the sequential scan on lane 0
enum { SKETCH_PATH_SMEM_PK = 0, SKETCH_PATH_SMEM = 1, SKETCH_PATH_ARENA = 2, SKETCH_PATH_SEQ = 3 };

// sring: NULL, or SKETCH_SMEM_BYTES of shared memory of this warp for the window rings
// pk: NULL, or the sequence 2 bits per base (see sketch_chunk); str is always there (the sequential scan below reads it)
// path: NULL, or where the way the list was made goes (SKETCH_PATH_*)
MG_HD inline int sketch_seq_w(Arena &A, const char *str, int len, int w, int k, uint32_t rid, AVec<u128> &out, int lane, u128 *sring = 0, const uint64_t *pk = 0,
							  int *path = 0)
{
	if (!(len > 0 && w > 0 && w < 256 && k > 0 && k <= 28)) return MGB_E_INTERNAL;
	const int min_chunk = w + 2 * k > 64? w + 2 * k : 64;
	const int n_ch = len / min_chunk < SKETCH_CHUNKS? len / min_chunk : SKETCH_CHUNKS;
	int fail = (k & 1) == 0 || n_ch < 2;
	if (!fail) {
		const uint64_t mark = A.top;
		const int chunk = (len + n_ch - 1) / n_ch, cap = chunk + w + 2;
		u128 *tmp, *ring;
		int32_t *cnt;
		MGB_ALLOC(A, tmp, u128, (int64_t)n_ch * cap);
		MGB_ALLOC(A, ring, u128, (int64_t)n_ch * w);
		MGB_ALLOC(A, cnt, int32_t, SKETCH_CHUNKS);
		for (int c = lane; c < n_ch; c += MGB_W) {
			const int p = c * chunk, e = p + chunk < len? p + chunk : len;
			int n = 0;
			if (p < e) {
				if (sring && w <= SKETCH_SMEM_W) {
					if (pk) fail |= sketch_chunk<32, 1>(str, pk, w, k, rid, p, e, c == 0, e == len, sring + lane, tmp + (int64_t)c * cap, cap, &n);
					else fail |= sketch_chunk<32, 0>(str, pk, w, k, rid, p, e, c == 0, e == len, sring + lane, tmp + (int64_t)c * cap, cap, &n);
				} else fail |= sketch_chunk<1, 0>(str, pk, w, k, rid, p, e, c == 0, e == len, ring + (int64_t)c * w, tmp + (int64_t)c * cap, cap, &n);
			}
			cnt[c] = n;
		}
		fail = warp_any(fail);
		warp_sync();
		if (!fail) {
			int64_t tot = 0;
			for (int c = 0; c < n_ch; ++c) tot += cnt[c];
			// the per-chunk lists are closed up in place (the first one already sits at the mark); a list only ever moves down
			u128 *dst = tmp;
			int64_t off = cnt[0];
			for (int c = 1; c < n_ch; ++c) {
				const u128 *src = tmp + (int64_t)c * cap;
				// read once, before the moves: past the last warp_sync below a lane may already be on to the caller, whose allocations
				// take the arena behind the list (cnt[] included) while another lane would still test its loop bound there
				const int32_t n_c = cnt[c];
				for (int j0 = 0; j0 < n_c; j0 += MGB_W) {
					const int j = j0 + lane;
					u128 e = {0, 0};
					if (j < n_c) e = src[j];
					warp_sync();
					if (j < n_c) dst[off + j] = e;
					warp_sync();
				}
				off += n_c;
			}
			A.top = mark + ((((uint64_t)tot + 16) * sizeof(u128) + 15) & ~(uint64_t)15);
			if (A.top > A.peak) A.peak = A.top;
			out.a = dst, out.n = tot, out.m = tot + 16;
			if (path) *path = !(sring && w <= SKETCH_SMEM_W)? SKETCH_PATH_ARENA : pk? SKETCH_PATH_SMEM_PK : SKETCH_PATH_SMEM;
			return 0;
		}
		A.top = mark;
	}
	// sequential scan on lane 0; its few scalar results are broadcast
	{
		Arena B = A;
		int rc = 0;
		if (lane == 0) rc = sketch_seq(B, str, len, w, k, rid, out);
		rc = warp_bcast_i32(rc, 0);
		out.a = (u128*)warp_bcast_u64((uint64_t)out.a, 0);
		out.n = (int64_t)warp_bcast_u64((uint64_t)out.n, 0);
		out.m = (int64_t)warp_bcast_u64((uint64_t)out.m, 0);
		A.top = warp_bcast_u64(B.top, 0);
		A.peak = warp_bcast_u64(B.peak, 0);
		warp_sync();
		if (path) *path = SKETCH_PATH_SEQ;
		return rc;
	}
}

struct SeedMatch {
	uint32_t n, q_pos, q_span;
	uint32_t seg_id, is_tandem;
	const uint64_t *cr;
};

// Index probe per minimizer with the high-occurrence filter (reference: map-algo.c:58-91 collect_matches()).
MG_HD inline int collect_matches(Arena &A, const IndexDev &ix, int max_occ, const AVec<u128> &mv, SeedMatch **m_, int *n_m_,
								 int64_t *n_a, int *rep_len, int32_t *mini_pos, int *n_mini_pos)
{
	int rep_st = 0, rep_en = 0, n_m = 0, n_mp = 0;
	SeedMatch *m;
	MGB_ALLOC(A, m, SeedMatch, mv.n);
	*rep_len = 0, *n_a = 0;
	for (int64_t i = 0; i < mv.n; ++i) {
		const u128 *p = &mv.a[i];
		uint32_t q_pos = (uint32_t)p->y, q_span = (uint32_t)(p->x & 0xff);
		int t;
		const uint64_t *cr = idx_get(ix, p->x >> 8, &t);
		if (t >= max_occ) {
			int en = (int)(q_pos >> 1) + 1, st = en - (int)q_span;
			if (st > rep_en) {
				*rep_len += rep_en - rep_st;
				rep_st = st, rep_en = en;
			} else rep_en = en;
		} else {
			SeedMatch *q = &m[n_m++];
			q->q_pos = q_pos, q->q_span = q_span, q->cr = cr, q->n = (uint32_t)t, q->seg_id = (uint32_t)(p->y >> 32);
			q->is_tandem = 0;
			if (i > 0 && p->x >> 8 == mv.a[i - 1].x >> 8) q->is_tandem = 1;
			if (i < mv.n - 1 && p->x >> 8 == mv.a[i + 1].x >> 8) q->is_tandem = 1;
			*n_a += q->n;
			mini_pos[n_mp++] = (int32_t)(q_pos >> 1);
		}
	}
	*rep_len += rep_en - rep_st;
	*m_ = m, *n_m_ = n_m, *n_mini_pos = n_mp;
	return 0;
}

// Expand matches to anchors (reference: map-algo.c:152-192 collect_seed_hits(), without the NO_DIAG branch):
//   a.x = seg<<33 | rev<<32 | tpos ;  a.y = occ<<56 | segid<<48 | tandem | q_span<<32 | qpos
MG_HD inline void expand_seeds(const GraphDev &g, int n_m, const SeedMatch *m, u128 *a)
{
	int64_t n = 0;
	for (int i = 0; i < n_m; ++i) {
		const SeedMatch *q = &m[i];
		const uint64_t *r = q->cr;
		for (uint32_t k = 0; k < q->n; ++k) {
			uint64_t rk = r[k];
			int32_t rpos = (int32_t)((uint32_t)rk >> 1);
			u128 *p = &a[n++];
			if ((rk & 1) == (q->q_pos & 1)) p->x = rk >> 32 << 33 | (uint64_t)(uint32_t)rpos;
			else p->x = rk >> 32 << 33 | 1ULL << 32 | (uint64_t)(uint32_t)(g.seg_len[rk >> 32] - (rpos + 1 - (int32_t)q->q_span) - 1);
			p->y = (uint64_t)q->q_span << 32 | (uint64_t)(q->q_pos >> 1);
			p->y |= (uint64_t)q->seg_id << SEED_SEG_SHIFT;
			if (q->is_tandem) p->y |= SEED_TANDEM;
			p->y |= (uint64_t)(q->n < 255? q->n : 255) << SEED_OCC_SHIFT;
		}
	}
}

// collect_matches() + the anchor offsets of expand_seeds(), entered by all lanes of a warp: the index probes (one random
// HBM access chain each) run 32 at a time; the lists are then compacted in order and the repeat-length rule, which is
// sequential over the rare high-occurrence minimizers, is replayed on their ballot.
MG_HD inline int collect_matches_w(Arena &A, const IndexDev &ix, int max_occ, const AVec<u128> &mv, SeedMatch **m_, int *n_m_,
								   int64_t *n_a, int *rep_len, int32_t *mini_pos, int *n_mini_pos, int32_t **a_off_, int lane)
{
	int rep_st = 0, rep_en = 0, rl = 0, n_m = 0;
	int32_t tot = 0;
	SeedMatch *m, *tm;
	int32_t *a_off;
	MGB_ALLOC(A, m, SeedMatch, mv.n);
	MGB_ALLOC(A, a_off, int32_t, mv.n);
	MGB_ALLOC(A, tm, SeedMatch, mv.n);
	for (int64_t i = lane; i < mv.n; i += MGB_W) {
		const u128 p = mv.a[i];
		int t;
		SeedMatch q;
		q.cr = idx_get(ix, p.x >> 8, &t);
		q.q_pos = (uint32_t)p.y, q.q_span = (uint32_t)(p.x & 0xff), q.n = (uint32_t)t, q.seg_id = (uint32_t)(p.y >> 32);
		q.is_tandem = 0;
		if (i > 0 && p.x >> 8 == mv.a[i - 1].x >> 8) q.is_tandem = 1;
		if (i < mv.n - 1 && p.x >> 8 == mv.a[i + 1].x >> 8) q.is_tandem = 1;
		tm[i] = q;
	}
	warp_sync();
	for (int64_t base = 0; base < mv.n; base += MGB_W) {
		const int64_t i = base + lane;
		SeedMatch q;
		q.n = 0, q.q_pos = q.q_span = q.seg_id = q.is_tandem = 0, q.cr = 0;
		if (i < mv.n) q = tm[i];
		const int high = i < mv.n && (int)q.n >= max_occ, keep = i < mv.n && !high;
		uint32_t mh = warp_ballot(high);
		const uint32_t mk = warp_ballot(keep);
		while (mh) { // reference: map-algo.c:73-80
			const int l = ctz32(mh);
			mh &= mh - 1;
			const SeedMatch h = tm[base + l];
			const int en = (int)(h.q_pos >> 1) + 1, st = en - (int)h.q_span;
			if (st > rep_en) {
				rl += rep_en - rep_st;
				rep_st = st, rep_en = en;
			} else rep_en = en;
		}
		const int32_t cnt = keep? (int32_t)q.n : 0;
		const int32_t incl = warp_incl_scan_i32(cnt, lane);
		if (keep) {
			const int at = n_m + mask_rank(mk, lane);
			m[at] = q;
			a_off[at] = tot + incl - cnt;
			mini_pos[at] = (int32_t)(q.q_pos >> 1);
		}
		n_m += mask_count(mk);
		tot += warp_bcast_i32(incl, MGB_W - 1);
	}
	rl += rep_en - rep_st;
	warp_sync();
	*rep_len = rl, *n_a = tot;
	*m_ = m, *n_m_ = n_m, *n_mini_pos = n_m, *a_off_ = a_off;
	return 0;
}

// expand_seeds() with the matches spread over the lanes; a_off[i] = number of anchors of the matches before i
MG_HD inline void expand_seeds_w(const GraphDev &g, int n_m, const SeedMatch *m, const int32_t *a_off, u128 *a, int lane)
{
	for (int i = lane; i < n_m; i += MGB_W) {
		const SeedMatch q = m[i];
		const uint64_t *r = q.cr;
		u128 *p = a + a_off[i];
		for (uint32_t k = 0; k < q.n; ++k, ++p) {
			uint64_t rk = r[k];
			int32_t rpos = (int32_t)((uint32_t)rk >> 1);
			u128 v;
			if ((rk & 1) == (q.q_pos & 1)) v.x = rk >> 32 << 33 | (uint64_t)(uint32_t)rpos;
			else v.x = rk >> 32 << 33 | 1ULL << 32 | (uint64_t)(uint32_t)(g.seg_len[rk >> 32] - (rpos + 1 - (int32_t)q.q_span) - 1);
			v.y = (uint64_t)q.q_span << 32 | (uint64_t)(q.q_pos >> 1);
			v.y |= (uint64_t)q.seg_id << SEED_SEG_SHIFT;
			if (q.is_tandem) v.y |= SEED_TANDEM;
			v.y |= (uint64_t)(q.n < 255? q.n : 255) << SEED_OCC_SHIFT;
			*p = v;
		}
	}
}

// Seeds by k-way merge of the occurrence lists (reference: map-algo.c:93-150 collect_seed_hits_heap, the `sr` preset).  The
// heap is klib's (ksort.h:43-70 with heap_lt = a.x > b.x): its sift order decides the order among equal target positions, so
// it is replayed as is.  Forward-strand anchors fill a[] from the front in pop order, reverse-strand ones from the back.
// One lane; no sort follows.
MG_HD inline void seed_heap_down(int64_t i, int64_t n, u128 *l)
{
	int64_t k = i;
	u128 tmp = l[i];
	while ((k = (k << 1) + 1) < n) {
		if (k != n - 1 && l[k].x > l[k+1].x) ++k;
		if (l[k].x > tmp.x) break;
		l[i] = l[k], i = k;
	}
	l[i] = tmp;
}
MG_HD inline int expand_seeds_heap(Arena &A, const GraphDev &g, int n_m, const SeedMatch *m, int64_t n_a, u128 *a)
{
	uint64_t mark = A.top;
	u128 *heap;
	MGB_ALLOC(A, heap, u128, n_m);
	int64_t heap_size = 0, n_for = 0, n_rev = 0;
	for (int i = 0; i < n_m; ++i)
		if (m[i].n > 0) heap[heap_size].x = m[i].cr[0], heap[heap_size].y = (uint64_t)i << 32, ++heap_size;
	for (int64_t i = (heap_size >> 1) - 1; i >= 0; --i) seed_heap_down(i, heap_size, heap);
	while (heap_size > 0) {
		const SeedMatch *q = &m[heap[0].y >> 32];
		const uint64_t r = heap[0].x;
		const int32_t rpos = (int32_t)((uint32_t)r >> 1);
		u128 *p;
		if ((r & 1) == (q->q_pos & 1)) {
			p = &a[n_for++];
			p->x = r >> 32 << 33 | (uint64_t)(uint32_t)rpos;
		} else {
			p = &a[n_a - (++n_rev)];
			p->x = r >> 32 << 33 | 1ULL << 32 | (uint64_t)(uint32_t)(g.seg_len[r >> 32] - (rpos + 1 - (int32_t)q->q_span) - 1);
		}
		p->y = (uint64_t)q->q_span << 32 | (uint64_t)(q->q_pos >> 1);
		p->y |= (uint64_t)q->seg_id << SEED_SEG_SHIFT;
		if (q->is_tandem) p->y |= SEED_TANDEM;
		p->y |= (uint64_t)(q->n < 255? q->n : 255) << SEED_OCC_SHIFT;
		if ((uint32_t)heap[0].y < q->n - 1) {
			++heap[0].y;
			heap[0].x = m[heap[0].y >> 32].cr[(uint32_t)heap[0].y];
		} else {
			heap[0] = heap[heap_size - 1];
			--heap_size;
		}
		seed_heap_down(0, heap_size, heap);
	}
	A.top = mark;
	return n_for + n_rev == n_a? 0 : MGB_E_INTERNAL;
}

// expand_seeds() with the self-diagonal filter of MG_M_NO_DIAG (reference: map-algo.c:160-188): a seed is dropped when the
// read carries the name its segment goes by and sits at its own position there.  One lane; returns the number of seeds kept.
MG_HD inline int64_t expand_seeds_nodiag(const GraphDev &g, int n_m, const SeedMatch *m, int32_t self_id, u128 *a)
{
	int64_t n = 0;
	for (int i = 0; i < n_m; ++i) {
		const SeedMatch *q = &m[i];
		const uint64_t *r = q->cr;
		for (uint32_t k = 0; k < q->n; ++k) {
			uint64_t rk = r[k];
			int32_t rpos = (int32_t)((uint32_t)rk >> 1);
			if (self_id >= 0 && g.seg_name_id[rk >> 32] == self_id && (uint32_t)(g.seg_soff[rk >> 32] + (int32_t)(uint32_t)rk) == q->q_pos) continue;
			u128 *p = &a[n++];
			if ((rk & 1) == (q->q_pos & 1)) p->x = rk >> 32 << 33 | (uint64_t)(uint32_t)rpos;
			else p->x = rk >> 32 << 33 | 1ULL << 32 | (uint64_t)(uint32_t)(g.seg_len[rk >> 32] - (rpos + 1 - (int32_t)q->q_span) - 1);
			p->y = (uint64_t)q->q_span << 32 | (uint64_t)(q->q_pos >> 1);
			p->y |= (uint64_t)q->seg_id << SEED_SEG_SHIFT;
			if (q->is_tandem) p->y |= SEED_TANDEM;
			p->y |= (uint64_t)(q->n < 255? q->n : 255) << SEED_OCC_SHIFT;
		}
	}
	return n;
}

} // namespace mgb
