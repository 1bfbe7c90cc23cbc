// mgb_records.cuh -- the results of a mapped batch as dense tables in device memory (mgb_map_batch_dev_rec, include/mgb200.h),
// written on the device from the result blobs in the output pool, as gaf_read() reads them.
//
// The host sizes every table but the CIGAR operations from the reads' ReadOut and builds SEQ_CSR.  Then, one warp per read:
//   * count pass: each record's CIGAR operations (scanned into CIGAR_CSR) and what its div needs (GafReq, as k_gaf_req lists
//     it for dv:f; the host computes div with its libm, SURVEY H3);
//   * write pass: the read's GChains transposed into its GC rows, one 32-bit cell per lane; its LLChains and anchors copied word by
//     word; each record's CIGAR operations copied to where CIGAR_CSR puts them.
// With the ds tables (mgb_map_batch_dev_rec_ds) the count pass also stores each record's ds bytes and offsets (scanned into DS_CSR),
// and the write pass copies them: the text 16 bytes per lane, the offsets one per lane.  Both passes are instantiated with and
// without them (DS), so that the tables without ds run the code they ran before.
#pragma once
#include "../../include/mgb200.h"
#include "mgb_gaf.cuh"
#include "mgb_ingest.cuh"

namespace mgb {

// GC columns up to MGB_GC_FLT are the GChain words of the same index; the later ones skip n_mini and q_span
static_assert(offsetof(GChain, flt) == 4 * MGB_GC_FLT && offsetof(GChain, has_cigar) == 4 * (MGB_GC_HAS_CIGAR + 2) &&
			  offsetof(GChain, c_ee) == 4 * (MGB_GC_C_EE + 2), "GChain words and GC columns");
static_assert(sizeof(LLChain) == 20 && sizeof(u128) == 16, "LC and A rows are LLChain and u128 verbatim");

struct RecArgs {
	const ReadOut *routs;
	const char *pool;        // output pool (blob_off and the chains' cigar_off point into it)
	int n;                   // reads of the part
	const int32_t *row_of;   // [n]: the SEQ_CSR row of read r's records; -1: none
	const int64_t *seq_csr;  // [n_seq + 1][3]
	uint64_t *cig_off;       // [n_rec + 1]: CIGAR operations of record k (count pass), then its first one (scan)
	GafReq *req;             // [n_rec]: what the div of record k needs
	int32_t *gc;             // the tables (write pass)
	uint32_t *lc;
	uint64_t *a, *cigar;
	unsigned int *next;      // work counter of the write pass
	// the ds tables (DS)
	uint64_t *ds_n;          // [n_rec + 1][2]: ds bytes and offsets of record k (count pass), then its first of each (scan): DS_CSR
	char *ds;                // the tables (write pass)
	int32_t *ds_off;
};

// Bytes src[0 .. len) to dst, by all lanes: lane l writes the 16-byte-aligned chunks l, l + 32, ... of the destination, each from
// the (at most two) aligned 16-byte chunks of the source that hold its bytes, whole where the chunk is all the string's and byte by
// byte at the ends.  A source chunk that holds none of the string's bytes is not loaded.  (Records' strings follow each other in
// DS at any byte; the blob's string starts 8-aligned.)
MG_HD inline void rec_copy_bytes(char *dst, const char *src, int64_t len, int lane)
{
	const int h = (int)((uintptr_t)dst & 15);
	char *d0 = dst - h;
	const int64_t n_chunk = (h + len + 15) >> 4;
	for (int64_t c = lane; c < n_chunk; c += MGB_W) {
		const int64_t o = 16 * c - h; // the string's byte at the chunk's start (negative in the first chunk)
		const char *base = (const char*)((uintptr_t)(src + o) & ~(uintptr_t)15);
		const int sh = (int)((uintptr_t)(src + o) & 15);
		uint32_t v[8];
		for (int k = 0; k < 2; ++k) {
			uint32_t *w = v + 4 * k;
			const char *p = base + 16 * k;
			if (p < src + len && p + 16 > src) {
#if MGB_ON_DEVICE
				const uint4 x = *(const uint4*)p;
				w[0] = x.x, w[1] = x.y, w[2] = x.z, w[3] = x.w;
#else
				memcpy(w, p, 16);
#endif
			} else w[0] = w[1] = w[2] = w[3] = 0;
		}
		const int ws = sh >> 2, bs = 8 * (sh & 3);
		uint32_t q[4];
		for (int j = 0; j < 4; ++j) { // (no indexing by a variable: registers)
			const uint32_t lo = ws == 0? v[j] : ws == 1? v[j + 1] : ws == 2? v[j + 2] : v[j + 3];
			const uint32_t hi = ws == 0? v[j + 1] : ws == 1? v[j + 2] : ws == 2? v[j + 3] : v[j + 4];
			q[j] = ingest_fshr(lo, hi, bs);
		}
		char *d = d0 + 16 * c;
		const int b0 = o < 0? (int)-o : 0, b1 = len - o < 16? (int)(len - o) : 16; // the chunk's bytes that are the string's
		if (b0 == 0 && b1 == 16) {
#if MGB_ON_DEVICE
			*(uint4*)d = make_uint4(q[0], q[1], q[2], q[3]);
#else
			memcpy(d, q, 16);
#endif
		} else {
			const uint64_t lo = (uint64_t)q[1] << 32 | q[0], hi = (uint64_t)q[3] << 32 | q[2]; // (no indexing by a variable)
			for (int b = b0; b < b1; ++b) d[b] = (char)((b < 8? lo : hi) >> 8 * (b & 7));
		}
	}
}

// the ds of the n_gc records of a read from k0 on (write pass)
MG_HD inline void rec_ds(const RecArgs &R, const GChain *gc, int64_t k0, int64_t n_gc, int lane)
{
	for (int64_t i = 0; i < n_gc; ++i) {
		const uint64_t *c = R.ds_n + 2 * (k0 + i);
		const int64_t nb = (int64_t)(c[2] - c[0]), no = (int64_t)(c[3] - c[1]);
		if (nb) rec_copy_bytes(R.ds + c[0], R.pool + gc[i].ds_off, nb, lane);
		const int32_t *so = no? (const int32_t*)(R.pool + gc[i].dsoff_off) : 0;
		for (int64_t j = lane; j < no; j += MGB_W) R.ds_off[c[1] + j] = so[j];
	}
}

// Read r (warp-uniform), count pass: each record's CIGAR operations and what its div needs (DS: and its ds bytes and offsets)
template<bool DS>
struct RecCount {
	const RecArgs &a;
	MG_HD int operator()(int r, int lane) const
	{
		const int32_t s = a.row_of[r];
		if (s < 0) return 0;
		const int64_t k0 = a.seq_csr[3 * (int64_t)s], n_gc = a.seq_csr[3 * (int64_t)s + 3] - k0;
		if (n_gc == 0) return 0;
		const GChain *gc = read_blob(a.pool, a.routs[r]).gc;
		for (int64_t i = lane; i < n_gc; i += MGB_W) {
			const GChain &p = gc[i];
			a.cig_off[k0 + i] = p.has_cigar? (uint64_t)p.n_cigar : 0;
			GafReq q; q.a = p.n_mini, q.b = p.n_anchor, q.q_span = p.q_span, q.kind = 0;
			a.req[k0 + i] = q;
			if (DS) a.ds_n[2 * (k0 + i)] = p.has_cigar? (uint64_t)p.ds_len : 0, a.ds_n[2 * (k0 + i) + 1] = p.has_cigar? (uint64_t)p.n_dsoff : 0;
		}
		return 0;
	}
};

// Read r (warp-uniform), write pass: its rows of every table
template<bool DS>
struct RecWrite {
	const RecArgs &a;
	MG_HD unsigned int *counter() const { return a.next; }
	MG_HD int operator()(int r, int lane) const
	{
		const int32_t s = a.row_of[r];
		if (s < 0) return 0;
		const int64_t *row = a.seq_csr + 3 * (int64_t)s;
		const int64_t k0 = row[0], n_gc = row[3] - row[0], n_lc = row[4] - row[1], n_a = row[5] - row[2];
		if (n_gc == 0) return 0;
		const ReadBlob B = read_blob(a.pool, a.routs[r]);
		const GChain *gc = B.gc;
		int32_t *dg = a.gc + k0 * MGB_GC_NCOL;
		for (int64_t w = lane; w < n_gc * MGB_GC_NCOL; w += MGB_W) {
			const int64_t i = w / MGB_GC_NCOL;
			const int c = (int)(w - i * MGB_GC_NCOL);
			const int32_t *src = (const int32_t*)(gc + i);
			int32_t v = src[c <= MGB_GC_FLT? c : c + 2];
			if (c == MGB_GC_MAPQ) v &= 0xff;                        // mg_gchain_t's bit fields
			else if (c == MGB_GC_FLT) v &= 1;
			else if (c > MGB_GC_HAS_CIGAR && !gc[i].has_cigar) v = 0; // no mg_cigar_t
			dg[w] = v;
		}
		const uint32_t *slc = (const uint32_t*)B.lc;
		uint32_t *dlc = a.lc + row[1] * 5;
		for (int64_t w = lane; w < n_lc * 5; w += MGB_W) dlc[w] = slc[w];
		const uint64_t *sa = (const uint64_t*)B.a;
		uint64_t *da = a.a + row[2] * 2;
		for (int64_t w = lane; w < n_a * 2; w += MGB_W) da[w] = sa[w];
		for (int64_t i = 0; i < n_gc; ++i) {
			const uint64_t c0 = a.cig_off[k0 + i], nc = a.cig_off[k0 + i + 1] - c0;
			const uint64_t *sc = nc? (const uint64_t*)(a.pool + gc[i].cigar_off) : 0;
			for (uint64_t j = lane; j < nc; j += MGB_W) a.cigar[c0 + j] = sc[j];
		}
		if (DS) rec_ds(a, gc, k0, n_gc, lane);
		return 0;
	}
};

// rows [0, rows) of a table of w int64 columns, column j raised by base[j] (the CSR tables of a part joined behind others), in n
// items of 32 rows
struct RecRebase { int64_t *v; int64_t rows; int w; int64_t base[3]; int n; };
MG_HD inline void rec_rebase_row(const RecRebase &B, int64_t i)
{
	for (int j = 0; j < 3; ++j) // (constant indices: base stays in registers)
		if (j < B.w) B.v[i * B.w + j] += B.base[j];
}
// item c: rows 32 c .. 32 c + 31, the lanes striding through them by MGB_W (one row per thread on the device)
struct RecRebaseRows {
	const RecRebase &a;
	MG_HD int operator()(int c, int lane) const
	{
		for (int j = lane; j < 32; j += MGB_W) { const int64_t i = 32 * (int64_t)c + j; if (i < a.rows) rec_rebase_row(a, i); }
		return 0;
	}
};

} // namespace mgb
