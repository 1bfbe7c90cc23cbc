// mgb_records.cuh -- the results of a mapped batch as dense tables in device memory (mgb_map_batch_dev_rec, include/mgb200.h),
// written on the device from the result blobs in the output pool, as gaf_read() reads them.
//
// The host sizes every table but the CIGAR operations from the reads' ReadOut and builds SEQ_CSR.  Then, one warp per read:
//   * count pass: each record's CIGAR operations (scanned into CIGAR_CSR) and what its div needs (GafReq, as k_gaf_req lists
//     it for dv:f; the host computes div with its libm, SURVEY H3);
//   * write pass: the read's GChains transposed into its GC rows, one 32-bit cell per lane; its LLChains and anchors copied word by
//     word; each record's CIGAR operations copied to where CIGAR_CSR puts them.
#pragma once
#include "../../include/mgb200.h"
#include "mgb_gaf.cuh"

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
};

// read r, warp-uniform; write == false: the count pass, otherwise the write pass
MG_HD inline void rec_read(const RecArgs &R, int r, int lane, bool write)
{
	const int32_t s = R.row_of[r];
	if (s < 0) return;
	const int64_t *row = R.seq_csr + 3 * (int64_t)s;
	const int64_t k0 = row[0], n_gc = row[3] - row[0], n_lc = row[4] - row[1], n_a = row[5] - row[2];
	if (n_gc == 0) return;
	const ReadBlob B = read_blob(R.pool, R.routs[r]);
	const GChain *gc = B.gc;
	if (!write) {
		for (int64_t i = lane; i < n_gc; i += MGB_W) {
			const GChain &p = gc[i];
			R.cig_off[k0 + i] = p.has_cigar? (uint64_t)p.n_cigar : 0;
			GafReq q; q.a = p.n_mini, q.b = p.n_anchor, q.q_span = p.q_span, q.kind = 0;
			R.req[k0 + i] = q;
		}
		return;
	}
	int32_t *dg = R.gc + k0 * MGB_GC_NCOL;
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
	uint32_t *dlc = R.lc + row[1] * 5;
	for (int64_t w = lane; w < n_lc * 5; w += MGB_W) dlc[w] = slc[w];
	const uint64_t *sa = (const uint64_t*)B.a;
	uint64_t *da = R.a + row[2] * 2;
	for (int64_t w = lane; w < n_a * 2; w += MGB_W) da[w] = sa[w];
	for (int64_t i = 0; i < n_gc; ++i) {
		const uint64_t c0 = R.cig_off[k0 + i], nc = R.cig_off[k0 + i + 1] - c0;
		const uint64_t *sc = nc? (const uint64_t*)(R.pool + gc[i].cigar_off) : 0;
		for (uint64_t j = lane; j < nc; j += MGB_W) R.cigar[c0 + j] = sc[j];
	}
}

// rows [0, n) of a table of w int64 columns, column j raised by base[j] (the CSR tables of a part joined behind others)
struct RecRebase { int64_t *v; int64_t n; int w; int64_t base[3]; };
MG_HD inline void rec_rebase_row(const RecRebase &B, int64_t i)
{
	for (int j = 0; j < 3; ++j) // (constant indices: base stays in registers)
		if (j < B.w) B.v[i * B.w + j] += B.base[j];
}

#ifndef MGB_HOSTSIM
__global__ void __launch_bounds__(256) k_rec_count(RecArgs R)
{
	const int lane = threadIdx.x & 31, warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), n_warp = (int)((gridDim.x * blockDim.x) >> 5);
	for (int r = warp; r < R.n; r += n_warp) rec_read(R, r, lane, false);
}
__global__ void __launch_bounds__(256) k_rec_write(RecArgs R)
{
	const int lane = threadIdx.x & 31;
	for (int r = gaf_next_read(R.next, lane); r < R.n; r = gaf_next_read(R.next, lane)) rec_read(R, r, lane, true);
}
__global__ void __launch_bounds__(256) k_rec_rebase(RecRebase B)
{
	for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B.n; i += (int64_t)gridDim.x * blockDim.x) rec_rebase_row(B, i);
}
#endif

} // namespace mgb
