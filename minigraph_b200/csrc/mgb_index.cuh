// mgb_index.cuh -- the minimizer table built from the segment sketch (reference: index.c:115-165 mg_idx_a2h, :74-93 mg_idx_cal_quantile).
// Input: the (x = hash << 8 | span, y = seg << 32 | pos << 1 | strand) records k_index_sketch left in device memory.  Output: the
// open-addressing table of mgb_model.cuh (one 16-byte slot per distinct minimizer), pos[] with the occurrence lists in ascending
// position order -- the order the reference's per-bucket radix sort leaves them in and seed expansion relies on -- and the sorted
// occurrence counts the quantiles of mg_opt_update() are read from.  build_index() (mgb_engine.cu) runs the passes below between
// two stable sorts, two prefix sums and a sort of the counts; only those three primitives have a second implementation in the
// CPU simulators.  Splitting, grouping, list layout and table insertion are the passes of this file, the same code on the device
// and in the simulators.
#pragma once
#include "mgb_model.cuh"

namespace mgb {

struct IdxArgs {
	const u128 *mz; uint64_t n_mz;    // the sketch's records
	uint64_t *key, *val;              // per record: its minimizer and position (split), then sorted by (minimizer, position)
	uint32_t *flag, *rank;            // sorted record i starts a run of one minimizer; the runs up to i (1-based)
	uint32_t n_keys;                  // runs: distinct minimizers
	uint32_t *start, *cnt, *multi, *pos_off; // per run: its first record, its length, its length when above 1, its start in pos[]
	uint64_t *pos; u128 *slot; uint64_t mask; // the table (n_slots = mask + 1)
	int n;                            // items of the pass: chunks of 32 records or runs
};

// A pass over the records (or the runs) of E in chunks of 32: item c holds elements 32 c .. 32 c + 31, the lanes stride through it by
// MGB_W.  In STRIDE order warp w takes element 32 w + lane first: one element per thread, as a grid-stride loop.
template<typename E> struct IdxChunk {
	const IdxArgs &a;
	MG_HD int operator()(int c, int lane) const
	{
		const uint64_t n = E::n(a);
		for (int j = lane; j < 32; j += MGB_W) { const uint64_t i = 32 * (uint64_t)c + j; if (i < n) E::at(a, i); }
		return 0;
	}
};
struct IdxSplit {
	MG_HD static uint64_t n(const IdxArgs &a) { return a.n_mz; }
	MG_HD static void at(const IdxArgs &a, uint64_t i) { a.key[i] = a.mz[i].x >> 8, a.val[i] = a.mz[i].y; }
};
struct IdxFlag {
	MG_HD static uint64_t n(const IdxArgs &a) { return a.n_mz; }
	MG_HD static void at(const IdxArgs &a, uint64_t i) { a.flag[i] = i == 0 || a.key[i] != a.key[i - 1]; }
};
struct IdxStarts {
	MG_HD static uint64_t n(const IdxArgs &a) { return a.n_mz; }
	MG_HD static void at(const IdxArgs &a, uint64_t i) { if (a.flag[i]) a.start[a.rank[i] - 1] = (uint32_t)i; }
};
struct IdxCounts { // a singleton lives in its slot, longer lists in pos[]
	MG_HD static uint64_t n(const IdxArgs &a) { return a.n_keys; }
	MG_HD static void at(const IdxArgs &a, uint64_t r)
	{
		const uint32_t c = (r + 1 < a.n_keys? a.start[r + 1] : (uint32_t)a.n_mz) - a.start[r];
		a.cnt[r] = c, a.multi[r] = c > 1? c : 0;
	}
};
struct IdxLists {
	MG_HD static uint64_t n(const IdxArgs &a) { return a.n_mz; }
	MG_HD static void at(const IdxArgs &a, uint64_t i)
	{
		const uint32_t r = a.rank[i] - 1;
		if (a.cnt[r] > 1) a.pos[a.pos_off[r] + ((uint32_t)i - a.start[r])] = a.val[i];
	}
};

// *p = x if *p is empty (all ones); true when it was.  The lanes of a simulated warp take turns only inside the warp helpers.
MG_HD inline bool idx_claim(uint64_t *p, uint64_t x)
{
#if MGB_ON_DEVICE
	return atomicCAS((unsigned long long*)p, ~0ULL, (unsigned long long)x) == ~0ULL;
#else
	if (*p != ~0ULL) return false;
	*p = x;
	return true;
#endif
}
struct IdxInsert { // keys are distinct: a taken slot is somebody else's
	MG_HD static uint64_t n(const IdxArgs &a) { return a.n_keys; }
	MG_HD static void at(const IdxArgs &a, uint64_t r)
	{
		const uint64_t k = a.key[a.start[r]], c = a.cnt[r];
		const uint64_t x = c == 1? k << 1 | 1 : k << 1, y = c == 1? a.val[a.start[r]] : (uint64_t)a.pos_off[r] << 32 | c;
		uint64_t h = idx_slot_hash(k) & a.mask;
		while (!idx_claim(&a.slot[h].x, x)) h = (h + 1) & a.mask;
		a.slot[h].y = y;
	}
};

} // namespace mgb
