// mgb_index.cuh -- the minimizer table built on the device (reference: index.c:115-165 mg_idx_a2h, :74-93 mg_idx_cal_quantile).
// Input: the (x = hash << 8 | span, y = seg << 32 | pos << 1 | strand) records k_index_sketch left in HBM.  Output: the open-addressing
// table of mgb_model.cuh (one 16-byte slot per distinct minimizer), pos[] with the occurrence lists in ascending position order --
// the order the reference's per-bucket radix sort leaves them in and seed expansion relies on -- and the sorted occurrence counts
// the quantiles of mg_opt_update() are read from.  Sorting and scans are CUB's (library code, index time only); grouping, list
// layout and table insertion are kernels of this file.  Not compiled into the CPU simulators of the tests (they keep the host build).
#pragma once
#include <cub/cub.cuh>
#include "mgb_model.cuh"

namespace mgb {

__global__ void k_idx_split(const u128 *mz, uint64_t n, uint64_t *key, uint64_t *val)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) key[i] = mz[i].x >> 8, val[i] = mz[i].y;
}
__global__ void k_idx_flag(const uint64_t *key, uint64_t n, uint32_t *flag)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) flag[i] = i == 0 || key[i] != key[i - 1];
}
// run r (1-based in rank[]) starts at element i
__global__ void k_idx_starts(const uint32_t *flag, const uint32_t *rank, uint64_t n, uint32_t *start)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) if (flag[i]) start[rank[i] - 1] = (uint32_t)i;
}
__global__ void k_idx_counts(const uint32_t *start, uint32_t n_keys, uint64_t n, uint32_t *cnt, uint32_t *multi)
{
	for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_keys; r += gridDim.x * blockDim.x) {
		const uint32_t c = (r + 1 < n_keys? start[r + 1] : (uint32_t)n) - start[r];
		cnt[r] = c, multi[r] = c > 1? c : 0; // a singleton lives in its slot, longer lists in pos[]
	}
}
__global__ void k_idx_lists(const uint32_t *rank, const uint32_t *start, const uint32_t *cnt, const uint32_t *pos_off, const uint64_t *val, uint64_t n, uint64_t *pos)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t r = rank[i] - 1;
		if (cnt[r] > 1) pos[pos_off[r] + ((uint32_t)i - start[r])] = val[i];
	}
}
__global__ void k_idx_insert(const uint64_t *key, const uint64_t *val, const uint32_t *start, const uint32_t *cnt, const uint32_t *pos_off, uint32_t n_keys,
							 u128 *slot, uint64_t mask)
{
	for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_keys; r += gridDim.x * blockDim.x) {
		const uint64_t k = key[start[r]], c = cnt[r];
		const uint64_t x = c == 1? k << 1 | 1 : k << 1, y = c == 1? val[start[r]] : (uint64_t)pos_off[r] << 32 | c;
		uint64_t h = idx_slot_hash(k) & mask;
		while (atomicCAS((unsigned long long*)&slot[h].x, ~0ULL, (unsigned long long)x) != ~0ULL) h = (h + 1) & mask; // keys are distinct: a taken slot is somebody else's
		slot[h].y = y;
	}
}

struct DevIndexOut { u128 *slot; uint64_t *pos; uint32_t *occ_sorted; uint64_t n_slots, n_pos; uint32_t n_keys; };

// everything on `stream`; the caller frees slot/pos/occ_sorted (cudaFree).  hash_bits = 2k.
inline cudaError_t build_index_device(const u128 *d_mz, uint64_t n, int hash_bits, cudaStream_t stream, DevIndexOut *out)
{
#define MGB_CU(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)
	memset(out, 0, sizeof(*out));
	uint64_t *key[2], *val[2];
	uint32_t *flag, *rank, *start = 0, *cnt = 0, *multi = 0, *pos_off = 0;
	const uint64_t n1 = n? n : 1;
	for (int b = 0; b < 2; ++b) { MGB_CU(cudaMalloc(&key[b], n1 * 8)); MGB_CU(cudaMalloc(&val[b], n1 * 8)); }
	MGB_CU(cudaMalloc(&flag, n1 * 4)); MGB_CU(cudaMalloc(&rank, n1 * 4));
	int dev = 0, n_sm = 0;
	MGB_CU(cudaGetDevice(&dev));
	MGB_CU(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	const int grid = n_sm * 8, blk = 256; // grid-stride loops: eight blocks per SM
	k_idx_split<<<grid, blk, 0, stream>>>(d_mz, n, key[0], val[0]);
	// order by (minimizer, position): a stable sort by position, then a stable sort by minimizer
	cub::DoubleBuffer<uint64_t> kb(val[0], val[1]), vb(key[0], key[1]); // first pass: positions are the keys
	size_t tmp_bytes = 0, t2 = 0;
	MGB_CU(cub::DeviceRadixSort::SortPairs(0, tmp_bytes, kb, vb, (int)n, 0, 64, stream));
	MGB_CU(cub::DeviceScan::InclusiveSum(0, t2, flag, rank, (int)n, stream));
	if (t2 > tmp_bytes) tmp_bytes = t2;
	void *tmp;
	MGB_CU(cudaMalloc(&tmp, tmp_bytes + 16));
	MGB_CU(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, kb, vb, (int)n, 0, 64, stream));
	cub::DoubleBuffer<uint64_t> kb2(vb.Current(), vb.Alternate()), vb2(kb.Current(), kb.Alternate()); // second pass: minimizers are the keys
	MGB_CU(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, kb2, vb2, (int)n, 0, hash_bits < 64? hash_bits : 64, stream));
	const uint64_t *skey = kb2.Current(), *sval = vb2.Current();
	k_idx_flag<<<grid, blk, 0, stream>>>(skey, n, flag);
	MGB_CU(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, flag, rank, (int)n, stream));
	uint32_t n_keys = 0;
	if (n) { MGB_CU(cudaMemcpyAsync(&n_keys, rank + (n - 1), 4, cudaMemcpyDeviceToHost, stream)); MGB_CU(cudaStreamSynchronize(stream)); }
	const uint32_t nk1 = n_keys? n_keys : 1;
	MGB_CU(cudaMalloc(&start, (size_t)nk1 * 4)); MGB_CU(cudaMalloc(&cnt, (size_t)nk1 * 4)); MGB_CU(cudaMalloc(&multi, (size_t)nk1 * 4)); MGB_CU(cudaMalloc(&pos_off, (size_t)nk1 * 4));
	k_idx_starts<<<grid, blk, 0, stream>>>(flag, rank, n, start);
	k_idx_counts<<<grid, blk, 0, stream>>>(start, n_keys, n, cnt, multi);
	MGB_CU(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, multi, pos_off, (int)n_keys, stream));
	uint32_t last_off = 0, last_multi = 0;
	if (n_keys) {
		MGB_CU(cudaMemcpyAsync(&last_off, pos_off + (n_keys - 1), 4, cudaMemcpyDeviceToHost, stream));
		MGB_CU(cudaMemcpyAsync(&last_multi, multi + (n_keys - 1), 4, cudaMemcpyDeviceToHost, stream));
		MGB_CU(cudaStreamSynchronize(stream));
	}
	out->n_keys = n_keys, out->n_pos = (uint64_t)last_off + last_multi;
	uint64_t n_slots = 16;
	while (n_slots < (uint64_t)n_keys * 2) n_slots <<= 1;
	out->n_slots = n_slots;
	MGB_CU(cudaMalloc(&out->slot, n_slots * sizeof(u128)));
	MGB_CU(cudaMalloc(&out->pos, (out->n_pos? out->n_pos : 1) * 8));
	MGB_CU(cudaMalloc(&out->occ_sorted, (size_t)nk1 * 4));
	MGB_CU(cudaMemsetAsync(out->slot, 0xff, n_slots * sizeof(u128), stream));
	k_idx_lists<<<grid, blk, 0, stream>>>(rank, start, cnt, pos_off, sval, n, out->pos);
	k_idx_insert<<<grid, blk, 0, stream>>>(skey, sval, start, cnt, pos_off, n_keys, out->slot, n_slots - 1);
	{ // ascending occurrence counts for the quantiles
		size_t t3 = 0;
		MGB_CU(cub::DeviceRadixSort::SortKeys(0, t3, cnt, out->occ_sorted, (int)n_keys, 0, 32, stream));
		void *tmp3 = tmp;
		if (t3 > tmp_bytes) MGB_CU(cudaMalloc(&tmp3, t3));
		MGB_CU(cub::DeviceRadixSort::SortKeys(tmp3, t3, cnt, out->occ_sorted, (int)n_keys, 0, 32, stream));
		MGB_CU(cudaStreamSynchronize(stream));
		if (tmp3 != tmp) cudaFree(tmp3);
	}
	MGB_CU(cudaGetLastError());
	for (int b = 0; b < 2; ++b) { cudaFree(key[b]); cudaFree(val[b]); }
	cudaFree(flag), cudaFree(rank), cudaFree(start), cudaFree(cnt), cudaFree(multi), cudaFree(pos_off), cudaFree(tmp);
#undef MGB_CU
	return cudaSuccess;
}

} // namespace mgb
