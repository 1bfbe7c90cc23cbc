// mgb_tma.cuh -- bulk asynchronous copies between HBM and shared memory (sm_90a: cp.async.bulk + mbarrier; SASS UBLKCP /
// SYNCS).  One lane issues a copy of a whole contiguous record array (a read's seeds, 16 bytes each) and the warp waits on the
// transaction barrier; the way back is a bulk store of the compacted array.  Addresses and sizes are multiples of 16 bytes.
// In the CPU simulators of the tests the same calls are plain copies.
#pragma once
#include "mgb_common.cuh"

namespace mgb {

#if MGB_ON_DEVICE
MG_D inline uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
MG_D inline void mbar_init(uint64_t *bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(count) : "memory");
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); // the async proxy must see the initialised barrier
}
// global -> shared, completion counted in bytes on the barrier
MG_D inline void bulk_load(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
				 :: "r"(smem_addr(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
MG_D inline void mbar_wait(uint64_t *bar, uint32_t parity)
{
	asm volatile("{\n .reg .pred P1;\n LAB_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n @P1 bra DONE;\n bra LAB_WAIT;\n DONE:\n }"
				 :: "r"(smem_addr(bar)), "r"(parity) : "memory");
}
// shared -> global; the shared source may be reused after bulk_store_wait()
MG_D inline void bulk_store(void *dst_gmem, const void *src_smem, uint32_t bytes)
{
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // the warp's ordinary stores to the source, before the async proxy reads it
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst_gmem), "r"(smem_addr(src_smem)), "r"(bytes) : "memory");
	asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
MG_D inline void bulk_store_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); } // complete: later kernels and this warp's own loads see the data
#else
inline void mbar_init(uint64_t *bar, uint32_t) { *bar = 0; }
inline void bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *) { memcpy(dst, src, bytes); }
inline void mbar_wait(uint64_t *, uint32_t) {}
inline void bulk_store(void *dst, const void *src, uint32_t bytes) { memcpy(dst, src, bytes); }
inline void bulk_store_wait() {}
#endif

} // namespace mgb
