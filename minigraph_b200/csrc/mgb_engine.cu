// mgb_engine.cu -- host side of libmgb200.so: model construction, batch dispatcher and the C ABI (include/mgb200.h).
//
// Compiled by nvcc for sm_90a (H100) into the product library.  With -DMGB_HOSTSIM the same file is compiled by g++ into
// the simulators of tests/hostsim, where "device memory" is host memory and a "launch" is a loop over the items, each run by
// one simulated warp: a single lane in libmgb_hostsim.so, 32 lanes as fibres in libmgb_hostsim32.so (-DMGB_SIM_LANES=32,
// mgb_simlanes.h).  Those builds exist only so that the CPU-only unit tests can exercise the control flow of the kernels.
// They are never loaded by the product path; the product library refuses to work without a CUDA device.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <vector>
#include <array>
#include <memory>
#include <algorithm>
#include <string>
#include <chrono>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <functional>
#include <optional>
#include <unordered_map>
#include "mgb_hostpool.h"

#include "../../include/mgb200.h"
#include "mgb_galign.cuh"
#include "mgb_gaf.cuh"
#include "mgb_ingest.cuh"
#include "mgb_fastx.cuh"
#include "mgb_records.cuh"

#ifndef MGB_HOSTSIM
#include <cuda_runtime.h>
#include "mgb_index.cuh"
#endif

using namespace mgb;

// ---------------------------------------------------------------------------------------------------------------
// errors, parameters
// ---------------------------------------------------------------------------------------------------------------

static std::string g_last_error;
static void set_error(const std::string &s) { g_last_error = s; fprintf(stderr, "[E::mgb200] %s\n", s.c_str()); }

// Per worker, first pass.  The slots' arenas take slots x SMs x workers_per_sm x arena_mb of HBM (3 x 132 x 32 x 3 MB = 37 GiB on an
// H100), which leaves the rest of its 80 GB to the output pools and the large-arena retry pass; a read needs far less than 3 MB
// (1.5 MB at most on the bench workloads), and one that needs more is redone with a large arena.
static int64_t p_arena_mb = 3;
static int64_t p_arena_big_mb = 1024; // per worker, retry pass
static int64_t p_workers_per_sm = 32;
static int64_t p_device = 0;
static int64_t p_host_threads = 0; // 0: min(16, hardware threads)
static int64_t p_slots = 3;            // mg_map_batch calls that may run at once on one index (each on its own slot: stream, buffers, arenas)
static int64_t p_slot_workers = 0;
static int64_t p_lab_cache = 1;        // 0: graph chaining searches its walks per read instead of keeping per-source labels in HBM (mgb_gclabel.cuh)

extern "C" const char *mgb_last_error(void) { return g_last_error.c_str(); }
extern "C" const char *mgb_version(void) { return "mgb200-r1"; }
extern "C" int mgb_set_param(const char *key, int64_t value)
{
	if (!strcmp(key, "arena_mb")) p_arena_mb = value;
	else if (!strcmp(key, "arena_big_mb")) p_arena_big_mb = value;
	else if (!strcmp(key, "workers_per_sm")) p_workers_per_sm = value;
	else if (!strcmp(key, "device")) p_device = value;
	else if (!strcmp(key, "host_threads")) p_host_threads = value;
	else if (!strcmp(key, "slots")) p_slots = value;
	else if (!strcmp(key, "slot_workers")) p_slot_workers = value;
	else if (!strcmp(key, "lab_cache")) p_lab_cache = value;
	else return -1;
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// device memory shim
// ---------------------------------------------------------------------------------------------------------------

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// A failed CUDA call (out of memory, a fault in a kernel) unwinds to the C entry point, which returns NULL / a negative code with
// the reason in mgb_last_error(); the library never ends the host process on its own.
struct MgbError { int code; };
#ifdef MGB_HOSTSIM
static bool dev_ok(int dev = -1) { (void)dev; return true; }
static void *dmalloc(size_t n) { void *p = malloc(n? n : 16); return p; }
static void dfree(void *p) { free(p); }
static void dzero(void *d, size_t n) { if (n) memset(d, 0, n); }
static void d2d(void *d, const void *s, size_t n) { if (n) memcpy(d, s, n); }
static void dfill(void *d, int v, size_t n) { if (n) memset(d, v, n); }
static void dsync() {}
static int dev_sm_count() { return 2; }
static size_t dev_free_mem() { return (size_t)8 << 30; }
typedef int DevStream;
typedef double DevEvent; // the host clock when it was recorded
static void dev_bind(int dev, DevStream s) { (void)dev, (void)s; }
static void h2d_async(void *d, const void *h, size_t n) { if (n) memcpy(d, h, n); }
static void d2h_async(void *h, const void *d, size_t n) { if (n) memcpy(h, d, n); }
static void d2d_peer(void *d, int d_dev, const void *s, int s_dev, size_t n) { (void)d_dev, (void)s_dev; if (n) memcpy(d, s, n); }
static void ev_record(DevEvent &e) { e = now_ms(); }
static void ev_wait(DevEvent &e) { (void)e; }
static double ev_ms(DevEvent &a, DevEvent &b) { return b - a; }
#else
#define CUDA_OK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { set_error(std::string(#call) + ": " + cudaGetErrorString(_e)); throw MgbError{MGB_E_INTERNAL}; } } while (0)
// every host thread that drives a slot of the batch pipeline works on its own stream
static thread_local cudaStream_t t_stream = 0;
static bool dev_ok(int dev = -1)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return false;
	if (cudaSetDevice(dev >= 0? dev : (int)p_device) != cudaSuccess) return false;
	return true;
}
static void *dmalloc(size_t n) { void *p = 0; CUDA_OK(cudaMalloc(&p, n? n : 16)); return p; }
static void dfree(void *p) { if (p) cudaFree(p); }
static void dsync() { CUDA_OK(cudaStreamSynchronize(t_stream)); }
static void dzero(void *d, size_t n) { if (n) CUDA_OK(cudaMemsetAsync(d, 0, n, t_stream)); }
static void d2d(void *d, const void *s, size_t n) { if (n) CUDA_OK(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToDevice, t_stream)); }
static void dfill(void *d, int v, size_t n) { if (n) CUDA_OK(cudaMemsetAsync(d, v, n, t_stream)); }
static int dev_sm_count() { static int v = 0; if (v == 0) { int d = 0; CUDA_OK(cudaGetDevice(&d)); CUDA_OK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d)); } return v; } // (the devices of one box are alike)
static size_t dev_free_mem() { size_t f = 0, t = 0; CUDA_OK(cudaMemGetInfo(&f, &t)); return f; }
typedef cudaStream_t DevStream;
typedef cudaEvent_t DevEvent;
// the calling thread's device and stream (0: the device's default stream)
static void dev_bind(int dev, DevStream s) { cudaSetDevice(dev); t_stream = s; }
// copies that do not wait: the host memory must be page-locked and stay untouched until the stream gets past them
static void h2d_async(void *d, const void *h, size_t n) { if (n) CUDA_OK(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, t_stream)); }
static void d2h_async(void *h, const void *d, size_t n) { if (n) CUDA_OK(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, t_stream)); }
// from another device's memory (or the same device's)
static void d2d_peer(void *d, int d_dev, const void *s, int s_dev, size_t n) { if (n) CUDA_OK(cudaMemcpyPeerAsync(d, d_dev, s, s_dev, n, t_stream)); }
static void ev_record(DevEvent &e) { CUDA_OK(cudaEventRecord(e, t_stream)); }
static void ev_wait(DevEvent &e) { CUDA_OK(cudaEventSynchronize(e)); }
static double ev_ms(DevEvent &a, DevEvent &b) { float t = 0; return cudaEventElapsedTime(&t, a, b) == cudaSuccess? t : 0; }
#endif
static void h2d(void *d, const void *h, size_t n) { if (n) h2d_async(d, h, n), dsync(); }
static void d2h(void *h, const void *d, size_t n) { if (n) d2h_async(h, d, n), dsync(); }
// kernels launched by the calling thread (every launcher counts its own): map_batch_on() counts those of a batch
static thread_local int64_t t_launches = 0;

// n elements of device memory, freed when the holder goes out of scope (also when a CUDA call throws) unless release()d
template<typename T> struct DevBuf {
	T *p;
	explicit DevBuf(size_t n) : p((T*)dmalloc(n * sizeof(T))) {}
	DevBuf(DevBuf &&o) : p(o.p) { o.p = 0; }
	DevBuf(const DevBuf &) = delete;
	DevBuf &operator=(const DevBuf &) = delete;
	~DevBuf() { dfree((void*)p); }
	operator T*() const { return p; }
	T *release() { T *r = p; p = 0; return r; }
};
// a device copy of the host array h[0..n)
template<typename T> static DevBuf<T> upload(const T *h, size_t n)
{
	DevBuf<T> d(n);
	h2d(d, h, n * sizeof(T));
	return d;
}

// grow-only buffers kept across batches: device memory, or page-locked host memory for fast H2D/D2H; freed with their owner
struct GrowBuf {
	void *p; size_t cap; bool host;
	GrowBuf(bool host_ = false) : p(0), cap(0), host(host_) {}
	GrowBuf(const GrowBuf &) = delete;
	GrowBuf &operator=(const GrowBuf &) = delete;
	~GrowBuf() { release(); }
	void release()
	{
		if (p == 0) return;
#ifdef MGB_HOSTSIM
		free(p);
#else
		if (host) cudaFreeHost(p); else cudaFree(p);
#endif
		p = 0, cap = 0;
	}
	void *ensure(size_t n)
	{
		if (n <= cap && p) return p;
		release();
		size_t c = n + n / 4 + 4096;
#ifdef MGB_HOSTSIM
		p = malloc(c);
#else
		if (host) CUDA_OK(cudaHostAlloc(&p, c, cudaHostAllocDefault)); else CUDA_OK(cudaMalloc(&p, c));
#endif
		cap = c;
		return p;
	}
};

// fn(0) .. fn(n - 1) on nt threads of pool; on the calling thread when there is little to do
static void pfor(mgb::HostPool &pool, int nt, int64_t n, const std::function<void(int64_t)> &fn)
{
	if (n < 256 || nt <= 1) { for (int64_t i = 0; i < n; ++i) fn(i); return; }
	pool.run(n, nt, fn);
}

// ---------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------

struct LaunchArgs {
	PipeCtx c;
	ReadOut *routs;
	const int32_t *rid_list; // NULL: reads 0..n-1
	int32_t n_work;
	const unsigned int *n_work_dev; // non-NULL: the number of items is read on the device (known only after the kernel in front)
	char *arena_base;
	uint64_t arena_bytes;
	uint64_t *arena_peak;    // per worker
	int64_t job_start;       // first job of this launch (bridging jobs, tier-1 gap jobs)
	// segment sketch (index build)
	Pool *pool_mz; u128 *mz;
};

// The stages of the pipeline, one kernel each (the table behind stage_loop_thread()).  Stages 0-9 index mgb_stats_t.t_kernel_ms
// and capi.KERNEL_NAMES.
enum Stage { S_SEED = 0, S_CHAIN = 1, S_GCHAIN = 2, S_INDEX_SKETCH = 3, S_WFA_SMALL = 4, S_FINISH = 5, S_WFA_MID = 6, S_WFA_BIG = 7, S_GWFA = 8,
             S_GCHAIN_GEN = 9, S_LABELS = 10, S_LABELS_BIG = 11, S_CHAIN_RESCUE = 12 };
// How one item of a stage runs: entered by all lanes of the warp, by lane 0 alone (with the warp's arena), or one item per
// thread (with 1/32 of the warp's arena)
enum class ItemMode { WARP, LANE0, THREAD };
// Where a failed item is recorded: on its read, found as the item itself, as rescue_list[item], through its bridging job or
// through its gap job of tier 1/2/3; in the one status word of the index build; or nowhere
enum class FailTo { READ, RESCUE_LIST, BRIDGE_JOB, GAP_JOB_T1, GAP_JOB_T2, GAP_JOB_T3, INDEX_STATUS, NOWHERE };
template<int S> struct StageSpec;

template<int S>
MG_HD inline int run_stage(const LaunchArgs &L, int item, Arena &A, int lane, int32_t *smem)
{
	if (S == S_SEED) return stage_seed(L.c, item, A, lane, smem);
	if (S == S_CHAIN) return stage_chain<0>(L.c, item, A, lane, smem);
	if (S == S_CHAIN_RESCUE) return stage_chain<1>(L.c, L.c.rescue_list[item], A, lane, smem); // the reads k_chain listed
	if (S == S_GCHAIN) return stage_gchain(L.c, L.routs, item, A, lane);
	if (S == S_LABELS) return label_job(A, L.c.g, L.c.lab, item, 0);
	if (S == S_LABELS_BIG) return label_job(A, L.c.g, L.c.lab, item, 1); // lane 0 with the whole arena of its warp
	if (S == S_FINISH) return stage_finish(L.c, L.routs, item, A, lane);
	if (S == S_GWFA) return gwfa_job_run(A, L.c, L.job_start + item, lane, smem);
	if (S == S_GCHAIN_GEN) return stage_gchain_gen(L.c, L.routs, item, A, lane);
	if (S == S_INDEX_SKETCH) { // sketch one graph segment for the index (reference: index.c:200-205)
		AVec<u128> mv;
		avec_init(mv);
		int32_t len = L.c.g.seg_len[item];
		if (len <= 0) return 0;
		MGB_TRY(sketch_seq(A, g_vseq(L.c.g, (uint32_t)item << 1), len, L.c.ix.w, L.c.ix.k, (uint32_t)item, mv));
		int64_t off = pool_alloc(L.pool_mz, (uint64_t)mv.n * sizeof(u128));
		if (off < 0) return MGB_E_POOL;
		u128 *dst = L.mz + off / (int64_t)sizeof(u128);
		for (int64_t i = 0; i < mv.n; ++i) dst[i] = mv.a[i];
		return 0;
	}
	return MGB_E_INTERNAL;
}

// record a failure: per read for the mapping stages, a single status word for the index build
template<int S>
MG_HD inline void stage_fail(const LaunchArgs &L, int item, int rc)
{
	constexpr FailTo f = StageSpec<S>::fail;
	if (f == FailTo::NOWHERE) return; // (labels) a source that could not be finished is searched again by the read that needs it
	if (f == FailTo::INDEX_STATUS) {
#if MGB_ON_DEVICE
		atomicMin((int*)L.routs, rc);
#else
		if (rc < *(int*)L.routs) *(int*)L.routs = rc;
#endif
		return;
	}
	int rid = f == FailTo::BRIDGE_JOB? L.c.gjobs[L.job_start + item].rid : f == FailTo::GAP_JOB_T1? L.c.jobs[L.job_start + item].rid : f == FailTo::GAP_JOB_T2? L.c.jobs[L.c.jobq[0][item]].rid
			: f == FailTo::GAP_JOB_T3? L.c.jobs[L.c.jobq[1][item]].rid : f == FailTo::RESCUE_LIST? L.c.rescue_list[item] : item;
	L.c.meta[rid].status = rc; // benign race between jobs of one read: any negative code triggers the redo
	L.routs[rid].status = rc;
}

// The gap jobs of the WFA stages, as the traceback batch of a warp sees them (WfaBatch): the items of k_wfa_small are jobs from
// job_start on, those of k_wfa_mid and k_wfa_big the queues tiers 1 and 2 filled.
MG_HD constexpr bool is_wfa_stage(int S) { return S == S_WFA_SMALL || S == S_WFA_MID || S == S_WFA_BIG; }
template<int S>
struct WfaStageGaps {
	const LaunchArgs &L;
	int32_t *smem;
	static constexpr int tier = S == S_WFA_SMALL? 1 : S == S_WFA_MID? 2 : 3;
	MG_HD int run(int item, Arena &A, WfTbJob *tb, int lane) const
	{
		return wfa_job_run(A, L.c, tier == 1? L.job_start + item : (int64_t)L.c.jobq[tier - 2][item], lane, smem, tier, tb);
	}
	MG_HD int done(const WfTbJob &b, int lane) const { return wfa_job_finish(L.c, b, smem, tier, lane); }
	MG_HD void fail(int item, int rc, int lane) const { if (lane == 0) stage_fail<S>(L, item, rc); }
	MG_HD void traced(unsigned long long cyc, int lane) const { if (lane == 0) prof_add(L.c, PROF_WFA_TB_CYC, cyc); }
};

// What a warp of stage S does to its slice of shared memory before its first item (S < 0: nothing).  Warp-uniform.
template<int S>
MG_HD inline void stage_warp_init(int32_t *smem, int lane)
{
	if (S == S_CHAIN || S == S_CHAIN_RESCUE) chain_smem_init(smem, lane);
	if ((S == S_WFA_SMALL || S == S_WFA_MID) && lane == 0) { unsigned long long *ck = wfa_cig_chunk(smem, S == S_WFA_SMALL? 1 : 2); ck[0] = ck[1] = 0; } // no slice of the CIGAR pool yet
}

#ifndef MGB_HOSTSIM
// One warp per work item; items are pulled from a global counter so that long items do not stall a wave.
// Every mapping stage is warp-uniform (all lanes enter the stage function, see mgb_common.cuh).
template<int S>
__device__ __forceinline__ void stage_loop(const LaunchArgs &L)
{
	typedef StageSpec<S> Spec;
	const int lane = threadIdx.x & 31;
	const int worker = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
	Arena A;
	arena_init(A, L.arena_base + (uint64_t)worker * L.arena_bytes, L.arena_bytes);
	extern __shared__ int4 dyn_smem[];
	int32_t *smem = Spec::smem? (int32_t*)((char*)dyn_smem + (size_t)(threadIdx.x >> 5) * Spec::smem) : 0;
	stage_warp_init<S>(smem, lane);
	prof_block_begin();
	const int n_work = L.n_work_dev? (int)*L.n_work_dev : L.n_work;
	const WfaStageGaps<S> gaps{L, smem};
	WfaBatch<WfaStageGaps<S>> batch; // the WFA stages keep the arena across the gaps of a batch
	if constexpr (is_wfa_stage(S)) batch.open(A);
	int next_item = 0, have = 0;
	for (;;) {
		if (have == 0) {
			if (lane == 0) next_item = (int)atomicAdd(L.c.next_read, (unsigned int)Spec::grab);
			next_item = __shfl_sync(0xffffffffu, next_item, 0);
			have = Spec::grab;
		}
		int item = next_item++;
		--have;
		if (item >= n_work) break;
		if (L.rid_list) item = L.rid_list[item];
		if constexpr (is_wfa_stage(S)) batch.add(gaps, item, A, lane);
		else if (Spec::mode == ItemMode::WARP) {
			A.top = 0;
			int rc = run_stage<S>(L, item, A, lane, smem);
			if (rc < 0 && lane == 0) stage_fail<S>(L, item, rc);
		} else if (lane == 0) {
			A.top = 0;
			int rc = run_stage<S>(L, item, A, 0, 0);
			if (rc < 0) stage_fail<S>(L, item, rc);
		}
		__syncwarp();
	}
	if constexpr (is_wfa_stage(S)) batch.flush(gaps, A, lane);
	if (lane == 0 && L.arena_peak) L.arena_peak[worker] = A.peak > L.arena_peak[worker]? A.peak : L.arena_peak[worker];
	prof_block_end(L.c.prof);
}

// Thread-per-item variant for the stages whose control flow is sequential: every THREAD pulls its own item and owns
// 1/32 of the warp's arena.  The 32 lanes of a warp diverge completely, but the hardware interleaves the diverged
// lanes, so 32x more items are in flight per warp and their memory latencies overlap.
template<int S>
__device__ __forceinline__ void stage_loop_thread(const LaunchArgs &L)
{
	const int lane = threadIdx.x & 31;
	const int worker = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
	const uint64_t sub = (L.arena_bytes / 32) & ~(uint64_t)15;
	Arena A;
	arena_init(A, L.arena_base + (uint64_t)worker * L.arena_bytes + (uint64_t)lane * sub, sub);
	prof_block_begin();
	const int n_work = L.n_work_dev? (int)*L.n_work_dev : L.n_work;
	for (;;) {
		int item = (int)atomicAdd(L.c.next_read, 1u);
		if (item >= n_work) break;
		if (L.rid_list) item = L.rid_list[item];
		A.top = 0;
		int rc = run_stage<S>(L, item, A, -1, 0);
		if (rc < 0) stage_fail<S>(L, item, rc);
	}
	if (L.arena_peak) atomicMax((unsigned long long*)&L.arena_peak[worker], (unsigned long long)A.peak);
	prof_block_end(L.c.prof);
}
#endif

// One row per stage: its kernel (named, so that profiles read well), warps per block, blocks per SM wanted, bytes of shared
// memory per warp, items taken per ticket of the work counter (the short jobs of the on-chip WFA tiers four at a time: one
// contended ticket per four jobs), how an item runs and where a failure is recorded.  The kernel's __launch_bounds__ are its
// launch shape; MGB_STAGE_BOUNDS gives a kernel bounds of its own.
#define MGB_STAGE(KERNEL, S, WARPS, MINB, SMEM, GRAB, MODE, FAIL) MGB_STAGE_BOUNDS(KERNEL, S, WARPS, MINB, SMEM, GRAB, MODE, FAIL, (WARPS) * 32, MINB)
#ifdef MGB_HOSTSIM
#define MGB_STAGE_KERNEL(KERNEL, S)
#else
#define MGB_STAGE_KERNEL(KERNEL, S) \
	__global__ void __launch_bounds__(StageSpec<S>::bound_threads, StageSpec<S>::bound_minb) KERNEL(LaunchArgs L) \
	{ if constexpr (StageSpec<S>::mode == ItemMode::THREAD) stage_loop_thread<S>(L); else stage_loop<S>(L); } \
	void (*StageSpec<S>::kernel())(LaunchArgs) { return KERNEL; }
#endif
#define MGB_STAGE_BOUNDS(KERNEL, S, WARPS, MINB, SMEM, GRAB, MODE, FAIL, BOUND_THREADS, BOUND_MINB) \
	template<> struct StageSpec<S> { \
		static constexpr int warps = WARPS, minb = MINB, smem = SMEM, grab = GRAB, bound_threads = BOUND_THREADS, bound_minb = BOUND_MINB; \
		static constexpr ItemMode mode = ItemMode::MODE; static constexpr FailTo fail = FailTo::FAIL; static void (*kernel())(LaunchArgs); \
	}; \
	MGB_STAGE_KERNEL(KERNEL, S)

//        kernel           stage           warps blocks shared memory per warp   grab  item   failure
MGB_STAGE(k_seed,          S_SEED,         4,    8,     SKETCH_SMEM_BYTES,       1,    WARP,  READ)         // K1-K3: sketch, index lookup, seed sort
MGB_STAGE(k_chain,         S_CHAIN,        7,    2,     CHAIN_SMEM_BYTES,        1,    WARP,  READ)         // K4/K5: linear chaining on chip (seeds bulk-loaded into shared memory), 2 x 7 slices of 16 KB per SM
MGB_STAGE(k_chain_rescue,  S_CHAIN_RESCUE, 6,    2,     CHAIN_RESCUE_SMEM_BYTES, 1,    WARP,  RESCUE_LIST)  // K5: long-join rescue (RMQ chaining) of the reads k_chain listed, 2 x 6 slices of 18 KB per SM
MGB_STAGE(k_gchain,        S_GCHAIN,       4,    8,     0,                       1,    WARP,  READ)         // K6: graph chaining DP + k-shortest walks, overlap resolution, bridging plan
MGB_STAGE(k_gwfa,          S_GWFA,         4,    4,     GWF_SHARED_BYTES,        1,    WARP,  BRIDGE_JOB)   // K7a: bridging alignments (graph wavefront), one warp per bridge
MGB_STAGE(k_gchain_gen,    S_GCHAIN_GEN,   4,    4,     0,                       1,    WARP,  READ)         // K7b: graph-chain materialisation, post filters, mapq, alignment plan
MGB_STAGE(k_index_sketch,  S_INDEX_SKETCH, 4,    8,     0,                       1,    LANE0, INDEX_STATUS) // index build: sketch of graph segments
MGB_STAGE(k_wfa_small,     S_WFA_SMALL,    4,    5,     WfTier1::STRIDE,         4,    WARP,  GAP_JOB_T1)   // K8a tier 1: small gaps, wavefronts + traceback bytes in shared memory
MGB_STAGE(k_wfa_mid,       S_WFA_MID,      2,    7,     WfTier2::STRIDE,         4,    WARP,  GAP_JOB_T2)   // K8a tier 2: mid-size gaps, wavefronts in shared memory, carried on in the arena ring of tier 3 past 254 diagonals; longer sides in that ring from the start (128 registers at 7 blocks per SM, no spills)
MGB_STAGE(k_wfa_big,       S_WFA_BIG,      4,    4,     0,                       1,    WARP,  GAP_JOB_T3)   // K8a tier 3: anything else, wavefronts in the worker arena (128 registers at 4 blocks per SM)
MGB_STAGE(k_finish,        S_FINISH,       4,    8,     0,                       1,    WARP,  READ)         // K8b: CIGAR stitching, ds strings, result blobs
MGB_STAGE(k_gc_labels,     S_LABELS,       4,    8,     0,                       1,    THREAD, NOWHERE)     // reachability labels of new source vertices, one search per thread (mgb_gclabel.cuh)
MGB_STAGE(k_gc_labels_big, S_LABELS_BIG,   4,    8,     0,                       1,    LANE0, NOWHERE)      // the few sources whose search outgrew a thread's share of the arena: one per warp

// Longest-first order of a job list (a tail of a few long jobs otherwise decides the kernel time).  Jobs are binned by
// size, four bins per octave, largest first; the order inside a bin does not matter (results do not depend on it).
MG_HD inline int order_bin(uint32_t key)
{
	uint32_t x = key + 1, lz = 0;
	while ((x >> lz) > 1) ++lz; // floor(log2(x))
	int b = (int)(lz * 4 + (lz >= 2? ((x >> (lz - 2)) & 3) : 0));
	return 63 - (b > 63? 63 : b);
}
// kind 0: bridging jobs [job_start, job_start+n), key = query length; kind 1: alignment jobs listed in q[0..n), key = tl + ql;
// kind 2: reads 0..n-1, key = number of linear chains
MG_HD inline uint32_t order_key(const LaunchArgs &L, int kind, const int32_t *q, int i)
{
	if (kind == 0) return (uint32_t)L.c.gjobs[L.job_start + i].ql;
	if (kind == 2) return (uint32_t)L.c.meta[i].n_lc; // reads by their number of linear chains (graph chaining is roughly quadratic in it)
	const WfaJob &J = L.c.jobs[q[i]];
	return (uint32_t)(J.tl + J.ql);
}
#ifndef MGB_HOSTSIM
__global__ void __launch_bounds__(1024) k_job_order(LaunchArgs L, int kind, const int32_t *q, int n, const unsigned int *n_dev, int32_t *order)
{
	if (n_dev) n = (int)*n_dev;
	__shared__ unsigned int cnt[64];
	const int tid = threadIdx.x;
	if (tid < 64) cnt[tid] = 0;
	__syncthreads();
	for (int i = tid; i < n; i += 1024) atomicAdd(&cnt[order_bin(order_key(L, kind, q, i))], 1u);
	__syncthreads();
	if (tid == 0) { unsigned int acc = 0; for (int b = 0; b < 64; ++b) { unsigned int c = cnt[b]; cnt[b] = acc; acc += c; } }
	__syncthreads();
	for (int i = tid; i < n; i += 1024) order[atomicAdd(&cnt[order_bin(order_key(L, kind, q, i))], 1u)] = i;
}
#endif
static void make_job_order(const LaunchArgs &L, int kind, const int32_t *q, int n, int32_t *order, const unsigned int *n_dev = 0)
{
#ifndef MGB_HOSTSIM
	k_job_order<<<1, 1024, 0, t_stream>>>(L, kind, q, n, n_dev, order);
	CUDA_OK(cudaGetLastError());
#else
	if (n_dev) n = (int)*n_dev;
	unsigned int cnt[65] = {0};
	for (int i = 0; i < n; ++i) ++cnt[order_bin(order_key(L, kind, q, i)) + 1];
	for (int b = 0; b < 64; ++b) cnt[b + 1] += cnt[b];
	for (int i = 0; i < n; ++i) order[cnt[order_bin(order_key(L, kind, q, i))]++] = i;
#endif
	++t_launches;
}

// ---- result blobs in read order ----
// The kernels allocate a read's two result blobs from the output pool in completion order.  Before the copy to the host they are
// closed up in read order, so that the copy can go in a few pieces and the host threads can build the mg_gchains_t of one piece
// while the next one is still on the wire.
struct PackArgs { ReadOut *routs; const ReadMeta *meta; int n; const char *pool; char *packed; uint64_t *off; };
MG_HD inline uint64_t pack_size(const PackArgs &P, int r)
{
	const ReadOut &ro = P.routs[r];
	if (P.meta[r].status != 0 || ro.status != 0 || ro.n_gc <= 0) return 0;
	return (((uint64_t)ro.blob_size + 15) & ~(uint64_t)15) + (((uint64_t)ro.blob2_size + 15) & ~(uint64_t)15);
}
// Read r's two blobs copied to their place in read order, and its chains' offsets into them moved along (warp-uniform)
struct PackRead {
	const PackArgs &a;
	MG_HD int operator()(int r, int lane) const
	{
		ReadOut &ro = a.routs[r];
		const uint64_t sz = a.off[r + 1] - a.off[r];
		if (sz == 0) return 0;
		const uint64_t n1 = ((uint64_t)ro.blob_size + 15) & ~(uint64_t)15, n2 = sz - n1;
		const uint64_t *s1 = (const uint64_t*)(a.pool + ro.blob_off), *s2 = (const uint64_t*)(a.pool + ro.blob2_off);
		uint64_t *d1 = (uint64_t*)(a.packed + a.off[r]), *d2 = d1 + n1 / 8;
		for (uint64_t i = lane; i < n1 / 8; i += MGB_W) d1[i] = s1[i];
		for (uint64_t i = lane; i < n2 / 8; i += MGB_W) d2[i] = s2[i];
		// every lane reads blob2_off before the sync, so that lane 0's store of the new offsets below comes after all the loads
		const int64_t delta = (int64_t)(a.off[r] + n1) - ro.blob2_off;
		warp_sync();
		GChain *gc = (GChain*)d1;
		for (int i = lane; i < ro.n_gc; i += MGB_W)
			if (gc[i].has_cigar) gc[i].cigar_off += delta, gc[i].ds_off += delta, gc[i].dsoff_off += delta;
		if (lane == 0) ro.blob_off = (int64_t)a.off[r], ro.blob2_off = (int64_t)(a.off[r] + n1);
		return 0;
	}
};

// ---- reads cross PCIe 2 bits per base ----
// Host: A/C/G/T -> 0..3 (the order of seq_nt4_table, sketch.c:9-26), 32 bases per 64-bit word, base i in bits 2*(i%32).  Returns false
// when the read holds any other byte (N, lower case, IUPAC): such a read travels as ASCII, because the alignment compares raw bytes.
static bool pack_read_scalar(const char *s, int len, uint64_t *out)
{
	static const struct Tab { uint8_t c[256]; Tab() { for (int i = 0; i < 256; ++i) c[i] = 4; c['A'] = 0, c['C'] = 1, c['G'] = 2, c['T'] = 3; } } T; // filled once: several host threads pack at once
	const uint8_t *tab = T.c;
	unsigned bad = 0;
	for (int w = 0; w * 32 < len; ++w) {
		uint64_t x = 0;
		const int n = len - w * 32 < 32? len - w * 32 : 32;
		for (int j = 0; j < n; ++j) { const unsigned c = tab[(uint8_t)s[w * 32 + j]]; bad |= c; x |= (uint64_t)(c & 3) << (2 * j); }
		out[w] = x;
	}
	return (bad & 4) == 0;
}
#if defined(__x86_64__) && !defined(MGB_NO_SIMD_PACK)
#include <immintrin.h>
// 16 bases per step: code = (b >> 1 & 3) with G and T swapped back, checked by mapping the codes to letters again
__attribute__((target("ssse3,sse4.1,bmi2"))) static bool pack_read_simd(const char *s, int len, uint64_t *out)
{
	const __m128i letters = _mm_setr_epi8('A', 'C', 'G', 'T', 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0), three = _mm_set1_epi8(3), one = _mm_set1_epi8(1);
	int i = 0;
	unsigned ok = 0xffffu;
	for (; i + 32 <= len; i += 32) {
		uint64_t word = 0;
		for (int h = 0; h < 2; ++h) {
			const __m128i x = _mm_loadu_si128((const __m128i*)(s + i + 16 * h));
			__m128i c = _mm_and_si128(_mm_srli_epi16(x, 1), three);              // A0 C1 T2 G3
			c = _mm_xor_si128(c, _mm_and_si128(_mm_srli_epi16(c, 1), one));       // A0 C1 G2 T3
			ok &= (unsigned)_mm_movemask_epi8(_mm_cmpeq_epi8(_mm_shuffle_epi8(letters, c), x));
			const uint64_t lo = _pext_u64((uint64_t)_mm_cvtsi128_si64(c), 0x0303030303030303ULL), hi = _pext_u64((uint64_t)_mm_extract_epi64(c, 1), 0x0303030303030303ULL);
			word |= (lo | hi << 16) << (32 * h);
		}
		out[i >> 5] = word;
	}
	bool good = ok == 0xffffu;
	if (i < len) good &= pack_read_scalar(s + i, len - i, out + (i >> 5));
	return good;
}
static bool pack_read(const char *s, int len, uint64_t *out)
{
	static const bool simd = __builtin_cpu_supports("ssse3") && __builtin_cpu_supports("bmi2") && __builtin_cpu_supports("sse4.1");
	return simd? pack_read_simd(s, len, out) : pack_read_scalar(s, len, out);
}
#else
static bool pack_read(const char *s, int len, uint64_t *out) { return pack_read_scalar(s, len, out); }
#endif

// Device: the ASCII copy of the packed reads (alignment, ds strings and the sequential sketch read bytes): one 64-bit word = 32 bases =
// two 16-byte stores per lane, a warp per read.
struct UnpackArgs { const uint64_t *pk, *pk_off, *seq_off; const int32_t *seq_len; char *seq; int n; };
MG_HD inline void unpack_word(const UnpackArgs &U, int r, int64_t wd)
{
	const int32_t len = U.seq_len[r];
	const uint64_t x = U.pk[U.pk_off[r] + (uint64_t)wd];
	uint32_t q[8];
	for (int j = 0; j < 8; ++j) { // four bases -> four letters: 'A' + {0, 2, 6, 19}
		uint32_t o = 0;
		for (int b = 0; b < 4; ++b) { const uint32_t c = (uint32_t)(x >> (2 * (4 * j + b))) & 3u; o |= (0x41u + ((0x13060200u >> (8 * c)) & 0xffu)) << (8 * b); }
		q[j] = o;
	}
	uint32_t *dst = (uint32_t*)(U.seq + U.seq_off[r] + (uint64_t)wd * 32);
	for (int h = 0; h < 2; ++h) // a half that starts at or behind the end of the read is not the read's to write
		if (wd * 32 + 16 * h < (int64_t)len) {
#if MGB_ON_DEVICE
			*(uint4*)(dst + 4 * h) = make_uint4(q[4 * h], q[4 * h + 1], q[4 * h + 2], q[4 * h + 3]);
#else
			for (int j = 0; j < 4; ++j) dst[4 * h + j] = q[4 * h + j];
#endif
		}
}
// read r (warp-uniform); a read uploaded as ASCII has no words
struct UnpackRead {
	const UnpackArgs &a;
	MG_HD int operator()(int r, int lane) const
	{
		if (a.pk_off[r] == ~0ULL) return 0;
		const int64_t nw = ((int64_t)a.seq_len[r] + 31) >> 5;
		for (int64_t wd = lane; wd < nw; wd += MGB_W) unpack_word(a, r, wd);
		return 0;
	}
};

// ---- the few words the host needs between two kernels (pool fill levels, queue lengths) ----
// They do not travel by cudaMemcpy: a copy of 16 bytes queues behind whatever another call in flight has put on the copy engines
// (a few hundred MB of results, tens of ms).  A one-warp kernel writes them into page-locked host memory the device can address.
struct Mail { Pool pools[16]; unsigned int jobq_n[2], lab_n[2]; unsigned long long prof[32]; unsigned int tier_hist[128]; unsigned long long arena_peak; };
struct MailSrc { const Pool *pools; const unsigned int *jobq_n, *lab_n; const unsigned long long *prof; const unsigned int *tier_hist; const uint64_t *peak; int n_workers; };
#ifndef MGB_HOSTSIM
__global__ void k_mail(MailSrc m, Mail *out)
{
	const int t = threadIdx.x;
	if (t < 16) out->pools[t] = m.pools[t];
	if (t < 2) out->jobq_n[t] = m.jobq_n[t], out->lab_n[t] = m.lab_n? m.lab_n[t] : 0;
	out->prof[t] = m.prof[t];
	for (int i = t; i < 128; i += 32) out->tier_hist[i] = m.tier_hist[i];
	unsigned long long pk = 0;
	for (int i = t; i < m.n_workers; i += 32) pk = m.peak[i] > pk? m.peak[i] : pk;
	for (int o = 16; o > 0; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xffffffffu, pk, o); pk = y > pk? y : pk; }
	if (t == 0) out->arena_peak = pk;
	__threadfence_system();
}
#endif
// how many bridging jobs / gap jobs the kernels in front have appended to their pools since `done`: the job kernels read it on the device
MG_HD inline void job_counts(const Pool *pools, int i_gjobs, int i_jobs, unsigned int gjobs_done, unsigned int jobs_done, unsigned int *cnt)
{
	const Pool &pg = pools[i_gjobs], &pj = pools[i_jobs];
	cnt[0] = (unsigned int)((pg.used < pg.cap? pg.used : pg.cap) / sizeof(GwfaJob)) - gjobs_done;
	cnt[1] = (unsigned int)((pj.used < pj.cap? pj.used : pj.cap) / sizeof(WfaJob)) - jobs_done;
}
#ifndef MGB_HOSTSIM
__global__ void k_job_counts(const Pool *pools, int i_gjobs, int i_jobs, unsigned int gjobs_done, unsigned int jobs_done, unsigned int *cnt) { job_counts(pools, i_gjobs, i_jobs, gjobs_done, jobs_done, cnt); }
#endif
static void count_jobs(const Pool *pools, int i_gjobs, int i_jobs, unsigned int gjobs_done, unsigned int jobs_done, unsigned int *cnt)
{
#ifndef MGB_HOSTSIM
	k_job_counts<<<1, 1, 0, t_stream>>>(pools, i_gjobs, i_jobs, gjobs_done, jobs_done, cnt);
	CUDA_OK(cudaGetLastError());
#else
	job_counts(pools, i_gjobs, i_jobs, gjobs_done, jobs_done, cnt);
#endif
	++t_launches;
}
static void fetch_mail(const MailSrc &m, Mail *mail)
{
	++t_launches;
#ifndef MGB_HOSTSIM
	k_mail<<<1, 32, 0, t_stream>>>(m, mail);
	CUDA_OK(cudaGetLastError());
	dsync();
#else
	memcpy(mail->pools, m.pools, sizeof(mail->pools));
	memcpy(mail->jobq_n, m.jobq_n, sizeof(mail->jobq_n));
	if (m.lab_n) memcpy(mail->lab_n, m.lab_n, sizeof(mail->lab_n)); else mail->lab_n[0] = mail->lab_n[1] = 0;
	memcpy(mail->prof, m.prof, sizeof(mail->prof));
	memcpy(mail->tier_hist, m.tier_hist, sizeof(mail->tier_hist));
	mail->arena_peak = 0;
	for (int i = 0; i < m.n_workers; ++i) if (m.peak[i] > mail->arena_peak) mail->arena_peak = m.peak[i];
#endif
}

struct Workers {
	int n_workers;
	uint64_t arena_bytes;
	char *arena;
	uint64_t *peak;
};

#ifdef MGB_HOSTSIM
// Runs fn(lane) on the MGB_W lanes of one simulated warp, which works on `item` of `stage` (for the simulator's messages), and
// returns lane 0's code; sets *differ when another lane returned a different one.
template<typename F>
static int sim_warp(int stage, int item, const F &fn, bool *differ)
{
#if MGB_W > 1
	int rcs[MGB_W];
	sim::tag()[0] = stage, sim::tag()[1] = item;
	sim::run_warp(MGB_W, [&](int lane) { rcs[lane] = fn(lane); });
	for (int l = 1; l < MGB_W; ++l) if (rcs[l] != rcs[0]) *differ = true;
	return rcs[0];
#else
	(void)stage, (void)item, (void)differ;
	return fn(0);
#endif
}

// One warp-uniform step fn(A, batch, lane) of a traceback batch (WfaBatch) on the simulated warp.  Every lane works on its own copy
// of the arena header and the batch (in registers on the device); lane 0's copies are kept.  *differ is set when the lanes end
// with different arena tops.
template<typename B, typename F>
static void sim_batch_step(int stage, int item, Arena &A, B &batch, const F &fn, bool *differ)
{
	Arena A0 = A;
	B b0 = batch;
	uint64_t peak = A.peak;
	sim_warp(stage, item, [&](int lane) {
		Arena Al = A;
		B bl = batch;
		fn(Al, bl, lane);
		peak = std::max(peak, Al.peak);
		if (lane == 0) A0 = Al, b0 = bl;
		return (int)(Al.top >> 4) ^ bl.n << 24;
	}, differ);
	A = A0, A.peak = peak, batch = b0;
}
#endif

template<int S>
static void launch_stage(LaunchArgs &L, const Workers &W)
{
	typedef StageSpec<S> Spec;
	L.arena_base = W.arena, L.arena_bytes = W.arena_bytes, L.arena_peak = W.peak;
	dzero(L.c.next_read, sizeof(unsigned int)); // in stream order: no host round trip per launch
	++t_launches;
#ifdef MGB_HOSTSIM
	Arena A;
	arena_init(A, W.arena, Spec::mode == ItemMode::THREAD? (W.arena_bytes / 32) & ~(uint64_t)15 : W.arena_bytes); // one item per thread: a thread's share, as on the device
	std::vector<int32_t> sim_smem(Spec::smem / 4);
	int32_t *smem = Spec::mode == ItemMode::WARP && Spec::smem? sim_smem.data() : 0; // the slice of one warp, as on the device
	bool differ = false;
	sim_warp(S, -1, [&](int lane) { stage_warp_init<S>(smem, lane); return 0; }, &differ);
	const int n_work_sim = L.n_work_dev? (int)*L.n_work_dev : L.n_work;
	if constexpr (is_wfa_stage(S)) { // the warp's traceback batch, as on the device
		const WfaStageGaps<S> gaps{L, smem};
		WfaBatch<WfaStageGaps<S>> batch;
		batch.open(A);
		for (int it = 0; it <= n_work_sim; ++it) {
			const int item = it == n_work_sim? -1 : L.rid_list? L.rid_list[it] : it;
			sim_batch_step(S, item, A, batch, [&](Arena &Al, WfaBatch<WfaStageGaps<S>> &bl, int lane) {
				if (item < 0) bl.flush(gaps, Al, lane);
				else bl.add(gaps, item, Al, lane);
			}, &differ);
			if (differ) { set_error("simulated warp: lanes of a WFA stage's batch went apart"); abort(); }
		}
		if (W.peak && A.peak > W.peak[0]) W.peak[0] = A.peak;
		return;
	}
	for (int it = 0; it < n_work_sim; ++it) {
		int item = L.rid_list? L.rid_list[it] : it;
		A.top = 0;
		// a WARP item: all lanes of the simulated warp enter, each with its own copy of the arena header (as in registers on the device)
		const int rc = Spec::mode != ItemMode::WARP? run_stage<S>(L, item, A, 0, smem) : sim_warp(S, item, [&](int lane) {
			Arena Al = A;
			const int r = run_stage<S>(L, item, Al, lane, smem);
			A.peak = std::max(A.peak, Al.peak);
			return r;
		}, &differ);
		if (differ) { set_error("simulated warp: lanes returned different codes from one stage"); abort(); }
		if (rc < 0 && getenv("MGB_HOSTSIM_TRACE")) fprintf(stderr, "[hostsim] stage %d item %d failed with %d\n", S, item, rc);
		if (rc < 0) stage_fail<S>(L, item, rc);
	}
	if (W.peak && A.peak > W.peak[0]) W.peak[0] = A.peak;
#else
	const int n_w = std::min(W.n_workers, dev_sm_count() * Spec::minb * Spec::warps); // resident warps this stage can keep on the chip
	const int blocks = std::max(1, n_w / Spec::warps);
	const size_t smem = (size_t)Spec::warps * Spec::smem;
	if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute(Spec::kernel(), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
	Spec::kernel()<<<blocks, Spec::warps * 32, smem, t_stream>>>(L);
	CUDA_OK(cudaGetLastError());
#endif
}

// ---- per-read passes ----
// A pass runs its body b(r, lane) on every read r < b.a.n, one warp per read; b.a are the arguments the kernel is launched with, held
// by reference (on the device: the kernel's parameter itself, not a copy).  The body is warp-uniform (all lanes enter it for read r,
// and it strides over its work by MGB_W) and returns a value on which the lanes agree.  Its warps take reads in one of two orders:
// STRIDE, warp w takes reads w, w + warps, ...; PULL, lane 0 takes the next read from the body's counter b.counter() and the warp
// gets it by shuffle, so that a long read holds up only its own warp.
enum class ReadOrder { STRIDE, PULL };
#ifndef MGB_HOSTSIM
__device__ inline int pass_next_read(unsigned int *next, int lane)
{
	unsigned int r = 0;
	if (lane == 0) r = atomicAdd(next, 1u);
	return (int)__shfl_sync(0xffffffffu, r, 0);
}
template<ReadOrder O, typename Body>
__device__ __forceinline__ void pass_loop(const Body &b)
{
	const int lane = threadIdx.x & 31;
	if constexpr (O == ReadOrder::PULL) {
		for (int r = pass_next_read(b.counter(), lane); r < b.a.n; r = pass_next_read(b.counter(), lane)) b(r, lane);
	} else {
		const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), n_warp = (int)((gridDim.x * blockDim.x) >> 5);
		for (int r = warp; r < b.a.n; r += n_warp) b(r, lane);
	}
}
#define MGB_PASS_KERNEL(KERNEL, ARGS, BODY, ORDER) __global__ void __launch_bounds__(256) KERNEL(ARGS a) { pass_loop<ReadOrder::ORDER>(BODY{a}); }
#define MGB_PASS_PTR(KERNEL) KERNEL
#else
#define MGB_PASS_KERNEL(KERNEL, ARGS, BODY, ORDER) void KERNEL(ARGS);
#define MGB_PASS_PTR(KERNEL) 0
#endif

// Runs pass b: dev_sm_count() * 8 blocks of 256 threads on the calling thread's stream, a PULL pass's counter zeroed in stream order
// first.  The simulators run the body on every read in order, on all lanes of a simulated warp.
template<ReadOrder O, typename K, typename Body>
static void launch_pass(K kernel, const char *name, const Body &b)
{
	if constexpr (O == ReadOrder::PULL) dzero(b.counter(), sizeof(unsigned int));
	++t_launches;
#ifdef MGB_HOSTSIM
	(void)kernel;
	bool differ = false;
	for (int r = 0; r < b.a.n; ++r) sim_warp(-1, r, [&](int lane) { return b(r, lane); }, &differ);
	if (differ) { set_error(std::string("simulated warp: lanes returned different values from ") + name); throw MgbError{MGB_E_INTERNAL}; }
#else
	(void)name;
	kernel<<<dev_sm_count() * 8, 256, 0, t_stream>>>(b.a);
	CUDA_OK(cudaGetLastError());
#endif
}

// One row per pass: its kernel (named, so that profiles read well), the arguments it is launched with, its body and the order in
// which its warps take reads.  A row defines the kernel and run_pass(body), which launches it.  MGB_PASS_DS: a body instantiated
// with and without the ds tables, one kernel template.
#define MGB_PASS_RUN(KERNEL, BODY, ORDER) static void run_pass(const BODY &b) { launch_pass<ReadOrder::ORDER>(MGB_PASS_PTR(KERNEL), #KERNEL, b); }
#define MGB_PASS(KERNEL, ARGS, BODY, ORDER) MGB_PASS_KERNEL(KERNEL, ARGS, BODY, ORDER) MGB_PASS_RUN(KERNEL, BODY, ORDER)
#define MGB_PASS_DS(KERNEL, ARGS, BODY, ORDER) \
	template<bool DS> MGB_PASS_KERNEL(KERNEL, ARGS, BODY<DS>, ORDER) \
	template<bool DS> MGB_PASS_RUN(KERNEL<DS>, BODY<DS>, ORDER)

// GAF text (mgb_gaf.cuh): what the dv:f values need; the bytes of each read's text (then scanned into offsets); the text
struct GafRequests { const GafArgs &a; MG_HD int operator()(int r, int lane) const { gaf_requests(a, r, lane); return 0; } };
struct GafCount {
	const GafArgs &a;
	MG_HD unsigned int *counter() const { return a.next; }
	MG_HD int operator()(int r, int lane) const { const uint64_t b = gaf_read(a, r, 0, lane); if (lane == 0) a.off[r] = b; return (int)b; }
};
struct GafWrite {
	const GafArgs &a;
	MG_HD unsigned int *counter() const { return a.next + 1; }
	MG_HD int operator()(int r, int lane) const { return (int)gaf_read(a, r, a.text + a.off[r], lane); }
};

//          kernel        arguments   body         reads
MGB_PASS(   k_unpack,     UnpackArgs, UnpackRead,  STRIDE) // the ASCII copy of the reads that crossed PCIe 2 bits per base
MGB_PASS(   k_out_pack,   PackArgs,   PackRead,    STRIDE) // the result blobs in read order
MGB_PASS(   k_gaf_req,    GafArgs,    GafRequests, STRIDE) // GAF text: what the dv:f values need,
MGB_PASS(   k_gaf_count,  GafArgs,    GafCount,    PULL)   // the bytes of each read's text,
MGB_PASS(   k_gaf_write,  GafArgs,    GafWrite,    PULL)   // the text
namespace mgb { // (the kernels of the headers' passes keep the names they had there)
MGB_PASS(   k_ingest,     IngestArgs, IngestRead,  STRIDE) // reads in device memory: their ASCII copy, words and flags (mgb_ingest.cuh)
MGB_PASS_DS(k_rec_count,  RecArgs,    RecCount,    STRIDE) // result tables (mgb_records.cuh): count pass,
MGB_PASS_DS(k_rec_write,  RecArgs,    RecWrite,    PULL)   // write pass
MGB_PASS(   k_fx_count,   FxArgs,     FxCount,     STRIDE) // FASTA/FASTQ text in device memory (mgb_fastx.cuh): list entries per chunk,
MGB_PASS(   k_fx_lists,   FxArgs,     FxLists,     STRIDE) // the lists,
MGB_PASS(   k_fx_succ,    FxArgs,     FxSucc,      STRIDE) // each candidate's successor,
MGB_PASS(   k_fx_jump,    FxArgs,     FxJump,      STRIDE) // a round of pointer jumping,
MGB_PASS(   k_fx_recs,    FxArgs,     FxRecs,      STRIDE) // the records,
MGB_PASS(   k_fx_tail,    FxArgs,     FxTail,      STRIDE) // those the call emits,
MGB_PASS(   k_fx_copy,    FxArgs,     FxCopy,      PULL)   // their bases and names
}

// ---- block scan ----
// The values src(r, j) of rows [0 .. n) of Src::W columns, their exclusive prefix sums written to out[W r + j] column by column, and
// row n = the totals.  Each thread sums a contiguous run of rows, then one thread per column scans the 1024 partial sums.
template<int W_> struct ScanCols { // in place: v = out
	static constexpr int W = W_;
	const uint64_t *v;
	MG_HD uint64_t operator()(int r, int j) const { return v[W * r + j]; }
};
struct PackSize { // the places of the result blobs in read order (out: PackArgs::off)
	static constexpr int W = 1;
	PackArgs P;
	MG_HD uint64_t operator()(int r, int) const { return pack_size(P, r); }
};
#ifndef MGB_HOSTSIM
template<typename Src>
__global__ void __launch_bounds__(1024) k_scan(Src src, uint64_t *out, int n)
{
	constexpr int W = Src::W;
	__shared__ uint64_t part[W][1024];
	const int tid = threadIdx.x, per = (n + 1023) / 1024;
	const int r0 = tid * per < n? tid * per : n, r1 = r0 + per < n? r0 + per : n;
	for (int j = 0; j < W; ++j) {
		uint64_t sum = 0;
		for (int r = r0; r < r1; ++r) sum += src(r, j);
		part[j][tid] = sum;
	}
	__syncthreads();
	if (tid < W) { uint64_t acc = 0; for (int i = 0; i < 1024; ++i) { uint64_t c = part[tid][i]; part[tid][i] = acc; acc += c; } out[W * n + tid] = acc; }
	__syncthreads();
	for (int j = 0; j < W; ++j) {
		uint64_t acc = part[j][tid];
		for (int r = r0; r < r1; ++r) { const uint64_t c = src(r, j); out[W * r + j] = acc; acc += c; }
	}
}
#endif
template<typename Src>
static void scan_u64(const Src &src, uint64_t *out, int n)
{
#ifndef MGB_HOSTSIM
	k_scan<<<1, 1024, 0, t_stream>>>(src, out, n);
	CUDA_OK(cudaGetLastError());
#else
	constexpr int W = Src::W;
	for (int j = 0; j < W; ++j) {
		uint64_t acc = 0;
		for (int r = 0; r < n; ++r) { const uint64_t c = src(r, j); out[W * r + j] = acc; acc += c; }
		out[W * n + j] = acc;
	}
#endif
	++t_launches;
}

// ---------------------------------------------------------------------------------------------------------------
// a batch on the device: where its reads go, its output pools, the timers of its spans
// ---------------------------------------------------------------------------------------------------------------

// Where the reads of a batch lie: the ASCII copy the kernels read (each read 16-byte aligned, with 8 bytes of slack behind it) and
// the 2-bit words in which they cross PCIe (a read's words start at pk_off[i], with one spare word behind them)
struct BatchLayout {
	std::vector<uint64_t> seq_off, pk_off;
	uint64_t seq_bytes = 0, n_words = 0;
	int64_t n_bases = 0;
	BatchLayout(int n, const int32_t *len) : seq_off((size_t)n), pk_off((size_t)n)
	{
		for (int i = 0; i < n; ++i) {
			const uint64_t l = len[i] > 0? (uint64_t)len[i] : 0;
			seq_off[(size_t)i] = seq_bytes, seq_bytes = (seq_bytes + l + 8 + 15) & ~(uint64_t)15;
			pk_off[(size_t)i] = n_words, n_words += (l + 31) / 32 + 1;
			n_bases += (int64_t)l;
		}
		seq_bytes += 16;
	}
};

// The page-locked host copies and the device copies of a batch's reads and per-read tables (upload_batch)
struct Staging {
	GrowBuf h_tables{true}, h_seq{true}, h_pk{true}, d_tables, d_seq, d_pk, d_segs;
	GrowBuf d_src; // reads in device memory that map on a peer device: their span of the caller's buffer (upload_batch_dev)
};

// The output pools of a batch (PipeCtx); an attempt at the batch that overflows one is run again with that pool grown
enum PoolId { P_ANCHOR, P_MINIPOS, P_LCHAIN, P_OUT, P_PLAN, P_JOBS, P_CIG, P_GSTATE, P_GJOBS, P_WALK, N_POOLS };
// their capacities at the first attempt
static std::array<uint64_t, N_POOLS> pool_caps(int n_reads, int64_t n_bases, int n_workers)
{
	std::array<uint64_t, N_POOLS> cap;
	cap[P_ANCHOR] = std::max<uint64_t>((uint64_t)n_bases / 4 * sizeof(u128), (uint64_t)1 << 22);
	cap[P_MINIPOS] = std::max<uint64_t>((uint64_t)n_bases * sizeof(int32_t) / 2, (uint64_t)1 << 20);
	cap[P_LCHAIN] = std::max<uint64_t>((uint64_t)n_reads * 64 * sizeof(LChain), (uint64_t)1 << 20);
	cap[P_OUT] = std::max<uint64_t>((uint64_t)n_bases * 4, (uint64_t)1 << 22);
	cap[P_PLAN] = std::max<uint64_t>((uint64_t)n_bases / 8 * 8, (uint64_t)1 << 20);
	cap[P_JOBS] = std::max<uint64_t>((uint64_t)n_bases / 40 * sizeof(WfaJob), (uint64_t)1 << 20);
	cap[P_CIG] = std::max<uint64_t>((uint64_t)n_bases, (uint64_t)1 << 20) + (uint64_t)n_workers * CIG_CHUNK_BYTES * 4; // + the unused ends of the warps' slices (three tier kernels per pass)
	cap[P_GSTATE] = std::max<uint64_t>((uint64_t)n_reads * 2048, (uint64_t)1 << 20);
	cap[P_GJOBS] = std::max<uint64_t>((uint64_t)n_reads * 24 * sizeof(GwfaJob), (uint64_t)1 << 20);
	cap[P_WALK] = std::max<uint64_t>((uint64_t)n_reads * 256, (uint64_t)1 << 20);
	return cap;
}

#ifndef MGB_HOSTSIM
struct EvTimer {
	cudaEvent_t a, b; bool used;
	EvTimer() : used(false) { cudaEventCreate(&a); cudaEventCreate(&b); }
	~EvTimer() { cudaEventDestroy(a); cudaEventDestroy(b); }
	void start() { cudaEventRecord(a, t_stream); used = true; }
	void stop() { cudaEventRecord(b, t_stream); }
	double ms() { if (!used) return 0; float t = 0; cudaEventSynchronize(b); cudaEventElapsedTime(&t, a, b); return t; }
	void clear() { used = false; }
};
#else
struct EvTimer { double t0 = 0, t1 = 0; void start() { t0 = now_ms(); } void stop() { t1 = now_ms(); } double ms() { return t1 - t0; } void clear() { t0 = t1 = 0; } };
#endif

struct SlotTimers {
	EvTimer h2d, seed, chain, align, wfa, fin, d2h, lab, k[10];
	void reset() { EvTimer *all[] = {&h2d, &seed, &chain, &align, &wfa, &fin, &d2h, &lab}; for (EvTimer *t : all) t->clear(); for (int i = 0; i < 10; ++i) k[i].clear(); }
	void to_stats(mgb_stats_t &S) // all but t_d2h_ms, which ends with the batch
	{
		S.t_h2d_ms = h2d.ms(), S.t_seed_ms = seed.ms(), S.t_chain_ms = chain.ms(), S.t_align_ms = align.ms();
		S.t_wfa_ms = wfa.ms(), S.t_finish_ms = fin.ms(), S.t_lab_ms = lab.ms();
		for (int i = 0; i < 10; ++i) S.t_kernel_ms[i] = k[i].ms();
	}
};

// t times the launches of one scope; NULL: an untimed scope
struct Span {
	EvTimer *t;
	explicit Span(EvTimer *t_) : t(t_) { if (t) t->start(); }
	~Span() { if (t) t->stop(); }
};

// ---------------------------------------------------------------------------------------------------------------
// model: flattened graph + minimizer index, host copy and device image
// ---------------------------------------------------------------------------------------------------------------

struct Model {
	// host copies
	std::vector<int32_t> seg_len;
	std::vector<uint64_t> vseq_off;
	std::vector<char> seq;
	std::vector<uint64_t> arc_idx;
	std::vector<DevArc> arc;
	std::vector<u128> slot;
	std::vector<uint64_t> pos;
	std::vector<uint32_t> occ;      // occurrences per distinct minimizer (for the quantiles)
	uint64_t n_slots_mask;
	int k, w;
	uint32_t *d_occ_sorted = 0; uint64_t n_keys = 0, n_pos = 0; // device-built index: ascending occurrence counts; host copies of slot/pos are made on demand
	std::mutex host_ix_mutex;
	// device image
	GraphDev g;
	IndexDev ix;
	GafGraph gafg; // names of the graph for the GAF kernels
	std::vector<void*> dev_ptrs;
	// per-model scratch reused across batches
	std::vector<int32_t> seg_name_id, seg_soff; // MG_M_NO_DIAG: the name a segment goes by (id into name_ids) and its offset there
	std::unordered_map<std::string, int32_t> name_ids;
	Workers W, Wbig;
	int32_t skip1_len = INT32_MAX; // WFA tier routing learned from earlier batches (wfa_job_run)
	std::vector<float> logf_tab; float *d_logf; int n_logf;
	mgb_stats_t stats;
	gfa_edseq_t *es;
	// the batch pipeline: a batch is cut into sub-batches, each driven by its own host thread on its own stream ("slot"),
	// so that kernels, copies and host-side result assembly of different sub-batches overlap
	struct Slot {
		Staging stage;
		GrowBuf h_out{true}, h_mail{true}, h_routs{true}, d_meta, d_routs, d_scratch, d_jobq, d_order, d_packed, d_packoff, d_lab_new, d_pool[N_POOLS];
		GrowBuf h_gaf{true}, d_gaf, d_gaf_text; // mgb_map_batch_gaf(): the reads' names and segments, requests and cells; the text
		GrowBuf h_rec{true}, d_rec; // mgb_map_batch_dev_rec(): SEQ_CSR, SEQ_INFO and the reads' rows; CIGAR counts, div requests and values
		mgb::HostPool host_pool; // packing and result assembly of the batch on this slot
		Workers W;
		mgb_stats_t st;
		DevStream stream;
		DevEvent ev_first, ev_last, ev_piece[4]; // first kernel start and last kernel end of the batch; the end of each piece's download
		std::unique_ptr<SlotTimers> timers; // the event pairs live in the slot: creating and destroying three dozen events per call contends on the driver's lock with the other calls in flight
		bool ready;
		Slot() : ready(false) { memset(&W, 0, sizeof(W)); }
	};
	enum { MAX_SLOTS = 8 };
	Slot slots[MAX_SLOTS];
	std::mutex big_mutex; // the large-arena retry pass, the label table and the learned routing are shared by the slots
	std::condition_variable slot_cv;
	std::mutex gpu_mutex;         // the kernels of one call at a time: calls in flight overlap their copies and host work with them, not with each other's kernels
	int device = 0;               // the GPU this image lives on
	std::vector<Model*> peers;    // MGB_DEVICES: the same index on further GPUs; a batch is cut into one contiguous part per device
	bool slot_busy[MAX_SLOTS] = {};
	int in_flight = 0;    // calls inside map_batch_impl
	bool lab_growing = false; // a call is waiting to replace the label pool: new calls wait
	// reachability labels of the graph (mgb_gclabel.cuh): built on demand, kept across batches, grown between them
	long long *d_lab_off = 0; Pool *d_lab_hdr = 0; char *d_lab_pool = 0;
	uint64_t lab_cap = 0; int32_t lab_max_dist_g = -1; int64_t lab_sources = 0;
	// mgb_reads_parse_dev(): one call at a time; the chunk table, the lists and the candidates' jumps and marks, the records
	struct FxScratch { std::mutex mu; GrowBuf tab, lists, recs; } fx;
};

static void model_free(Model *M)
{
	for (Model *P : M->peers) model_free(P);
	M->peers.clear();
#ifndef MGB_HOSTSIM
	cudaSetDevice(M->device);
#endif
	for (void *p : M->dev_ptrs) dfree(p);
	if (M->W.arena) dfree(M->W.arena);
	if (M->W.peak) dfree(M->W.peak);
	if (M->Wbig.arena) dfree(M->Wbig.arena);
	if (M->Wbig.peak) dfree(M->Wbig.peak);
	if (M->d_logf) dfree(M->d_logf);
	dfree(M->d_lab_off), dfree(M->d_lab_hdr), dfree(M->d_lab_pool), dfree(M->d_occ_sorted);
	for (int k = 0; k < Model::MAX_SLOTS; ++k) {
		Model::Slot &sl = M->slots[k];
		if (sl.W.arena) dfree(sl.W.arena);
		if (sl.W.peak) dfree(sl.W.peak);
#ifndef MGB_HOSTSIM
		if (sl.ready) { cudaStreamDestroy(sl.stream); cudaEventDestroy(sl.ev_first); cudaEventDestroy(sl.ev_last); for (int i = 0; i < 4; ++i) cudaEventDestroy(sl.ev_piece[i]); }
#endif
	}
	delete M; // (with it the slots' buffers and timers, on this device)
}

// reference: gfa-base.c:509-526 gfa_comp_table.  Filled once: with MGB_DEVICES, mg_index() builds the models of the further devices
// on several threads at once, and a table filled anew by each of them was read half-filled by another (reverse strands of segments
// left uncomplemented on one device).
static const unsigned char *comp_tab()
{
	static const struct Tab {
		unsigned char c[256];
		Tab()
		{
			const char *from = "ABCDEFGHIJKLMNOPQRSTUVWXYZ", *to = "TVGHEFCDIJMLKNOPQYSAABWXRZ";
			for (int i = 0; i < 256; ++i) c[i] = (unsigned char)i;
			for (int i = 0; i < 26; ++i) {
				c[(unsigned char)from[i]] = (unsigned char)to[i];
				c[(unsigned char)(from[i] + 32)] = (unsigned char)(to[i] + 32);
			}
		}
	} tab;
	return tab.c;
}

static void ensure_workers(Workers &W, int n_workers, uint64_t arena_bytes)
{
	if (W.arena && W.n_workers == n_workers && W.arena_bytes == arena_bytes) return;
	if (W.arena) dfree(W.arena);
	if (W.peak) dfree(W.peak);
	W.n_workers = n_workers, W.arena_bytes = arena_bytes;
	W.arena = (char*)dmalloc((size_t)n_workers * arena_bytes);
	W.peak = (uint64_t*)dmalloc((size_t)n_workers * sizeof(uint64_t));
	dzero(W.peak, (size_t)n_workers * sizeof(uint64_t));
}

static int default_workers()
{
#ifdef MGB_HOSTSIM
	return 1;
#else
	return dev_sm_count() * (int)p_workers_per_sm;
#endif
}

// The slot on the model's device: its stream and events made at its first batch, its arenas sized; then the calling thread works on
// its stream
static void slot_prepare(Model *M, Model::Slot &sl, int n_workers)
{
#ifndef MGB_HOSTSIM
	cudaSetDevice(M->device);
	if (!sl.ready) {
		CUDA_OK(cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking));
		CUDA_OK(cudaEventCreate(&sl.ev_first));
		CUDA_OK(cudaEventCreate(&sl.ev_last));
		for (int i = 0; i < 4; ++i) CUDA_OK(cudaEventCreateWithFlags(&sl.ev_piece[i], cudaEventDisableTiming));
	}
#endif
	sl.ready = true;
	ensure_workers(sl.W, n_workers, (uint64_t)p_arena_mb << 20);
	dev_bind(M->device, sl.stream);
}

static Model *model_build(gfa_t *g, int k, int w)
{
	Model *M = new Model();
	M->k = k, M->w = w, M->d_logf = 0, M->n_logf = 0, M->es = 0;
	memset(&M->W, 0, sizeof(Workers)), memset(&M->Wbig, 0, sizeof(Workers));
	memset(&M->stats, 0, sizeof(M->stats));
	const unsigned char *comp = comp_tab();
	const uint32_t n_seg = g->n_seg, n_vtx = n_seg * 2;
	M->seg_len.resize(n_seg);
	M->vseq_off.resize(n_vtx);
	uint64_t tot = 0;
	for (uint32_t i = 0; i < n_seg; ++i) {
		M->seg_len[i] = g->seg[i].len;
		M->vseq_off[i << 1] = tot, tot += (uint64_t)g->seg[i].len + 8;   // 8 bytes of slack after every copy
		M->vseq_off[i << 1 | 1] = tot, tot += (uint64_t)g->seg[i].len + 8;
	}
	M->seq.assign(tot + 16, 0);
	for (uint32_t i = 0; i < n_seg; ++i) {
		const gfa_seg_t *s = &g->seg[i];
		char *f = &M->seq[M->vseq_off[i << 1]], *r = &M->seq[M->vseq_off[i << 1 | 1]];
		for (int32_t j = 0; j < s->len; ++j) f[j] = s->seq[j];
		for (int32_t j = 0; j < s->len; ++j) r[s->len - j - 1] = (char)comp[(uint8_t)s->seq[j]]; // reference: gfa-ed.c:33-36
	}
	M->arc_idx.assign(g->idx, g->idx + n_vtx);
	M->arc.resize(g->n_arc);
	for (uint64_t i = 0; i < g->n_arc; ++i) { // verbatim order (SURVEY H10b)
		DevArc a;
		a.w = g->arc[i].w, a.lv = (uint32_t)g->arc[i].v_lv, a.rank = g->arc[i].rank, a.ow = g->arc[i].ow;
		M->arc[i] = a;
	}
	M->seg_name_id.resize(n_seg), M->seg_soff.resize(n_seg);
	for (uint32_t i = 0; i < n_seg; ++i) { // reference: map-algo.c:168-174
		const gfa_seg_t *s = &g->seg[i];
		const bool stable = s->snid >= 0 && g->sseq;
		const char *gname = stable? g->sseq[s->snid].name : s->name;
		auto it = M->name_ids.emplace(std::string(gname? gname : ""), (int32_t)M->name_ids.size()).first;
		M->seg_name_id[i] = it->second, M->seg_soff[i] = stable? s->soff : 0;
	}
	// upload the graph
	M->g.n_seg = (int32_t)n_seg;
	M->g.seg_name_id = upload(M->seg_name_id.data(), M->seg_name_id.size()).release(), M->dev_ptrs.push_back((void*)M->g.seg_name_id);
	M->g.seg_soff = upload(M->seg_soff.data(), M->seg_soff.size()).release(), M->dev_ptrs.push_back((void*)M->g.seg_soff);
	M->g.seg_len = upload(M->seg_len.data(), M->seg_len.size()).release(), M->dev_ptrs.push_back((void*)M->g.seg_len);
	M->g.vseq_off = upload(M->vseq_off.data(), M->vseq_off.size()).release(), M->dev_ptrs.push_back((void*)M->g.vseq_off);
	M->g.seq = upload(M->seq.data(), M->seq.size()).release(), M->dev_ptrs.push_back((void*)M->g.seq);
	M->g.arc_idx = upload(M->arc_idx.data(), M->arc_idx.size()).release(), M->dev_ptrs.push_back((void*)M->g.arc_idx);
	M->g.arc = upload(M->arc.data(), M->arc.size()).release(), M->dev_ptrs.push_back((void*)M->g.arc);
	M->ix.k = k, M->ix.w = w, M->ix.slot = 0, M->ix.pos = 0, M->ix.n_slots_mask = 0;
	{ // names of segments and stable sequences for the GAF kernels: concatenated bytes + offsets
		auto names = [&](uint32_t n, const std::function<const char*(uint32_t)> &nm, const char **d_name, const int64_t **d_off) {
			std::vector<int64_t> off((size_t)n + 1, 0);
			std::string b;
			for (uint32_t i = 0; i < n; ++i) { const char *s = nm(i); if (s) b += s; off[(size_t)i + 1] = (int64_t)b.size(); }
			*d_name = upload(b.data(), b.size()).release(), M->dev_ptrs.push_back((void*)*d_name);
			*d_off = upload(off.data(), off.size()).release(), M->dev_ptrs.push_back((void*)*d_off);
		};
		const uint32_t n_sseq = g->sseq? g->n_sseq : 0;
		names(n_seg, [&](uint32_t i) { return (const char*)g->seg[i].name; }, &M->gafg.seg_name, &M->gafg.seg_name_off);
		names(n_sseq, [&](uint32_t i) { return (const char*)g->sseq[i].name; }, &M->gafg.sseq_name, &M->gafg.sseq_name_off);
		std::vector<int32_t> snid(n_seg), soff(n_seg), smin(n_sseq + 1), smax(n_sseq + 1), srank(n_sseq + 1);
		for (uint32_t i = 0; i < n_seg; ++i) snid[i] = g->seg[i].snid, soff[i] = g->seg[i].soff;
		for (uint32_t i = 0; i < n_sseq; ++i) smin[i] = g->sseq[i].min, smax[i] = g->sseq[i].max, srank[i] = g->sseq[i].rank;
		auto put = [&](const std::vector<int32_t> &v, const int32_t **d) { *d = upload(v.data(), v.size()).release(), M->dev_ptrs.push_back((void*)*d); };
		put(snid, &M->gafg.snid), put(soff, &M->gafg.soff), put(smin, &M->gafg.sseq_min), put(smax, &M->gafg.sseq_max), put(srank, &M->gafg.sseq_rank);
		M->gafg.seg_len = M->g.seg_len;
	}

	// sketch every segment on the device (K1 reused), then build the table: on the device (the simulators: on the host)
#ifdef MGB_HOSTSIM
	std::vector<u128> mz;
#endif
	{
		uint64_t tot_len = 0;
		int32_t max_len = 1;
		for (uint32_t i = 0; i < n_seg; ++i) { tot_len += (uint64_t)g->seg[i].len; if (g->seg[i].len > max_len) max_len = g->seg[i].len; }
		uint64_t cap = (tot_len / 2 + 64 * (uint64_t)n_seg + 1024) * sizeof(u128);
		// a worker sketches one whole segment inside its arena: ~ (len/w + growth slack) records
		uint64_t need = (uint64_t)max_len * 16 + ((uint64_t)1 << 20);
		uint64_t arena_b = std::max<uint64_t>((uint64_t)p_arena_mb << 20, need);
		int nw = default_workers();
		while (nw > 1 && (uint64_t)nw * arena_b > dev_free_mem() / 2) nw /= 2;
		for (;;) {
			ensure_workers(M->W, nw, arena_b);
			Pool hp; hp.used = 0, hp.cap = cap;
			Pool *d_pool = (Pool*)dmalloc(sizeof(Pool));
			u128 *d_mz = (u128*)dmalloc(cap);
			int *d_status = (int*)dmalloc(sizeof(int));
			unsigned int *d_next = (unsigned int*)dmalloc(sizeof(unsigned int));
			int st0 = 0;
			h2d(d_pool, &hp, sizeof(Pool));
			h2d(d_status, &st0, sizeof(int));
			LaunchArgs L;
			memset(&L, 0, sizeof(L));
			L.c.g = M->g, L.c.ix = M->ix, L.c.next_read = d_next;
			L.routs = (ReadOut*)d_status, L.rid_list = 0, L.n_work = (int32_t)n_seg, L.pool_mz = d_pool, L.mz = d_mz;
			launch_stage<S_INDEX_SKETCH>(L, M->W);
			dsync();
			d2h(&st0, d_status, sizeof(int));
			d2h(&hp, d_pool, sizeof(Pool));
			bool retry = false;
			if (st0 == MGB_E_POOL) cap *= 2, retry = true;
			else if (st0 == MGB_E_ARENA) arena_b *= 2, nw = std::max(1, nw / 2), retry = true;
			else if (st0 < 0) { set_error("segment sketch failed with code " + std::to_string(st0)); throw MgbError{st0}; }
#ifndef MGB_HOSTSIM
			if (!retry) { // group, lay out and insert on the device (mgb_index.cuh)
				DevIndexOut out;
				dfree(M->W.arena), dfree(M->W.peak); // the sketch arenas are not needed again; the sort wants the memory
				memset(&M->W, 0, sizeof(Workers));
				cudaError_t e = build_index_device(d_mz, hp.used / sizeof(u128), 2 * k, t_stream, &out);
				dfree(d_pool), dfree(d_mz), dfree(d_status), dfree(d_next);
				if (e != cudaSuccess) { set_error(std::string("index build on the device: ") + cudaGetErrorString(e)); throw MgbError{MGB_E_INTERNAL}; }
				M->n_slots_mask = out.n_slots - 1, M->n_keys = out.n_keys, M->n_pos = out.n_pos, M->d_occ_sorted = out.occ_sorted;
				M->ix.n_slots_mask = M->n_slots_mask, M->ix.slot = out.slot, M->ix.pos = out.pos;
				M->dev_ptrs.push_back((void*)out.slot), M->dev_ptrs.push_back((void*)out.pos);
				return M;
			}
#else
			if (!retry) {
				mz.resize(hp.used / sizeof(u128));
				d2h(mz.data(), d_mz, hp.used);
			}
#endif
			dfree(d_pool), dfree(d_mz), dfree(d_status), dfree(d_next);
			if (!retry) break;
		}
	}
#ifdef MGB_HOSTSIM
	// the sketch arenas are not needed again (every mapping slot owns its arenas)
	dfree(M->W.arena), dfree(M->W.peak);
	memset(&M->W, 0, sizeof(Workers));
	// group by minimizer; occurrence lists ascending (reference: index.c:115-165 mg_idx_a2h)
	std::sort(mz.begin(), mz.end(), [](const u128 &a, const u128 &b) { return (a.x >> 8) != (b.x >> 8)? (a.x >> 8) < (b.x >> 8) : a.y < b.y; });
	size_t n_keys = 0;
	for (size_t i = 0; i < mz.size(); ++i) if (i == 0 || (mz[i].x >> 8) != (mz[i-1].x >> 8)) ++n_keys;
	uint64_t n_slots = 16;
	while (n_slots < n_keys * 2) n_slots <<= 1;
	M->n_slots_mask = n_slots - 1;
	M->slot.assign(n_slots, u128{~0ULL, ~0ULL});
	M->occ.reserve(n_keys);
	for (size_t i = 0; i < mz.size();) {
		size_t j = i;
		uint64_t key = mz[i].x >> 8;
		while (j < mz.size() && (mz[j].x >> 8) == key) ++j;
		uint64_t h = idx_slot_hash(key) & M->n_slots_mask;
		while (M->slot[h].x != ~0ULL) h = (h + 1) & M->n_slots_mask;
		if (j - i == 1) {
			M->slot[h].x = key << 1 | 1, M->slot[h].y = mz[i].y;
			M->occ.push_back(1);
		} else {
			M->slot[h].x = key << 1, M->slot[h].y = (uint64_t)M->pos.size() << 32 | (uint64_t)(j - i);
			for (size_t t = i; t < j; ++t) M->pos.push_back(mz[t].y);
			M->occ.push_back((uint32_t)(j - i));
		}
		i = j;
	}
	M->ix.n_slots_mask = M->n_slots_mask;
	M->ix.slot = upload(M->slot.data(), M->slot.size()).release(), M->dev_ptrs.push_back((void*)M->ix.slot);
	M->ix.pos = upload(M->pos.data(), M->pos.size()).release(), M->dev_ptrs.push_back((void*)M->ix.pos);
#endif
	return M;
}

static const Model *model_of(const mg_idx_t *gi) { return (const Model*)gi->B; }

// ---------------------------------------------------------------------------------------------------------------
// C ABI: index
// ---------------------------------------------------------------------------------------------------------------

extern "C" void mg_idx_cal_quantile(const mg_idx_t *gi, int32_t m, float f[], int32_t q[])
{
	const Model *M = model_of(gi);
#ifndef MGB_HOSTSIM
	if (M->d_occ_sorted) { // the table was built on the device: the counts are there, sorted
		const uint64_t n = M->n_keys;
		for (int32_t i = 0; i < m; ++i) {
			size_t kk = (size_t)((1.0 - (double)f[i]) * (double)n);
			if (n == 0) { q[i] = 0; continue; }
			if (kk >= n) kk = n - 1;
			uint32_t v = 0;
			cudaSetDevice(M->device);
			cudaMemcpy(&v, M->d_occ_sorted + kk, 4, cudaMemcpyDeviceToHost);
			q[i] = (int32_t)v;
		}
		return;
	}
#endif
	std::vector<uint32_t> a(M->occ);
	uint64_t n = a.size();
	for (int32_t i = 0; i < m; ++i) {
		size_t kk = (size_t)((1.0 - (double)f[i]) * (double)n);
		if (n == 0) { q[i] = 0; continue; }
		if (kk >= n) kk = n - 1;
		std::nth_element(a.begin(), a.begin() + kk, a.end());
		q[i] = (int32_t)a[kk];
	}
}

extern "C" const uint64_t *mg_idx_get(const mg_idx_t *gi, uint64_t minier, int *n)
{
	Model *M = (Model*)model_of(gi);
#ifndef MGB_HOSTSIM
	if (M->slot.empty() && M->ix.slot) { // device-built table: the host view is fetched the first time somebody asks for it
		std::lock_guard<std::mutex> lk(M->host_ix_mutex);
		if (M->slot.empty()) {
			cudaSetDevice(M->device);
			M->pos.resize(M->n_pos? M->n_pos : 1);
			cudaMemcpy(M->pos.data(), M->ix.pos, M->n_pos * 8, cudaMemcpyDeviceToHost);
			std::vector<u128> sl(M->n_slots_mask + 1);
			cudaMemcpy(sl.data(), M->ix.slot, sl.size() * sizeof(u128), cudaMemcpyDeviceToHost);
			M->slot.swap(sl);
		}
	}
#endif
	IndexDev ix;
	ix.k = M->k, ix.w = M->w, ix.n_slots_mask = M->n_slots_mask, ix.slot = M->slot.data(), ix.pos = M->pos.data();
	return idx_get(ix, minier, n);
}

extern "C" mg_idx_t *mg_index(gfa_t *g, const mg_idxopt_t *io, int n_threads, mg_mapopt_t *mo)
{
	(void)n_threads;
	// MGB_DEVICES=0-7 | 0,2,5: the index is replicated on every listed GPU and each batch is cut into one part per GPU (the reference's
	// "-t": gmap.c:163-211 hands its mini-batch to n_threads workers; here the workers are devices).  Unset: the "device" parameter.
	std::vector<int> devs;
	if (const char *e = getenv("MGB_DEVICES")) {
		for (const char *q = e; *q;) {
			char *end;
			long a = strtol(q, &end, 10), b2 = a;
			if (end == q) break;
			if (*end == '-') { q = end + 1; b2 = strtol(q, &end, 10); }
			for (long d = a; d <= b2 && devs.size() < 64; ++d) devs.push_back((int)d);
			q = *end == ','? end + 1 : end;
			if (*end && *end != ',') break;
		}
	}
	if (devs.empty()) devs.push_back((int)p_device);
	for (int d : devs) if (!dev_ok(d)) { set_error("no CUDA device " + std::to_string(d) + " available: libmgb200 has no CPU path"); return 0; }
	dev_ok(devs[0]);
	for (uint32_t i = 0; i < g->n_seg; ++i) { // reference: index.c:215-220
		gfa_seg_t *s = &g->seg[i];
		for (int32_t j = 0; j < s->len; ++j)
			if (s->seq[j] >= 'a' && s->seq[j] <= 'z') s->seq[j] -= 32;
	}
	for (uint64_t i = 0; i < g->n_arc; ++i) // reference: index.c:176-183,192-196
		if (g->arc[i].ov != 0 || g->arc[i].ow != 0) {
			fprintf(stderr, "[E::%s] minigraph doesn't work with graphs containing overlapping segments\n", __func__);
			return 0;
		}
	int k = io->k, w = io->w, b = io->bucket_bits;
	if (k * 2 < b) b = k * 2;
	if (w < 1) w = 1;
	Model *M = 0;
	try { M = model_build(g, k, w); } catch (const MgbError &) { return 0; }
	M->device = devs[0];
	if (devs.size() > 1) { // every further device builds its own copy, all at once
		M->peers.resize(devs.size() - 1, (Model*)0);
		std::vector<std::thread> th;
		for (size_t i = 1; i < devs.size(); ++i)
			th.emplace_back([&, i]() { try { if (dev_ok(devs[i])) { M->peers[i - 1] = model_build(g, k, w); M->peers[i - 1]->device = devs[i]; } } catch (const MgbError &) {} });
		for (auto &t : th) t.join();
		dev_ok(devs[0]);
		for (Model *P : M->peers) if (P == 0) { model_free(M); return 0; } // mgb_last_error() has the reason
	}
	mg_idx_t *gi = (mg_idx_t*)calloc(1, sizeof(mg_idx_t));
	gi->g = g, gi->b = b, gi->w = w, gi->k = k, gi->n_seg = (int32_t)g->n_seg;
	gi->B = (struct mg_idx_bucket_s*)M;
	// host view of both strands for callers that read gi->es (reference: gfa-ed.c:24-42)
	gi->es = (gfa_edseq_t*)malloc(sizeof(gfa_edseq_t) * 2 * (size_t)g->n_seg);
	for (uint32_t i = 0; i < g->n_seg; ++i) {
		gi->es[i << 1].seq = g->seg[i].seq, gi->es[i << 1].len = g->seg[i].len;
		gi->es[i << 1 | 1].seq = &M->seq[M->vseq_off[i << 1 | 1]], gi->es[i << 1 | 1].len = g->seg[i].len;
	}
	if (mo) { // reference: options.c:120-134 mg_opt_update
		float f[2];
		int32_t q[2];
		f[0] = 0.1f, f[1] = mo->occ_max1_frac;
		mg_idx_cal_quantile(gi, 2, f, q);
		if (q[0] > mo->lc_max_occ) mo->lc_max_occ = q[0];
		if (mo->lc_max_occ > mo->occ_max1_cap) mo->lc_max_occ = mo->occ_max1_cap;
		if (q[1] > mo->occ_max1) mo->occ_max1 = q[1];
		if (mo->occ_max1 > mo->occ_max1_cap) mo->occ_max1 = mo->occ_max1_cap;
		if (mo->bw_long < mo->bw) mo->bw_long = mo->bw;
	}
	return gi;
}

extern "C" void mg_idx_destroy(mg_idx_t *gi)
{
	if (gi == 0) return;
	if (gi->B) model_free((Model*)gi->B);
	free(gi->es);
	free(gi);
}

extern "C" void mg_idx_hfree(void *h) { (void)h; } // reference callers only pass NULL (shortk.c:191)

struct mg_tbuf_s { int dummy; };
extern "C" mg_tbuf_t *mg_tbuf_init(void) { return (mg_tbuf_t*)calloc(1, sizeof(mg_tbuf_t)); }
extern "C" void mg_tbuf_destroy(mg_tbuf_t *b) { free(b); }

extern "C" void mg_gchain_free(mg_gchains_t *gs)
{
	if (gs == 0) return;
	for (int32_t i = 0; i < gs->n_gc; ++i) {
		free(gs->gc[i].p);
		free(gs->gc[i].ds.ds);
		free(gs->gc[i].ds.off);
	}
	free(gs->gc); free(gs->a); free(gs->lc);
	free(gs);
}

extern "C" void mgb_free_batch(int n_reads, mg_gchains_t **gcs)
{
	for (int i = 0; i < n_reads; ++i) { mg_gchain_free(gcs[i]); gcs[i] = 0; }
}

// ---------------------------------------------------------------------------------------------------------------
// batch dispatcher
// ---------------------------------------------------------------------------------------------------------------

static void fill_opt(MapOptDev &o, const mg_mapopt_t *opt, int k)
{
	memset(&o, 0, sizeof(o));
	o.flag = opt->flag, o.seed = opt->seed, o.max_qlen = opt->max_qlen, o.occ_max1 = opt->occ_max1;
	o.bw = opt->bw, o.bw_long = opt->bw_long, o.rmq_size_cap = opt->rmq_size_cap, o.rmq_rescue_size = opt->rmq_rescue_size;
	o.rmq_rescue_ratio = opt->rmq_rescue_ratio;
	o.max_gap_pre = opt->max_gap_pre, o.max_gap = opt->max_gap, o.max_gap_ref = opt->max_gap_ref, o.max_frag_len = opt->max_frag_len;
	{ // reference: map-algo.c:388-390; expf() must be the host libm (SURVEY H3)
		float tmp = expf(-opt->div * k);
		o.chn_pen_gap = opt->chn_pen_gap * tmp;
		o.chn_pen_skip = opt->chn_pen_skip * tmp;
	}
	o.max_lc_skip = opt->max_lc_skip, o.max_lc_iter = opt->max_lc_iter, o.max_gc_skip = opt->max_gc_skip;
	o.min_lc_cnt = opt->min_lc_cnt, o.min_lc_score = opt->min_lc_score, o.min_gc_cnt = opt->min_gc_cnt, o.min_gc_score = opt->min_gc_score;
	o.gdp_max_ed = opt->gdp_max_ed, o.lc_max_trim = opt->lc_max_trim, o.lc_max_occ = opt->lc_max_occ;
	o.mask_level = opt->mask_level, o.sub_diff = opt->sub_diff, o.best_n = opt->best_n, o.pri_ratio = opt->pri_ratio, o.ref_bonus = opt->ref_bonus;
}

// dv:f of a graph chain (reference: gchain1.c:295; host libm log, SURVEY H3): mg_gchain_t::div here and in the GAF cells
static float gc_div(int32_t n_mini, int32_t n_anchor, int32_t q_span)
{
	return n_mini >= n_anchor? (float)(log((double)n_mini / n_anchor) / q_span) : (float)(log((double)n_anchor / n_mini) / q_span);
}

static mg_gchains_t *build_result(const ReadOut &ro, const char *pool)
{
	mg_gchains_t *gs = (mg_gchains_t*)calloc(1, sizeof(mg_gchains_t));
	gs->rep_len = ro.rep_len;
	if (ro.n_gc == 0) return gs; // reference: gchain1.c:460 returns the bare struct
	gs->n_gc = ro.n_gc, gs->n_lc = ro.n_lc, gs->n_a = ro.n_a;
	gs->gc = (mg_gchain_t*)calloc((size_t)ro.n_gc, sizeof(mg_gchain_t));
	gs->lc = (mg_llchain_t*)malloc((size_t)(ro.n_lc > 0? ro.n_lc : 1) * sizeof(mg_llchain_t));
	gs->a = (mg128_t*)malloc((size_t)(ro.n_a > 0? ro.n_a : 1) * sizeof(mg128_t));
	const ReadBlob B = read_blob(pool, ro);
	const GChain *d = B.gc;
	memcpy(gs->lc, B.lc, (size_t)ro.n_lc * sizeof(mg_llchain_t));
	memcpy(gs->a, B.a, (size_t)ro.n_a * sizeof(mg128_t));
	for (int32_t i = 0; i < ro.n_gc; ++i) {
		mg_gchain_t *p = &gs->gc[i];
		const GChain *s = &d[i];
		p->id = s->id, p->parent = s->parent, p->off = s->off, p->cnt = s->cnt, p->n_anchor = s->n_anchor, p->score = s->score;
		p->qs = s->qs, p->qe = s->qe, p->plen = s->plen, p->ps = s->ps, p->pe = s->pe, p->blen = s->blen, p->mlen = s->mlen;
		p->hash = s->hash, p->subsc = s->subsc, p->n_sub = s->n_sub, p->mapq = (uint32_t)s->mapq, p->flt = (uint32_t)s->flt;
		p->div = gc_div(s->n_mini, s->n_anchor, s->q_span);
		if (s->has_cigar) {
			p->p = (mg_cigar_t*)calloc(1, (size_t)s->n_cigar * 8 + sizeof(mg_cigar_t));
			p->p->n_cigar = s->n_cigar, p->p->mlen = s->c_mlen, p->p->blen = s->c_blen, p->p->aplen = s->c_aplen, p->p->ss = s->c_ss, p->p->ee = s->c_ee;
			memcpy(p->p->cigar, pool + s->cigar_off, (size_t)s->n_cigar * 8);
			p->ds.len = s->ds_len, p->ds.n_off = s->n_dsoff;
			p->ds.ds = (char*)calloc((size_t)s->ds_len + 1, 1);
			memcpy(p->ds.ds, pool + s->ds_off, (size_t)s->ds_len);
			p->ds.off = (int32_t*)calloc((size_t)(s->n_dsoff > 0? s->n_dsoff : 1), sizeof(int32_t));
			memcpy(p->ds.off, pool + s->dsoff_off, (size_t)s->n_dsoff * sizeof(int32_t));
		}
	}
	return gs;
}


// The label table of graph chaining: allocated at the first batch, emptied when a batch asks for longer walks than it was built for.
static bool lab_prepare(Model *M, int32_t max_dist_g)
{
	std::unique_lock<std::mutex> lock(M->big_mutex);
	const size_t n_vtx = (size_t)M->g.n_seg * 2;
	if (M->lab_max_dist_g >= max_dist_g && M->d_lab_off) return true; // labels are exact for every bound up to the one they were searched with
	// (re)start the table: it must be ours alone.  No new call starts until those in flight are done; a second call that gets here
	// meanwhile searches per read this once (it is one of those the first is waiting for).
	if (M->lab_growing) return false;
	M->lab_growing = true;
	M->slot_cv.wait(lock, [&]() { return M->in_flight <= 1; });
	struct Done { Model *M; ~Done() { M->lab_growing = false; M->slot_cv.notify_all(); } } done{M};
	if (M->d_lab_off == 0) {
		M->d_lab_off = (long long*)dmalloc(n_vtx * sizeof(long long));
		M->d_lab_hdr = (Pool*)dmalloc(sizeof(Pool));
		M->lab_cap = std::min<uint64_t>(std::max<uint64_t>((uint64_t)256 << 20, (uint64_t)n_vtx * 8192), std::max<uint64_t>((uint64_t)64 << 20, dev_free_mem() / 16));
		M->d_lab_pool = (char*)dmalloc(M->lab_cap);
	}
	dfill(M->d_lab_off, 0xff, n_vtx * sizeof(long long));
	Pool hp; hp.used = 0, hp.cap = M->lab_cap;
	h2d(M->d_lab_hdr, &hp, sizeof(Pool));
	M->lab_max_dist_g = max_dist_g;
	dsync();
	return true;
}
// after a batch: a label pool that overflowed is enlarged for the batches to come (the sources that did not fit were searched per read)
static void lab_after_batch(Model *M, unsigned int n_new)
{
	std::unique_lock<std::mutex> lock(M->big_mutex);
	M->lab_sources += n_new;
	Pool hp;
	d2h(&hp, M->d_lab_hdr, sizeof(Pool));
	if (hp.used <= hp.cap || M->lab_growing) return;
	// kernels of other calls may be reading the pool: no new call starts until those in flight are done, then the pool is replaced
	M->lab_growing = true;
	M->slot_cv.wait(lock, [&]() { return M->in_flight <= 1; });
	struct Done { Model *M; ~Done() { M->lab_growing = false; M->slot_cv.notify_all(); } } done{M};
	const uint64_t want = std::max<uint64_t>((uint64_t)hp.used * 2, M->lab_cap * 2);
	if (want > dev_free_mem() / 2) return;
	char *np = (char*)dmalloc(want);
	d2d(np, M->d_lab_pool, M->lab_cap);
	dsync();
	dfree(M->d_lab_pool);
	hp.used = M->lab_cap, hp.cap = want; // everything that was written lies below the old capacity
	M->d_lab_pool = np, M->lab_cap = want;
	h2d(M->d_lab_hdr, &hp, sizeof(Pool));
}

// Reads that are already in device memory (mgb_map_batch_dev*): read i of a batch is src[src_off[i] .. + its length) on device
// src_dev.  copy: the batch maps on a peer (MGB_DEVICES), which takes its span of src into the slot's staging first.  t_off_ms: the
// host time of the copy of the caller's offsets, counted in the batch's t_h2d_ms.
struct DevReads { const char *src; const int64_t *src_off; int src_dev; bool copy; double t_off_ms; };

// What a call maps (make_batch).  The reads as the kernels see them: n of them, of lengths qlens, from seqs on the host or from dev,
// named names[i] (names may be NULL).  A fragment of several segments is one read, its segments concatenated: their lengths are
// seg_len[seg_off[f] .. seg_off[f + 1]), and the fragment is entries seg_first[f] .. + n_seg[f] of the caller's arrays, whose
// per-segment lengths are seg_qlens.  When every fragment has one segment, seg_off and n_seg are NULL and read i is entry i.
struct Batch {
	int n = 0;
	const int *qlens = 0;
	const char *const *seqs = 0, *const *names = 0;
	std::optional<DevReads> dev;
	const int32_t *seg_off = 0, *seg_len = 0;
	const int *n_seg = 0;
	const int64_t *seg_first = 0;
	const int *seg_qlens = 0;
	// what the fields point to when the fragments have segments
	std::vector<std::string> cat;
	std::vector<int> qsum;
	std::vector<const char*> sq;
	std::vector<int32_t> off, len;
	std::vector<int64_t> first, src;
	// reads [b, e) of a batch without segments, mapped on device d of the index (MGB_DEVICES): a peer takes its span of dev first
	Batch part(int b, int e, int d) const
	{
		Batch p;
		p.n = e - b, p.qlens = qlens + b, p.seqs = seqs? seqs + b : 0, p.names = names? names + b : 0;
		if (dev) p.dev = *dev, p.dev->src_off += b, p.dev->copy = d > 0;
		return p;
	}
};

// The batch of n_frag fragments, fragment f of n_seg[f] consecutive entries of qlens / seqs (n_seg NULL: one each), from seqs on the
// host or from dev (with the caller's offset of every entry), named names[f]
static Batch make_batch(int n_frag, const int *n_seg, const int *qlens, const char *const *seqs, const char *const *names, const DevReads *dev)
{
	Batch B;
	bool single = true;
	for (int f = 0; f < n_frag && n_seg; ++f) if (n_seg[f] != 1) single = false;
	B.n = n_frag, B.names = names;
	if (dev) B.dev = *dev;
	if (single) { B.qlens = qlens, B.seqs = seqs; return B; }
	const size_t nf = (size_t)n_frag;
	B.cat.resize(nf), B.qsum.resize(nf), B.sq.resize(nf), B.off.resize(nf + 1), B.first.resize(nf);
	int64_t at = 0;
	for (size_t f = 0; f < nf; ++f) {
		B.off[f] = (int32_t)B.len.size();
		B.first[f] = at;
		const int ns = n_seg[f] > 0 && n_seg[f] <= 255? n_seg[f] : 0; // more than MG_MAX_SEG segments: no result (map-algo.c:359)
		int sum = 0;
		for (int j = 0; j < ns; ++j) {
			const int l = qlens[at + j] > 0? qlens[at + j] : 0;
			B.len.push_back(l);
			if (l > 0 && seqs) B.cat[f].append(seqs[at + j], (size_t)l);
			sum += l;
		}
		B.qsum[f] = sum, B.sq[f] = B.cat[f].data();
		at += n_seg[f] > 0? n_seg[f] : 0;
	}
	B.off[nf] = (int32_t)B.len.size();
	B.qlens = B.qsum.data(), B.seqs = seqs? B.sq.data() : 0;
	B.seg_off = B.off.data(), B.seg_len = B.len.data();
	B.n_seg = n_seg, B.seg_first = B.first.data(), B.seg_qlens = qlens;
	if (dev) { // a fragment's segments follow each other in src: it is mapped from there as one read
		for (size_t f = 0; f < nf; ++f) B.src.push_back(dev->src_off[B.first[f]]);
		B.dev->src_off = B.src.data();
	}
	return B;
}

// What the last pass over a sub-batch left: the reads' outcomes on the host (on the device: the slot's d_routs), the output pool
struct Last { const ReadMeta *meta; ReadOut *routs; const char *d_out; uint64_t out_used; };

// Where the results of a call go, one kind per output format: mg_gchains_t objects (GcsSink), GAF text (GafSink), tables in device
// memory (RecSink).  The dispatcher hands them over without knowing the format; each entry point ends with its sink's end(rc).
struct Sink {
	virtual ~Sink() {}
	// sub-batch B after its last pass on slot sl, whose stats (sl.st) and copy-back timer (sl.timers->d2h) it adds to.  0 or a negative code
	virtual int results(Model *M, Model::Slot &sl, const Batch &B, const Last &L, int host_threads) = 0;
	// the sink of reads [b, e) of a call split over the devices, which map on device `device`; made in input order before any maps
	virtual Sink &part(int b, int e, int device) = 0;
	// once every part has mapped: their results joined in input order, on M's device
	virtual int join(Model *M) = 0;
	// the result of a call without reads
	virtual int empty(Model *M) = 0;
};

// GAF text formatted on the device (mgb_map_batch_gaf, mgb_map_batch_dev_gaf) into the caller's (out, out_len, out_cap): its
// buffer, reused and grown, or with out_cap NULL a fresh block.  A part keeps its text (out NULL) until the join.
struct GafSink : Sink {
	uint64_t flag;
	char **out; size_t *out_len, *out_cap; // the caller's; out NULL: a part
	char *fresh = 0;
	std::vector<char> text; // a part's
	size_t len = 0;
	std::vector<std::unique_ptr<GafSink>> parts;
	GafSink(uint64_t flag_, char **out_, size_t *out_len_, size_t *out_cap_) : flag(flag_), out(out_), out_len(out_len_), out_cap(out_cap_) {}
	static int refuse(const mg_mapopt_t *opt) // --cov and independent segments (minigraph.h:19,22): no per-fragment GAF record
	{
		if ((opt->flag & (0x4000 | 0x20000)) == 0) return 0;
		set_error("mgb_map_batch_gaf: --cov and independent segments print no per-fragment GAF record");
		return MGB_E_UNSUPPORTED;
	}
	// room for n bytes of text and a closing 0, or NULL
	char *dest(size_t n)
	{
		if (out == 0) { text.resize(n + 1); return text.data(); }
		if (out_cap == 0) return fresh = (char*)malloc(n + 1);
		if (*out == 0 || *out_cap < n + 1) {
			free(*out);
			*out_cap = n + n / 8 + 1;
			*out = (char*)malloc(*out_cap);
			if (*out == 0) *out_cap = 0;
		}
		return *out;
	}
	int results(Model *M, Model::Slot &sl, const Batch &B, const Last &L, int host_threads) override;
	Sink &part(int, int, int) override { parts.emplace_back(new GafSink(flag, 0, 0, 0)); return *parts.back(); }
	int join(Model *) override
	{
		size_t tot = 0;
		for (const auto &p : parts) tot += p->len;
		char *o = dest(tot);
		if (o == 0) { set_error("mgb_map_batch_gaf: out of host memory for the text"); return MGB_E_INTERNAL; }
		size_t at = 0;
		for (const auto &p : parts) { if (p->len) memcpy(o + at, p->text.data(), p->len); at += p->len; }
		o[tot] = 0;
		len = tot;
		return 0;
	}
	int empty(Model *) override
	{
		char *o = dest(0);
		if (o == 0) { set_error("mgb_map_batch_gaf: out of host memory"); return MGB_E_INTERNAL; }
		o[0] = 0;
		return 0;
	}
	// the text's length to the caller; on failure no partial text: *out_len = 0, and an empty caller's buffer or no block
	int end(int rc)
	{
		if (rc < 0) free(fresh), fresh = 0, len = 0;
		if (out_cap == 0) *out = fresh;
		else if (rc < 0 && *out && *out_cap) (*out)[0] = 0;
		*out_len = len;
		return rc < 0? rc : 0;
	}
};

// A batch of 2048 reads or more goes up and comes back in 4 pieces, so that the host threads pack or assemble one piece while
// another is on the wire.  Piece pc holds reads [r0(pc), r0(pc + 1)).
struct Pieces {
	int n_reads, n;
	explicit Pieces(int n_reads_) : n_reads(n_reads_), n(n_reads_ >= 2048? 4 : 1) {}
	int64_t r0(int pc) const { return (int64_t)n_reads * pc / n; }
};

// Bytes [off[r0], off[r1]) of each piece of the reads from d to h, each piece followed by the event the host waits for before it
// reads them
static void download_in_pieces(Model::Slot &sl, int n_reads, const uint64_t *off, char *h, const char *d)
{
	const Pieces pcs(n_reads);
	for (int pc = 0; pc < pcs.n; ++pc) {
		const uint64_t b0 = off[pcs.r0(pc)], b1 = off[pcs.r0(pc + 1)];
		d2h_async(h + b0, d + b0, b1 - b0);
		ev_record(sl.ev_piece[pc]);
	}
}

// a read's outcome: the code of the stage that failed it, or else ReadOut::status (1: not mapped)
static int read_status(const ReadMeta &m, const ReadOut &o) { return m.status < 0? m.status : o.status; }

// The GAF text of a mapped sub-batch, formatted on the device from the blobs in the output pool (mgb_gaf.cuh): requests for the dv:f
// values, cells formatted by the host, count, scan, write; then the text goes to the host in pieces, each copied on to dest() by the
// host threads while the next is on the wire.  t_d2h_ms: the GAF kernels and the pieces of the copy.
int GafSink::results(Model *M, Model::Slot &sl, const Batch &B, const Last &L, int host_threads)
{
	const int n_reads = B.n;
	const char *const *names = B.names;
	const ReadOut *routs = L.routs;
	const size_t n = (size_t)n_reads;
	const bool lchain = (flag & F_WRITE_LCHAIN) != 0;
	size_t n_segs = 0, name_bytes = 0, n_req = 0;
	for (size_t i = 0; i < n; ++i) {
		n_segs += B.n_seg? (size_t)std::max(B.n_seg[i], 0) : 1;
		name_bytes += names && names[i]? strlen(names[i]) : 1;
		if (routs[i].n_gc > 0) n_req += (size_t)routs[i].n_gc + (lchain? (size_t)routs[i].n_lc : 0);
	}
	auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
	// one block on both sides: name_off | req_off | n_seg | seg_first | seg_len | names (uploaded), then requests | cells | off | counters
	const size_t o_req_off = al(8 * (n + 1)), o_nseg = o_req_off + al(8 * (n + 1)), o_first = o_nseg + al(4 * n), o_len = o_first + al(4 * n);
	const size_t o_names = o_len + al(4 * n_segs), o_req = o_names + al(name_bytes), o_cells = o_req + al(sizeof(GafReq) * n_req);
	const size_t o_off = o_cells + al((size_t)GAF_CELL * n_req), o_next = o_off + al(8 * (n + 1)), tot = o_next + 16;
	char *h = (char*)sl.h_gaf.ensure(tot), *d = (char*)sl.d_gaf.ensure(tot);
	{
		int64_t *name_off = (int64_t*)h, *req_off = (int64_t*)(h + o_req_off);
		int32_t *nseg = (int32_t*)(h + o_nseg), *first = (int32_t*)(h + o_first), *slen = (int32_t*)(h + o_len);
		char *nm = h + o_names;
		int64_t at = 0, rq = 0, sg = 0;
		for (size_t i = 0; i < n; ++i) {
			const char *s = names && names[i]? names[i] : "*";
			const size_t l = strlen(s);
			memcpy(nm + at, s, l);
			name_off[i] = at, at += (int64_t)l;
			req_off[i] = rq;
			if (routs[i].n_gc > 0) rq += routs[i].n_gc + (lchain? routs[i].n_lc : 0);
			const int ns = B.n_seg? std::max(B.n_seg[i], 0) : 1;
			const int *ql = B.n_seg? B.seg_qlens + B.seg_first[i] : B.qlens + i;
			nseg[i] = ns, first[i] = (int32_t)sg;
			for (int j = 0; j < ns; ++j) slen[sg++] = ql[j];
		}
		name_off[n] = at, req_off[n] = rq;
	}
	h2d(d, h, o_req);
	GafArgs G;
	G.g = M->gafg;
	G.q.name = d + o_names, G.q.name_off = (const int64_t*)d, G.q.n_seg = (const int32_t*)(d + o_nseg), G.q.seg_first = (const int32_t*)(d + o_first);
	G.q.seg_len = (const int32_t*)(d + o_len);
	G.routs = (const ReadOut*)sl.d_routs.p, G.pool = L.d_out, G.n = n_reads, G.flag = flag;
	G.req_off = (const int64_t*)(d + o_req_off), G.req = (GafReq*)(d + o_req), G.cells = d + o_cells;
	G.off = (uint64_t*)(d + o_off), G.text = 0, G.next = (unsigned int*)(d + o_next);
	const Pieces pcs(n_reads);
	const uint64_t *hoff = (const uint64_t*)(h + o_off);
	char *htext;
	{
		Span span(&sl.timers->d2h);
		// dv:f values: the device lists what each needs, the host formats them with its libm (SURVEY H3)
		if (n_req) run_pass(GafRequests{G});
		d2h(h + o_req, d + o_req, sizeof(GafReq) * n_req);
		const GafReq *hreq = (const GafReq*)(h + o_req);
		char *hcells = h + o_cells;
		pfor(sl.host_pool, host_threads, (int64_t)n_req, [&](int64_t k) {
			const GafReq &q = hreq[k];
			char *c = hcells + (size_t)GAF_CELL * (size_t)k;
			c[0] = 0;
			if (q.kind == 0) { // format.c:204-209
				const float div = gc_div(q.a, q.b, q.q_span);
				if (div >= 0.0f && div <= 1.0f) { if (div == 0.0f) c[0] = '0', c[1] = 0; else snprintf(c, GAF_CELL, "%.4f", div); }
			} else if (q.kind == 1) { // format.c:256-263
				const double div = q.a == q.b? 0.0 : (q.a > q.b? log((double)q.a / q.b) : log((double)q.b / q.a)) / q.q_span;
				if (div == 0.0) c[0] = '0', c[1] = 0; else snprintf(c, GAF_CELL, "%.4f", div);
			}
		});
		h2d(d + o_cells, hcells, (size_t)GAF_CELL * n_req);
		// text: sizes, offsets in read order, bytes
		run_pass(GafCount{G});
		scan_u64(ScanCols<1>{G.off}, G.off, G.n);
		d2h(h + o_off, G.off, 8 * (n + 1));
		G.text = (char*)sl.d_gaf_text.ensure(hoff[n] + 64);
		htext = (char*)sl.h_out.ensure(hoff[n] + 64);
		run_pass(GafWrite{G});
		download_in_pieces(sl, n_reads, hoff, htext, G.text);
	}
	const uint64_t total = hoff[n];
	const double t_asm0 = now_ms();
	char *dst = dest((size_t)total);
	if (dst == 0) { dsync(); set_error("mgb_map_batch_gaf: out of host memory for the text"); return MGB_E_INTERNAL; }
	const uint64_t chunk = 1 << 20;
	for (int pc = 0; pc < pcs.n; ++pc) {
		const uint64_t b0 = hoff[pcs.r0(pc)], b1 = hoff[pcs.r0(pc + 1)];
		ev_wait(sl.ev_piece[pc]);
		pfor(sl.host_pool, host_threads, (int64_t)((b1 - b0 + chunk - 1) / chunk), [&](int64_t k) {
			const uint64_t c0 = b0 + (uint64_t)k * chunk, c1 = std::min(b1, c0 + chunk);
			memcpy(dst + c0, htext + c0, c1 - c0);
		});
	}
	dst[total] = 0;
	len = (size_t)total;
	sl.st.out_bytes = (int64_t)total;
	sl.st.t_asm_ms = now_ms() - t_asm0;
	return 0;
}

// Every table's offset in the block (256-byte aligned) and the block's size, from the rows r.n_* (and x.n_*: the ds tables after
// the others; x NULL: none)
static void rec_layout(mgb_records_t &r, mgb_records_ds_t *x)
{
	const int64_t bytes[MGB_REC_NTAB] = {24 * (r.n_seq + 1), 8 * r.n_seq, 4 * MGB_GC_NCOL * r.n_rec, 4 * r.n_rec, 8 * (r.n_rec + 1), 20 * r.n_lc, 16 * r.n_a, 8 * r.n_cigar};
	int64_t at = 0;
	for (int t = 0; t < MGB_REC_NTAB; ++t) r.off[t] = at, at += (bytes[t] + 255) & ~(int64_t)255;
	if (x) {
		const int64_t ds_bytes[MGB_REC_DS_NTAB] = {16 * (r.n_rec + 1), x->n_ds, 4 * x->n_ds_off};
		for (int t = 0; t < MGB_REC_DS_NTAB; ++t) x->off[t] = at, at += (ds_bytes[t] + 255) & ~(int64_t)255;
	}
	r.bytes = at;
}

// Tables in device memory (mgb_map_batch_dev_rec, with_ds: mgb_map_batch_dev_rec_ds), R and X, in one block from the caller's
// allocator on the index's device, ordered after the work queued on the caller's stream.  A part (alloc NULL) writes its tables into
// a block of its own on its device, freed with it, and the join copies them into the caller's block.
struct RecSink : Sink {
	mgb_dev_alloc_fn alloc;
	void *alloc_ctx, *stream;
	int device;       // where the block is
	bool with_ds;
	mgb_records_t R;  // the tables as written
	mgb_records_ds_t X;
	std::vector<std::unique_ptr<RecSink>> parts;
	RecSink(mgb_dev_alloc_fn alloc_, void *alloc_ctx_, void *stream_, int device_, bool with_ds_)
		: alloc(alloc_), alloc_ctx(alloc_ctx_), stream(stream_), device(device_), with_ds(with_ds_) { memset(&R, 0, sizeof(R)), memset(&X, 0, sizeof(X)); }
	~RecSink() // (the calling thread is left on the device of the first part, the index's)
	{
		if (alloc == 0 && R.block) dev_ok(device), dfree(R.block);
		if (!parts.empty()) { const int d0 = parts[0]->device; parts.clear(); dev_ok(d0); }
	}
	// R's block, ordered after the caller's stream; false when there is none
	bool block()
	{
		rec_layout(R, with_ds? &X : 0);
		R.block = alloc? alloc(alloc_ctx, (size_t)R.bytes) : dmalloc((size_t)R.bytes);
		if (R.block == 0) { set_error("mgb_map_batch_dev_rec: the allocator returned no block of " + std::to_string(R.bytes) + " bytes"); return false; }
#ifndef MGB_HOSTSIM
		CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream)); // a block the caller's allocator reuses may still be read by work queued there
#endif
		return true;
	}
	int results(Model *M, Model::Slot &sl, const Batch &B, const Last &L, int host_threads) override;
	Sink &part(int, int, int device_) override { parts.emplace_back(new RecSink(0, 0, stream, device_, with_ds)); return *parts.back(); }
	int join(Model *M) override;
	int empty(Model *M) override // the two rows of totals alone, all 0: the join of no part
	{
		int rc;
		try { rc = join(M); } catch (const MgbError &e) { rc = e.code; }
		dev_bind(M->device, 0);
		return rc;
	}
	int end(mgb_records_t *out, mgb_records_ds_t *ds_out, int rc) // no block handed back on failure
	{
		if (rc == 0) { *out = R; if (ds_out) *ds_out = X; }
		return rc;
	}
};

// The tables of a mapped sub-batch, written on the device from the blobs in the output pool (mgb_records.cuh): SEQ_CSR and the
// reads' rows from the host, the CIGAR operations (with_ds: and the ds bytes and offsets, of which only the totals come back) counted
// and scanned, the div requests to the host and the values back up, then the block and the write pass.  t_d2h_ms: the table kernels, their copies and the host work between them; t_asm_ms stays 0: the
// tables are final when the write pass ends.
int RecSink::results(Model *, Model::Slot &sl, const Batch &B, const Last &L, int host_threads)
{
	const int n_reads = B.n;
	const ReadOut *routs = L.routs;
	mgb_stats_t &S = sl.st;
	const size_t n = (size_t)n_reads;
	auto has_result = [&](size_t f) { return (B.n_seg == 0 || B.n_seg[f] > 0) && read_status(L.meta[f], routs[f]) != 1; }; // mgb_map_batch_dev() leaves one
	memset(&R, 0, sizeof(R)), memset(&X, 0, sizeof(X));
	for (size_t f = 0; f < n; ++f) {
		R.n_seq += B.n_seg? std::max(B.n_seg[f], 0) : 1;
		if (has_result(f)) R.n_rec += std::max(routs[f].n_gc, 0);
	}
	if (R.n_rec >= INT32_MAX) { set_error("mgb_map_batch_dev_rec: more than INT32_MAX records in one batch"); return MGB_E_UNSUPPORTED; }
	const size_t n_seq = (size_t)R.n_seq, n_rec = (size_t)R.n_rec;
	auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
	// host and device: seq_csr | seq_info | row_of (uploaded), then on the device cig_off | req | next [| ds_n], on the host
	// req | div [| the two ds totals]
	const size_t o_info = al(24 * (n_seq + 1)), o_row = o_info + al(8 * n_seq), o_up = o_row + al(4 * n);
	const size_t o_cig = o_up, o_req = o_cig + al(8 * (n_rec + 1)), o_next = o_req + al(sizeof(GafReq) * n_rec), o_ds = o_next + al(16);
	const size_t o_hdiv = o_up + al(sizeof(GafReq) * n_rec), o_htot = o_hdiv + al(4 * n_rec);
	char *h = (char*)sl.h_rec.ensure(with_ds? o_htot + 16 : o_hdiv + 4 * n_rec + 16);
	char *d = (char*)sl.d_rec.ensure(with_ds? o_ds + 16 * (n_rec + 1) : o_next + 16);
	int64_t *csr = (int64_t*)h;
	int32_t *info = (int32_t*)(h + o_info), *row_of = (int32_t*)(h + o_row);
	GafReq *hreq = (GafReq*)(h + o_up);
	float *hdiv = (float*)(h + o_hdiv);
	int64_t rec = 0, lc = 0, a = 0;
	for (size_t f = 0, s = 0; f < n; ++f) {
		const int ns = B.n_seg? std::max(B.n_seg[f], 0) : 1;
		const bool has = has_result(f);
		const ReadOut &o = routs[f];
		row_of[f] = has? (int32_t)s : -1;
		for (int j = 0; j < ns; ++j, ++s) {
			csr[3 * s] = rec, csr[3 * s + 1] = lc, csr[3 * s + 2] = a;
			info[2 * s] = has && j == 0, info[2 * s + 1] = has && j == 0? o.rep_len : 0;
			if (has && j == 0 && o.n_gc > 0) rec += o.n_gc, lc += o.n_lc, a += o.n_a;
		}
	}
	csr[3 * n_seq] = rec, csr[3 * n_seq + 1] = R.n_lc = lc, csr[3 * n_seq + 2] = R.n_a = a;
	RecArgs A;
	A.routs = (const ReadOut*)sl.d_routs.p, A.pool = L.d_out, A.n = n_reads;
	A.row_of = (const int32_t*)(d + o_row), A.seq_csr = (const int64_t*)d;
	A.cig_off = (uint64_t*)(d + o_cig), A.req = (GafReq*)(d + o_req), A.next = (unsigned int*)(d + o_next);
	A.ds_n = with_ds? (uint64_t*)(d + o_ds) : 0, A.ds = 0, A.ds_off = 0;
	{
		Span span(&sl.timers->d2h);
		h2d(d, h, o_up);
		S.h2d_bytes += (int64_t)o_up;
		if (with_ds) run_pass(RecCount<true>{A}); else run_pass(RecCount<false>{A});
		scan_u64(ScanCols<1>{A.cig_off}, A.cig_off, (int)n_rec);
		int64_t *htot = (int64_t*)(h + o_htot);
		if (with_ds) scan_u64(ScanCols<2>{A.ds_n}, A.ds_n, (int)n_rec), d2h_async(htot, A.ds_n + 2 * n_rec, 16);
		d2h_async(hreq, A.req, sizeof(GafReq) * n_rec);
		d2h(&R.n_cigar, A.cig_off + n_rec, 8);
		S.out_bytes = (int64_t)(sizeof(GafReq) * n_rec + 8);
		if (with_ds) X.n_ds = htot[0], X.n_ds_off = htot[1], S.out_bytes += 16;
		pfor(sl.host_pool, host_threads, (int64_t)n_rec, [&](int64_t k) { hdiv[k] = gc_div(hreq[k].a, hreq[k].b, hreq[k].q_span); });
		if (!block()) return MGB_E_INTERNAL;
		char *b = (char*)R.block;
		d2d(b + R.off[MGB_REC_SEQ_CSR], d, 24 * (n_seq + 1));
		d2d(b + R.off[MGB_REC_SEQ_INFO], d + o_info, 8 * n_seq);
		d2d(b + R.off[MGB_REC_CIGAR_CSR], A.cig_off, 8 * (n_rec + 1));
		if (with_ds) {
			d2d(b + X.off[MGB_REC_DS_CSR], A.ds_n, 16 * (n_rec + 1));
			A.ds = b + X.off[MGB_REC_DS], A.ds_off = (int32_t*)(b + X.off[MGB_REC_DS_OFF]);
		}
		h2d_async(b + R.off[MGB_REC_GC_DIV], hdiv, 4 * n_rec);
		S.h2d_bytes += (int64_t)(4 * n_rec);
		A.gc = (int32_t*)(b + R.off[MGB_REC_GC]), A.lc = (uint32_t*)(b + R.off[MGB_REC_LC]);
		A.a = (uint64_t*)(b + R.off[MGB_REC_A]), A.cigar = (uint64_t*)(b + R.off[MGB_REC_CIGAR]);
		if (with_ds) run_pass(RecWrite<true>{A}); else run_pass(RecWrite<false>{A});
	}
	dsync();
	return 0;
}

// The rows of totals of R's block (SEQ_CSR row n_seq, CIGAR_CSR row n_rec; x: DS_CSR row n_rec), on the calling thread's stream,
// which is synchronised
static void rec_totals(const mgb_records_t &R, const mgb_records_ds_t *x)
{
	const int64_t tot[6] = {R.n_rec, R.n_lc, R.n_a, R.n_cigar, x? x->n_ds : 0, x? x->n_ds_off : 0};
	char *b = (char*)R.block;
	h2d_async(b + R.off[MGB_REC_SEQ_CSR] + 24 * R.n_seq, tot, 24);
	h2d_async(b + R.off[MGB_REC_CIGAR_CSR] + 8 * R.n_rec, tot + 3, 8);
	if (x) h2d_async(b + x->off[MGB_REC_DS_CSR] + 16 * R.n_rec, tot + 4, 16);
	dsync();
}

#ifndef MGB_HOSTSIM
namespace mgb { // (named as in mgb_records.cuh, which holds its row function)
__global__ void __launch_bounds__(256) k_rec_rebase(RecRebase B)
{
	for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B.n; i += (int64_t)gridDim.x * blockDim.x) rec_rebase_row(B, i);
}
}
#endif
// The tables of the parts (each in its own block on its device) joined in input order into R's block on M's device: every table
// copied behind those of the parts before, the CSR rows raised by the rows before, the totals written last.  On the caller's stream.
int RecSink::join(Model *M)
{
	memset(&R, 0, sizeof(R)), memset(&X, 0, sizeof(X));
	for (const auto &p : parts) {
		R.n_seq += p->R.n_seq, R.n_rec += p->R.n_rec, R.n_lc += p->R.n_lc, R.n_a += p->R.n_a, R.n_cigar += p->R.n_cigar;
		X.n_ds += p->X.n_ds, X.n_ds_off += p->X.n_ds_off;
	}
#ifndef MGB_HOSTSIM
	dev_bind(M->device, (cudaStream_t)stream);
#endif
	if (!block()) return MGB_E_INTERNAL;
	// the tables of R, then those of X
	enum { SEQ, REC, LC, A, CIG, DS, DSO, N_KIND };
	const int n_tab = MGB_REC_NTAB + (with_ds? MGB_REC_DS_NTAB : 0);
	static const int kind[MGB_REC_NTAB + MGB_REC_DS_NTAB] = {SEQ, SEQ, REC, REC, REC, LC, A, CIG, REC, DS, DSO};
	static const int64_t row_bytes[MGB_REC_NTAB + MGB_REC_DS_NTAB] = {24, 8, 4 * MGB_GC_NCOL, 4, 8, 20, 16, 8, 16, 1, 4};
	auto off = [](const mgb_records_t &r, const mgb_records_ds_t &x, int t) { return t < MGB_REC_NTAB? r.off[t] : x.off[t - MGB_REC_NTAB]; };
	char *b = (char*)R.block;
	int64_t at[N_KIND] = {0, 0, 0, 0, 0, 0, 0}; // rows of the parts before
	for (size_t d = 0; d < parts.size(); ++d) {
		const mgb_records_t &p = parts[d]->R;
		const mgb_records_ds_t &px = parts[d]->X;
		const int64_t rows[N_KIND] = {p.n_seq, p.n_rec, p.n_lc, p.n_a, p.n_cigar, px.n_ds, px.n_ds_off};
		if (p.block)
			for (int t = 0; t < n_tab; ++t)
				d2d_peer(b + off(R, X, t) + at[kind[t]] * row_bytes[t], M->device, (const char*)p.block + off(p, px, t), parts[d]->device, (size_t)(rows[kind[t]] * row_bytes[t]));
		const RecRebase rb[3] = {{(int64_t*)(b + R.off[MGB_REC_SEQ_CSR]) + 3 * at[SEQ], p.n_seq, 3, {at[REC], at[LC], at[A]}},
								 {(int64_t*)(b + R.off[MGB_REC_CIGAR_CSR]) + at[REC], p.n_rec, 1, {at[CIG], 0, 0}},
								 {(int64_t*)(b + X.off[MGB_REC_DS_CSR]) + 2 * at[REC], with_ds? p.n_rec : 0, 2, {at[DS], at[DSO], 0}}};
		for (const RecRebase &B : rb) {
			if (B.n == 0 || (B.base[0] == 0 && B.base[1] == 0 && B.base[2] == 0)) continue;
#ifndef MGB_HOSTSIM
			k_rec_rebase<<<(int)std::min<int64_t>((B.n + 255) / 256, dev_sm_count() * 8), 256, 0, t_stream>>>(B);
			CUDA_OK(cudaGetLastError());
#else
			for (int64_t i = 0; i < B.n; ++i) rec_rebase_row(B, i);
#endif
		}
		for (int k = 0; k < N_KIND; ++k) at[k] += rows[k];
	}
	rec_totals(R, with_ds? &X : 0);
	return 0;
}

// seq_off, seq_len and name_hash of a batch in one page-locked block (they go up in one copy, upload_tables)
static uint64_t *batch_tables(Staging &B, const BatchLayout &lay, int n_reads, const int *qlens, const char *const *names)
{
	const size_t n = (size_t)n_reads;
	uint64_t *seq_off = (uint64_t*)B.h_tables.ensure(n * 16 + 256);
	int32_t *seq_len = (int32_t*)(seq_off + n);
	uint32_t *name_hash = (uint32_t*)(seq_len + n);
	memcpy(seq_off, lay.seq_off.data(), n * 8);
	for (size_t i = 0; i < n; ++i) seq_len[i] = qlens[i], name_hash[i] = names && names[i]? hash_str(names[i]) : 0;
	return seq_off;
}

// those tables to the device, into b (with room behind them for self_id)
static void upload_tables(Staging &B, BatchDev &b, int n_reads, const uint64_t *h_tables, char *d_seq, mgb_stats_t &S)
{
	const size_t n = (size_t)n_reads;
	uint64_t *d_seq_off = (uint64_t*)B.d_tables.ensure(n * 20 + 64); // seq_off, seq_len, name_hash, self_id
	h2d(d_seq_off, h_tables, n * 16);
	S.h2d_bytes += (int64_t)n * 16;
	b.n_reads = n_reads, b.seq = d_seq, b.seq_off = d_seq_off, b.seq_len = (const int32_t*)(d_seq_off + n), b.name_hash = (const uint32_t*)(b.seq_len + n);
}

// what follows the reads of every batch: which segment name, if any, is each read's own (MG_M_NO_DIAG; exact string match on the
// host), and the segments of the fragments (seg_off, seg_len: as BatchDev has them, or NULL)
static void upload_read_extras(Staging &B, BatchDev &b, const Model *M, const char *const *names, bool no_diag, const int32_t *seg_off, const int32_t *seg_len)
{
	const size_t n = (size_t)b.n_reads;
	if (no_diag) {
		std::vector<int32_t> self(n, -1);
		for (size_t i = 0; i < n; ++i)
			if (names && names[i]) { auto it = M->name_ids.find(names[i]); if (it != M->name_ids.end()) self[i] = it->second; }
		int32_t *d_self_id = (int32_t*)(b.name_hash + n);
		h2d(d_self_id, self.data(), sizeof(int32_t) * n);
		b.self_id = d_self_id;
	}
	if (seg_off) {
		const size_t n_len = (size_t)seg_off[n];
		int32_t *d_segs = (int32_t*)B.d_segs.ensure(sizeof(int32_t) * (n + 1 + n_len));
		h2d(d_segs, seg_off, sizeof(int32_t) * (n + 1));
		h2d(d_segs + n + 1, seg_len, sizeof(int32_t) * n_len);
		b.seg_off = d_segs, b.seg_len = d_segs + n + 1;
	}
}

// Copies a batch laid out as lay says to the device and returns what the kernels read of it.  The reads go up 2 bits per base (a
// quarter of the bytes) and k_unpack writes their ASCII copy on the device; a read with any byte other than A/C/G/T goes up as
// ASCII, and so does the whole batch when such reads are many or the fragments have segments (seg_off, seg_len: as BatchDev has
// them, or NULL).  t (or NULL) times the reads, the per-read tables and k_unpack.
static BatchDev upload_batch(Staging &B, const BatchLayout &lay, const Model *M, int n_reads, const int *qlens, const char *const *seqs,
							 const char *const *names, bool no_diag, const int32_t *seg_off, const int32_t *seg_len, mgb::HostPool &pool, int nt,
							 EvTimer *t, mgb_stats_t &S)
{
	const size_t n = (size_t)n_reads;
	const uint64_t *seq_off = batch_tables(B, lay, n_reads, qlens, names);
	char *hseq = (char*)B.h_seq.ensure(lay.seq_bytes), *d_seq = (char*)B.d_seq.ensure(lay.seq_bytes);
	const Pieces pcs(n_reads);
	BatchDev b;
	memset(&b, 0, sizeof(b));
	{
		Span span(t);
		// put(r) for the reads of each piece, then the piece's copy; returns the host's time
		auto in_pieces = [&](const std::function<void(int64_t)> &put, char *d, const char *h, const uint64_t *off, uint64_t end, uint64_t unit) {
			double t_pack = 0;
			for (int pc = 0; pc < pcs.n; ++pc) {
				const int64_t r0 = pcs.r0(pc), r1 = pcs.r0(pc + 1);
				const double tp0 = now_ms();
				pfor(pool, nt, r1 - r0, [&](int64_t i) { put(r0 + i); });
				t_pack += now_ms() - tp0;
				const uint64_t b0 = off[r0] * unit, b1 = (r1 < n_reads? off[r1] : end) * unit;
				h2d_async(d + b0, h + b0, b1 - b0);
			}
			return t_pack;
		};
		bool packed = seg_off == 0;
		uint64_t *pk_off = 0, *d_pk = 0, *d_pk_off = 0;
		if (packed) {
			const size_t n8 = (n + 7) & ~(size_t)7;
			pk_off = (uint64_t*)B.h_pk.ensure(n * 8 + 64 + (size_t)(lay.n_bases / 4) + n * 16);
			memcpy(pk_off, lay.pk_off.data(), n * 8);
			uint64_t *hpk = pk_off + n8;
			d_pk_off = (uint64_t*)B.d_pk.ensure((n8 + lay.n_words + 8) * 8);
			d_pk = d_pk_off + n8;
			std::vector<uint8_t> raw(n, 0);
			const double t_pack = in_pieces([&](int64_t r) { if (qlens[r] > 0 && !pack_read(seqs[r], qlens[r], hpk + pk_off[r])) raw[(size_t)r] = 1; },
											(char*)d_pk, (const char*)hpk, pk_off, lay.n_words, 8);
			int64_t n_raw = 0;
			for (size_t i = 0; i < n; ++i) n_raw += raw[i];
			if (n_raw > 64) packed = false; // not worth a copy per read
			else {
				S.t_pack_ms = t_pack;
				S.h2d_bytes = (int64_t)(lay.n_words * 8);
				for (size_t i = 0; i < n; ++i)
					if (raw[i]) {
						memcpy(hseq + seq_off[i], seqs[i], (size_t)qlens[i]);
						h2d_async(d_seq + seq_off[i], hseq + seq_off[i], (size_t)qlens[i]);
						pk_off[i] = ~0ULL, S.h2d_bytes += qlens[i];
					}
				h2d(d_pk_off, pk_off, n * 8);
			}
		}
		if (!packed) {
			S.t_pack_ms += in_pieces([&](int64_t r) { if (qlens[r] > 0) memcpy(hseq + seq_off[r], seqs[r], (size_t)qlens[r]); }, d_seq, hseq, seq_off, lay.seq_bytes, 1);
			dsync();
			S.h2d_bytes = (int64_t)lay.seq_bytes;
		}
		upload_tables(B, b, n_reads, seq_off, d_seq, S);
		b.pk = packed? d_pk : 0, b.pk_off = packed? d_pk_off : 0;
		if (packed) run_pass(UnpackRead{UnpackArgs{d_pk, d_pk_off, b.seq_off, b.seq_len, d_seq, n_reads}});
	}
	upload_read_extras(B, b, M, names, no_diag, seg_off, seg_len);
	return b;
}

// upload_batch() for reads in device memory: no base crosses PCIe.  The per-read tables and the reads' offsets go up, and k_ingest
// writes the ASCII copy, the 2-bit words (none for fragments with segments) and, for a read that holds any other byte than
// A/C/G/T, pk_off = ~0.  d_raw (or NULL) receives those flags.  t (or NULL) times the peer copy, the tables and k_ingest.
static BatchDev upload_batch_dev(Staging &B, const BatchLayout &lay, const Model *M, int n_reads, const int *qlens, const DevReads &R,
								 const char *const *names, bool no_diag, const int32_t *seg_off, const int32_t *seg_len, EvTimer *t, mgb_stats_t &S,
								 int32_t *d_raw = 0)
{
	const size_t n = (size_t)n_reads, n8 = (n + 7) & ~(size_t)7;
	const bool packed = seg_off == 0;
	const uint64_t *h_tables = batch_tables(B, lay, n_reads, qlens, names);
	char *d_seq = (char*)B.d_seq.ensure(lay.seq_bytes);
	BatchDev b;
	memset(&b, 0, sizeof(b));
	{
		Span span(t);
		uint64_t *h = (uint64_t*)B.h_pk.ensure(n8 * 16 + 64); // pk_off, then the reads' offsets in src
		memcpy(h, lay.pk_off.data(), n * 8);
		int64_t *src_off = (int64_t*)(h + n8);
		const char *src = R.src;
		if (R.copy) {
			int64_t lo = INT64_MAX, hi = 0;
			for (size_t i = 0; i < n; ++i) if (qlens[i] > 0) lo = std::min(lo, R.src_off[i]), hi = std::max(hi, R.src_off[i] + qlens[i]);
			if (lo > hi) lo = hi = 0;
			char *d_src = (char*)B.d_src.ensure((size_t)(hi - lo) + 16);
			d2d_peer(d_src, M->device, R.src + lo, R.src_dev, (size_t)(hi - lo));
			src = d_src;
			for (size_t i = 0; i < n; ++i) src_off[i] = R.src_off[i] - lo;
		} else memcpy(src_off, R.src_off, n * 8);
		uint64_t *d_pk_off = (uint64_t*)B.d_pk.ensure((2 * n8 + (packed? lay.n_words : 0) + 8) * 8);
		h2d(d_pk_off, h, n8 * 16);
		S.h2d_bytes = (int64_t)n * 16;
		upload_tables(B, b, n_reads, h_tables, d_seq, S);
		b.pk = packed? d_pk_off + 2 * n8 : 0, b.pk_off = packed? d_pk_off : 0;
		run_pass(IngestRead{IngestArgs{src, (const int64_t*)(d_pk_off + n8), b.seq_off, b.seq_len, d_seq, (uint64_t*)b.pk, d_pk_off, d_raw, n_reads}});
	}
	upload_read_extras(B, b, M, names, no_diag, seg_off, seg_len);
	return b;
}

// The slot's device scratch for a batch: the read list of the retry pass, the reads k_chain hands to k_chain_rescue, work counters,
// profile counters, pool headers and the tier histogram
struct PassScratch {
	int32_t *list, *rescue;
	unsigned int *next, *jobq_n, *rescue_n, *cnt, *tier_hist; // cnt: [0] bridging jobs, [1] gap jobs the next job kernel has to take
	unsigned long long *prof;
	Pool *pools;
	PassScratch(GrowBuf &buf, int n_reads)
	{
		list = (int32_t*)buf.ensure((size_t)n_reads * 8 + 4096 + 1024), rescue = list + n_reads;
		char *dsm = (char*)(((uintptr_t)(rescue + n_reads) + 255) & ~(uintptr_t)255);
		next = (unsigned int*)dsm, jobq_n = next + 4, rescue_n = next + 8, cnt = next + 10;
		prof = (unsigned long long*)(dsm + 64);
		pools = (Pool*)(dsm + 64 + sizeof(unsigned long long) * PROF_N);
		tier_hist = (unsigned int*)((char*)(pools + 16) + 64); // 32 x 4 counters behind the pool headers
	}
};

// One attempt at a batch: its pools, emptied, and one pass of the pipeline over its reads (run), or over the list of the
// large-arena retry.  Every kernel after k_gchain reads its number of items on the device, so a pass is queued without a host round
// trip, and nothing another thread does in the driver (large copies, blocking waits) can open gaps between its kernels; the mailbox
// at its end is its one wait.
struct Pass {
	Model::Slot &sl;
	const PassScratch &D;
	LaunchArgs L;
	int64_t max_jobs, jobs_done = 0, gjobs_done = 0;
	int32_t *jobq, *order; // the queues of tiers 2 and 3 (max_jobs each); the order of a job list
	unsigned int *lab_n;   // the sources k_chain listed for the label searches; NULL: no label table
	MailSrc msrc;
	Mail *mail;
	Pass(Model *M, Model::Slot &sl_, const MapOptDev &o, const BatchDev &b, const PassScratch &D_, const std::array<uint64_t, N_POOLS> &cap,
		 unsigned int *lab_n_, int32_t skip1) : sl(sl_), D(D_), lab_n(lab_n_)
	{
		void *buf[N_POOLS];
		Pool hp[N_POOLS];
		for (int i = 0; i < N_POOLS; ++i) buf[i] = sl.d_pool[i].ensure(cap[i]), hp[i].used = 0, hp[i].cap = cap[i];
		h2d(D.pools, hp, sizeof(hp));
		dfill(buf[P_GJOBS], 0xff, cap[P_GJOBS]); // reserved-but-unused bridging job slots read as rid == -1
		dfill(buf[P_JOBS], 0xff, cap[P_JOBS]);   // the same for gap jobs: slots of an allocation that overflowed the pool are never written
		memset(&L, 0, sizeof(L));
		L.c.g = M->g, L.c.ix = M->ix, L.c.opt = o, L.c.b = b;
		L.c.meta = (ReadMeta*)sl.d_meta.p, L.routs = (ReadOut*)sl.d_routs.p;
		L.c.pool_anchor = &D.pools[P_ANCHOR], L.c.anchor = (u128*)buf[P_ANCHOR];
		L.c.pool_minipos = &D.pools[P_MINIPOS], L.c.minipos = (int32_t*)buf[P_MINIPOS];
		L.c.pool_lchain = &D.pools[P_LCHAIN], L.c.lchain = (LChain*)buf[P_LCHAIN];
		L.c.pool_out = &D.pools[P_OUT], L.c.out = (char*)buf[P_OUT];
		L.c.pool_plan = &D.pools[P_PLAN], L.c.plan = (uint64_t*)buf[P_PLAN];
		L.c.pool_jobs = &D.pools[P_JOBS], L.c.jobs = (WfaJob*)buf[P_JOBS];
		L.c.pool_cig = &D.pools[P_CIG], L.c.cig = (uint32_t*)buf[P_CIG];
		L.c.pool_gstate = &D.pools[P_GSTATE], L.c.gstate = (char*)buf[P_GSTATE];
		L.c.pool_gjobs = &D.pools[P_GJOBS], L.c.gjobs = (GwfaJob*)buf[P_GJOBS];
		L.c.pool_walk = &D.pools[P_WALK], L.c.walk = (int32_t*)buf[P_WALK];
		L.c.next_read = D.next;
		L.c.rescue_list = D.rescue, L.c.rescue_n = D.rescue_n;
		if (lab_n) {
			L.c.lab.src_off = M->d_lab_off, L.c.lab.pool_hdr = M->d_lab_hdr, L.c.lab.pool = M->d_lab_pool, L.c.lab.new_src = (int32_t*)(lab_n + 4), L.c.lab.n_new = lab_n;
			L.c.lab.max_dist_g = M->lab_max_dist_g, L.c.lab.cap_new = M->g.n_seg * 2;
			dzero(lab_n, 2 * sizeof(unsigned int));
		}
		L.c.prof = D.prof;
		L.c.tier_hist = D.tier_hist, L.c.skip1_len = skip1;
		L.c.jobq_n = D.jobq_n;
		max_jobs = (int64_t)(cap[P_JOBS] / sizeof(WfaJob)) + 1;
		const int64_t max_gjobs = (int64_t)(cap[P_GJOBS] / sizeof(GwfaJob)) + 1;
		jobq = (int32_t*)sl.d_jobq.ensure(sizeof(int32_t) * 2 * (size_t)max_jobs);
		order = (int32_t*)sl.d_order.ensure(sizeof(int32_t) * (size_t)std::max<int64_t>(std::max<int64_t>(max_jobs, max_gjobs), b.n_reads));
		msrc.pools = D.pools, msrc.jobq_n = D.jobq_n, msrc.lab_n = lab_n, msrc.prof = D.prof, msrc.tier_hist = D.tier_hist, msrc.peak = sl.W.peak, msrc.n_workers = sl.W.n_workers;
		mail = (Mail*)sl.h_mail.p;
	}
	// list: the reads to run (NULL: all n_list of the batch); T: the timers of the spans (NULL: untimed)
	void run(const int32_t *list, int32_t n_list, const Workers &W, SlotTimers *T)
	{
		auto tk = [&](int s) { return T? &T->k[s] : (EvTimer*)0; };
		auto tm = [&](EvTimer SlotTimers::*m) { return T? &(T->*m) : (EvTimer*)0; };
		L.rid_list = list, L.n_work = n_list;
		{ Span t(tm(&SlotTimers::seed)), k(tk(S_SEED)); launch_stage<S_SEED>(L, W); }
		{
			Span t(tm(&SlotTimers::chain)), k(tk(S_CHAIN));
			dzero(D.rescue_n, sizeof(unsigned int));
			launch_stage<S_CHAIN>(L, W);
			L.n_work_dev = D.rescue_n, L.rid_list = 0; // the reads k_chain put on the rescue list (count known on the device only)
			launch_stage<S_CHAIN_RESCUE>(L, W);
			L.n_work_dev = 0, L.rid_list = list;
		}
		{
			Span t(tm(&SlotTimers::align));
			if (lab_n) { // labels of the sources k_chain listed (count known on the device only)
				L.n_work_dev = lab_n, L.rid_list = 0;
				Span tl(tm(&SlotTimers::lab));
				launch_stage<S_LABELS>(L, W);
				L.n_work_dev = lab_n + 1;
				launch_stage<S_LABELS_BIG>(L, W);
				L.n_work_dev = 0, L.rid_list = list;
			}
			{
				Span k(tk(S_GCHAIN));
				if (list == 0 && n_list >= 1024) { // whole batch: reads with many linear chains first (a few of them set the time of this kernel)
					make_job_order(L, 2, 0, n_list, order);
					L.rid_list = order;
				}
				launch_stage<S_GCHAIN>(L, W);
				L.rid_list = list;
			}
			// bridging jobs planned by k_gchain, then materialisation
			count_jobs(D.pools, (int)P_GJOBS, (int)P_JOBS, (unsigned int)gjobs_done, (unsigned int)jobs_done, D.cnt);
			L.rid_list = 0, L.job_start = gjobs_done, L.n_work = 0, L.n_work_dev = D.cnt;
			{ Span k(tk(S_GWFA)); make_job_order(L, 0, 0, 0, order, D.cnt); L.rid_list = order; launch_stage<S_GWFA>(L, W); }
			L.rid_list = list, L.n_work = n_list, L.n_work_dev = 0;
			{ Span k(tk(S_GCHAIN_GEN)); launch_stage<S_GCHAIN_GEN>(L, W); }
		}
		{ // three tiers; a job that does not fit one tier is queued for the next
			Span t(tm(&SlotTimers::wfa));
			count_jobs(D.pools, (int)P_GJOBS, (int)P_JOBS, (unsigned int)gjobs_done, (unsigned int)jobs_done, D.cnt);
			L.c.jobq[0] = jobq, L.c.jobq[1] = jobq + max_jobs;
			dzero(D.jobq_n, 2 * sizeof(unsigned int));
			L.rid_list = 0, L.job_start = jobs_done, L.n_work = 0, L.n_work_dev = D.cnt + 1;
			{ Span k(tk(S_WFA_SMALL)); launch_stage<S_WFA_SMALL>(L, W); }
			L.n_work_dev = D.jobq_n;
			{ // longest first: the long gaps, which run on one warp each, start early
				Span k(tk(S_WFA_MID));
				make_job_order(L, 1, L.c.jobq[0], 0, order, D.jobq_n);
				L.rid_list = order;
				launch_stage<S_WFA_MID>(L, W);
			}
			L.rid_list = 0, L.n_work_dev = D.jobq_n + 1;
			{ Span k(tk(S_WFA_BIG)); make_job_order(L, 1, L.c.jobq[1], 0, order, D.jobq_n + 1); L.rid_list = order; launch_stage<S_WFA_BIG>(L, W); }
			L.rid_list = 0, L.n_work_dev = 0;
		}
		L.rid_list = list, L.n_work = n_list;
		{ Span t(tm(&SlotTimers::fin)), k(tk(S_FINISH)); launch_stage<S_FINISH>(L, W); }
		ev_record(sl.ev_last);
		fetch_mail(msrc, mail); // (also the one wait of the pass)
		gjobs_done = (int64_t)(std::min<uint64_t>(mail->pools[P_GJOBS].used, mail->pools[P_GJOBS].cap) / sizeof(GwfaJob));
		jobs_done = (int64_t)(std::min<uint64_t>(mail->pools[P_JOBS].used, mail->pools[P_JOBS].cap) / sizeof(WfaJob));
	}
};

// The result blobs of a batch closed up in read order (k_scan, k_out_pack), then to the host in pieces, each followed by the event the
// assembly of its reads waits for.  routs gets the blobs' new places.  Returns the host copy.
static const char *download_blobs(Model::Slot &sl, int n_reads, ReadOut *routs, const char *d_out, uint64_t out_used, EvTimer &tm_d2h, mgb_stats_t &S)
{
	Span span(&tm_d2h);
	const size_t n = (size_t)n_reads;
	PackArgs P;
	P.routs = (ReadOut*)sl.d_routs.p, P.meta = (const ReadMeta*)sl.d_meta.p, P.n = n_reads, P.pool = d_out;
	P.packed = (char*)sl.d_packed.ensure(out_used + 64), P.off = (uint64_t*)sl.d_packoff.ensure(sizeof(uint64_t) * (n + 1));
	scan_u64(PackSize{P}, P.off, n_reads);
	run_pass(PackRead{P});
	d2h(routs, P.routs, sizeof(ReadOut) * n);
	std::vector<uint64_t> off(n + 1);
	d2h(off.data(), P.off, sizeof(uint64_t) * (n + 1));
	char *hout = (char*)sl.h_out.ensure(off[n] + 64);
	download_in_pieces(sl, n_reads, off.data(), hout, P.packed);
	S.out_bytes = (int64_t)off[n];
	return hout;
}

// mg_gchains_t objects (mg_map_batch, mg_map_batch_frag, mg_map_frag, mgb_map_batch_dev): fragment f's result in gcs[seg_first[f]]
// (gcs[f] without segments), every other entry of the n the caller passes NULL.  Parts write theirs in place.
struct GcsSink : Sink {
	mg_gchains_t **gcs;
	int64_t n;
	std::vector<std::unique_ptr<GcsSink>> parts;
	GcsSink(mg_gchains_t **gcs_, int64_t n_) : gcs(gcs_), n(n_) { for (int64_t i = 0; i < n; ++i) gcs[i] = 0; }
	int results(Model *M, Model::Slot &sl, const Batch &B, const Last &L, int host_threads) override;
	Sink &part(int b, int e, int) override { parts.emplace_back(new GcsSink(gcs + b, e - b)); return *parts.back(); }
	int join(Model *) override { return 0; }
	int empty(Model *) override { return 0; }
	int end(int rc) { if (rc < 0) mgb_free_batch((int)n, gcs); return rc; } // no partial results are left behind
};

// The blobs to the host (download_blobs, counted in w_download_ms), then the results built from them piece by piece as the pieces
// arrive.  t_d2h_ms: the pack kernels and the pieces of the copy (they overlap the assembly).
int GcsSink::results(Model *, Model::Slot &sl, const Batch &B, const Last &L, int host_threads)
{
	mgb_stats_t &S = sl.st;
	const double t0 = now_ms();
	const char *hout = download_blobs(sl, B.n, L.routs, L.d_out, L.out_used, sl.timers->d2h, S);
	const double t_asm0 = now_ms();
	S.w_download_ms += t_asm0 - t0;
	const Pieces pcs(B.n);
	for (int pc = 0; pc < pcs.n; ++pc) {
		const int64_t r0 = pcs.r0(pc);
		ev_wait(sl.ev_piece[pc]);
		pfor(sl.host_pool, host_threads, pcs.r0(pc + 1) - r0, [&](int64_t k) {
			const int64_t i = r0 + k; // an empty or over-long read (status 1): the reference returns before allocating (map-algo.c:359-360)
			if (B.n_seg && B.n_seg[i] <= 0) return; // (a fragment without segments has no entry)
			gcs[B.n_seg? B.seg_first[i] : i] = read_status(L.meta[i], L.routs[i]) == 1? 0 : build_result(L.routs[i], hout);
		});
	}
	S.t_asm_ms = now_ms() - t_asm0;
	return 0;
}

// Tier-1 routing for the batches to come: the first length bucket in which the sampled gaps mostly ended beyond tier 1
static void learn_tier_routing(Model *M, const unsigned int *h)
{
	int32_t t1 = INT32_MAX;
	for (int b = 0; b < 32 && t1 == INT32_MAX; ++b) { unsigned int in = h[b * 4 + 1], out = h[b * 4 + 2] + h[b * 4 + 3]; if (in + out >= 8 && in < out) t1 = b * 16; }
	unsigned int tot = 0;
	for (int i = 0; i < 128; ++i) tot += h[i];
	if (tot >= 64) { std::lock_guard<std::mutex> lock(M->big_mutex); M->skip1_len = t1; }
}

// Map the reads of sub-batch B on the calling thread's stream (slot `sl`): upload, passes until no output pool overflows, then the
// results through K
static int map_range(Model *M, Model::Slot &sl, const MapOptDev &o, const Batch &B, Sink &K, int host_threads)
{
	mgb_stats_t &S = sl.st;
	memset(&S, 0, sizeof(S));
	const int n_reads = B.n;
	const int *qlens = B.qlens;
	const char *const *names = B.names;
	const size_t n = (size_t)n_reads;
	const int32_t L_skip1 = M->skip1_len; // threshold this batch runs with
	const double t_host0 = now_ms();
	if (!sl.timers) sl.timers.reset(new SlotTimers());
	SlotTimers &TM = *sl.timers;
	TM.reset();
	const BatchLayout lay(n_reads, qlens);
	S.n_reads = n_reads, S.n_bases = lay.n_bases;
	const bool no_diag = (o.flag & F_NO_DIAG) != 0;
	const BatchDev b = B.dev? upload_batch_dev(sl.stage, lay, M, n_reads, qlens, *B.dev, names, no_diag, B.seg_off, B.seg_len, &TM.h2d, S)
							: upload_batch(sl.stage, lay, M, n_reads, qlens, B.seqs, names, no_diag, B.seg_off, B.seg_len, sl.host_pool, host_threads, &TM.h2d, S);
	// ---- device buffers (all persistent: cudaMalloc/cudaFree would serialise the slots) ----
	const PassScratch D(sl.d_scratch, n_reads);
	void *d_meta = sl.d_meta.ensure(sizeof(ReadMeta) * n), *d_routs = sl.d_routs.ensure(sizeof(ReadOut) * n);
	dzero(d_meta, sizeof(ReadMeta) * n);
	dzero(d_routs, sizeof(ReadOut) * n);
	dzero(D.prof, sizeof(unsigned long long) * PROF_N);
	dzero(D.tier_hist, sizeof(unsigned int) * 128);
	std::array<uint64_t, N_POOLS> cap = pool_caps(n_reads, lay.n_bases, sl.W.n_workers);
	for (int i = 0; i < N_POOLS; ++i) if (sl.d_pool[i].cap > cap[i]) cap[i] = sl.d_pool[i].cap & ~(size_t)4095; // keep what earlier batches needed
	ReadOut *routs = (ReadOut*)sl.h_routs.ensure((sizeof(ReadOut) + sizeof(ReadMeta)) * n + 64); // page-locked: a pageable destination makes the copy a blocking, staged one
	ReadMeta *meta = (ReadMeta*)(routs + n_reads);
	const bool use_lab = p_lab_cache && lab_prepare(M, o.bw_long);
	Mail *mail = (Mail*)sl.h_mail.ensure(sizeof(Mail));
	unsigned int *lab_n = use_lab? (unsigned int*)sl.d_lab_new.ensure(((size_t)M->g.n_seg * 2 + 4) * sizeof(int32_t)) : 0; // 2 counts, then the list
	const char *d_out = 0; // the output pool of the last attempt
	int rc = 0;
	for (int attempt = 0;; ++attempt) {
		Pass P(M, sl, o, b, D, cap, lab_n, L_skip1);
		{
			const double tq = now_ms();
			if (attempt == 0) S.w_upload_ms = tq - t_host0;
			std::lock_guard<std::mutex> gpu(M->gpu_mutex);
			const double tw = now_ms();
			S.w_gpu_wait_ms += tw - tq;
			if (attempt == 0) ev_record(sl.ev_first);
			P.run(0, n_reads, sl.W, &TM);
			S.w_pass_ms += now_ms() - tw;
		}
		S.n_jobs = P.jobs_done, S.n_jobs_mid = mail->jobq_n[0], S.n_jobs_big = mail->jobq_n[1];
		d2h(routs, P.L.routs, sizeof(ReadOut) * n);
		d2h(meta, P.L.c.meta, sizeof(ReadMeta) * n);
		// reads whose worker arena overflowed: run them again with large arenas and few workers (shared by the slots)
		std::vector<int32_t> redo;
		bool pool_full = false;
		for (int i = 0; i < n_reads; ++i) {
			const int st = read_status(meta[i], routs[i]);
			if (st == MGB_E_ARENA) redo.push_back(i);
			else if (st == MGB_E_POOL) pool_full = true;
		}
		if (!pool_full && !redo.empty()) {
			std::lock_guard<std::mutex> lock(M->big_mutex);
			uint64_t big = (uint64_t)p_arena_big_mb << 20;
			int nw = (int)std::min<uint64_t>(16, std::max<uint64_t>(1, dev_free_mem() / 2 / big)); // a handful of reads per batch at most come here
			if (M->Wbig.arena == 0 || M->Wbig.arena_bytes != big) ensure_workers(M->Wbig, std::max(1, nw), big);
			h2d(D.list, redo.data(), redo.size() * sizeof(int32_t));
			{ std::lock_guard<std::mutex> gpu(M->gpu_mutex); const double tw = now_ms(); P.run(D.list, (int32_t)redo.size(), M->Wbig, 0); S.w_redo_ms += now_ms() - tw; }
			S.n_retry += (int64_t)redo.size();
			d2h(routs, P.L.routs, sizeof(ReadOut) * n);
			d2h(meta, P.L.c.meta, sizeof(ReadMeta) * n);
			for (int i = 0; i < n_reads; ++i) if (read_status(meta[i], routs[i]) == MGB_E_POOL) pool_full = true;
		}
		fetch_mail(P.msrc, mail);
		if (use_lab) { S.n_lab_new = (int64_t)mail->lab_n[0], S.n_lab_big = (int64_t)mail->lab_n[1]; lab_after_batch(M, mail->lab_n[0]); }
		d_out = P.L.c.out;
		if (!pool_full) break;
		// grow whatever overflowed (used counts keep growing past cap, so they tell how much was wanted)
		for (int i = 0; i < N_POOLS; ++i) if (mail->pools[i].used > cap[i]) cap[i] = (mail->pools[i].used * 3 / 2 + 4095) & ~(uint64_t)4095;
		if (attempt == 7) { set_error("output pools kept overflowing"); rc = -2; break; }
	}
	TM.to_stats(S);
	if (B.dev) S.t_h2d_ms += B.dev->t_off_ms;
	S.arena_peak = mail->arena_peak; // (the mailbox was last filled after the last pass of the batch)
	for (int i = 0; i < 32; ++i) S.prof[i] = (uint64_t)mail->prof[i];
	learn_tier_routing(M, mail->tier_hist);
	S.skip1_len = L_skip1, S.skip2_len = INT32_MAX; // every gap that fits tier 2's lengths is aligned there
	if (rc < 0) return rc;

	// ---- results ----
	S.w_download_ms = now_ms() - t_host0 - S.w_upload_ms - S.w_pass_ms - S.w_redo_ms - S.w_gpu_wait_ms;
	for (int i = 0; i < n_reads; ++i) {
		const int st = read_status(meta[i], routs[i]);
		if (st < 0) {
			char buf[256];
			snprintf(buf, sizeof(buf), "read '%s' (%d bp) failed on the device with code %d%s", names && names[i]? names[i] : "", qlens[i], st,
					 st == MGB_E_ARENA? " (worker arena exhausted even in the retry pass; raise arena_big_mb)" : "");
			set_error(buf);
			return st;
		}
		S.n_seeds += meta[i].n_seed0, S.n_anchors_out += meta[i].n_a, S.n_chains_out += meta[i].n_u0, S.n_minimizers += meta[i].n_mz;
	}
	rc = K.results(M, sl, B, Last{meta, routs, d_out, std::min<uint64_t>(mail->pools[P_OUT].used, cap[P_OUT])}, host_threads);
	S.t_d2h_ms = TM.d2h.ms();
	S.t_host_ms = now_ms() - t_host0;
	return rc;
}

static thread_local mgb_stats_t t_last_stats; // of the last batch mapped by the calling thread
static thread_local bool t_has_stats = false;

// The glibc logf table of mapq (reference: gcmisc.c:216-217) for reads of up to max_qlen bases, into o.  Grown under the lock; old
// copies are kept until the model dies.
static void logf_prepare(Model *M, int32_t max_qlen, MapOptDev &o)
{
	std::lock_guard<std::mutex> lk(M->big_mutex);
	int need = std::max(1 << 16, max_qlen + 4096);
	if (M->n_logf < need) {
		M->logf_tab.resize(need);
		for (int i = 0; i < need; ++i) M->logf_tab[i] = logf((float)i);
		if (M->d_logf) M->dev_ptrs.push_back(M->d_logf); // a call in flight may still read it
		M->d_logf = upload(M->logf_tab.data(), M->logf_tab.size()).release();
		M->n_logf = need;
	}
	o.logf_tab = M->d_logf, o.n_logf_tab = M->n_logf;
}

// One call = one slot: its own stream, staging buffers, pools and worker arenas.  Up to "slots" calls run at once on one index
// (callers beyond that wait), so a host that maps mini-batch i+1 on a second thread overlaps its packing, copies and result
// assembly with the kernels of mini-batch i -- what the reference's kt_pipeline does with its step threads (gmap.c:176).
static int map_batch_on(Model *M, const Batch &B, Sink &K, const mg_mapopt_t *opt)
{
	double t0 = now_ms();
	int32_t max_qlen = 0;
	for (int i = 0; i < B.n; ++i) if (B.qlens[i] > max_qlen) max_qlen = B.qlens[i];
	int k = -1;
	{ // take a slot
		std::unique_lock<std::mutex> lk(M->big_mutex);
		const int max_slots = (int)std::max<int64_t>(1, std::min<int64_t>(p_slots, Model::MAX_SLOTS));
		M->slot_cv.wait(lk, [&]() { if (M->lab_growing) return false; for (int i = 0; i < max_slots; ++i) if (!M->slot_busy[i]) return true; return false; });
		for (int i = 0; i < max_slots && k < 0; ++i) if (!M->slot_busy[i]) k = i;
		M->slot_busy[k] = true, ++M->in_flight;
	}
	Model::Slot &sl = M->slots[k];
	const double t_slot = now_ms();
	int rc = 0;
	try {
		slot_prepare(M, sl, p_slot_workers > 0? (int)p_slot_workers : default_workers());
		MapOptDev o;
		fill_opt(o, opt, M->k);
		logf_prepare(M, max_qlen, o);
		int nt = (int)p_host_threads;
		if (nt <= 0) { nt = (int)std::thread::hardware_concurrency(); if (nt > 16) nt = 16; if (nt < 1) nt = 1; }
		t_launches = 0;
		rc = map_range(M, sl, o, B, K, nt);
	} catch (const MgbError &e) {
		rc = e.code;
	}
	dev_bind(M->device, 0); // the slot's stream dies with the model; later calls on this thread (mg_index of another graph) use the default one
	mgb_stats_t S = sl.st;
	S.n_launches = t_launches;
	S.w_slot_wait_ms = t_slot - t0;
	if (rc == 0) S.t_dev_span_ms = ev_ms(sl.ev_first, sl.ev_last);
	S.n_slots = k;
	S.t_host_ms = now_ms() - t0;
	t_last_stats = S, t_has_stats = true;
	{
		std::lock_guard<std::mutex> lk(M->big_mutex);
		M->stats = S;
		M->slot_busy[k] = false, --M->in_flight;
	}
	M->slot_cv.notify_all();
	return rc;
}

// The batch on every device of the index: contiguous parts of about equal bases, one host thread per device, each part's results
// into its part of K, joined by K in input order.  A batch with segments, or too small to split, maps on the index's device alone.
static int map_batch_impl(Model *M, const Batch &B, Sink &K, const mg_mapopt_t *opt)
{
	if (B.n <= 0) return K.empty(M);
	const int n_dev = 1 + (int)M->peers.size();
	if (n_dev == 1 || B.seg_off || B.n < 2 * n_dev) return map_batch_on(M, B, K, opt);
	for (Model *P : M->peers) if (P == 0) { set_error("the index is missing on one of the MGB_DEVICES"); return MGB_E_INTERNAL; }
	int64_t tot = 0;
	for (int i = 0; i < B.n; ++i) tot += B.qlens[i] > 0? B.qlens[i] : 0;
	std::vector<int> bound((size_t)n_dev + 1, B.n);
	bound[0] = 0;
	{
		int64_t acc = 0; int k = 1;
		for (int i = 0; i < B.n && k < n_dev; ++i) {
			acc += B.qlens[i] > 0? B.qlens[i] : 0;
			if (acc >= tot * k / n_dev) bound[(size_t)k++] = i + 1;
		}
	}
	auto on = [&](int d) { return d == 0? M : M->peers[(size_t)d - 1]; };
	std::vector<Batch> parts;
	std::vector<Sink*> sinks;
	for (int d = 0; d < n_dev; ++d) {
		parts.push_back(B.part(bound[(size_t)d], bound[(size_t)d + 1], d));
		sinks.push_back(&K.part(bound[(size_t)d], bound[(size_t)d + 1], on(d)->device));
	}
	std::vector<int> rcs((size_t)n_dev, 0);
	std::vector<std::thread> th;
	for (int d = 0; d < n_dev; ++d)
		th.emplace_back([&, d]() { if (parts[(size_t)d].n > 0) rcs[(size_t)d] = map_batch_on(on(d), parts[(size_t)d], *sinks[(size_t)d], opt); });
	for (auto &t : th) t.join();
	int rc = 0;
	for (int d = 0; d < n_dev; ++d) if (rcs[(size_t)d] < 0 && rc == 0) rc = rcs[(size_t)d];
	if (rc == 0) try { rc = K.join(M); } catch (const MgbError &e) { rc = e.code; }
	dev_bind(M->device, 0);
	return rc;
}

// The eight entry points below check their input, describe the reads (make_batch) and where the results go (a sink), and map.

extern "C" int mg_map_batch(const mg_idx_t *gi, int n_reads, const int *qlens, const char *const *seqs, const char *const *names,
							mg_gchains_t **gcs, const mg_mapopt_t *opt)
{
	GcsSink K(gcs, std::max(n_reads, 0));
	return K.end(map_batch_impl((Model*)gi->B, make_batch(n_reads, 0, qlens, seqs, names, 0), K, opt));
}

// Fragments of several segments (read pairs) in one go: fragment f has n_seg[f] consecutive entries of qlens/seqs/gcs starting at
// seg_off[f] = n_seg[0] + ... + n_seg[f-1]; gcs[seg_off[f]] receives the result of the concatenated fragment and the other
// entries NULL, exactly what worker_for() leaves behind without MG_M_INDEPEND_SEG (gmap.c:46-48).  names[f] is per fragment.
extern "C" int mg_map_batch_frag(const mg_idx_t *gi, int n_frag, const int *n_seg, const int *qlens, const char *const *seqs, const char *const *names,
								 mg_gchains_t **gcs, const mg_mapopt_t *opt)
{
	int64_t n_tot = 0;
	for (int f = 0; f < n_frag; ++f) n_tot += n_seg[f] > 0? n_seg[f] : 0;
	GcsSink K(gcs, n_tot);
	return K.end(map_batch_impl((Model*)gi->B, make_batch(n_frag, n_seg, qlens, seqs, names, 0), K, opt));
}

// Map a batch and return its GAF text, formatted on the device.
extern "C" int mgb_map_batch_gaf(const mg_idx_t *gi, int n_frag, const int *n_seg, const int *qlens, const char *const *seqs, const char *const *names,
								 const mg_mapopt_t *opt, char **out, size_t *out_len, size_t *out_cap)
{
	GafSink K(opt->flag, out, out_len, out_cap);
	if (int rc = GafSink::refuse(opt)) return K.end(rc);
	return K.end(map_batch_impl((Model*)gi->B, make_batch(n_frag, n_seg, qlens, seqs, names, 0), K, opt));
}

// ---- reads in device memory (mgb_map_batch_dev, mgb_map_batch_dev_gaf, mgb_map_batch_dev_rec, mgb_map_batch_dev_rec_ds) ----
// A batch whose n_seq + 1 offsets d_off (sequence i is d_seq[d_off[i] .. d_off[i+1])) are in device memory: checks the buffers, copies
// the offsets back once the caller's stream has got past the work queued on it, checks them, and gives the sequences' lengths and
// their DevReads.  Returns 0, or a negative code with the reason set.
struct DevBatch {
	std::vector<int64_t> off;
	std::vector<int> qlen;
	DevReads R;
};
static int dev_batch_prepare(const mg_idx_t *gi, const char *who, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
							 const int64_t *d_off, const mg_mapopt_t *opt, void *stream, DevBatch &D)
{
	auto refuse = [&](const std::string &why) { set_error(std::string(who) + ": " + why); return (int)MGB_E_UNSUPPORTED; };
	if (gi == 0 || opt == 0 || n_frag < 0 || n_seq < 0 || seq_bytes < 0 || d_off == 0 || (seq_bytes > 0 && d_seq == 0))
		return refuse("an index, options, the offsets, and counts and seq_bytes at least 0");
	if (n_seg == 0 && n_seq != n_frag) return refuse("n_seq must be n_frag when n_seg is NULL");
	if (n_seg) {
		int64_t tot = 0;
		for (int f = 0; f < n_frag; ++f) tot += n_seg[f] > 0? n_seg[f] : 0;
		if (tot != n_seq) return refuse("the fragments' segments add up to " + std::to_string(tot) + ", not n_seq = " + std::to_string(n_seq));
	}
	const Model *M = model_of(gi);
	D.off.assign((size_t)n_seq + 1, 0);
	D.R.src = d_seq, D.R.src_off = D.off.data(), D.R.src_dev = M->device, D.R.copy = false, D.R.t_off_ms = 0;
#ifdef MGB_HOSTSIM
	(void)stream;
	memcpy(D.off.data(), d_off, sizeof(int64_t) * ((size_t)n_seq + 1));
#else
	CUDA_OK(cudaSetDevice(M->device));
	const void *bufs[2] = {d_off, seq_bytes > 0? (const void*)d_seq : 0};
	for (int k = 0; k < 2; ++k) {
		if (bufs[k] == 0) continue;
		cudaPointerAttributes a;
		const bool ok = cudaPointerGetAttributes(&a, bufs[k]) == cudaSuccess && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == M->device;
		cudaGetLastError();
		if (!ok) return refuse(std::string(k? "d_seq" : "d_off") + " is not device or managed memory on the index's device " + std::to_string(M->device));
	}
	CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
	const double t0 = now_ms();
	CUDA_OK(cudaMemcpy(D.off.data(), d_off, sizeof(int64_t) * ((size_t)n_seq + 1), cudaMemcpyDeviceToHost));
	D.R.t_off_ms = now_ms() - t0;
#endif
	D.qlen.resize((size_t)std::max(n_seq, 1));
	for (int i = 0; i <= n_seq; ++i)
		if (D.off[(size_t)i] < 0 || D.off[(size_t)i] > seq_bytes) return refuse("offset " + std::to_string(i) + " lies outside [0, seq_bytes]");
	for (int i = 0; i < n_seq; ++i) {
		const int64_t l = D.off[(size_t)i + 1] - D.off[(size_t)i];
		if (l < 0) return refuse("the offsets decrease at sequence " + std::to_string(i));
		if (l > INT32_MAX) return refuse("sequence " + std::to_string(i) + " is longer than INT32_MAX");
		D.qlen[(size_t)i] = (int)l;
	}
	if (n_seg) { // a fragment's segments follow each other in d_seq: it is mapped from there as one read
		for (int f = 0, i = 0; f < n_frag; ++f) {
			const int ns = n_seg[f] > 0? n_seg[f] : 0;
			if (D.off[(size_t)(i + ns)] - D.off[(size_t)i] > INT32_MAX) return refuse("fragment " + std::to_string(f) + " is longer than INT32_MAX");
			i += ns;
		}
	}
	return 0;
}

extern "C" int mgb_map_batch_dev(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
								 const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream, mg_gchains_t **gcs)
{
	GcsSink K(gcs, std::max(n_seq, 0));
	try {
		DevBatch D;
		if (int rc = dev_batch_prepare(gi, "mgb_map_batch_dev", n_frag, n_seg, n_seq, d_seq, seq_bytes, d_off, opt, stream, D)) return rc;
		return K.end(map_batch_impl((Model*)gi->B, make_batch(n_frag, n_seg, D.qlen.data(), 0, names, &D.R), K, opt));
	} catch (const MgbError &e) { return K.end(e.code); }
}

extern "C" int mgb_map_batch_dev_gaf(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
									 const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream, char **out, size_t *out_len,
									 size_t *out_cap)
{
	GafSink K(opt? opt->flag : 0, out, out_len, out_cap);
	try {
		DevBatch D;
		if (int rc = dev_batch_prepare(gi, "mgb_map_batch_dev_gaf", n_frag, n_seg, n_seq, d_seq, seq_bytes, d_off, opt, stream, D)) return K.end(rc);
		if (int rc = GafSink::refuse(opt)) return K.end(rc);
		return K.end(map_batch_impl((Model*)gi->B, make_batch(n_frag, n_seg, D.qlen.data(), 0, names, &D.R), K, opt));
	} catch (const MgbError &e) { return K.end(e.code); }
}

// mgb_map_batch_dev_rec(), and with ds_out mgb_map_batch_dev_rec_ds()
static int dev_rec(const char *who, const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
				   const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream, mgb_dev_alloc_fn alloc, void *alloc_ctx,
				   mgb_records_t *out, mgb_records_ds_t *ds_out, bool with_ds)
{
	if (out) memset(out, 0, sizeof(*out));
	if (ds_out) memset(ds_out, 0, sizeof(*ds_out));
	try {
		if (alloc == 0 || out == 0 || (with_ds && ds_out == 0)) {
			set_error(std::string(who) + (with_ds? ": an allocator, an mgb_records_t and an mgb_records_ds_t for the tables" : ": an allocator and an mgb_records_t for the tables"));
			return MGB_E_UNSUPPORTED;
		}
		DevBatch D;
		if (int rc = dev_batch_prepare(gi, who, n_frag, n_seg, n_seq, d_seq, seq_bytes, d_off, opt, stream, D)) return rc;
		RecSink K(alloc, alloc_ctx, stream, model_of(gi)->device, with_ds);
		return K.end(out, ds_out, map_batch_impl((Model*)gi->B, make_batch(n_frag, n_seg, D.qlen.data(), 0, names, &D.R), K, opt));
	} catch (const MgbError &e) { return e.code; }
}

extern "C" int mgb_map_batch_dev_rec(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
									 const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream,
									 mgb_dev_alloc_fn alloc, void *alloc_ctx, mgb_records_t *out)
{
	return dev_rec("mgb_map_batch_dev_rec", gi, n_frag, n_seg, n_seq, d_seq, seq_bytes, d_off, names, opt, stream, alloc, alloc_ctx, out, 0, false);
}

extern "C" int mgb_map_batch_dev_rec_ds(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
										const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream,
										mgb_dev_alloc_fn alloc, void *alloc_ctx, mgb_records_t *out, mgb_records_ds_t *ds_out)
{
	return dev_rec("mgb_map_batch_dev_rec_ds", gi, n_frag, n_seg, n_seq, d_seq, seq_bytes, d_off, names, opt, stream, alloc, alloc_ctx, out, ds_out, true);
}

// ---- FASTA/FASTQ text in device memory (mgb_reads_parse_dev, mgb_fastx.cuh) ----
// The passes of mgb_fastx.cuh on the caller's stream, with the scratch of M; the host reads back the list totals, one jump per
// round, the number of records and the call's FxSum.  Returns 0, or a negative code with the reason set and nothing in R.
static int reads_parse(Model *M, const char *text, int64_t n, int64_t max_bases, int final, void *stream, mgb_dev_alloc_fn alloc,
					   void *alloc_ctx, mgb_dev_reads_t &R)
{
	auto refuse = [&](const std::string &why) { set_error("mgb_reads_parse_dev: " + why); return (int)MGB_E_UNSUPPORTED; };
	auto al = [](uint64_t x) { return (x + 255) & ~(uint64_t)255; };
#ifndef MGB_HOSTSIM
	CUDA_OK(cudaSetDevice(M->device));
	if (n > 0) {
		cudaPointerAttributes pa;
		const bool ok = cudaPointerGetAttributes(&pa, text) == cudaSuccess && (pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged) && pa.device == M->device;
		cudaGetLastError();
		if (!ok) return refuse("the text is not device or managed memory on the index's device " + std::to_string(M->device));
	}
#endif
	dev_bind(M->device, (DevStream)(uintptr_t)stream);
	const int64_t n_chunks = (n + FX_CHUNK - 1) / FX_CHUNK;
	if (n_chunks >= INT32_MAX) return refuse("a text of " + std::to_string(n) + " bytes");
	FxArgs A;
	memset(&A, 0, sizeof(A));
	A.text = text, A.n_text = n, A.n_chunks = (int)n_chunks, A.max_bases = max_bases, A.final_ = final != 0;
	Model::FxScratch &X = M->fx;
	A.tab = (uint64_t*)X.tab.ensure(8 * FX_NLIST * ((size_t)n_chunks + 1));
	uint64_t tot[FX_NLIST] = {0, 0, 0, 0};
	if (n_chunks > 0) {
		A.n = A.n_chunks;
		run_pass(FxCount{A});
		scan_u64(ScanCols<FX_NLIST>{A.tab}, A.tab, A.n_chunks);
		d2h(tot, A.tab + FX_NLIST * n_chunks, sizeof(tot));
	}
	if (tot[FX_HD] >= (uint64_t)INT32_MAX) return refuse("more than INT32_MAX - 1 '>' and '@' bytes in one text");
	const int64_t C = (int64_t)tot[FX_HD], n_groups = (C + 1 + 31) / 32;
	// the lists | the jumps, twice | the marks | the records before each group
	uint64_t o = 0, o_list[FX_NLIST];
	for (int k = 0; k < FX_NLIST; ++k) o_list[k] = o, o += al(8 * tot[k]);
	const uint64_t o_j0 = o, o_j1 = o_j0 + al(4 * (C + 1)), o_mark = o_j1 + al(4 * (C + 1)), o_grp = o_mark + al(C + 1);
	char *d = (char*)X.lists.ensure(o_grp + 8 * (n_groups + 1));
	for (int k = 0; k < FX_NLIST; ++k) A.list[k] = (int64_t*)(d + o_list[k]);
	int32_t *J[2] = {(int32_t*)(d + o_j0), (int32_t*)(d + o_j1)};
	A.mark = (uint8_t*)(d + o_mark);
	uint64_t *grp = (uint64_t*)(d + o_grp);
	A.n_cand = C;
	if (n_chunks > 0) run_pass(FxLists{A});
	A.n = (int)n_groups, A.jout = J[0];
	run_pass(FxSucc{A});
	for (int k = 0; C > 0; ++k) { // until the first candidate's jump passes the end: then every record is marked
		int32_t j0 = 0;
		d2h(&j0, J[k & 1], 4);
		if (j0 == (int32_t)C) break;
		A.jin = J[k & 1], A.jout = J[(k + 1) & 1];
		run_pass(FxJump{A});
	}
	scan_u64(FxMarks{A}, grp, (int)n_groups);
	uint64_t K = 0;
	d2h(&K, grp + n_groups, 8);
	// per record: its row | bases and name bytes | the call's FxSum and FxCopy's counter
	const uint64_t o_lens = al(sizeof(FxRow) * K), o_sum = o_lens + al(16 * (K + 1));
	char *e = (char*)X.recs.ensure(o_sum + sizeof(FxSum) + 16);
	A.grp = grp, A.rows = (FxRow*)e, A.lens = (uint64_t*)(e + o_lens), A.sum = (FxSum*)(e + o_sum), A.next = (unsigned int*)(A.sum + 1);
	A.n_rec = (int64_t)K;
	dfill(A.sum, 0x7f, sizeof(FxSum)); // first_long: none
	run_pass(FxRecs{A});
	scan_u64(ScanCols<2>{A.lens}, A.lens, (int)K);
	A.n = 1;
	run_pass(FxTail{A});
	FxSum s;
	d2h(&s, A.sum, sizeof(s));
	if (s.first_long < s.n_reads) return refuse("record " + std::to_string(s.first_long) + " is longer than INT32_MAX bases");
	const int64_t bytes[MGB_DR_NTAB] = {s.n_bases, 8 * (s.n_reads + 1), s.name_bytes, 8 * (s.n_reads + 1)};
	int64_t at = 0;
	for (int t = 0; t < MGB_DR_NTAB; ++t) R.off[t] = at, at += (int64_t)al((uint64_t)bytes[t]);
	char *b = (char*)alloc(alloc_ctx, (size_t)at);
	if (b == 0) { set_error("mgb_reads_parse_dev: the allocator returned no block of " + std::to_string(at) + " bytes"); return MGB_E_INTERNAL; }
	A.seq = b + R.off[MGB_DR_SEQ], A.name = b + R.off[MGB_DR_NAME];
	A.off = (int64_t*)(b + R.off[MGB_DR_OFF]), A.name_off = (int64_t*)(b + R.off[MGB_DR_NAME_OFF]);
	A.n = (int)s.n_reads;
	run_pass(FxCopy{A});
	h2d_async(A.off + s.n_reads, &s.n_bases, 8); // the rows of totals
	h2d_async(A.name_off + s.n_reads, &s.name_bytes, 8);
	dsync();
	R.n_reads = s.n_reads, R.n_bases = s.n_bases, R.name_bytes = s.name_bytes, R.used = s.used, R.block = b, R.bytes = at;
	return 0;
}

extern "C" int mgb_reads_parse_dev(const mg_idx_t *gi, const char *d_text, int64_t text_bytes, int64_t max_bases, int final, void *stream,
								   mgb_dev_alloc_fn alloc, void *alloc_ctx, mgb_dev_reads_t *out)
{
	if (out) memset(out, 0, sizeof(*out));
	if (gi == 0 || alloc == 0 || out == 0 || text_bytes < 0 || (text_bytes > 0 && d_text == 0)) {
		set_error("mgb_reads_parse_dev: an index, an allocator, an mgb_dev_reads_t, and text_bytes at least 0 with the text");
		return MGB_E_UNSUPPORTED;
	}
	Model *M = (Model*)gi->B;
	std::lock_guard<std::mutex> lk(M->fx.mu);
	mgb_dev_reads_t R;
	memset(&R, 0, sizeof(R));
	int rc;
	try { rc = reads_parse(M, d_text, text_bytes, max_bases, final, stream, alloc, alloc_ctx, R); } catch (const MgbError &e) { rc = e.code; }
	dev_bind(M->device, 0);
	if (rc == 0) *out = R;
	return rc;
}

extern "C" void mg_map_frag(const mg_idx_t *gi, int n_segs, const int *qlens, const char **seqs, mg_gchains_t **gcs, mg_tbuf_t *b, const mg_mapopt_t *opt, const char *qname)
{
	(void)b;
	GcsSink K(gcs, std::max(n_segs, 0));
	if (n_segs <= 0) return;
	const Batch B = make_batch(1, &n_segs, qlens, seqs, &qname, 0); // segments: one result, concatenated, no CIGAR (map-algo.c:356-360,366,457-464)
	if (B.seg_off && B.qlens[0] == 0) return; // (also more than MG_MAX_SEG segments)
	if (map_batch_impl((Model*)gi->B, B, K, opt) < 0) abort(); // the reference aborts on internal errors too
}

extern "C" mg_gchains_t *mg_map(const mg_idx_t *gi, int qlen, const char *seq, mg_tbuf_t *b, const mg_mapopt_t *opt, const char *qname)
{
	mg_gchains_t *gcs;
	mg_map_frag(gi, 1, &qlen, &seq, &gcs, b, opt, qname);
	return gcs;
}

// ---------------------------------------------------------------------------------------------------------------
// test hooks: one piece of device code run on inputs from the tests, launched as its pipeline kernel launches it
// ---------------------------------------------------------------------------------------------------------------
static const int NO_STAGE = -1;                              // a hook that mirrors no stage: its slice is not set up
static const uint32_t TEST_SMEM_FILL = 0x00050005u;          // two cells holding offset 5, a value a real wavefront holds

// A hook's body(i, slice, A, worker, lane) runs item i on all lanes of a warp, with the warp's slice of shared memory (NULL: none),
// its arena and its number, and returns a code on which the lanes agree.
#ifndef MGB_HOSTSIM
template<int S, typename Body>
__global__ void k_test(Body body, int n, int smem, char *arena, uint64_t arena_bytes)
{
	extern __shared__ int4 dyn_smem[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
	for (int j = threadIdx.x; j < n_warps * smem / 4; j += blockDim.x) ((uint32_t*)dyn_smem)[j] = TEST_SMEM_FILL;
	__syncthreads();
	int32_t *slice = smem? (int32_t*)((char*)dyn_smem + (size_t)warp * smem) : 0;
	stage_warp_init<S>(slice, lane);
	const int worker = blockIdx.x * n_warps + warp;
	Arena A;
	arena_init(A, arena + (uint64_t)worker * arena_bytes, arena_bytes);
	for (int i = worker; i < n; i += gridDim.x * n_warps) body(i, slice, A, worker, lane);
}
#endif

// Runs body on items 0..n-1 in blocks of `warps` warps (by default stage S's) with `smem` bytes of shared memory per warp (by default
// stage S's slice), n_workers warps rounded up to whole blocks.  Each warp's slice starts out filled with junk and is then set up as
// stage S sets it up; each warp has an arena of arena_bytes.  Warp w runs items w, w + (warps launched), ... in this order, so that
// the results also show that a warp reuses its slice dirty and keeps to its own.  The simulators run the warps one after the
// other, each on its own slice and arena.  Returns 0, or MGB_E_INTERNAL when the lanes of a simulated warp returned different codes.
template<int S, typename Body>
static int test_launch(int n, int n_workers, uint64_t arena_bytes, const Body &body, int warps = StageSpec<S>::warps, int smem = StageSpec<S>::smem)
{
	const int blocks = (n_workers + warps - 1) / warps, n_warps = blocks * warps;
	DevBuf<char> arena((size_t)arena_bytes * n_warps);
#ifdef MGB_HOSTSIM
	std::vector<uint32_t> sim_smem((size_t)n_warps * smem / 4 + 1, TEST_SMEM_FILL);
	bool differ = false;
	for (int w = 0; w < n_warps; ++w) {
		int32_t *slice = smem? (int32_t*)((char*)sim_smem.data() + (size_t)w * smem) : 0;
		sim_warp(S, -1, [&](int lane) { stage_warp_init<S>(slice, lane); return 0; }, &differ);
		for (int i = w; i < n; i += n_warps)
			sim_warp(S, i, [&](int lane) { Arena A; arena_init(A, arena + (uint64_t)w * arena_bytes, arena_bytes); return body(i, slice, A, w, lane); }, &differ);
	}
	if (differ) { set_error("simulated warp: lanes returned different codes from a test hook"); return MGB_E_INTERNAL; }
#else
	const size_t smem_b = (size_t)warps * smem;
	if (smem_b > 48 * 1024) CUDA_OK(cudaFuncSetAttribute(k_test<S, Body>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_b));
	k_test<S, Body><<<blocks, warps * 32, smem_b, t_stream>>>(body, n, smem, arena, arena_bytes);
	CUDA_OK(cudaGetLastError());
	dsync();
#endif
	return 0;
}

// the hooks run only where their kernels run
static int test_no_device(int dev = -1)
{
	if (dev_ok(dev)) return 0;
	set_error("no CUDA device available: libmgb200 has no CPU path");
	return -100;
}

static int64_t test_seq_bytes(int n, const int64_t *off, const int32_t *len)
{
	int64_t end = 0;
	for (int i = 0; i < n; ++i) end = std::max(end, off[i] + len[i]);
	return end;
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: one gap alignment through the tier-3 path (exact WFA capped at max_iter cells, then the chaining
// heuristic with low-memory checkpoints every `step` scores), reference: miniwfa.c:824-834 mwf_wfa_auto
// ---------------------------------------------------------------------------------------------------------------
struct TestWfa {
	const char *ts, *qs; int32_t tl, ql, step, cap; int64_t max_iter; uint32_t *cigar; int32_t *out;
	MG_HD int operator()(int, int32_t *, Arena &A, int, int lane) const
	{
		WfResult r;
		WfTbJob *tb = (WfTbJob*)arena_alloc(A, sizeof(WfTbJob)); // a batch of one
		int rc = wfa_exact(A, tl, ts, ql, qs, max_iter, &r, lane, step);
		if (rc == 0) {
			wfa_tb_keep(tb, r, tl, ts, ql, qs, 0, lane);
			wfa_tb_batch(tb, 1, lane);
			rc = tb->rc;
		}
		const int32_t n_cig = rc == 0? tb->n_cigar : 0;
		if (rc == 0 && n_cig <= cap) for (int32_t i = lane; i < n_cig; i += MGB_W) cigar[i] = tb->cig[tb->first + i];
		if (lane == 0) out[0] = rc, out[1] = n_cig, out[2] = rc == 0? r.s : 0;
		return 0;
	}
};
static int test_wfa_impl(const char *ts, int tl, const char *qs, int ql, int64_t max_iter, int step, uint32_t *cigar, int cap, int *score)
{
	if (int e = test_no_device()) return e;
	DevBuf<char> ts_d((size_t)tl + 64), qs_d((size_t)ql + 64);
	h2d(ts_d, ts, (size_t)tl), h2d(qs_d, qs, (size_t)ql);
	DevBuf<uint32_t> cigar_d(cap);
	DevBuf<int32_t> out_d(4);
	TestWfa t;
	t.ts = ts_d, t.qs = qs_d, t.tl = tl, t.ql = ql, t.step = step, t.cap = cap, t.max_iter = max_iter, t.cigar = cigar_d, t.out = out_d;
	if (int e = test_launch<NO_STAGE>(1, 1, (uint64_t)1 << 30, t, 1, 0)) return e;
	int32_t out[4] = {0, 0, 0, 0};
	d2h(out, out_d, sizeof(out));
	if (out[0] == 0 && out[1] <= cap) d2h(cigar, cigar_d, sizeof(uint32_t) * (size_t)out[1]);
	*score = out[2];
	return out[0] < 0? out[0] : out[1];
}

extern "C" int mgb_test_wfa(const char *ts, int tl, const char *qs, int ql, int64_t max_iter, int step, uint32_t *cigar, int cap, int *score)
{
	try { return test_wfa_impl(ts, tl, qs, ql, max_iter, step, cigar, cap, score); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: a batch of gaps through one on-chip WFA tier, wfa_smem() with the template arguments of k_wfa_small (tier 1)
// or k_wfa_mid (tier 2), launched as those kernels are (test_launch), the tracebacks in the batches those kernels run (WfaBatch):
// warp w takes gaps w, w + n_workers, ...  The junk in the slices is cells that are not -inf, so the results also show that
// wfa_smem() clears the slices it reads.
// ---------------------------------------------------------------------------------------------------------------
struct TestTier {
	int tier, cap, n, n_workers;
	const char *ts, *qs;
	const int64_t *t_off, *q_off;
	const int32_t *tl, *ql;
	int64_t *out;       // per gap: rc (0: aligned, 1: does not fit the tier), score, n_iter, n_cigar
	uint32_t *cigar;    // per gap: cap entries
	struct Gaps { // what the gaps are to the batch
		const TestTier &t;
		int32_t *smem;
		MG_HD void put(int i, int64_t rc, int64_t s, int64_t n_iter, int64_t n_cigar, int lane) const
		{
			if (lane == 0) { int64_t *o = t.out + 4 * (int64_t)i; o[0] = rc, o[1] = s, o[2] = n_iter, o[3] = n_cigar; }
		}
		MG_HD int run(int i, Arena &A, WfTbJob *tb, int lane) const
		{
			WfResult r;
			const char *ts_i = t.ts + t.t_off[i], *qs_i = t.qs + t.q_off[i];
			int64_t cont_cells = 0;
			const int rc = t.tier == 1? wfa_smem<WfTier1::W_, WfTier1::MAXLEN_, WfTier1::TBCAP_>(A, smem, t.tl[i], ts_i, t.ql[i], qs_i, &r, lane)
					: t.tier == 2? wfa_smem<WfTier2::W_, WfTier2::MAXLEN_, WfTier2::TBCAP_>(A, smem, t.tl[i], ts_i, t.ql[i], qs_i, &r, lane)
								 : wfa_smem<WfTier2::W_, WfTier2::MAXLEN_, WfTier2::TBCAP_, true>(A, smem, t.tl[i], ts_i, t.ql[i], qs_i, &r, lane, &cont_cells);
			if (rc == 1) put(i, 1, -1, 0, 0, lane);
			if (rc != 0) return rc < 0? rc : 0;
			wfa_tb_keep(tb, r, t.tl[i], ts_i, t.ql[i], qs_i, i, lane);
			return 1;
		}
		MG_HD int done(const WfTbJob &b, int lane) const
		{
			if (b.rc < 0) return b.rc;
			if (b.n_cigar > t.cap) return MGB_E_INTERNAL;
			for (int32_t j = lane; j < b.n_cigar; j += MGB_W) t.cigar[b.job * t.cap + j] = b.cig[b.first + j];
			put((int)b.job, 0, b.s, b.n_iter, b.n_cigar, lane);
			return 0;
		}
		MG_HD void fail(int i, int rc, int lane) const { put(i, rc, -1, 0, 0, lane); }
		MG_HD void traced(unsigned long long, int) const {}
	};
	MG_HD int operator()(int w, int32_t *smem, Arena &A, int, int lane) const
	{
		const Gaps g{*this, smem};
		WfaBatch<Gaps> batch;
		batch.open(A);
		for (int i = w; i < n; i += n_workers) batch.add(g, i, A, lane);
		batch.flush(g, A, lane);
		warp_sync();
		return 0;
	}
};

static int test_wfa_tier_impl(int tier, int n, const char *ts, const int64_t *t_off, const int32_t *tl, const char *qs, const int64_t *q_off,
							  const int32_t *ql, int64_t *out, uint32_t *cigar, int cap)
{
	if ((tier != 1 && tier != 2 && tier != MGB_TEST_TIER2_CONT) || n < 0 || cap < 0) {
		set_error("mgb_test_wfa_tier: tier must be 1, 2 or MGB_TEST_TIER2_CONT, n and cap at least 0");
		return MGB_E_UNSUPPORTED;
	}
	for (int i = 0; i < n; ++i) // the gaps of real jobs are never empty on either side (galign.c:97-99 emits plain I/D for those)
		if (tl[i] < 1 || ql[i] < 1 || t_off[i] < 0 || q_off[i] < 0) { set_error("mgb_test_wfa_tier: gap " + std::to_string(i) + " has an empty side"); return MGB_E_UNSUPPORTED; }
	if (n == 0) return 0;
	if (int e = test_no_device()) return e;
	auto ts_d = upload(ts, test_seq_bytes(n, t_off, tl)), qs_d = upload(qs, test_seq_bytes(n, q_off, ql));
	auto t_off_d = upload(t_off, n), q_off_d = upload(q_off, n);
	auto tl_d = upload(tl, n), ql_d = upload(ql, n);
	DevBuf<int64_t> out_d(4 * (size_t)n);
	DevBuf<uint32_t> cigar_d((size_t)n * cap + 1);
	TestTier t;
	const int warps = tier == 1? StageSpec<S_WFA_SMALL>::warps : StageSpec<S_WFA_MID>::warps;
	t.tier = tier, t.cap = cap, t.n = n, t.n_workers = (std::min(n, 64 * warps) + warps - 1) / warps * warps; // whole blocks, as launched
	t.ts = ts_d, t.qs = qs_d, t.t_off = t_off_d, t.q_off = q_off_d, t.tl = tl_d, t.ql = ql_d, t.out = out_d, t.cigar = cigar_d;
	// a tier-2 gap needs at most 8 KB of CIGAR and 70 KB of traceback rows; one carried on in the arena at most 230 KB of ring and
	// 4.3 MB of traceback rows (scores below tl + ql + 30, rows of at most tl + ql + 1 bytes).  A batch is flushed once it keeps a
	// quarter of the arena.
	const uint64_t arena_bytes = tier == MGB_TEST_TIER2_CONT? (uint64_t)5 << 20 : (uint64_t)256 << 10;
	const int rc = tier == 1? test_launch<S_WFA_SMALL>(t.n_workers, t.n_workers, arena_bytes, t)
							: test_launch<S_WFA_MID>(t.n_workers, t.n_workers, arena_bytes, t);
	if (rc) return rc;
	d2h(out, out_d, sizeof(int64_t) * 4 * (size_t)n);
	d2h(cigar, cigar_d, sizeof(uint32_t) * (size_t)n * cap);
	return 0;
}

extern "C" int mgb_test_wfa_tier(int tier, int n, const char *ts, const int64_t *t_off, const int32_t *tl, const char *qs, const int64_t *q_off,
								 const int32_t *ql, int64_t *out, uint32_t *cigar, int cap)
{
	try { return test_wfa_tier_impl(tier, n, ts, t_off, tl, qs, q_off, ql, out, cigar, cap); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: bridging alignments (reference: gchain1.c:349-381 bridge_gwfa) on the device graph of an index, with the
// options bridge_gwfa gives gfa_ed_init/gfa_ed_step.  mode 0: gwf_align_w() on one warp, the alignment state in shared
// memory and the arena in global memory, as k_gwfa runs it (gwfa_job_run); mode 1: the sequential gwf_align() on lane 0,
// as graph chaining runs it (gc_bridge_gwfa).
// ---------------------------------------------------------------------------------------------------------------
struct TestGwfa {
	GraphDev g;
	int mode, walk_cap;
	const char *q;
	const int64_t *q_off;
	const int32_t *ql, *off0, *off1, *max_ed;
	const uint32_t *v0, *v1;
	int64_t *out;       // per bridge: rc, s, end_v, end_off, nv, n_iter
	int32_t *walk;      // per bridge: walk_cap vertices
	MG_HD int operator()(int i, int32_t *smem, Arena &A, int, int lane) const
	{
		GwfShared *sh = (GwfShared*)smem;
		GwfOpt opt;
		opt.traceback = 1, opt.max_chk = 1000, opt.bw_dyn = 1000, opt.max_lag = max_ed[i] / 2, opt.s_term = -1;
		opt.i_term = 500000000LL;
		A.top = 0, A.peak = 0;
		const char *q_i = q + q_off[i];
		int rc = 0;
		GwfResult rs;
		const GwfResult *r = &rs;
		if (mode == 0) {
			if (lane == 0) sh->A = A;
			warp_sync();
			rc = gwf_align_w(sh, g, opt, ql[i], q_i, v0[i], off0[i], v1[i], off1[i], max_ed[i], lane); // s_term: max_ed
			r = &sh->r;
		} else {
			if (lane == 0) rc = gwf_align(A, g, opt, ql[i], q_i, v0[i], off0[i], v1[i], off1[i], max_ed[i], &rs);
			rc = warp_bcast_i32(rc, 0);
		}
		if (lane == 0) {
			int64_t *o = out + 6 * (int64_t)i;
			const int32_t nv = rc == 0 && r->s >= 0? r->nv : 0;
			if (nv > walk_cap) rc = MGB_E_INTERNAL;
			o[0] = rc;
			o[1] = rc == 0? r->s : -1, o[2] = rc == 0? (int64_t)r->end_v : -1, o[3] = rc == 0? r->end_off : -1;
			o[4] = rc == 0? nv : 0, o[5] = rc == 0? r->n_iter : 0;
			if (rc == 0) for (int32_t j = 0; j < nv; ++j) walk[(int64_t)i * walk_cap + j] = r->v[j];
		}
		warp_sync();
		return 0;
	}
};

static int test_gwfa_impl(const mg_idx_t *gi, int mode, int n, const char *q, const int64_t *q_off, const int32_t *ql, const uint32_t *v0,
						  const int32_t *off0, const uint32_t *v1, const int32_t *off1, const int32_t *max_ed, int64_t *out, int32_t *walk, int walk_cap)
{
	if (gi == 0 || (mode != 0 && mode != 1) || n < 0 || walk_cap < 0) { set_error("mgb_test_gwfa: an index, mode 0 or 1, n and walk_cap at least 0"); return MGB_E_UNSUPPORTED; }
	const Model *M = model_of(gi);
	for (int i = 0; i < n; ++i)
		if (ql[i] < 1 || q_off[i] < 0 || (v0[i] >> 1) >= (uint32_t)M->g.n_seg || (v1[i] >> 1) >= (uint32_t)M->g.n_seg || off0[i] < 0 || off0[i] >= M->seg_len[v0[i] >> 1]
			|| off1[i] < 0 || off1[i] >= M->seg_len[v1[i] >> 1]) {
			set_error("mgb_test_gwfa: bridge " + std::to_string(i) + " has an empty query or an end outside the graph");
			return MGB_E_UNSUPPORTED;
		}
	if (n == 0) return 0;
	if (int e = test_no_device(M->device)) return e;
	auto q_d = upload(q, test_seq_bytes(n, q_off, ql));
	auto q_off_d = upload(q_off, n);
	auto ql_d = upload(ql, n), off0_d = upload(off0, n), off1_d = upload(off1, n), max_ed_d = upload(max_ed, n);
	auto v0_d = upload(v0, n), v1_d = upload(v1, n);
	DevBuf<int64_t> out_d(6 * (size_t)n);
	DevBuf<int32_t> walk_d((size_t)n * walk_cap + 1);
	TestGwfa t;
	t.g = M->g, t.mode = mode, t.walk_cap = walk_cap;
	t.q = q_d, t.q_off = q_off_d, t.ql = ql_d, t.off0 = off0_d, t.off1 = off1_d, t.max_ed = max_ed_d, t.v0 = v0_d, t.v1 = v1_d, t.out = out_d, t.walk = walk_d;
	if (int e = test_launch<S_GWFA>(n, std::min(n, 8 * StageSpec<S_GWFA>::warps), (uint64_t)64 << 20, t)) return e;
	d2h(out, out_d, sizeof(int64_t) * 6 * (size_t)n);
	d2h(walk, walk_d, sizeof(int32_t) * (size_t)n * walk_cap);
	return 0;
}

extern "C" int mgb_test_gwfa(const mg_idx_t *gi, int mode, int n, const char *q, const int64_t *q_off, const int32_t *ql, const uint32_t *v0,
							 const int32_t *off0, const uint32_t *v1, const int32_t *off1, const int32_t *max_ed, int64_t *out, int32_t *walk, int walk_cap)
{
	try { return test_gwfa_impl(gi, mode, n, q, q_off, ql, v0, off0, v1, off1, max_ed, out, walk, walk_cap); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: the warp-wide exact radix sort on an array of 16-byte records, in place or with the digit walk, on one warp with
// `hot_bytes` of shared memory for the range stack and bin tables (0: everything in the arena in global memory), as k_seed sorts
// its seeds; tests/cases.py holds it against klib's.
// ---------------------------------------------------------------------------------------------------------------
struct TestRadix {
	u128 *a; int64_t n; int walk, hot_bytes; int32_t *rc;
	MG_HD int operator()(int, int32_t *hot, Arena &A, int, int lane) const
	{
		Arena H;
		arena_init(H, hot, hot_bytes > 0? (uint64_t)hot_bytes : 0);
		const int r = radix_sort_128x_w(hot_bytes > 0? H : A, a, n, lane, &A, walk != 0);
		if (lane == 0) *rc = r;
		return r;
	}
};

static int test_radix128_impl(u128 *a, int64_t n, int walk, int hot_bytes)
{
	if (n < 0 || hot_bytes < 0 || hot_bytes > 200 * 1024) { set_error("mgb_test_radix128: n >= 0 and 0 <= hot_bytes <= 200 KB"); return MGB_E_UNSUPPORTED; }
	if (int e = test_no_device()) return e;
	auto a_d = upload(a, n);
	DevBuf<int32_t> rc_d(1);
	TestRadix t;
	t.a = a_d, t.n = n, t.walk = walk, t.hot_bytes = hot_bytes, t.rc = rc_d;
	if (int e = test_launch<NO_STAGE>(1, 1, (uint64_t)n * 64 + (1 << 20), t, 1, hot_bytes)) return e;
	int32_t rc = 0;
	d2h(&rc, rc_d, sizeof(rc));
	if (rc == 0) d2h(a, a_d, sizeof(u128) * (size_t)n);
	return rc;
}

extern "C" int mgb_test_radix128(mg128_t *a, int64_t n, int walk, int hot_bytes)
{
	static_assert(sizeof(mg128_t) == sizeof(u128), "mg128_t and u128 are the same record");
	try { return test_radix128_impl((u128*)a, n, walk, hot_bytes); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: the linear chaining of k_chain (mode 0: DP, 1: RMQ) or k_chain_rescue (mode 2: sort into target order, RMQ) on
// anchor sets with options of their own, launched as those kernels are (test_launch), the anchors staged into the slice when
// they fit (chain_staged, chain_run: the code of stage_chain).  Each warp chains several sets in a row, so it reuses its slice
// dirty, flips the parity of its barrier and moves between staged and unstaged sets.  Set i goes to worker i % n_workers.
// ---------------------------------------------------------------------------------------------------------------
struct TestLchain {
	int mode;
	uint64_t slice;       // bytes of shared memory per warp
	u128 *a;              // every set's anchors, chained in place: the compacted anchors are read back from here
	const int64_t *off;
	const int32_t *cnt;
	const LChainOpt *opt;
	int32_t *out;         // per set: rc, n_u, n_v, staged, path, worker
	uint64_t *u;          // per set: the chains at u[off[i]..]
	MG_HD int operator()(int i, int32_t *smem, Arena &A, int worker, int lane) const
	{
		A.top = 0;
		u128 *a_i = a + off[i];
		const int64_t n = cnt[i];
		const LChainOpt &co = opt[i];
		int32_t n_u = 0, n_v = 0;
		uint64_t *u_i = 0;
		int path = -1, staged = 0;
		const int rc = chain_staged(smem, slice, A, a_i, n, lane, &staged, [&](Arena &H, u128 *aw, int32_t *n_keep) {
			const int r = mode == 2? chain_run<1>(H, A, 1, co, n, aw, &n_u, &u_i, &n_v, lane, &path) : chain_run<0>(H, A, mode == 1, co, n, aw, &n_u, &u_i, &n_v, lane, &path);
			*n_keep = n_u > 0? n_v : 0;
			return r;
		});
		if (rc == 0) for (int32_t j = lane; j < n_u; j += MGB_W) u[off[i] + j] = u_i[j];
		if (lane == 0) {
			int32_t *o = out + 6 * (int64_t)i;
			o[0] = rc, o[1] = n_u, o[2] = n_v, o[3] = staged, o[4] = path, o[5] = worker;
		}
		warp_sync();
		return 0;
	}
};

static int test_lchain_impl(int mode, int n, const u128 *a, const int64_t *off, const int32_t *cnt, const mgb_lchain_opt_t *opt, int32_t *out, uint64_t *u, u128 *a_out)
{
#define MGB_SAME_FIELD(f) static_assert(offsetof(mgb_lchain_opt_t, f) == offsetof(LChainOpt, f) && sizeof(mgb_lchain_opt_t::f) == sizeof(LChainOpt::f), "mgb_lchain_opt_t and LChainOpt differ in " #f)
	MGB_SAME_FIELD(max_dist_x); MGB_SAME_FIELD(max_dist_y); MGB_SAME_FIELD(bw); MGB_SAME_FIELD(max_skip); MGB_SAME_FIELD(max_iter); MGB_SAME_FIELD(min_cnt);
	MGB_SAME_FIELD(min_sc); MGB_SAME_FIELD(pen_gap); MGB_SAME_FIELD(pen_skip); MGB_SAME_FIELD(is_cdna); MGB_SAME_FIELD(n_seg); MGB_SAME_FIELD(max_dist_inner);
	MGB_SAME_FIELD(cap_rmq_size);
#undef MGB_SAME_FIELD
	static_assert(sizeof(mgb_lchain_opt_t) == sizeof(LChainOpt), "mgb_lchain_opt_t and LChainOpt are the same record");
	if (mode < 0 || mode > 2 || n < 0) { set_error("mgb_test_lchain: mode 0, 1 or 2 and n at least 0"); return MGB_E_UNSUPPORTED; }
	int64_t max_cnt = 0;
	for (int i = 0; i < n; ++i) {
		if (cnt[i] < 0 || off[i] < 0) { set_error("mgb_test_lchain: set " + std::to_string(i) + " has a negative offset or count"); return MGB_E_UNSUPPORTED; }
		max_cnt = std::max(max_cnt, (int64_t)cnt[i]);
	}
	if (n == 0) return 0;
	if (int e = test_no_device()) return e;
	const int64_t n_a = test_seq_bytes(n, off, cnt);
	auto a_d = upload(a, n_a);
	auto off_d = upload(off, n);
	auto cnt_d = upload(cnt, n);
	auto opt_d = upload((const LChainOpt*)opt, n);
	DevBuf<int32_t> out_d(6 * (size_t)n);
	DevBuf<uint64_t> u_d((size_t)n_a + 1);
	TestLchain t;
	t.mode = mode, t.slice = mode == 2? StageSpec<S_CHAIN_RESCUE>::smem : StageSpec<S_CHAIN>::smem;
	t.a = a_d, t.off = off_d, t.cnt = cnt_d, t.opt = opt_d, t.out = out_d, t.u = u_d;
	// per anchor at most ~200 bytes: f/p/v/t, the RMQ window, priorities and block summaries, the end-point list, the compaction's
	// copy, and the two AVL trees of the sequential fill
	const uint64_t arena_bytes = (uint64_t)max_cnt * 512 + ((uint64_t)1 << 20);
	const int rc = mode == 2? test_launch<S_CHAIN_RESCUE>(n, std::min(n, 2 * StageSpec<S_CHAIN_RESCUE>::warps), arena_bytes, t)
							: test_launch<S_CHAIN>(n, std::min(n, 2 * StageSpec<S_CHAIN>::warps), arena_bytes, t);
	if (rc) return rc;
	d2h(out, out_d, sizeof(int32_t) * 6 * (size_t)n);
	d2h(u, u_d, sizeof(uint64_t) * (size_t)n_a);
	d2h(a_out, a_d, sizeof(u128) * (size_t)n_a);
	return 0;
}

extern "C" int mgb_test_lchain(int mode, int n, const mg128_t *a, const int64_t *off, const int32_t *cnt, const mgb_lchain_opt_t *opt, int32_t *out,
							   uint64_t *u, mg128_t *a_out)
{
	try { return test_lchain_impl(mode, n, (const u128*)a, off, cnt, opt, out, u, (u128*)a_out); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: the minimizer sketch of n sequences, launched as k_seed is (test_launch).  mode 0: sketch_seq_w() on the warp, the
// window rings in the warp's slice and, for a sequence that is all A/C/G/T, the 2-bit words of the host packer of the batch upload
// (stage_seed); mode 1: sketch_seq() on lane 0 (k_index_sketch).  Sequence i is sketched with rid i.
// ---------------------------------------------------------------------------------------------------------------
struct TestSketch {
	int k, w, mode;
	const char *seq;
	const int64_t *off, *pk_off, *mz_off; // pk_off[i] < 0: sequence i has other letters and no 2-bit words
	const int32_t *len;
	const uint64_t *pk;
	int32_t *out;         // per sequence: rc, n, path
	u128 *mz;             // list i at mz[mz_off[i]..mz_off[i+1])
	MG_HD int operator()(int i, int32_t *smem, Arena &A, int, int lane) const
	{
		A.top = 0;
		AVec<u128> mv;
		avec_init(mv);
		const char *s = seq + off[i];
		int rc = 0, path = -1;
		if (mode == 0) rc = sketch_seq_w(A, s, len[i], w, k, (uint32_t)i, mv, lane, (u128*)smem, pk_off[i] >= 0? pk + pk_off[i] : 0, &path);
		else if (lane == 0) rc = sketch_seq(A, s, len[i], w, k, (uint32_t)i, mv); // the list is lane 0's alone
		rc = warp_bcast_i32(rc, 0);
		const int64_t n = rc == 0? (int64_t)warp_bcast_u64((uint64_t)mv.n, 0) : 0;
		if (n <= mz_off[i + 1] - mz_off[i]) {
			if (mode == 0) for (int64_t j = lane; j < n; j += MGB_W) mz[mz_off[i] + j] = mv.a[j];
			else if (lane == 0) for (int64_t j = 0; j < n; ++j) mz[mz_off[i] + j] = mv.a[j];
		}
		if (lane == 0) out[3 * (int64_t)i] = rc, out[3 * (int64_t)i + 1] = (int32_t)n, out[3 * (int64_t)i + 2] = path;
		warp_sync();
		return 0;
	}
};

static int test_sketch_impl(int k, int w, int n, const char *seq, const int64_t *off, const int32_t *len, int mode, int32_t *out, u128 *mz, const int64_t *mz_off)
{
	static_assert(SKETCH_PATH_SMEM_PK == MGB_SKETCH_PATH_SMEM_PK && SKETCH_PATH_SMEM == MGB_SKETCH_PATH_SMEM && SKETCH_PATH_ARENA == MGB_SKETCH_PATH_ARENA
				  && SKETCH_PATH_SEQ == MGB_SKETCH_PATH_SEQ, "the sketch paths of mgb200.h are mgb_seed.cuh's");
	if (k < 1 || k > 28 || w < 1 || w > 255 || (mode != 0 && mode != 1) || n < 0) {
		set_error("mgb_test_sketch: 1 <= k <= 28, 1 <= w <= 255, mode 0 or 1 and n at least 0");
		return MGB_E_UNSUPPORTED;
	}
	int32_t max_len = 0;
	for (int i = 0; i < n; ++i) { // the sketch of an empty sequence is not defined (sketch.c:63 asserts)
		if (len[i] < 1 || off[i] < 0 || mz_off[i] < 0 || mz_off[i + 1] < mz_off[i]) {
			set_error("mgb_test_sketch: sequence " + std::to_string(i) + " is empty or has a bad offset");
			return MGB_E_UNSUPPORTED;
		}
		max_len = std::max(max_len, len[i]);
	}
	if (n == 0) return 0;
	if (int e = test_no_device()) return e;
	const BatchLayout lay(n, len); // the words as a batch lays them out
	std::vector<int64_t> pk_off((size_t)n);
	std::vector<uint64_t> hpk(lay.n_words);
	for (int i = 0; i < n; ++i) pk_off[(size_t)i] = pack_read(seq + off[i], len[i], hpk.data() + lay.pk_off[(size_t)i])? (int64_t)lay.pk_off[(size_t)i] : -1;
	auto seq_d = upload(seq, test_seq_bytes(n, off, len));
	auto off_d = upload(off, n), pk_off_d = upload(pk_off.data(), n), mz_off_d = upload(mz_off, (size_t)n + 1);
	auto len_d = upload(len, n);
	auto pk_d = upload(hpk.data(), hpk.size());
	DevBuf<int32_t> out_d(3 * (size_t)n);
	DevBuf<u128> mz_d((size_t)mz_off[n] + 1);
	TestSketch t;
	t.k = k, t.w = w, t.mode = mode, t.seq = seq_d, t.off = off_d, t.pk_off = pk_off_d, t.mz_off = mz_off_d, t.len = len_d, t.pk = pk_d;
	t.out = out_d, t.mz = mz_d;
	// the chunk lists and rings (about 16 bytes per base and window slot), or the sequential list grown in the arena
	const uint64_t arena_bytes = (uint64_t)max_len * 256 + ((uint64_t)1 << 20);
	if (int e = test_launch<S_SEED>(n, std::min(n, 2 * StageSpec<S_SEED>::warps), arena_bytes, t)) return e;
	d2h(out, out_d, sizeof(int32_t) * 3 * (size_t)n);
	d2h(mz, mz_d, sizeof(u128) * (size_t)mz_off[n]);
	return 0;
}

extern "C" int mgb_test_sketch(int k, int w, int n, const char *seq, const int64_t *off, const int32_t *len, int mode, int32_t *out, mg128_t *mz, const int64_t *mz_off)
{
	try { return test_sketch_impl(k, w, n, seq, off, len, mode, out, (u128*)mz, mz_off); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: the ingest step of reads in device memory as mgb_map_batch_dev uploads them (upload_batch_dev, k_ingest): sequence i is
// seq[off[i] .. off[i+1]), copied to the device first.  Its ASCII copy goes to ascii_out[off[i]..], its 2-bit words (unless segmented)
// follow those of sequence i-1 in pk_out, its flag to raw_out[i].  pk_off must be ~0 exactly for the flagged reads.
// ---------------------------------------------------------------------------------------------------------------
static int test_ingest_impl(int n, const char *seq, const int64_t *off, int segmented, char *ascii_out, uint64_t *pk_out, int32_t *raw_out)
{
	if (n < 0 || (n > 0 && (off == 0 || off[0] < 0))) { set_error("mgb_test_ingest: n at least 0 and offsets from 0"); return MGB_E_UNSUPPORTED; }
	std::vector<int> qlen((size_t)std::max(n, 1));
	for (int i = 0; i < n; ++i) {
		if (off[i + 1] < off[i] || off[i + 1] - off[i] > INT32_MAX) { set_error("mgb_test_ingest: sequence " + std::to_string(i) + " has a bad length"); return MGB_E_UNSUPPORTED; }
		qlen[(size_t)i] = (int)(off[i + 1] - off[i]);
	}
	if (n == 0) return 0;
	if (int e = test_no_device()) return e;
	auto seq_d = upload(seq, (size_t)off[n]);
	const BatchLayout lay(n, qlen.data());
	std::vector<int32_t> seg_off((size_t)n + 1), seg_len(qlen.begin(), qlen.begin() + n); // segmented: one segment per read
	for (int i = 0; i <= n; ++i) seg_off[(size_t)i] = i;
	DevReads R;
	R.src = seq_d, R.src_off = off, R.src_dev = (int)p_device, R.copy = false, R.t_off_ms = 0;
	DevBuf<int32_t> raw_d((size_t)n);
	Staging stg;
	mgb_stats_t st = {};
	const BatchDev b = upload_batch_dev(stg, lay, 0, n, qlen.data(), R, 0, false, segmented? seg_off.data() : 0, segmented? seg_len.data() : 0, 0, st, raw_d);
	std::vector<char> hseq(lay.seq_bytes);
	d2h(hseq.data(), b.seq, lay.seq_bytes);
	d2h(raw_out, raw_d, sizeof(int32_t) * (size_t)n);
	for (int i = 0; i < n; ++i) memcpy(ascii_out + off[i], hseq.data() + lay.seq_off[(size_t)i], (size_t)qlen[(size_t)i]);
	if (segmented) {
		if (b.pk || b.pk_off) { set_error("mgb_test_ingest: words of fragments with segments"); return MGB_E_INTERNAL; }
		return 0;
	}
	std::vector<uint64_t> pk(lay.n_words + 1), pk_off((size_t)n);
	d2h(pk.data(), b.pk, sizeof(uint64_t) * lay.n_words);
	d2h(pk_off.data(), b.pk_off, sizeof(uint64_t) * (size_t)n);
	int64_t at = 0;
	for (int i = 0; i < n; ++i) {
		const int nw = (qlen[(size_t)i] + 31) / 32;
		memcpy(pk_out + at, pk.data() + lay.pk_off[(size_t)i], sizeof(uint64_t) * (size_t)nw);
		at += nw;
		if (pk_off[(size_t)i] != (raw_out[i]? ~0ULL : lay.pk_off[(size_t)i])) {
			set_error("mgb_test_ingest: read " + std::to_string(i) + ": pk_off does not follow its flag");
			return MGB_E_INTERNAL;
		}
	}
	return 0;
}

extern "C" int mgb_test_ingest(int n, const char *seq, const int64_t *off, int segmented, char *ascii_out, uint64_t *pk_out, int32_t *raw_out)
{
	try { return test_ingest_impl(n, seq, off, segmented, ascii_out, pk_out, raw_out); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: stage_seed() itself on a batch uploaded as mg_map_batch uploads it (upload_batch), with the graph and index of gi and
// the options flag, occ_max1 and max_qlen, launched as k_seed is (test_launch).  The seeds and mini_pos of each read are read back
// from the pools.
// ---------------------------------------------------------------------------------------------------------------
struct TestSeed {
	PipeCtx c;
	MG_HD int operator()(int i, int32_t *smem, Arena &A, int, int lane) const
	{
		A.top = 0;
		const int rc = stage_seed(c, i, A, lane, smem);
		if (rc < 0 && lane == 0) c.meta[i].status = rc; // as stage_fail records a failed read
		warp_sync();
		return 0;
	}
};

static int test_seed_impl(const mg_idx_t *gi, int n, const int *qlens, const char *const *seqs, const int32_t *seg_off, const int32_t *seg_len,
						  const char *const *names, uint64_t flag, int occ_max1, int max_qlen, int32_t *out, u128 *a, int64_t a_cap, int32_t *mini_pos, int64_t mp_cap)
{
	if (gi == 0 || n < 0 || a_cap < 0 || mp_cap < 0) { set_error("mgb_test_seed: an index, n and the capacities at least 0"); return MGB_E_UNSUPPORTED; }
	for (int i = 0; i < n; ++i) {
		int64_t sum = 0;
		if (seg_off) {
			if (seg_off[i] < 0 || seg_off[i + 1] <= seg_off[i]) { set_error("mgb_test_seed: read " + std::to_string(i) + " has no segment"); return MGB_E_UNSUPPORTED; }
			for (int32_t j = seg_off[i]; j < seg_off[i + 1]; ++j) {
				if (seg_len[j] < 1) { set_error("mgb_test_seed: read " + std::to_string(i) + " has an empty segment"); return MGB_E_UNSUPPORTED; } // map-algo.c:34-45 sketches every one
				sum += seg_len[j];
			}
		}
		if (qlens[i] < 0 || (seg_off && sum != qlens[i]) || (qlens[i] > 0 && seqs[i] == 0)) {
			set_error("mgb_test_seed: read " + std::to_string(i) + " has a bad length");
			return MGB_E_UNSUPPORTED;
		}
	}
	if (n == 0) return 0;
	const Model *M = model_of(gi);
	if (int e = test_no_device(M->device)) return e;
	DevBuf<ReadMeta> meta_d((size_t)n);
	DevBuf<Pool> pools_d(2);
	TestSeed t;
	memset(&t.c, 0, sizeof(t.c));
	t.c.g = M->g, t.c.ix = M->ix;
	t.c.opt.flag = flag, t.c.opt.occ_max1 = occ_max1, t.c.opt.max_qlen = max_qlen;
	const BatchLayout lay(n, qlens);
	Staging stg;
	mgb::HostPool one;
	mgb_stats_t st = {};
	t.c.b = upload_batch(stg, lay, M, n, qlens, seqs, names, (flag & F_NO_DIAG) != 0, seg_off, seg_len, one, 1, 0, st);
	t.c.meta = meta_d, t.c.pool_anchor = pools_d, t.c.pool_minipos = pools_d + 1;
	// the first pools of a batch, doubled while a read runs out of them (the batch's retry)
	const std::array<uint64_t, N_POOLS> cap = pool_caps(n, lay.n_bases, 0);
	uint64_t cap_a = cap[P_ANCHOR], cap_mp = cap[P_MINIPOS];
	std::vector<ReadMeta> meta((size_t)n);
	for (;;) {
		DevBuf<u128> anchor_d(cap_a / sizeof(u128));
		DevBuf<int32_t> mp_d(cap_mp / sizeof(int32_t));
		Pool hp[2];
		hp[0].used = 0, hp[0].cap = cap_a, hp[1].used = 0, hp[1].cap = cap_mp;
		h2d(pools_d, hp, sizeof(hp));
		dzero(meta_d, sizeof(ReadMeta) * (size_t)n);
		t.c.anchor = anchor_d, t.c.minipos = mp_d;
		// a read's lists in the arena: minimizers and matches (~120 bytes per base at w = 1), the sort's scratch when off chip
		int32_t max_len = 0;
		for (int i = 0; i < n; ++i) max_len = std::max(max_len, qlens[i]);
		const uint64_t arena_bytes = (uint64_t)max_len * 256 + ((uint64_t)16 << 20);
		if (int e = test_launch<S_SEED>(n, std::min(n, 2 * StageSpec<S_SEED>::warps), arena_bytes, t)) return e;
		d2h(meta.data(), meta_d, sizeof(ReadMeta) * (size_t)n);
		bool pool_full = false;
		for (int i = 0; i < n; ++i) pool_full |= meta[(size_t)i].status == MGB_E_POOL;
		if (pool_full) { cap_a *= 2, cap_mp *= 2; continue; }
		int64_t sum_a = 0, sum_mp = 0;
		for (int i = 0; i < n; ++i) {
			const ReadMeta &m = meta[(size_t)i];
			int32_t *o = out + 5 * (int64_t)i;
			o[0] = m.status, o[1] = m.n_mz, o[2] = m.rep_len, o[3] = m.n_a, o[4] = m.n_mp;
			if (m.status != 0) continue;
			if (sum_a + m.n_a <= a_cap) d2h(a + sum_a, (const u128*)anchor_d + m.a_off, sizeof(u128) * (size_t)m.n_a);
			if (sum_mp + m.n_mp <= mp_cap) d2h(mini_pos + sum_mp, (const int32_t*)mp_d + m.mp_off, sizeof(int32_t) * (size_t)m.n_mp);
			sum_a += m.n_a, sum_mp += m.n_mp;
		}
		if (sum_a > a_cap || sum_mp > mp_cap) { set_error("mgb_test_seed: the seeds or mini_pos do not fit a_cap / mp_cap"); return MGB_E_POOL; }
		return 0;
	}
}

extern "C" int mgb_test_seed(const mg_idx_t *gi, int n, const int *qlens, const char *const *seqs, const int32_t *seg_off, const int32_t *seg_len,
							 const char *const *names, uint64_t flag, int occ_max1, int max_qlen, int32_t *out, mg128_t *a, int64_t a_cap, int32_t *mini_pos, int64_t mp_cap)
{
	try { return test_seed_impl(gi, n, qlens, seqs, seg_off, seg_len, names, flag, occ_max1, max_qlen, out, (u128*)a, a_cap, mini_pos, mp_cap); } catch (const MgbError &e) { return e.code; }
}

// ---------------------------------------------------------------------------------------------------------------
// test hook: K7b on reads whose graph chaining is given (u, lc, a), run in the order of a pass (Pass::run) with the graph of gi and
// the options opt: the batch uploaded by upload_batch; the bridging plan of stage_gchain_plan on lane 0, as stage_gchain ends
// (k_gchain); the bridging jobs in make_job_order's order through gwfa_job_run (k_gwfa); stage_gchain_gen (k_gchain_gen), each
// launched as its kernel is (test_launch).  The results are built by build_result, as mg_map_batch builds them.
// ---------------------------------------------------------------------------------------------------------------
struct TestGcPlan {
	PipeCtx c;
	ReadOut *routs;
	const uint64_t *u;    // read i's chains at u[u_off[i]..+n_u[i]); its linear chains are c.lchain[meta.lc_off..]
	const int64_t *u_off;
	const int32_t *n_u;
	MG_HD int operator()(int i, int32_t *, Arena &A, int, int lane) const
	{
		ReadMeta &m = c.meta[i];
		A.top = 0;
		if (lane == 0) gchain_out_init(routs[i], m);
		LChain *lc;
		uint32_t *gc_hash;
		MGB_ALLOC(A, lc, LChain, m.n_lc);
		MGB_ALLOC(A, gc_hash, uint32_t, m.n_lc);
		for (int32_t j = lane; j < m.n_lc; j += MGB_W) lc[j] = c.lchain[m.lc_off + j];
		warp_sync();
		const int rc = stage_gchain_tail(c, m, i, A, m.n_lc, lc, n_u[i], u + u_off[i], c.anchor + m.a_off, gc_hash, lane);
		if (rc < 0 && lane == 0) m.status = rc, routs[i].status = rc; // as stage_fail records a failed read
		warp_sync();
		return 0;
	}
};

struct TestGcBridge {
	PipeCtx c;
	ReadOut *routs;
	const int32_t *order; // the jobs in the order k_gwfa takes them
	MG_HD int operator()(int i, int32_t *smem, Arena &A, int, int lane) const
	{
		A.top = 0;
		const int rc = gwfa_job_run(A, c, order[i], lane, smem);
		if (rc < 0 && lane == 0) { const int rid = c.gjobs[order[i]].rid; c.meta[rid].status = rc, routs[rid].status = rc; }
		warp_sync();
		return 0;
	}
};

struct TestGcGen {
	PipeCtx c;
	ReadOut *routs;
	int32_t *out; // per read: rc, bridging jobs, of which aligned, pairs bridged again in place
	MG_HD int operator()(int i, int32_t *, Arena &A, int, int lane) const
	{
		int32_t *o = out + 4 * (int64_t)i;
		const ReadMeta &m = c.meta[i];
		A.top = 0;
		if (lane == 0 && m.status == 0) {
			const GState *gsb = (const GState*)(c.gstate + m.gstate_off);
			o[1] = gsb->n_jobs, o[2] = 0;
			for (int32_t j = 0; j < gsb->n_jobs; ++j) o[2] += c.gjobs[gsb->job_first + j].s >= 0;
		}
		const int rc = stage_gchain_gen(c, routs, i, A, lane, &o[3]);
		if (rc < 0 && lane == 0) c.meta[i].status = rc, routs[i].status = rc;
		warp_sync();
		return 0;
	}
};

static int test_gchain_gen_impl(const mg_idx_t *gi, const mg_mapopt_t *opt, int n, const int *qlens, const char *const *seqs, const int32_t *seg_off,
								const int32_t *seg_len, const uint32_t *hash, const int32_t *rep_len, const int32_t *n_mz, const int32_t *n_u, const uint64_t *u,
								const int32_t *n_lc, const mg_lchain_t *lc, const int32_t *n_a, const u128 *a, int32_t *out, mg_gchains_t **gcs)
{
	auto refuse = [](const std::string &why) { set_error("mgb_test_gchain_gen: " + why); return (int)MGB_E_UNSUPPORTED; };
	if (gi == 0 || opt == 0 || n < 0) return refuse("an index, options and n at least 0");
	const Model *M = model_of(gi);
	std::vector<ReadMeta> meta((size_t)n);
	std::vector<LChain> hlc;
	std::vector<int64_t> u_off((size_t)n);
	int64_t su = 0, sa = 0;
	int32_t max_qlen = 0;
	for (int i = 0; i < n; ++i) {
		const std::string r = "read " + std::to_string(i);
		if (qlens[i] < 1 || seqs[i] == 0) return refuse(r + " is empty");
		if (seg_off) {
			if (seg_off[i] < 0 || seg_off[i + 1] <= seg_off[i]) return refuse(r + " has no segment");
			int64_t sum = 0;
			for (int32_t j = seg_off[i]; j < seg_off[i + 1]; ++j) {
				if (seg_len[j] < 1) return refuse(r + " has an empty segment");
				sum += seg_len[j];
			}
			if (sum != qlens[i]) return refuse(r + ": its segments do not add up to its length");
		}
		if (n_u[i] < 0 || n_lc[i] < 0 || n_a[i] < 0 || n_mz[i] < 0 || rep_len[i] < 0) return refuse(r + " has a negative count");
		int64_t sum = 0;
		for (int32_t j = 0; j < n_u[i]; ++j) {
			if ((uint32_t)u[su + j] == 0) return refuse(r + " has a chain of no linear chains");
			sum += (uint32_t)u[su + j];
		}
		if (sum != n_lc[i]) return refuse(r + ": the linear chains counted by u do not add up to n_lc");
		if (n_lc[i] > 0 && n_a[i] == 0) return refuse(r + " has linear chains but no anchors");
		ReadMeta &m = meta[(size_t)i];
		m.hash = hash[i], m.rep_len = rep_len[i], m.n_mz = n_mz[i], m.n_a = n_a[i], m.a_off = sa, m.n_lc = n_lc[i], m.lc_off = (int64_t)hlc.size();
		for (int32_t j = 0; j < n_lc[i]; ++j) {
			const mg_lchain_t &l = lc[m.lc_off + j];
			if ((l.v >> 1) >= (uint32_t)M->g.n_seg) return refuse(r + " has a vertex outside the graph");
			const int32_t vlen = M->seg_len[l.v >> 1];
			if (l.off < 0 || l.cnt < 0 || (int64_t)l.off + l.cnt > n_a[i] || l.rs < 0 || l.rs > l.re || l.re > vlen || l.qs < 0 || l.qs > l.qe || l.qe > qlens[i])
				return refuse(r + " has a linear chain outside its anchors, its vertex or the read");
			for (int32_t t = l.off; t < l.off + l.cnt; ++t)
				if ((int32_t)a[sa + t].x < 0 || (int32_t)a[sa + t].x >= vlen || (int32_t)a[sa + t].y < 0 || (int32_t)a[sa + t].y >= qlens[i])
					return refuse(r + " has an anchor outside its vertex or the read");
			LChain q;
			q.off = l.off, q.cnt = l.cnt, q.v = l.v, q.rs = l.rs, q.re = l.re, q.qs = l.qs, q.qe = l.qe, q.score = l.score, q.dist_pre = l.dist_pre;
			q.hash_pre = l.hash_pre, q.inner_pre = l.inner_pre;
			hlc.push_back(q);
		}
		u_off[(size_t)i] = su;
		su += n_u[i], sa += n_a[i];
		max_qlen = std::max(max_qlen, qlens[i]);
	}
	if (n == 0) return 0;
	if (int e = test_no_device(M->device)) return e;
	PipeCtx c;
	memset(&c, 0, sizeof(c));
	c.g = M->g, c.ix = M->ix;
	fill_opt(c.opt, opt, M->k);
	c.opt.flag &= ~(uint64_t)F_CIGAR; // the alignment plan and what follows it are left out
	logf_prepare((Model*)M, max_qlen, c.opt);
	const BatchLayout lay(n, qlens);
	Staging stg;
	mgb::HostPool one;
	mgb_stats_t st = {};
	c.b = upload_batch(stg, lay, M, n, qlens, seqs, 0, false, seg_off, seg_len, one, 1, 0, st);
	std::vector<u128> ha(a, a + sa);
	std::vector<uint64_t> hu(u, u + su);
	ha.resize((size_t)sa + 1), hu.resize((size_t)su + 1), hlc.resize(hlc.size() + 1); // no empty device buffers
	auto a_d = upload(ha.data(), ha.size());
	auto u_d = upload(hu.data(), hu.size());
	auto lc_d = upload(hlc.data(), hlc.size());
	auto u_off_d = upload(u_off.data(), (size_t)n);
	auto n_u_d = upload(n_u, (size_t)n);
	DevBuf<ReadMeta> meta_d((size_t)n);
	DevBuf<ReadOut> routs_d((size_t)n);
	DevBuf<int32_t> out_d(4 * (size_t)n);
	DevBuf<Pool> pools_d(4);
	c.meta = meta_d, c.anchor = a_d, c.lchain = lc_d;
	c.pool_out = pools_d, c.pool_gstate = pools_d + 1, c.pool_gjobs = pools_d + 2, c.pool_walk = pools_d + 3;
	const std::array<uint64_t, N_POOLS> cap0 = pool_caps(n, lay.n_bases, 0);
	uint64_t cap[4] = {cap0[P_OUT], cap0[P_GSTATE], cap0[P_GJOBS], cap0[P_WALK]};
	const uint64_t arena_bytes = (uint64_t)32 << 20; // (the pipeline's workers have 3 MB and retry a read that outgrows them with 1 GB)
	std::vector<ReadOut> routs((size_t)n);
	for (;;) {
		DevBuf<char> out_pool(cap[0]), gstate(cap[1]);
		DevBuf<GwfaJob> gjobs(cap[2] / sizeof(GwfaJob) + 1);
		DevBuf<int32_t> walk(cap[3] / sizeof(int32_t) + 1);
		Pool hp[4];
		for (int p = 0; p < 4; ++p) hp[p].used = 0, hp[p].cap = cap[p];
		h2d(pools_d, hp, sizeof(hp));
		dfill(gjobs, 0xff, cap[2]); // reserved-but-unused bridging job slots read as rid == -1 (as in Pass)
		h2d(meta_d, meta.data(), sizeof(ReadMeta) * (size_t)n);
		dzero(routs_d, sizeof(ReadOut) * (size_t)n);
		dzero(out_d, sizeof(int32_t) * 4 * (size_t)n);
		c.out = out_pool, c.gstate = gstate, c.gjobs = gjobs, c.walk = walk;
		const TestGcPlan tp{c, routs_d, u_d, u_off_d, n_u_d};
		if (int e = test_launch<S_GCHAIN>(n, std::min(n, StageSpec<S_GCHAIN>::warps), arena_bytes, tp)) return e;
		d2h(hp, pools_d, sizeof(hp));
		const int n_jobs = (int)(std::min(hp[2].used, hp[2].cap) / sizeof(GwfaJob));
		if (n_jobs > 0) {
			LaunchArgs L;
			memset(&L, 0, sizeof(L));
			L.c = c;
			DevBuf<int32_t> order((size_t)n_jobs);
			make_job_order(L, 0, 0, n_jobs, order);
			const TestGcBridge tb{c, routs_d, order};
			if (int e = test_launch<S_GWFA>(n_jobs, std::min(n_jobs, 2 * StageSpec<S_GWFA>::warps), arena_bytes, tb)) return e;
		}
		const TestGcGen tg{c, routs_d, out_d};
		if (int e = test_launch<S_GCHAIN_GEN>(n, std::min(n, StageSpec<S_GCHAIN_GEN>::warps), arena_bytes, tg)) return e;
		std::vector<ReadMeta> m_out((size_t)n);
		d2h(m_out.data(), meta_d, sizeof(ReadMeta) * (size_t)n);
		d2h(routs.data(), routs_d, sizeof(ReadOut) * (size_t)n);
		d2h(hp, pools_d, sizeof(hp));
		bool pool_full = false;
		for (int i = 0; i < n; ++i) pool_full |= read_status(m_out[(size_t)i], routs[(size_t)i]) == MGB_E_POOL;
		if (pool_full) { for (int p = 0; p < 4; ++p) cap[p] *= 2; continue; }
		std::vector<char> hout(std::min(hp[0].used, hp[0].cap) + 64);
		d2h(hout.data(), out_pool, std::min(hp[0].used, hp[0].cap));
		d2h(out, out_d, sizeof(int32_t) * 4 * (size_t)n);
		for (int i = 0; i < n; ++i) {
			out[4 * (int64_t)i] = read_status(m_out[(size_t)i], routs[(size_t)i]);
			gcs[i] = out[4 * (int64_t)i] == 0? build_result(routs[(size_t)i], hout.data()) : 0;
		}
		return 0;
	}
}

extern "C" int mgb_test_gchain_gen(const mg_idx_t *gi, const mg_mapopt_t *opt, int n, const int *qlens, const char *const *seqs, const int32_t *seg_off,
								   const int32_t *seg_len, const uint32_t *hash, const int32_t *rep_len, const int32_t *n_mz, const int32_t *n_u, const uint64_t *u,
								   const int32_t *n_lc, const mg_lchain_t *lc, const int32_t *n_a, const mg128_t *a, int32_t *out, mg_gchains_t **gcs)
{
	for (int i = 0; i < n; ++i) gcs[i] = 0;
	try { return test_gchain_gen_impl(gi, opt, n, qlens, seqs, seg_off, seg_len, hash, rep_len, n_mz, n_u, u, n_lc, lc, n_a, (const u128*)a, out, gcs); }
	catch (const MgbError &e) { return e.code; }
}

extern "C" void mgb_get_stats(const mg_idx_t *gi, mgb_stats_t *st) { *st = t_has_stats? t_last_stats : model_of(gi)->stats; } // the calling thread's last batch
