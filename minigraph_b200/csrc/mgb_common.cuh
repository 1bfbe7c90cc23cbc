// mgb_common.cuh -- shared device-side building blocks of the mapping engine.
//
// Everything in csrc/*.cuh is written once as warp-cooperative device code.  The functions are
// marked MG_HD so that the *same* source can also be compiled by g++ into tests/hostsim (a
// single-lane simulator used only by the CPU-side unit tests to debug control flow in the
// GPU-less build container).  The shipped library (libmgb200.so) contains only the CUDA build.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#if defined(__CUDACC__)
#define MG_HD __host__ __device__
#define MG_D __device__
#else
#define MG_HD
#define MG_D
#endif

#if defined(__CUDA_ARCH__)
#define MGB_ON_DEVICE 1
#else
#define MGB_ON_DEVICE 0
#endif

// a function kept out of line: rare paths (container growth, table rebuilds, large sorts) of kernels whose hot loop has to
// stay small -- the L1.5 instruction cache holds 2048 instructions and the warps of an SM are all in different places
#if defined(__CUDACC__)
#define MG_NOINLINE __noinline__
#define MGB_NO_UNROLL _Pragma("unroll 1")
#else
#define MG_NOINLINE __attribute__((noinline))
#define MGB_NO_UNROLL
#endif

namespace mgb {

// ---- error codes (per read) ----
enum {
	MGB_OK = 0,
	MGB_E_ARENA = -1,    // per-worker arena exhausted: the read is retried by the host with a larger arena
	MGB_E_POOL = -2,     // a global output pool is exhausted: the batch is retried with larger pools
	MGB_E_INTERNAL = -3, // invariant violated (the reference would assert/abort here)
	MGB_E_UNSUPPORTED = -4
};

// ---- the universal 16-byte record (reference: minigraph.h:41 mg128_t) ----
struct u128 { uint64_t x, y; };

// seed flag bits (reference: mgpriv.h:18-27)
static const uint64_t SEED_IGNORE = 1ULL << 41;
static const uint64_t SEED_TANDEM = 1ULL << 42;
static const uint64_t SEED_FIXED = 1ULL << 43;
static const int SEED_SEG_SHIFT = 48;
static const uint64_t SEED_SEG_MASK = 0xffULL << 48;
static const int SEED_OCC_SHIFT = 56;
static const int MAX_SHORT_K = 15;

// ---- warp-cooperative helpers ----
// Warp-uniform functions take `lane` and are entered by all lanes of a warp together: scalar control flow is
// replicated on every lane (identical values, identical branches), data-parallel loops stride by MGB_W, and
// phases that exchange data through memory are separated by warp_sync().  The CPU simulator runs with one lane.
#if MGB_ON_DEVICE
#define MGB_W 32
MG_D inline void warp_sync() { __syncwarp(); }
MG_D inline int warp_any(int pred) { return __any_sync(0xffffffffu, pred); }
MG_D inline int32_t warp_bcast_i32(int32_t x, int src) { return __shfl_sync(0xffffffffu, x, src); }
MG_D inline uint64_t warp_bcast_u64(uint64_t x, int src) { return __shfl_sync(0xffffffffu, x, src); }
MG_D inline int32_t warp_min_i32(int32_t x) { return __reduce_min_sync(0xffffffffu, x); } // one REDUX instead of five shuffle + select steps
MG_D inline int32_t warp_max_i32(int32_t x) { return __reduce_max_sync(0xffffffffu, x); }
MG_D inline int32_t warp_sum_i32(int32_t x) { return __reduce_add_sync(0xffffffffu, x); }
MG_D inline uint32_t warp_ballot(int pred) { return __ballot_sync(0xffffffffu, pred); }
MG_D inline uint64_t warp_or_u64(uint64_t x) { return (uint64_t)__reduce_or_sync(0xffffffffu, (uint32_t)(x >> 32)) << 32 | __reduce_or_sync(0xffffffffu, (uint32_t)x); }
MG_D inline uint64_t warp_and_u64(uint64_t x) { return (uint64_t)__reduce_and_sync(0xffffffffu, (uint32_t)(x >> 32)) << 32 | __reduce_and_sync(0xffffffffu, (uint32_t)x); }
MG_D inline void lane_atomic_inc(int32_t *p) { atomicAdd(p, 1); }
// maximum over this lane and the lanes below it
MG_D inline uint64_t warp_incl_scan_max_u64(uint64_t x, int lane)
{
	for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o && y > x) x = y; }
	return x;
}
MG_D inline uint64_t warp_shfl_up1_u64(uint64_t x) { return __shfl_up_sync(0xffffffffu, x, 1); } // value of the lane below (own value on lane 0)
// sum over this lane and the lanes below it
MG_D inline int32_t warp_incl_scan_i32(int32_t x, int lane)
{
	for (int o = 1; o < 32; o <<= 1) { int32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
	return x;
}
// maximum over the lanes below this one (INT32_MIN on lane 0)
MG_D inline int32_t warp_excl_prefix_max_i32(int32_t x, int lane)
{
	for (int o = 1; o < 32; o <<= 1) { int32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o && y > x) x = y; }
	x = __shfl_up_sync(0xffffffffu, x, 1);
	return lane == 0? INT32_MIN : x;
}
MG_D inline int mask_rank(uint32_t mask, int lane) { return __popc(mask & ((1u << lane) - 1u)); } // set bits below `lane`
MG_D inline int mask_count(uint32_t mask) { return __popc(mask); }
#elif defined(MGB_SIM_LANES)
// test infrastructure: the lanes of a warp as fibres on one CPU thread (mgb_simlanes.h)
} // namespace mgb
#include "mgb_simlanes.h"
namespace mgb {
#define MGB_W MGB_SIM_LANES
inline void warp_sync() { uint64_t o[32]; sim::exchange(0, o, 1); }
inline int warp_any(int pred) { uint64_t o[32]; sim::exchange(pred != 0, o, 2); for (int i = 0; i < MGB_W; ++i) if (o[i]) return 1; return 0; }
inline int32_t warp_bcast_i32(int32_t x, int src) { uint64_t o[32]; sim::exchange((uint64_t)(uint32_t)x, o, 3); return (int32_t)(uint32_t)o[src]; }
inline uint64_t warp_bcast_u64(uint64_t x, int src) { uint64_t o[32]; sim::exchange(x, o, 4); return o[src]; }
inline int32_t warp_min_i32(int32_t x) { uint64_t o[32]; sim::exchange((uint64_t)(uint32_t)x, o, 5); int32_t r = x; for (int i = 0; i < MGB_W; ++i) if ((int32_t)(uint32_t)o[i] < r) r = (int32_t)(uint32_t)o[i]; return r; }
inline int32_t warp_max_i32(int32_t x) { uint64_t o[32]; sim::exchange((uint64_t)(uint32_t)x, o, 6); int32_t r = x; for (int i = 0; i < MGB_W; ++i) if ((int32_t)(uint32_t)o[i] > r) r = (int32_t)(uint32_t)o[i]; return r; }
inline int32_t warp_sum_i32(int32_t x) { uint64_t o[32]; sim::exchange((uint64_t)(uint32_t)x, o, 7); uint32_t r = 0; for (int i = 0; i < MGB_W; ++i) r += (uint32_t)o[i]; return (int32_t)r; }
inline uint32_t warp_ballot(int pred) { uint64_t o[32]; sim::exchange(pred != 0, o, 8); uint32_t m = 0; for (int i = 0; i < MGB_W; ++i) if (o[i]) m |= 1u << i; return m; }
inline uint64_t warp_or_u64(uint64_t x) { uint64_t o[32]; sim::exchange(x, o, 9); uint64_t r = 0; for (int i = 0; i < MGB_W; ++i) r |= o[i]; return r; }
inline uint64_t warp_and_u64(uint64_t x) { uint64_t o[32]; sim::exchange(x, o, 10); uint64_t r = ~0ULL; for (int i = 0; i < MGB_W; ++i) r &= o[i]; return r; }
inline void lane_atomic_inc(int32_t *p) { ++*p; }
inline uint64_t warp_incl_scan_max_u64(uint64_t x, int lane) { uint64_t o[32]; sim::exchange(x, o, 11); uint64_t r = o[0]; for (int i = 1; i <= lane; ++i) if (o[i] > r) r = o[i]; return r; }
inline uint64_t warp_shfl_up1_u64(uint64_t x) { uint64_t o[32]; sim::exchange(x, o, 12); const int l = sim::lane(); return l > 0? o[l - 1] : x; }
inline int32_t warp_incl_scan_i32(int32_t x, int lane) { uint64_t o[32]; sim::exchange((uint64_t)(uint32_t)x, o, 13); uint32_t r = 0; for (int i = 0; i <= lane; ++i) r += (uint32_t)o[i]; return (int32_t)r; }
inline int32_t warp_excl_prefix_max_i32(int32_t x, int lane) { uint64_t o[32]; sim::exchange((uint64_t)(uint32_t)x, o, 14); int32_t r = INT32_MIN; for (int i = 0; i < lane; ++i) if ((int32_t)(uint32_t)o[i] > r) r = (int32_t)(uint32_t)o[i]; return r; }
inline int mask_rank(uint32_t mask, int lane) { return __builtin_popcount(mask & ((1u << lane) - 1u)); }
inline int mask_count(uint32_t mask) { return __builtin_popcount(mask); }
#else
#define MGB_W 1
inline void warp_sync() {}
inline int warp_any(int pred) { return pred; }
inline int32_t warp_bcast_i32(int32_t x, int) { return x; }
inline uint64_t warp_bcast_u64(uint64_t x, int) { return x; }
inline int32_t warp_min_i32(int32_t x) { return x; }
inline int32_t warp_max_i32(int32_t x) { return x; }
inline int32_t warp_sum_i32(int32_t x) { return x; }
inline uint32_t warp_ballot(int pred) { return pred? 1u : 0u; }
inline int32_t warp_excl_prefix_max_i32(int32_t, int) { return INT32_MIN; }
inline int32_t warp_incl_scan_i32(int32_t x, int) { return x; }
inline uint64_t warp_incl_scan_max_u64(uint64_t x, int) { return x; }
inline uint64_t warp_shfl_up1_u64(uint64_t x) { return x; }
inline uint64_t warp_or_u64(uint64_t x) { return x; }
inline uint64_t warp_and_u64(uint64_t x) { return x; }
inline void lane_atomic_inc(int32_t *p) { ++*p; }
inline int mask_rank(uint32_t, int) { return 0; }
inline int mask_count(uint32_t mask) { return (int)(mask & 1u); }
#endif

// ---- bump arena: one per worker (warp), stack discipline via mark/release ----
struct Arena {
	char *base;
	uint64_t cap, top, peak;
};

MG_HD inline void arena_init(Arena &A, void *base, uint64_t cap) { A.base = (char*)base, A.cap = cap, A.top = 0, A.peak = 0; }

MG_HD inline void *arena_alloc(Arena &A, uint64_t n_bytes)
{
	uint64_t n = (n_bytes + 15) & ~(uint64_t)15;
	if (A.top + n > A.cap) return 0;
	void *p = A.base + A.top;
	A.top += n;
	if (A.top > A.peak) A.peak = A.top;
	return p;
}

#define MGB_ALLOC(A, ptr, type, n) do { \
		(ptr) = (type*)mgb::arena_alloc((A), (uint64_t)sizeof(type) * (uint64_t)((n) > 0? (n) : 1)); \
		if ((ptr) == 0) return mgb::MGB_E_ARENA; \
	} while (0)

#define MGB_TRY(expr) do { int _mgb_rc = (expr); if (_mgb_rc < 0) return _mgb_rc; } while (0)

// growable vector living in an arena; growth abandons the old block (reclaimed when the caller releases its mark)
template<typename T>
struct AVec {
	T *a;
	int64_t n, m;
};

template<typename T>
MG_HD inline void avec_init(AVec<T> &v) { v.a = 0, v.n = v.m = 0; }

template<typename T>
MG_HD inline int avec_reserve(Arena &A, AVec<T> &v, int64_t want)
{
	if (want <= v.m) return 0;
	int64_t m = v.m? v.m : 16;
	while (m < want) m += (m >> 1) + 16;
	// extend in place when the vector is the topmost allocation of the arena
	uint64_t old_bytes = ((uint64_t)sizeof(T) * (uint64_t)v.m + 15) & ~(uint64_t)15;
	if (v.a && (char*)v.a + old_bytes == A.base + A.top) {
		uint64_t new_bytes = ((uint64_t)sizeof(T) * (uint64_t)m + 15) & ~(uint64_t)15;
		if ((uint64_t)((char*)v.a - A.base) + new_bytes > A.cap) return MGB_E_ARENA;
		A.top = (uint64_t)((char*)v.a - A.base) + new_bytes;
		if (A.top > A.peak) A.peak = A.top;
		v.m = m;
		return 0;
	}
	T *b = (T*)arena_alloc(A, (uint64_t)sizeof(T) * (uint64_t)m);
	if (b == 0) return MGB_E_ARENA;
	for (int64_t i = 0; i < v.n; ++i) b[i] = v.a[i];
	v.a = b, v.m = m;
	return 0;
}

// warp-uniform variant: every lane holds an identical copy of A and v; the element copy is split across lanes
template<typename T>
MG_HD inline int avec_reserve_w(Arena &A, AVec<T> &v, int64_t want, int lane)
{
	if (want <= v.m) return 0;
	int64_t m = v.m? v.m : 16;
	while (m < want) m += (m >> 1) + 16;
	uint64_t old_bytes = ((uint64_t)sizeof(T) * (uint64_t)v.m + 15) & ~(uint64_t)15;
	if (v.a && (char*)v.a + old_bytes == A.base + A.top) {
		uint64_t new_bytes = ((uint64_t)sizeof(T) * (uint64_t)m + 15) & ~(uint64_t)15;
		if ((uint64_t)((char*)v.a - A.base) + new_bytes > A.cap) return MGB_E_ARENA;
		A.top = (uint64_t)((char*)v.a - A.base) + new_bytes;
		if (A.top > A.peak) A.peak = A.top;
		v.m = m;
		return 0;
	}
	T *b = (T*)arena_alloc(A, (uint64_t)sizeof(T) * (uint64_t)m);
	if (b == 0) return MGB_E_ARENA;
	for (int64_t i = lane; i < v.n; i += MGB_W) b[i] = v.a[i];
	warp_sync();
	v.a = b, v.m = m;
	return 0;
}

template<typename T>
MG_HD inline int avec_push(Arena &A, AVec<T> &v, const T &x)
{
	if (v.n == v.m) { int rc = avec_reserve(A, v, v.n + 1); if (rc < 0) return rc; }
	v.a[v.n++] = x;
	return 0;
}

// The same growth out of line and independent of the element type (avec_reserve_c / avec_push_c): same capacities, same arena
// traffic, one copy of the code per kernel instead of one per call site.
MG_HD MG_NOINLINE inline int avec_grow_cold(Arena &A, void **pa, int64_t n, int64_t *pm, uint32_t elem, int64_t want)
{
	int64_t m = *pm? *pm : 16;
	while (m < want) m += (m >> 1) + 16;
	char *a = (char*)*pa;
	const uint64_t old_bytes = ((uint64_t)elem * (uint64_t)*pm + 15) & ~(uint64_t)15;
	if (a && a + old_bytes == A.base + A.top) {
		const uint64_t new_bytes = ((uint64_t)elem * (uint64_t)m + 15) & ~(uint64_t)15;
		if ((uint64_t)(a - A.base) + new_bytes > A.cap) return MGB_E_ARENA;
		A.top = (uint64_t)(a - A.base) + new_bytes;
		if (A.top > A.peak) A.peak = A.top;
		*pm = m;
		return 0;
	}
	char *b = (char*)arena_alloc(A, (uint64_t)elem * (uint64_t)m);
	if (b == 0) return MGB_E_ARENA;
	const uint64_t n_words = (uint64_t)elem * (uint64_t)n / 4; // element sizes are multiples of four bytes, blocks 16-byte aligned
	MGB_NO_UNROLL
	for (uint64_t i = 0; i < n_words; ++i) ((uint32_t*)b)[i] = ((const uint32_t*)a)[i];
	*pa = b, *pm = m;
	return 0;
}
template<typename T>
MG_HD inline int avec_reserve_c(Arena &A, AVec<T> &v, int64_t want)
{
	static_assert(sizeof(T) % 4 == 0, "avec_grow_cold copies words");
	if (want <= v.m) return 0;
	return avec_grow_cold(A, (void**)&v.a, v.n, &v.m, (uint32_t)sizeof(T), want);
}
template<typename T>
MG_HD inline int avec_push_c(Arena &A, AVec<T> &v, const T &x)
{
	if (v.n == v.m) { int rc = avec_reserve_c(A, v, v.n + 1); if (rc < 0) return rc; }
	v.a[v.n++] = x;
	return 0;
}

// ---- global bump pool shared by all workers of one launch ----
struct Pool {
	unsigned long long used; // bytes
	unsigned long long cap;
};

MG_HD inline int64_t pool_alloc(Pool *p, uint64_t n_bytes) // returns byte offset or -1
{
	unsigned long long n = (n_bytes + 15) & ~15ULL, off;
#if MGB_ON_DEVICE
	off = atomicAdd(&p->used, n);
#else
	off = p->used, p->used += n;
#endif
	if (off + n > p->cap) return -1;
	return (int64_t)off;
}

// ---- hash functions that leak into results (reference: khashl.h:321-346, sketch.c:28-38) ----
MG_HD inline uint32_t hash32(uint32_t key)
{
	key += ~(key << 15);
	key ^= (key >> 10);
	key += (key << 3);
	key ^= (key >> 6);
	key += ~(key << 11);
	key ^= (key >> 16);
	return key;
}

MG_HD inline uint32_t hash_str(const char *s)
{
	uint32_t h = (uint32_t)(int32_t)*s; // NB: plain char is signed on x86-64
	if (h) for (++s; *s; ++s) h = (h << 5) - h + (uint32_t)(int32_t)*s;
	return h;
}

MG_HD inline uint64_t hash64_mask(uint64_t key, uint64_t mask) // invertible integer hash restricted to 2k bits
{
	key = (~key + (key << 21)) & mask;
	key = key ^ key >> 24;
	key = ((key + (key << 3)) + (key << 8)) & mask;
	key = key ^ key >> 14;
	key = ((key + (key << 2)) + (key << 4)) & mask;
	key = key ^ key >> 28;
	key = (key + (key << 31)) & mask;
	return key;
}

// fast log2 approximation used by the chaining penalties (reference: mgpriv.h:63-71); valid for x>=2
MG_HD inline float fast_log2(float x)
{
	uint32_t i;
#if MGB_ON_DEVICE
	i = __float_as_uint(x);
#else
	memcpy(&i, &x, 4);
#endif
	float log_2 = (float)(int)(((i >> 23) & 255) - 128);
	i &= ~(255u << 23);
	i += 127u << 23;
	float f;
#if MGB_ON_DEVICE
	f = __uint_as_float(i);
	// no FMA contraction: the reference is built with -ffp-contract=off (SURVEY H3)
	log_2 = __fadd_rn(log_2, __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(-0.34484843f, f), 2.02466578f), f), -0.67487759f));
#else
	memcpy(&f, &i, 4);
	log_2 += (-0.34484843f * f + 2.02466578f) * f - 0.67487759f;
#endif
	return log_2;
}

// unaligned 32-bit load assembled from two aligned ones (may touch up to 7 bytes behind p: buffers carry slack)
MG_HD inline uint32_t ld32_unaligned(const char *p)
{
	uintptr_t a = (uintptr_t)p;
	const uint32_t *w = (const uint32_t*)(a & ~(uintptr_t)3);
	int sh = (int)(a & 3) << 3;
	uint32_t lo = w[0], hi = w[1];
#if MGB_ON_DEVICE
	return __funnelshift_r(lo, hi, sh);
#else
	return sh? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}
MG_HD inline int ctz32_nz(uint32_t x)
{
#if MGB_ON_DEVICE
	return __ffs((int)x) - 1;
#else
	return __builtin_ctz(x);
#endif
}
// position of the k-th set bit of mask (k >= 1), 32 when there are fewer
MG_HD inline int nth_set_bit(uint32_t mask, int k)
{
#if MGB_ON_DEVICE
	const unsigned r = __fns(mask, 0, k);
	return r > 31? 32 : (int)r;
#else
	for (int b = 0; b < 32; ++b) if ((mask >> b & 1) && --k == 0) return b;
	return 32;
#endif
}
// Replay of the "skip" counter of the chaining loops over one chunk of candidates in visiting order (lchain.c:185-190, 336-343):
// a candidate that improves the best score lowers the counter by one (not below zero), one that is already on a better chain
// raises it, and the walk stops at the candidate that takes it above max_skip.  imp / mk: lanes of the two kinds.  Returns the
// lane the walk stops at, or -1; *n_skip is the counter after the chunk (or at the stop).
MG_HD inline int replay_skips(uint32_t imp, uint32_t mk, int max_skip, int32_t *n_skip)
{
	int32_t ns = *n_skip;
	for (;;) { // one round per improving candidate: the marks in front of it in one step
		const int nxt = imp? ctz32_nz(imp) : 32;
		const uint32_t seg = nxt >= 32? mk : mk & ((1u << nxt) - 1u);
		const int c = mask_count(seg);
		if (ns + c > max_skip) { *n_skip = max_skip + 1; return nth_set_bit(seg, max_skip - ns + 1); }
		ns += c;
		if (nxt >= 32) break;
		if (ns > 0) --ns;
		imp &= imp - 1, mk &= ~((2u << nxt) - 1u);
	}
	*n_skip = ns;
	return -1;
}
MG_HD inline int ctz32(uint32_t x)
{
#if MGB_ON_DEVICE
	return __ffs((int)x) - 1;
#else
	return __builtin_ctz(x);
#endif
}

MG_HD inline int nt4(uint8_t c) // reference: sketch.c:9-26 seq_nt4_table (A/C/G/T/U in either case and the raw codes 0..3; 4 otherwise)
{
	const uint32_t idx = c & 0x1fu; // position in the alphabet for 0x40..0x7f
	const uint64_t code = (1ULL << 2 * 3) | (2ULL << 2 * 7) | (3ULL << 2 * 20) | (3ULL << 2 * 21); // C, G, T, U (A is 0)
	const uint32_t letters = (1u << 1) | (1u << 3) | (1u << 7) | (1u << 20) | (1u << 21);
	if ((c & 0xc0u) == 0x40u && (letters >> idx & 1u)) return (int)(code >> 2 * idx & 3u);
	return c < 4? (int)c : 4;
}

// ---- bit-exact emulation of klib's in-place MSD radix sort (reference: ksort.h:112-162) ----
// The sort is NOT stable; its tie order reaches the output (SURVEY H1), hence the exact replay of
// the cycle-leader permutation.  Recursion is turned into an explicit range stack (children are
// disjoint, so their processing order is irrelevant).  A digit on which all keys agree permutes
// nothing, so such levels are skipped.
template<typename T, typename KeyFn>
MG_HD inline void rs_insertsort(T *beg, T *end, KeyFn key)
{
	for (T *i = beg + 1; i < end; ++i) {
		if (key(*i) < key(*(i - 1))) {
			T *j, tmp = *i;
			for (j = i; j > beg && key(tmp) < key(*(j - 1)); --j) *j = *(j - 1);
			*j = tmp;
		}
	}
}

struct RsRange { int32_t beg, end, s; };

template<typename T, typename KeyFn>
MG_HD inline int radix_sort_exact(Arena &A, T *a, int64_t n, int sizeof_key, KeyFn key)
{
	const int MIN_SIZE = 64;
	if (n <= MIN_SIZE) { rs_insertsort(a, a + n, key); return 0; }
	uint64_t mark = A.top;
	RsRange *stack;
	int64_t m_stack = n / MIN_SIZE + 4; // pending ranges are disjoint and each holds more than MIN_SIZE elements
	MGB_ALLOC(A, stack, RsRange, m_stack);
	int32_t *bb, *be; // bin tables in the arena, not on the thread's stack
	MGB_ALLOC(A, bb, int32_t, 512);
	be = bb + 256;
	int64_t top = 0;
	stack[top].beg = 0, stack[top].end = (int32_t)n, stack[top].s = (sizeof_key - 1) * 8, ++top;
	while (top > 0) {
		RsRange r = stack[--top];
		int s = r.s;
		// which digits vary inside this range?
		uint64_t k_or = 0, k_and = ~0ULL;
		for (int32_t i = r.beg; i < r.end; ++i) { uint64_t k = (uint64_t)key(a[i]); k_or |= k, k_and &= k; }
		uint64_t diff = k_or ^ k_and;
		while (s > 0 && ((diff >> s) & 0xff) == 0) s -= 8; // identity levels
		if (s < 0) s = 0;
		if (((diff >> s) & 0xff) == 0) continue; // s == 0 and nothing varies: all keys equal, order untouched
		for (int k = 0; k < 256; ++k) bb[k] = 0;
		for (int32_t i = r.beg; i < r.end; ++i) ++bb[(key(a[i]) >> s) & 0xff];
		{
			int32_t acc = r.beg;
			for (int k = 0; k < 256; ++k) { int32_t c = bb[k]; bb[k] = acc; acc += c; be[k] = acc; }
		}
		for (int k = 0; k < 256;) { // cycle-leader permutation
			if (bb[k] != be[k]) {
				int l = (int)((key(a[bb[k]]) >> s) & 0xff);
				if (l != k) {
					T tmp = a[bb[k]], swap;
					do {
						swap = tmp; tmp = a[bb[l]]; a[bb[l]++] = swap;
						l = (int)((key(tmp) >> s) & 0xff);
					} while (l != k);
					a[bb[k]++] = tmp;
				} else ++bb[k];
			} else ++k;
		}
		if (s) {
			int s2 = s > 8? s - 8 : 0;
			int32_t st = r.beg;
			for (int k = 0; k < 256; ++k) {
				int32_t en = be[k];
				if (en - st > MIN_SIZE) {
					if (top >= m_stack) { A.top = mark; return MGB_E_INTERNAL; }
					stack[top].beg = st, stack[top].end = en, stack[top].s = s2, ++top;
				} else if (en - st > 1) rs_insertsort(a + st, a + en, key);
				st = en;
			}
		}
	}
	A.top = mark;
	return 0;
}

struct KeyX128 { MG_HD uint64_t operator()(const u128 &p) const { return p.x; } };
struct KeyU64 { MG_HD uint64_t operator()(const uint64_t &p) const { return p; } };

MG_HD inline int radix_sort_128x(Arena &A, u128 *a, int64_t n) { return radix_sort_exact(A, a, n, 8, KeyX128()); }
MG_HD inline int radix_sort_64(Arena &A, uint64_t *a, int64_t n) { return radix_sort_exact(A, a, n, 8, KeyU64()); }

// At most 64 elements, entered by all lanes: klib sorts these by insertion, i.e. stably, so every element's final place is a
// count (keys below it, equal keys in front of it); two elements per lane.  No arena, no scratch.
template<typename T, typename KeyFn>
MG_HD inline void small_sort_stable_w(T *a, int64_t n, KeyFn key, int lane)
{
	if (MGB_W < 32) { if (lane == 0) rs_insertsort(a, a + n, key); warp_sync(); return; }
	T e[2];
	int32_t r[2] = {-1, -1};
	for (int h = 0; h < 2; ++h) {
		const int64_t i = lane + 32 * h;
		if (i >= n) continue;
		e[h] = a[i];
		const uint64_t ki = (uint64_t)key(e[h]);
		int32_t c = 0;
#if MGB_ON_DEVICE
#pragma unroll 2
#endif
		for (int64_t j = 0; j < n; ++j) { const uint64_t kj = (uint64_t)key(a[j]); c += kj < ki || (kj == ki && j < i); }
		r[h] = c;
	}
	warp_sync();
	for (int h = 0; h < 2; ++h) if (r[h] >= 0) a[r[h]] = e[h];
	warp_sync();
}

// radix_sort_exact() entered by all lanes of a warp.  Only the cycle-leader permutation is inherently sequential (its
// tie order is what has to be reproduced); it runs on lane 0 over the non-empty bins.  The digit census, the bin
// offsets, the child ranges and the insertion sorts of the small bins are spread over the lanes.
// The permutation as a walk over DIGITS: every read of the cycle-leader loop is of an element still at its original place (a bin's
// frontier only moves forward and the home slot of a chain is not read before the chain ends), so where each element ends up
// follows from the digits alone.  Lane 0 walks a byte per element (kept in the hot arena A, on chip where the caller has the room)
// and notes the destinations; all lanes then move the elements through a copy in the arena `cold`.  Same moves, same result; the
// dependent load of the walk is a byte that stays in L1 / shared memory instead of a 16-byte element in L2.  Asked for by the caller
// (`walk`): it pays where the elements are in global memory (the seeds of k_seed), not where the list is already on chip.
template<typename T, typename KeyFn>
MG_HD inline int radix_sort_exact_w(Arena &A, T *a, int64_t n, int sizeof_key, KeyFn key, int lane, Arena *cold = 0, bool walk = false)
{
	const int MIN_SIZE = 64, MIN_WALK = 192; // ranges shorter than MIN_WALK are permuted in place as before
	if (n <= MIN_SIZE) { small_sort_stable_w(a, n, key, lane); return 0; }
	Arena &C = cold? *cold : A;
	uint64_t mark = A.top;
	RsRange *stack;
	int64_t m_stack = n / MIN_SIZE + 4; // pending ranges are disjoint and each holds more than MIN_SIZE elements
	MGB_ALLOC(A, stack, RsRange, m_stack);
	int32_t *bb, *be, *nz;
	MGB_ALLOC(A, bb, int32_t, 256);
	MGB_ALLOC(A, be, int32_t, 256);
	MGB_ALLOC(A, nz, int32_t, 256);
	int64_t top = 0;
	if (lane == 0) stack[0].beg = 0, stack[0].end = (int32_t)n, stack[0].s = (sizeof_key - 1) * 8;
	top = 1;
	warp_sync();
	while (top > 0) {
		const RsRange r = stack[--top];
		int s = r.s;
		uint64_t k_or = 0, k_and = ~0ULL;
		for (int32_t i = r.beg + lane; i < r.end; i += MGB_W) { uint64_t k = (uint64_t)key(a[i]); k_or |= k, k_and &= k; }
		k_or = warp_or_u64(k_or), k_and = warp_and_u64(k_and);
		const uint64_t diff = k_or ^ k_and;
		while (s > 0 && ((diff >> s) & 0xff) == 0) s -= 8;
		if (s < 0) s = 0;
		if (((diff >> s) & 0xff) == 0) continue;
		for (int k = lane; k < 256; k += MGB_W) bb[k] = 0;
		warp_sync();
		// scratch of the digit walk: digits (hot if there is room), destinations and the copy of the range (cold)
		const int32_t n_r = r.end - r.beg;
		const uint64_t mark_hot = A.top, mark_cold = C.top;
		uint8_t *dg = 0;
		int32_t *dst = 0;
		T *cp = 0;
		if (walk && n_r >= MIN_WALK) {
			dg = (uint8_t*)arena_alloc(A, (uint64_t)n_r);
			if (dg == 0 && &C != &A) dg = (uint8_t*)arena_alloc(C, (uint64_t)n_r);
			dst = (int32_t*)arena_alloc(C, (uint64_t)n_r * sizeof(int32_t));
			cp = (T*)arena_alloc(C, (uint64_t)n_r * sizeof(T));
			if (dg == 0 || dst == 0 || cp == 0) dg = 0; // no room: in place
		}
		for (int32_t i = r.beg + lane; i < r.end; i += MGB_W) {
			const int d = (int)((key(a[i]) >> s) & 0xff);
			lane_atomic_inc(&bb[d]);
			if (dg) dg[i - r.beg] = (uint8_t)d, cp[i - r.beg] = a[i];
		}
		warp_sync();
		int32_t acc = r.beg, n_nz = 0;
		for (int k0 = 0; k0 < 256; k0 += MGB_W) {
			const int k = k0 + lane;
			const int32_t c = bb[k];
			const int32_t incl = warp_incl_scan_i32(c, lane);
			const uint32_t mz = warp_ballot(c > 0);
			warp_sync();
			bb[k] = acc + incl - c, be[k] = acc + incl;
			if (c > 0) nz[n_nz + mask_rank(mz, lane)] = k;
			n_nz += mask_count(mz);
			acc += warp_bcast_i32(incl, MGB_W - 1);
		}
		warp_sync();
		if (dg) {
			if (lane == 0) {
				const uint8_t *dgr = dg - r.beg;
				int32_t *dstr = dst - r.beg;
				for (int z = 0; z < n_nz;) { // the walk of the cycle-leader permutation over the digits
					const int k = nz[z];
					if (bb[k] != be[k]) {
						int32_t cur = bb[k];
						int l = dgr[cur];
						if (l != k) {
							do { // the element held (cur) goes to the frontier of its bin, whose occupant is held next
								const int32_t nxt = bb[l];
								dstr[cur] = nxt, bb[l] = nxt + 1;
								cur = nxt, l = dgr[cur];
							} while (l != k);
							dstr[cur] = bb[k]++;
						} else dstr[cur] = cur, ++bb[k];
					} else ++z;
				}
			}
			warp_sync();
			for (int32_t i = lane; i < n_r; i += MGB_W) a[dst[i]] = cp[i];
			A.top = mark_hot, C.top = mark_cold;
		} else if (lane == 0) {
			for (int z = 0; z < n_nz;) { // cycle-leader permutation (empty bins have nothing to do)
				const int k = nz[z];
				if (bb[k] != be[k]) {
					int l = (int)((key(a[bb[k]]) >> s) & 0xff);
					if (l != k) {
						T tmp = a[bb[k]], swap;
						do {
							swap = tmp; tmp = a[bb[l]]; a[bb[l]++] = swap;
							l = (int)((key(tmp) >> s) & 0xff);
						} while (l != k);
						a[bb[k]++] = tmp;
					} else ++bb[k];
				} else ++z;
			}
		}
		warp_sync();
		if (s) {
			const int s2 = s > 8? s - 8 : 0;
			for (int k0 = 0; k0 < 256; k0 += MGB_W) {
				const int k = k0 + lane;
				const int32_t st = k == 0? r.beg : be[k - 1], en = be[k];
				const int big = en - st > MIN_SIZE;
				const uint32_t mb = warp_ballot(big);
				if (top + mask_count(mb) > m_stack) { A.top = mark; return MGB_E_INTERNAL; }
				if (big) { RsRange c; c.beg = st, c.end = en, c.s = s2; stack[top + mask_rank(mb, lane)] = c; }
				else if (en - st > 1) rs_insertsort(a + st, a + en, key); // bins are disjoint: one lane each
				top += mask_count(mb);
			}
		}
		warp_sync();
	}
	A.top = mark;
	return 0;
}

MG_HD inline int radix_sort_128x_w(Arena &A, u128 *a, int64_t n, int lane, Arena *cold = 0, bool walk = false) { return radix_sort_exact_w(A, a, n, 8, KeyX128(), lane, cold, walk); }

} // namespace mgb
