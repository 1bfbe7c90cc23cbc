// mgb_ingest.cuh -- reads that are already in device memory, laid out as the kernels read a batch (mgb_map_batch_dev*).
//
// k_ingest leaves what upload_batch() and k_unpack leave for reads that come from host strings: the upper-case ASCII copy of read r
// at seq_off[r] (16-byte aligned) and, unless the batch has segments, its 2-bit words at pk_off[r] (A/C/G/T -> 0..3, the order of
// seq_nt4_table, sketch.c:9-26, base j in bits 2*(j%32)).  A read that holds any byte other than A/C/G/T after upper-casing gets
// pk_off[r] = ~0 and is read as ASCII.  Upper-casing is gmap.c:81 mg_toupper's: only 'a'..'z' change.
#pragma once
#include "mgb_common.cuh"

namespace mgb {

// read r is src[src_off[r] .. + seq_len[r]); pk == NULL: no words (fragments with segments); raw (or NULL): 1 for a read that holds
// a byte other than A/C/G/T
struct IngestArgs {
	const char *src; const int64_t *src_off;
	const uint64_t *seq_off; const int32_t *seq_len; char *seq;
	uint64_t *pk, *pk_off; int32_t *raw; int n;
};

// bits [s, s + 32) of hi:lo
MG_HD inline uint32_t ingest_fshr(uint32_t lo, uint32_t hi, int s)
{
#if MGB_ON_DEVICE
	return __funnelshift_r(lo, hi, (unsigned)s);
#else
	return (uint32_t)((((uint64_t)hi << 32) | lo) >> s);
#endif
}

// 0x80 in each byte of x that is 0, 0 elsewhere
MG_HD inline uint32_t ingest_zero_bytes(uint32_t x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu); }

// Word wd of read r: bases [32 wd, 32 wd + 32) from three aligned 16-byte loads (the read may start at any byte), upper-cased, four
// bytes per step.  Writes the ASCII copy in 16-byte halves (a half that starts at or behind the end of the read is not the read's to
// write; the bytes past the end in the last half are 0) and the 2-bit word.  Returns non-zero when a base is not A/C/G/T.
MG_HD inline uint32_t ingest_word(const IngestArgs &I, int r, int64_t wd)
{
	const int64_t len = I.seq_len[r], b0 = wd * 32;
	const int n = len - b0 < 32? (int)(len - b0) : 32;
	const char *a = I.src + I.src_off[r] + b0;
	const char *base = (const char*)((uintptr_t)a & ~(uintptr_t)15);
	const int sh = (int)((uintptr_t)a & 15);
	uint32_t v[12];
	for (int c = 0; c < 3; ++c) { // a chunk that holds no byte of the word is not loaded: it may lie past the end of the buffer
		uint32_t *d = v + 4 * c;
		if (base + 16 * c < a + n) {
#if MGB_ON_DEVICE
			const uint4 x = *(const uint4*)(base + 16 * c);
			d[0] = x.x, d[1] = x.y, d[2] = x.z, d[3] = x.w;
#else
			memcpy(d, base + 16 * c, 16);
#endif
		} else d[0] = d[1] = d[2] = d[3] = 0;
	}
	const int ws = sh >> 2, bs = 8 * (sh & 3);
	uint32_t u[9];
	for (int j = 0; j < 9; ++j) u[j] = ws == 0? v[j] : ws == 1? v[j + 1] : ws == 2? v[j + 2] : v[j + 3]; // (no indexing by a variable: registers)
	uint32_t q[8], bad = 0;
	uint64_t word = 0;
	for (int j = 0; j < 8; ++j) {
		const int m = n - 4 * j; // bytes of this step that are the read's
		const uint32_t valid = m >= 4? 0xffffffffu : m <= 0? 0u : (1u << (8 * m)) - 1;
		uint32_t x = ingest_fshr(u[j], u[j + 1], bs) & valid;
		const uint32_t t = x & 0x7f7f7f7fu; // 'a'..'z' (0x61..0x7a, high bit clear) lose 0x20
		const uint32_t lower = (t + 0x1f1f1f1fu) & ~(t + 0x05050505u) & ~x & 0x80808080u;
		x ^= lower >> 2;
		const uint32_t acgt = ingest_zero_bytes(x ^ 0x41414141u) | ingest_zero_bytes(x ^ 0x43434343u) | ingest_zero_bytes(x ^ 0x47474747u) | ingest_zero_bytes(x ^ 0x54545454u);
		const uint32_t b = ~acgt & valid & 0x80808080u;
		bad |= b;
		uint32_t c = (x >> 1) & 0x03030303u;        // A0 C1 T2 G3
		c ^= (c >> 1) & 0x01010101u;                // A0 C1 G2 T3
		c &= ~((b >> 7) * 3u);                      // any other byte: 0, as the host's table gives (4 & 3)
		const uint32_t p = c | (c >> 6);            // four codes -> one byte
		word |= (uint64_t)((p & 0x0fu) | ((p >> 12) & 0xf0u)) << (8 * j);
		q[j] = x;
	}
	char *dst = I.seq + I.seq_off[r] + b0;
	for (int h = 0; h < 2; ++h)
		if (b0 + 16 * h < len) {
#if MGB_ON_DEVICE
			*(uint4*)(dst + 16 * h) = make_uint4(q[4 * h], q[4 * h + 1], q[4 * h + 2], q[4 * h + 3]);
#else
			memcpy(dst + 16 * h, q + 4 * h, 16);
#endif
		}
	if (I.pk) I.pk[I.pk_off[r] + (uint64_t)wd] = word;
	return bad;
}

// after every word of read r: the OR of their flags
MG_HD inline void ingest_flag(const IngestArgs &I, int r, bool raw)
{
	if (I.raw) I.raw[r] = raw;
	if (raw && I.pk) I.pk_off[r] = ~0ULL;
}

// read r (warp-uniform): each lane whole words, long reads strided over the lanes; returns the read's flag
struct IngestRead {
	const IngestArgs &a;
	MG_HD int operator()(int r, int lane) const
	{
		const int64_t nw = ((int64_t)a.seq_len[r] + 31) >> 5;
		uint32_t bad = 0;
		for (int64_t wd = lane; wd < nw; wd += MGB_W) bad |= ingest_word(a, r, wd);
		const bool raw = warp_any(bad != 0); // (every lane has read pk_off[r] by now)
		if (lane == 0) ingest_flag(a, r, raw);
		return raw;
	}
};

} // namespace mgb
