// mgb_fastx.cuh -- FASTA/FASTQ text in device memory parsed into reads on the device (mgb_reads_parse_dev).
//
// The records are those mgb_reads_load() (mgb_gfa.cpp) finds in the same bytes: from the first '>' or '@', a record's name runs to the
// first white space and its header line to the first '\n' (L); its sequence is every byte but '\n' and '\r' from there to the first
// line that starts with '>', '+' or '@' (S), upper-cased ('a'..'z' only); after an '@' header whose S line starts with '+', as many
// non-CR/LF bytes as the sequence has bases are skipped from the end of that line, then the rest of their line; the next record
// starts at the next '>' or '@'.  A quality string is full of '>', '+' and '@' (Q29, Q10, Q31), so where records start cannot be
// told locally.  Every '>' / '@' byte is a candidate instead, and each candidate's successor (where the next record would start if
// one started there) is found from four sorted position lists of the text in O(log) steps; the records are the chain of successors
// from the first candidate, marked by pointer jumping.
//
// The passes, in order (launched by mgb_engine.cu, each one warp per item):
//   FxCount  (item: a chunk of FX_CHUNK bytes)   how many entries of each list the chunk holds; scanned into each chunk's first entry
//   FxLists  (chunk)                              the lists: '\n'; '\n' or '\r'; line starts with '>' / '+' / '@'; '>' or '@'
//   FxSucc   (32 candidates)                      jump[0][c] = the successor of candidate c (n_cand: none), mark[c] = (c == 0)
//   FxJump   (32 candidates, log rounds)          every marked candidate marks its 2^k-th successor, the jumps double
//   FxRecs   (32 candidates)                      the marked candidates, numbered by a scan of the marks, as records with their lengths
//   FxTail   (one item)                           which records the call emits (final, max_bases) and where the next call starts
//   FxCopy   (a record)                           its bases without CR/LF, upper-cased, and its name into the caller's block
#pragma once
#include "mgb_common.cuh"

namespace mgb {

static const int FX_CHUNK = 4096; // bytes of text per item of the list passes
enum { FX_NL, FX_BRK, FX_CL, FX_HD, FX_NLIST }; // the lists: '\n'; '\n' or '\r'; line starts with '>' / '+' / '@'; '>' or '@'

// what a call emits and where the next one starts (written by FxTail)
struct FxSum {
	int64_t n_reads, n_bases, name_bytes, used;
	int64_t first_long; // the first record longer than INT32_MAX bases (INT64_MAX: none)
};

// a record: the header byte h, the end of its name ne, the end of its header line L and the start of the line that ends its sequence S
struct FxRow { int64_t h, ne, L, S; };

struct FxArgs {
	const char *text; int64_t n_text; // the text, n_text bytes
	int n_chunks;
	uint64_t *tab;                    // [n_chunks + 1][FX_NLIST]: entries per chunk, scanned in place into the chunk's first entry
	int64_t *list[FX_NLIST];          // positions in the text, ascending
	int64_t n_cand;                   // entries of list[FX_HD]
	const int32_t *jin; int32_t *jout; // candidate -> its successor (n_cand: none, and n_cand -> n_cand), in / out of a round
	uint8_t *mark;                    // [n_cand + 1]: the candidate starts a record
	const uint64_t *grp;              // [groups + 1]: records in the groups of 32 candidates before
	FxRow *rows; uint64_t *lens;      // per record: its row; [n_rec + 1][2]: bases and name bytes, scanned in place into offsets
	int64_t n_rec, max_bases; int final_;
	FxSum *sum;
	char *seq, *name; int64_t *off, *name_off; // the caller's tables
	unsigned int *next;               // FxCopy's read counter
	int n;                            // items of the pass
};

MG_HD inline bool fx_space(unsigned char c) { return c == ' ' || (c >= '\t' && c <= '\r'); } // C-locale isspace

// index of the first entry of list k at or after x (the list's length when there is none): a search among the entries of x's chunk
MG_HD inline int64_t fx_lb(const FxArgs &a, int k, int64_t x)
{
	if (x >= a.n_text) return (int64_t)a.tab[(int64_t)FX_NLIST * a.n_chunks + k];
	const int64_t q = x / FX_CHUNK;
	int64_t lo = (int64_t)a.tab[FX_NLIST * q + k], hi = (int64_t)a.tab[FX_NLIST * (q + 1) + k];
	const int64_t *L = a.list[k];
	while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (L[m] < x) lo = m + 1; else hi = m; }
	return lo;
}
// the first entry of list k at or after x, or n_text
MG_HD inline int64_t fx_next(const FxArgs &a, int k, int64_t x)
{
	const int64_t i = fx_lb(a, k, x);
	return i < (int64_t)a.tab[(int64_t)FX_NLIST * a.n_chunks + k]? a.list[k][i] : a.n_text;
}
// bytes other than '\n' and '\r' before x
MG_HD inline int64_t fx_rank(const FxArgs &a, int64_t x) { return x - fx_lb(a, FX_BRK, x); }
// the position of the byte other than '\n' / '\r' of rank r (r < fx_rank(a, n_text)): r plus the CR/LF bytes before it, which are the
// entries j of the CR/LF list with list[j] - j (the rank of entry j) <= r; they all lie in or before the last chunk that starts at rank <= r
MG_HD inline int64_t fx_unrank(const FxArgs &a, int64_t r)
{
	int64_t lo = 0, hi = a.n_chunks - 1;
	while (lo < hi) {
		const int64_t m = (lo + hi + 1) >> 1;
		if (m * FX_CHUNK - (int64_t)a.tab[FX_NLIST * m + FX_BRK] <= r) lo = m; else hi = m - 1;
	}
	int64_t b = (int64_t)a.tab[FX_NLIST * lo + FX_BRK], e = (int64_t)a.tab[FX_NLIST * (lo + 1) + FX_BRK];
	const int64_t *D = a.list[FX_BRK];
	while (b < e) { const int64_t m = (b + e) >> 1; if (D[m] - m <= r) b = m + 1; else e = m; }
	return r + b;
}

// the record that would start at header byte h: its L, S and bases, and where the record after it starts (n_text: none)
struct FxRec { int64_t L, S, len, next; };
MG_HD inline FxRec fx_record(const FxArgs &a, int64_t h)
{
	const int64_t n = a.n_text;
	FxRec r;
	r.L = fx_next(a, FX_NL, h + 1);
	r.S = r.L < n? fx_next(a, FX_CL, r.L + 1) : n;
	r.len = fx_rank(a, r.S) - fx_rank(a, r.L);
	int64_t e = r.S;
	if (a.text[h] == '@' && r.S < n && a.text[r.S] == '+') { // the quality: from the end of the '+' line, r.len bytes other than CR/LF
		const int64_t q0 = fx_next(a, FX_NL, r.S);
		int64_t q1 = n;
		if (q0 < n) {
			const int64_t last = fx_rank(a, q0) + r.len - 1; // the rank of its last byte
			q1 = r.len == 0? q0 : last < fx_rank(a, n)? fx_unrank(a, last) + 1 : n;
		}
		e = q1 < n? fx_next(a, FX_NL, q1) : n;
	}
	r.next = e < n? fx_next(a, FX_HD, e) : n;
	return r;
}

// bytes [p, p + 16) of the text (0 past its end): one 16-byte load where the address allows
MG_HD inline void fx_load16(const FxArgs &a, int64_t p, unsigned char *c)
{
	const char *s = a.text + p;
	if (p + 16 <= a.n_text && ((uintptr_t)s & 15) == 0) {
#if MGB_ON_DEVICE
		*(uint4*)c = *(const uint4*)s;
#else
		memcpy(c, s, 16);
#endif
		return;
	}
	for (int i = 0; i < 16; ++i) c[i] = p + i < a.n_text? (unsigned char)s[i] : 0;
}

// chunk q, 16 bytes per lane and step: with write, the positions of each list's entries go to a.list at the chunk's first entry;
// returns (on every lane) the entries of list k in the chunk in cnt[k]
MG_HD inline void fx_chunk(const FxArgs &a, int q, int lane, bool write, uint64_t *cnt)
{
	uint64_t at[FX_NLIST];
	for (int k = 0; k < FX_NLIST; ++k) cnt[k] = 0, at[k] = write? a.tab[(int64_t)FX_NLIST * q + k] : 0;
	const int64_t c0 = (int64_t)q * FX_CHUNK, c1 = c0 + FX_CHUNK < a.n_text? c0 + FX_CHUNK : a.n_text;
	for (int64_t s = c0; s < c1; s += 16 * MGB_W) {
		const int64_t p = s + 16 * lane;
		unsigned char c[16];
		uint32_t m[FX_NLIST] = {0, 0, 0, 0};
		if (p < c1) {
			fx_load16(a, p, c);
			const int nb = c1 - p < 16? (int)(c1 - p) : 16;
			bool prev_nl = p > 0 && a.text[p - 1] == '\n';
			for (int i = 0; i < nb; ++i) {
				const unsigned char x = c[i];
				if (x == '\n') m[FX_NL] |= 1u << i;
				if (x == '\n' || x == '\r') m[FX_BRK] |= 1u << i;
				if (prev_nl && (x == '>' || x == '+' || x == '@')) m[FX_CL] |= 1u << i;
				if (x == '>' || x == '@') m[FX_HD] |= 1u << i;
				prev_nl = x == '\n';
			}
		}
		for (int k = 0; k < FX_NLIST; ++k) {
			int cn = 0;
			for (uint32_t v = m[k]; v; v &= v - 1) ++cn;
			const int incl = warp_incl_scan_i32(cn, lane);
			if (write && m[k]) {
				int64_t *o = a.list[k] + at[k] + (uint64_t)(incl - cn);
				for (int i = 0; i < 16; ++i) if ((m[k] >> i) & 1u) *o++ = p + i;
			}
			const uint64_t tot = (uint64_t)(uint32_t)warp_bcast_i32(incl, MGB_W - 1);
			cnt[k] += tot, at[k] += tot;
		}
	}
}

struct FxCount {
	const FxArgs &a;
	MG_HD int operator()(int q, int lane) const
	{
		uint64_t cnt[FX_NLIST];
		fx_chunk(a, q, lane, false, cnt);
		if (lane == 0) for (int k = 0; k < FX_NLIST; ++k) a.tab[(int64_t)FX_NLIST * q + k] = cnt[k];
		return 0;
	}
};
struct FxLists {
	const FxArgs &a;
	MG_HD int operator()(int q, int lane) const { uint64_t cnt[FX_NLIST]; fx_chunk(a, q, lane, true, cnt); return 0; }
};

// group g: candidates [32 g, 32 g + 32) and the end node n_cand, one per lane
struct FxSucc {
	const FxArgs &a;
	MG_HD int operator()(int g, int lane) const
	{
		for (int64_t c = 32 * (int64_t)g + lane; c < 32 * (int64_t)g + 32 && c <= a.n_cand; c += MGB_W) {
			int32_t s = (int32_t)a.n_cand;
			if (c < a.n_cand) {
				const FxRec r = fx_record(a, a.list[FX_HD][c]);
				s = (int32_t)fx_lb(a, FX_HD, r.next);
			}
			a.jout[c] = s;
			a.mark[c] = c == 0;
		}
		return 0;
	}
};
// one round: a marked candidate marks its 2^k-th successor, which lies on the chain too (a candidate that another round marks in
// the meantime may pass its mark on early: every mark stays on the chain), and the jumps double
struct FxJump {
	const FxArgs &a;
	MG_HD int operator()(int g, int lane) const
	{
		for (int64_t c = 32 * (int64_t)g + lane; c < 32 * (int64_t)g + 32 && c <= a.n_cand; c += MGB_W) {
			const int32_t j = a.jin[c];
			a.jout[c] = a.jin[j];
			if (a.mark[c]) a.mark[j] = 1;
		}
		return 0;
	}
};
// the records among the candidates of group g (the end node excluded)
MG_HD inline int fx_group_marks(const FxArgs &a, int64_t g)
{
	int k = 0;
	for (int64_t c = 32 * g; c < 32 * g + 32 && c < a.n_cand; ++c) k += a.mark[c];
	return k;
}
struct FxMarks { // scan_u64 source: records per group
	static constexpr int W = 1;
	FxArgs a;
	MG_HD uint64_t operator()(int g, int) const { return (uint64_t)fx_group_marks(a, g); }
};

MG_HD inline void fx_first_long(const FxArgs &a, int64_t k)
{
#if MGB_ON_DEVICE
	atomicMin((unsigned long long*)&a.sum->first_long, (unsigned long long)k);
#else
	if (k < a.sum->first_long) a.sum->first_long = k;
#endif
}

struct FxRecs {
	const FxArgs &a;
	MG_HD int operator()(int g, int lane) const
	{
		uint64_t k0 = a.grp[g];
		for (int i = 0; i < 32; i += MGB_W) {
			const int64_t c = 32 * (int64_t)g + i + lane;
			const bool rec = c < a.n_cand && a.mark[c];
			const uint32_t m = warp_ballot(rec);
			if (rec) {
				const int64_t k = (int64_t)k0 + mask_rank(m, lane), h = a.list[FX_HD][c];
				const FxRec r = fx_record(a, h);
				int64_t ne = h + 1;
				while (ne < r.L && !fx_space((unsigned char)a.text[ne])) ++ne;
				a.rows[k] = FxRow{h, ne, r.L, r.S};
				a.lens[2 * k] = (uint64_t)r.len, a.lens[2 * k + 1] = (uint64_t)(ne - h - 1);
				if (r.len > INT32_MAX) fx_first_long(a, k);
			}
			k0 += (uint64_t)mask_count(m);
		}
		return 0;
	}
};

// which records the call emits: without final, not the last (its end may lie past the text); with max_bases, none after the one
// that reaches it.  The next call starts at the record after the last one emitted, or at the first header.
struct FxTail {
	const FxArgs &a;
	MG_HD int operator()(int, int lane) const
	{
		if (lane != 0) return 0;
		const int64_t K = a.n_rec;
		int64_t k = a.final_? K : K > 0? K - 1 : 0;
		if (a.max_bases > 0 && K > 0 && (int64_t)a.lens[2 * K] >= a.max_bases) { // the first record whose end reaches max_bases
			int64_t lo = 0, hi = K - 1;
			while (lo < hi) { const int64_t m = (lo + hi) >> 1; if ((int64_t)a.lens[2 * (m + 1)] >= a.max_bases) hi = m; else lo = m + 1; }
			if (lo + 1 < k) k = lo + 1;
		}
		FxSum &s = *a.sum;
		s.n_reads = k, s.n_bases = (int64_t)a.lens[2 * k], s.name_bytes = (int64_t)a.lens[2 * k + 1];
		s.used = k > 0? fx_record(a, a.rows[k - 1].h).next : a.n_cand > 0? a.list[FX_HD][0] : a.n_text;
		return 0;
	}
};

// record k: its name, then its bases, 16 bytes per lane and step from the 16-byte boundary at or before L, without CR/LF and upper-cased
struct FxCopy {
	const FxArgs &a;
	MG_HD unsigned int *counter() const { return a.next; }
	MG_HD int operator()(int k, int lane) const
	{
		const FxRow r = a.rows[k];
		char *nm = a.name + a.lens[2 * k + 1];
		for (int64_t i = lane; i < r.ne - r.h - 1; i += MGB_W) nm[i] = a.text[r.h + 1 + i];
		char *dst = a.seq + a.lens[2 * k];
		uint64_t w = 0;
		for (int64_t s = r.L & ~(int64_t)15; s < r.S; s += 16 * MGB_W) {
			const int64_t p = s + 16 * lane;
			unsigned char c[16];
			uint32_t keep = 0;
			if (p < r.S) {
				fx_load16(a, p, c);
				for (int i = 0; i < 16; ++i)
					if (p + i >= r.L && p + i < r.S && c[i] != '\n' && c[i] != '\r') keep |= 1u << i;
			}
			int cn = 0;
			for (uint32_t v = keep; v; v &= v - 1) ++cn;
			const int incl = warp_incl_scan_i32(cn, lane);
			char *o = dst + w + (uint64_t)(incl - cn);
			for (int i = 0; i < 16; ++i)
				if ((keep >> i) & 1u) { const unsigned char x = c[i]; *o++ = (char)(x >= 'a' && x <= 'z'? x - 32 : x); }
			w += (uint64_t)(uint32_t)warp_bcast_i32(incl, MGB_W - 1);
		}
		if (lane == 0) a.off[k] = (int64_t)a.lens[2 * k], a.name_off[k] = (int64_t)a.lens[2 * k + 1];
		return 0;
	}
};

} // namespace mgb
