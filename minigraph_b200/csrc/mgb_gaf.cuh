// mgb_gaf.cuh -- GAF text of a mapped batch, formatted on the device from the result blobs in the output pool
// (reference: format.c:121-291 mg_write_gaf).
//
// gaf_read() is warp-uniform: all lanes enter with the same read and run the same scalar control flow.  With dst == NULL it only
// counts the read's bytes; with dst it writes them there.  Size and bytes come from the same code, so they cannot disagree.
//   * fixed fields and the path column are short and sequential: every lane follows them, lane 0 writes the bytes;
//   * names (query, segments, stable sequences) are copied by all lanes;
//   * CIGAR ops and the anchor deltas of --write-mz: one item per lane, places from a warp prefix sum of their widths;
//   * ds:Z: the forward text is a plain copy; reversed, every op keeps its length, so each byte's place follows from the op
//     offsets alone and all lanes write at once.
// The dv:f values are computed by the host with its libm (gchain1.c:295, format.c:258-263): gaf_requests() lists what each value
// needs, the host formats each into a 16-byte cell (the reference's buf[16]), and gaf_read() copies the cells.
#pragma once
#include "mgb_galign.cuh"

namespace mgb {

static const uint64_t F_FRAG_MERGE = 0x80, F_VERTEX_COOR = 0x800, F_PRINT_2ND = 0x2000, F_SHOW_UNMAP = 0x100000, F_NO_COMP_PATH = 0x200000;
static const uint64_t F_WRITE_LCHAIN = 0x800000, F_WRITE_MZ = 0x1000000;
static const int GAF_CELL = 16;

// the names of the graph (uploaded at mg_index): concatenated bytes, name i at name[off[i] .. off[i+1])
struct GafGraph {
	const char *seg_name; const int64_t *seg_name_off;
	const int32_t *seg_len, *snid, *soff;            // gfa_seg_t len / snid / soff
	const char *sseq_name; const int64_t *sseq_name_off;
	const int32_t *sseq_min, *sseq_max, *sseq_rank;  // gfa_sseq_t
};

// the reads of one call: names ("*" for a NULL name) and the lengths of every read's segments
struct GafQuery {
	const char *name; const int64_t *name_off;       // [n + 1]
	const int32_t *n_seg, *seg_first;                // [n]
	const int32_t *seg_len;
};

// what one dv:f value needs: kind 0, a graph chain (a = n_mini, b = n_anchor); kind 1, a linear chain of -S (a = n, b = cnt);
// kind -1, nothing is printed
struct GafReq { int32_t a, b, q_span, kind; };

struct GafArgs {
	GafGraph g;
	GafQuery q;
	const ReadOut *routs;
	const char *pool;       // output pool (blob_off / blob2_off and the chains' cigar/ds offsets point into it)
	int n;
	uint64_t flag;
	const int64_t *req_off; // [n + 1]: read r owns requests and cells req_off[r] .. req_off[r+1]: n_gc of them, then n_lc under -S
	GafReq *req;
	const char *cells;      // GAF_CELL bytes per request, 0-terminated; empty: no dv:f field
	uint64_t *off;          // [n + 1]: bytes of read r (count pass), then its offset in the text (scan)
	char *text;
	unsigned int *next;     // [2] work counters of the count and the write pass
};

MG_HD inline int gaf_dec_len(uint32_t x) { int l = 1; while (x >= 10) x /= 10, ++l; return l; }

// reference: gfa-base.c:509-526 gfa_comp_table
MG_HD inline char gaf_comp(char c)
{
	const char *to = "TVGHEFCDIJMLKNOPQYSAABWXRZ";
	if (c >= 'A' && c <= 'Z') return to[c - 'A'];
	if (c >= 'a' && c <= 'z') return (char)(to[c - 'a'] + 32);
	return c;
}

struct GafOut {
	char *p;     // NULL: count only
	uint64_t n;
	int lane;
	MG_HD void c(char ch) { if (p && lane == 0) p[n] = ch; ++n; }
	MG_HD void lit(const char *z) { while (*z) c(*z++); }
	MG_HD void s(const char *src, uint64_t len) { if (p) for (uint64_t i = (uint64_t)lane; i < len; i += MGB_W) p[n + i] = src[i]; n += len; }
	MG_HD void d(int32_t v)
	{
		uint32_t x = v < 0? 0u - (uint32_t)v : (uint32_t)v;
		const int l = gaf_dec_len(x) + (v < 0);
		if (p && lane == 0) {
			char *q = p + n + l;
			do { *--q = (char)('0' + x % 10); x /= 10; } while (x);
			if (v < 0) *--q = '-';
		}
		n += (uint64_t)l;
	}
	MG_HD void cell(const char *z) { uint64_t l = 0; while (l < GAF_CELL - 1 && z[l]) ++l; s(z, l); }
};

// n items, each [pre] decimal [suf] (a 0 char is left out), one item per lane; item(i, &val, &pre, &suf)
template<typename F>
MG_HD inline void gaf_list(GafOut &o, int32_t n, const F &item)
{
	for (int32_t b = 0; b < n; b += MGB_W) {
		const int32_t i = b + o.lane;
		int32_t val = 0, w = 0;
		char pre = 0, suf = 0;
		uint32_t x = 0;
		if (i < n) {
			item(i, &val, &pre, &suf);
			x = val < 0? 0u - (uint32_t)val : (uint32_t)val;
			w = (pre != 0) + gaf_dec_len(x) + (val < 0) + (suf != 0);
		}
		const int32_t incl = warp_incl_scan_i32(w, o.lane);
		const int32_t tot = warp_bcast_i32(incl, MGB_W - 1);
		if (o.p && i < n) {
			char *q = o.p + o.n + (incl - w);
			if (pre) *q++ = pre;
			q += gaf_dec_len(x) + (val < 0);
			char *e = q;
			do { *--q = (char)('0' + x % 10); x /= 10; } while (x);
			if (val < 0) *--q = '-';
			if (suf) *e = suf;
		}
		o.n += (uint64_t)tot;
	}
}

// the requests of read r (warp-uniform)
MG_HD inline void gaf_requests(const GafArgs &G, int r, int lane)
{
	const ReadOut &ro = G.routs[r];
	if (ro.n_gc == 0) return;
	const ReadBlob B = read_blob(G.pool, ro);
	GafReq *q = G.req + G.req_off[r];
	for (int32_t i = lane; i < ro.n_gc; i += MGB_W) {
		GafReq t; t.a = B.gc[i].n_mini, t.b = B.gc[i].n_anchor, t.q_span = B.gc[i].q_span, t.kind = 0;
		q[i] = t;
	}
	if (G.flag & F_WRITE_LCHAIN)
		for (int32_t j = lane; j < ro.n_lc; j += MGB_W) {
			const LLChain &l = B.lc[j];
			GafReq t; t.a = t.b = t.q_span = 0, t.kind = -1;
			if (l.cnt > 0) { // format.c:256-258
				t.q_span = (int32_t)(B.a[l.off].y >> 32 & 0xff);
				t.a = (int32_t)(B.a[l.off + l.cnt - 1].x >> 32) - (int32_t)(B.a[l.off].x >> 32) + 1;
				t.b = l.cnt, t.kind = 1;
			}
			q[ro.n_gc + j] = t;
		}
}

// GAF records of read r (format.c:121-291); returns their bytes, written to dst unless it is NULL (warp-uniform)
MG_HD inline uint64_t gaf_read(const GafArgs &G, int r, char *dst, int lane)
{
	GafOut o;
	o.p = dst, o.n = 0, o.lane = lane;
	const uint64_t flag = G.flag;
	const GafGraph &g = G.g;
	const ReadOut &ro = G.routs[r];
	const char *qn = G.q.name + G.q.name_off[r];
	const int64_t qn_len = G.q.name_off[r + 1] - G.q.name_off[r];
	const int32_t ns = G.q.n_seg[r];
	const int32_t *ql = G.q.seg_len + G.q.seg_first[r];
	int32_t qlen = 0;
	for (int32_t j = 0; j < ns; ++j) qlen += ql[j];
	// "/1" is dropped from a merged pair's name once the text so far (this read's) is longer than 2 bytes (format.c:128,138)
	const bool trim = (flag & F_FRAG_MERGE) && ns == 2 && qn_len >= 2 && qn[qn_len - 2] == '/' && qn[qn_len - 1] == '1';
	auto put_qname = [&]() { o.s(qn, (uint64_t)(trim && o.n + (uint64_t)qn_len > 2? qn_len - 2 : qn_len)); };
	auto put_seg = [&](uint32_t v) { o.c("><"[v & 1]); const uint32_t s = v >> 1; o.s(g.seg_name + g.seg_name_off[s], (uint64_t)(g.seg_name_off[s + 1] - g.seg_name_off[s])); };
	auto put_sseq = [&](int32_t k) { o.s(g.sseq_name + g.sseq_name_off[k], (uint64_t)(g.sseq_name_off[k + 1] - g.sseq_name_off[k])); };
	auto put_stable = [&](int32_t rev, int32_t k, int32_t st, int32_t en) { o.c("><"[rev]); put_sseq(k); o.c(':'); o.d(st); o.c('-'); o.d(en); };
	if (ro.n_gc == 0) { // no result object (empty or over-long read) or no graph chain
		if (flag & F_SHOW_UNMAP) { put_qname(); o.c('\t'); o.d(qlen); o.lit("\t0\t0\t*\t*\t0\t0\t0\t0\t0\t0\n"); }
		return o.n;
	}
	const ReadBlob B = read_blob(G.pool, ro);
	const char *cells = G.cells + (uint64_t)GAF_CELL * (uint64_t)G.req_off[r];
	int rev_sign = 0; // sticky across the records of the read (format.c:123,193)
	for (int32_t i = 0; i < ro.n_gc; ++i) {
		const GChain &p = B.gc[i];
		if (p.id != p.parent && !(flag & F_PRINT_2ND)) continue;
		if (p.cnt == 0) continue;
		put_qname();
		o.c('\t'); o.d(qlen); o.c('\t'); o.d(p.qs); o.c('\t'); o.d(p.qe); o.lit("\t+\t");
		const uint64_t sign_pos = o.n - 2;
		int compact;
		if (flag & F_VERTEX_COOR) {
			compact = 0;
			for (int32_t j = 0; j < p.cnt; ++j) put_seg(B.lc[p.off + j].v);
		} else {
			int32_t last = -1, st = -1, en = -1, rev = -1;
			compact = flag & F_NO_COMP_PATH? 0 : 1;
			for (int32_t j = 0; j < p.cnt; ++j) {
				const uint32_t v = B.lc[p.off + j].v, sid = v >> 1;
				const int32_t snid = g.snid[sid];
				if (snid < 0) { // no stable name: the segment itself
					compact = 0;
					if (last >= 0) put_stable(rev, last, st, en);
					last = -1, st = -1, en = -1, rev = -1;
					put_seg(v);
				} else {
					const int32_t soff = g.soff[sid], len = g.seg_len[sid];
					int cont = 0;
					if (last >= 0 && snid == last && (int32_t)(v & 1) == rev) { // same stable sequence, same strand
						if (!(v & 1)) { if (soff == en) en = soff + len, cont = 1; }
						else { if (soff + len == st) st = soff, cont = 1; }
					}
					if (cont == 0) {
						if (last >= 0) compact = 0, put_stable(rev, last, st, en);
						last = snid, rev = (int32_t)(v & 1), st = soff, en = st + len;
					}
				}
			}
			if (last >= 0) {
				if (g.sseq_rank[last] != 0 || g.sseq_min[last] != 0) compact = 0;
				if (!compact) put_stable(rev, last, st, en);
			} else compact = 0;
		}
		if (compact) {
			const int32_t rev = (int32_t)(B.lc[p.off].v & 1);
			const uint32_t sid = B.lc[rev? p.off + p.cnt - 1 : p.off].v >> 1;
			const int32_t snid = g.snid[sid], soff = g.soff[sid];
			put_sseq(snid); o.c('\t'); o.d(g.sseq_max[snid]); o.c('\t');
			if (rev) {
				rev_sign = 1;
				if (o.p && lane == 0) o.p[sign_pos] = '-';
				o.d(soff + (p.plen - p.pe)); o.c('\t'); o.d(soff + (p.plen - p.ps));
			} else {
				o.d(soff + p.ps); o.c('\t'); o.d(soff + p.pe);
			}
		} else { o.c('\t'); o.d(p.plen); o.c('\t'); o.d(p.ps); o.c('\t'); o.d(p.pe); }
		o.c('\t'); o.d(p.has_cigar? p.c_mlen : p.mlen); o.c('\t'); o.d(p.has_cigar? p.c_blen : p.blen); o.c('\t'); o.d(p.mapq & 0xff);
		o.lit("\ttp:A:"); o.c(p.id == p.parent? 'P' : 'S');
		if (p.has_cigar) { o.lit("\tNM:i:"); o.d(p.c_blen - p.c_mlen); }
		o.lit("\tcm:i:"); o.d(p.n_anchor); o.lit("\ts1:i:"); o.d(p.score); o.lit("\ts2:i:"); o.d(p.subsc);
		if (cells[GAF_CELL * i]) { o.lit("\tdv:f:"); o.cell(cells + GAF_CELL * i); }
		if (ns > 1) { o.lit("\tql:B:i"); for (int32_t j = 0; j < ns; ++j) { o.c(','); o.d(ql[j]); } }
		if (p.has_cigar) {
			o.lit("\tcg:Z:");
			const uint64_t *cg = (const uint64_t*)(G.pool + p.cigar_off);
			const int32_t nc = p.n_cigar;
			gaf_list(o, nc, [&](int32_t k, int32_t *val, char *pre, char *suf) {
				const uint64_t op = cg[rev_sign? nc - 1 - k : k];
				*val = (int32_t)(op >> 4), *pre = 0, *suf = "MIDNSHP=XB"[op & 0xf];
			});
			o.lit("\tds:Z:");
			const char *ds = G.pool + p.ds_off;
			const int32_t len = p.ds_len, n_off = p.n_dsoff;
			if (!rev_sign) o.s(ds, (uint64_t)len);
			else if (n_off > 0) { // format.c:226-246: ops in reverse order, each op's bytes in place of the same length
				const int32_t *off = (const int32_t*)(G.pool + p.dsoff_off);
				if (o.p)
					for (int32_t j = off[0] + lane; j < len; j += MGB_W) {
						int32_t lo = 0, hi = n_off - 1; // the op holding byte j
						while (lo < hi) { const int32_t mid = (lo + hi + 1) >> 1; if (off[mid] <= j) lo = mid; else hi = mid - 1; }
						const int32_t ok = off[lo], ek = lo < n_off - 1? off[lo + 1] : len;
						const char op = ds[ok], c = ds[j];
						char *base = o.p + o.n + (len - ek);
						if (j == ok) base[0] = op;
						else if (op == ':') base[j - ok] = c;
						else if (op == '*') base[j - ok] = gaf_comp(c);
						else base[1 + (ek - 1 - j)] = c == '['? ']' : c == ']'? '[' : gaf_comp(c);
					}
				o.n += (uint64_t)(len - off[0]);
			}
		}
		o.c('\n');
		if (flag & F_WRITE_LCHAIN) { // -S / --write-mz (format.c:252-289)
			for (int32_t j = 0; j < p.cnt; ++j) {
				const LLChain &l = B.lc[p.off + j];
				o.lit("*\t"); put_seg(l.v); o.c('\t'); o.d(g.seg_len[l.v >> 1]); o.c('\t'); o.d(l.cnt);
				if (l.cnt > 0) {
					const u128 *a = B.a + l.off;
					const int32_t q_span = (int32_t)(a[0].y >> 32 & 0xff);
					o.c('\t'); o.cell(cells + GAF_CELL * (ro.n_gc + p.off + j));
					o.c('\t'); o.d((int32_t)a[0].x + 1 - q_span); o.c('\t'); o.d((int32_t)a[l.cnt - 1].x + 1);
					o.c('\t'); o.d((int32_t)a[0].y + 1 - q_span); o.c('\t'); o.d((int32_t)a[l.cnt - 1].y + 1);
					if (flag & F_WRITE_MZ) {
						o.c('\t'); o.d(q_span); o.c('\t');
						gaf_list(o, l.cnt - 1, [&](int32_t k, int32_t *val, char *pre, char *suf) {
							*val = (int32_t)((uint32_t)a[k + 1].x - (uint32_t)a[k].x), *pre = k > 0? ',' : 0, *suf = 0;
						});
						o.c('\t');
						gaf_list(o, l.cnt - 1, [&](int32_t k, int32_t *val, char *pre, char *suf) {
							*val = (int32_t)((uint32_t)a[k + 1].y - (uint32_t)a[k].y), *pre = k > 0? ',' : 0, *suf = 0;
						});
					}
				}
				o.c('\n');
			}
		}
	}
	return o.n;
}

} // namespace mgb
