/* mgb200.h -- C ABI of libmgb200.so, the GPU-native (H100) replacement of minigraph's seed-chain-align hot path.
 *
 * The library is a drop-in for the mapping entry points of the reference: it keeps the symbol names, argument
 * meaning and ownership rules of minigraph.h so that the unmodified C host (main.c, gfa-*.c, bseq.c, format.c,
 * options.c, kthread.c ...) links against it.  Struct layouts below are binary compatible with the reference
 * headers they cite; they are restated here (not included) so that the library builds without the reference tree.
 * If the reference headers are included first (MINIGRAPH_H / __GFA_H__ defined), the restated types are skipped.
 *
 * Every entry point needs a CUDA device (an H100, sm_90a); there is no CPU fallback: without a device mg_index() returns
 * NULL after printing an error, and mgb_last_error() tells why.
 */
#ifndef MGB200_H
#define MGB200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------------------
 * Types restated from the reference (binary compatible)
 * ---------------------------------------------------------------------------------------------------------- */
#ifndef __GFA_H__
#define __GFA_H__ /* the restated declarations below stand in for gfa.h */
typedef struct { /* gfa.h:33-39 */
	uint64_t v_lv;
	uint32_t w;
	int32_t rank;
	int32_t ov, ow;
	uint64_t link_id:61, strong:1, del:1, comp:1;
} gfa_arc_t;

typedef struct { uint32_t m_aux, l_aux; uint8_t *aux; } gfa_aux_t; /* gfa.h:50-53 */

typedef struct gfa_utg_s gfa_utg_t; /* gfa.h:55-63, opaque here */

typedef struct { /* gfa.h:65-74 */
	int32_t len;
	uint32_t del:16, circ:16;
	int32_t snid;
	int32_t soff;
	int32_t rank;
	char *name, *seq;
	gfa_utg_t *utg;
	gfa_aux_t aux;
} gfa_seg_t;

typedef struct { char *name; int32_t min, max, rank; } gfa_sseq_t; /* gfa.h:82-85 */

typedef struct { /* gfa.h:89-101 */
	uint32_t m_seg, n_seg, max_rank;
	gfa_seg_t *seg;
	void *h_names;
	uint32_t m_sseq, n_sseq;
	gfa_sseq_t *sseq;
	void *h_snames;
	uint64_t m_arc, n_arc;
	gfa_arc_t *arc;
	gfa_aux_t *link_aux;
	uint64_t *idx;
} gfa_t;

typedef struct { const char *seq; int32_t len; } gfa_edseq_t; /* gfa.h:103-106 */
#endif

#ifndef MINIGRAPH_H
#define MINIGRAPH_H /* the restated declarations below stand in for minigraph.h */
#define MG_M_RMQ    0x8000      /* minigraph.h:24 */
#define MG_M_CIGAR  0x4000000   /* minigraph.h:35 */

typedef struct { uint64_t x, y; } mg128_t; /* minigraph.h:41 */

typedef struct { int w, k; int bucket_bits; } mg_idxopt_t; /* minigraph.h:46-49 */

typedef struct { /* minigraph.h:51-77 */
	uint64_t flag;
	int64_t mini_batch_size;
	int seed;
	int max_qlen;
	int pe_ori;
	int occ_max1, occ_max1_cap;
	float occ_max1_frac;
	int bw, bw_long;
	int rmq_size_cap;
	int rmq_rescue_size;
	float rmq_rescue_ratio;
	int max_gap_pre, max_gap, max_gap_ref, max_frag_len;
	float div;
	float chn_pen_gap, chn_pen_skip;
	int max_lc_skip, max_lc_iter, max_gc_skip;
	int min_lc_cnt, min_lc_score;
	int min_gc_cnt, min_gc_score;
	int gdp_max_ed, lc_max_trim, lc_max_occ;
	float mask_level;
	int sub_diff;
	int best_n;
	float pri_ratio;
	int ref_bonus;
	int64_t cap_kalloc;
	int min_cov_mapq, min_cov_blen;
} mg_mapopt_t;

typedef struct { /* minigraph.h:93-98 */
	const gfa_t *g;
	gfa_edseq_t *es;
	int32_t b, w, k, flag, n_seg;
	struct mg_idx_bucket_s *B; /* hidden: here it points to the engine's model (host copy + device image) */
} mg_idx_t;

typedef struct { /* minigraph.h:100-106 */
	int32_t off, cnt:31, inner_pre:1;
	uint32_t v;
	int32_t rs, re, qs, qe;
	int32_t score, dist_pre;
	uint32_t hash_pre;
} mg_lchain_t;

typedef struct { int32_t off, cnt; uint32_t v; int32_t score; int32_t ed; } mg_llchain_t; /* minigraph.h:108-113 */

typedef struct { /* minigraph.h:115-118 */
	int32_t n_cigar, mlen, blen, aplen, ss, ee;
	uint64_t cigar[];
} mg_cigar_t;

typedef struct { int32_t len, n_off, *off; char *ds; } mg_ds_t; /* minigraph.h:120-123 */

typedef struct { /* minigraph.h:125-138 */
	int32_t id, parent;
	int32_t off, cnt;
	int32_t n_anchor, score;
	int32_t qs, qe;
	int32_t plen, ps, pe;
	int32_t blen, mlen;
	float div;
	uint32_t hash;
	int32_t subsc, n_sub;
	uint32_t mapq:8, flt:1, dummy:23;
	mg_cigar_t *p;
	mg_ds_t ds;
} mg_gchain_t;

typedef struct { /* minigraph.h:140-146 */
	void *km;
	int32_t n_gc, n_lc, n_a, rep_len;
	mg_gchain_t *gc;
	mg_llchain_t *lc;
	mg128_t *a;
} mg_gchains_t;

typedef struct mg_tbuf_s mg_tbuf_t; /* minigraph.h:148, opaque */
#endif

/* ------------------------------------------------------------------------------------------------------------
 * Entry points that replace reference symbols one to one
 * ---------------------------------------------------------------------------------------------------------- */

/* replaces index.c:211-230 mg_index(): upper-cases the segments of g (index.c:215-220), returns NULL when the graph
 * has overlapping links (index.c:192-196), builds the minimizer index, uploads graph+index to the GPU and updates
 * mo->occ_max1 / lc_max_occ / bw_long exactly like options.c:120-134 mg_opt_update(). n_threads is ignored.
 * The GPU is the engine parameter "device" (default 0); with the environment variable MGB_DEVICES ("0-7", "0,2,5") the index is
 * replicated on every listed GPU and each mg_map_batch*() call is cut into one contiguous part per GPU (results in input order).
 * Returns NULL on failure (no CUDA device, out of device memory, overlapping links) with the reason in mgb_last_error(). */
mg_idx_t *mg_index(gfa_t *g, const mg_idxopt_t *io, int n_threads, mg_mapopt_t *mo);

/* replaces index.c:30-46 mg_idx_destroy() */
void mg_idx_destroy(mg_idx_t *gi);

/* replaces index.c:67-72 mg_idx_get(): host view of one occurrence list (ascending seg<<32|pos<<1|strand) */
const uint64_t *mg_idx_get(const mg_idx_t *gi, uint64_t minier, int *n);

/* replaces index.c:74-93 mg_idx_cal_quantile() */
void mg_idx_cal_quantile(const mg_idx_t *gi, int32_t m, float f[], int32_t q[]);

/* replaces index.c:108-113 mg_idx_hfree(): the one other index.c symbol the remaining host files reference
 * (shortk.c:191, always with a NULL handle); a no-op here */
void mg_idx_hfree(void *h);

/* replace map-algo.c:14-27 mg_tbuf_init()/mg_tbuf_destroy(): the per-thread arena becomes a handle without state */
mg_tbuf_t *mg_tbuf_init(void);
void mg_tbuf_destroy(mg_tbuf_t *b);

/* replaces map-algo.c:340-495 mg_map_frag(): gcs[0] receives a malloc()ed result owned by the caller (free with
 * mg_gchain_free), or NULL when the fragment is empty, has more than 255 segments or is longer than opt->max_qlen
 * (map-algo.c:359-360); gcs[i>0] = NULL. With n_segs > 1 the concatenated fragment is mapped and no CIGAR is produced
 * (map-algo.c:34-45,464,475). One fragment per launch: correct but slow -- use mg_map_batch for single-segment reads.
 * Re-entrancy: like the reference's (which needs one mg_tbuf_t per thread, map-algo.c:9-12), any number of host threads may call
 * mg_map_frag()/mg_map()/mg_map_batch*() on one mg_idx_t at the same time.  Every call in flight owns a "slot" (stream, staging
 * buffers, pools, worker arenas); at most "slots" calls (engine parameter, default 3) run at once, further callers wait.
 * This entry point has no error return (the reference's has none): an internal failure ends the process as an assert would. */
void mg_map_frag(const mg_idx_t *gi, int n_segs, const int *qlens, const char **seqs, mg_gchains_t **gcs, mg_tbuf_t *b, const mg_mapopt_t *opt, const char *qname);

/* replaces map-algo.c:497-502 mg_map() */
mg_gchains_t *mg_map(const mg_idx_t *gi, int qlen, const char *seq, mg_tbuf_t *b, const mg_mapopt_t *opt, const char *qname);

/* replaces gchain1.c:522-535 mg_gchain_free() (results are plain malloc/calloc blocks, km == NULL) */
void mg_gchain_free(mg_gchains_t *gs);

/* ------------------------------------------------------------------------------------------------------------
 * New entry point: the GPU batch dispatcher that replaces kt_for(worker_for) at gmap.c:99
 * ---------------------------------------------------------------------------------------------------------- */

/* Map n_reads single-segment reads in one go. seqs[i] must be upper-case (gmap.c:81) and need not be 0-terminated;
 * names[i] may be NULL. gcs[i] is filled exactly as worker_for() (gmap.c:29-64) would fill s->gcs[off].
 * Returns 0, or a negative code after printing the reason (no partial results are left behind; a CUDA failure -- out of memory,
 * a fault -- is reported this way too, the library never ends the process from here).  A host that maps mini-batch i+1 from a
 * second thread while the first is still inside the call for mini-batch i overlaps packing, copies and result assembly of one
 * with the kernels of the other, as the reference's kt_pipeline overlaps its steps (gmap.c:176-177). */
int mg_map_batch(const mg_idx_t *gi, int n_reads, const int *qlens, const char *const *seqs, const char *const *names,
				 mg_gchains_t **gcs, const mg_mapopt_t *opt);

/* The same for fragments of several segments (read pairs, the `sr` preset): fragment f owns n_seg[f] consecutive entries of
 * qlens/seqs/gcs; the result of the concatenated fragment goes to its first gcs entry, the others are NULL -- what
 * worker_for() leaves without MG_M_INDEPEND_SEG (gmap.c:46-48). names[] is per fragment. The caller reverse-complements
 * mates beforehand as gmap.c:38-40 does. */
int mg_map_batch_frag(const mg_idx_t *gi, int n_frag, const int *n_seg, const int *qlens, const char *const *seqs, const char *const *names,
					  mg_gchains_t **gcs, const mg_mapopt_t *opt);

/* mg_gchain_free() over a whole batch (what step 2 of the reference pipeline does read by read, gmap.c:130); entries are set to NULL */
void mgb_free_batch(int n_reads, mg_gchains_t **gcs);

/* Map a batch and return its GAF text, formatted on the device: byte for byte what mg_map_batch_frag() followed by the
 * reference's mg_write_gaf() (format.c:121-291) on every fragment in input order gives, with opt->flag as the writer's flag.
 * n_seg == NULL: one segment per read (n_frag reads).  names[f] may be NULL ("*", as mgb_write_gaf_batch).  The text is
 * 0-terminated; (out, out_len, out_cap) follow mgb_write_gaf_batch(): out_cap == NULL gives a fresh malloc() block, otherwise a
 * caller-owned buffer that is reused and grown.  Returns 0, or a negative code with the reason in mgb_last_error() and
 * *out_len = 0 (no partial text).  MG_M_CAL_COV and MG_M_INDEPEND_SEG are refused: the reference prints no per-fragment GAF
 * record under them.  Slots, host threads and MGB_DEVICES work as for mg_map_batch(); no mg_gchains_t is built.  In the
 * stats of such a call, out_bytes is the number of text bytes copied back, t_d2h_ms covers the GAF kernels plus that copy,
 * and t_asm_ms is the host time after the copy (the text copied on into the caller's buffer). */
int mgb_map_batch_gaf(const mg_idx_t *gi, int n_frag, const int *n_seg, const int *qlens, const char *const *seqs,
					  const char *const *names, const mg_mapopt_t *opt, char **out, size_t *out_len, size_t *out_cap);

/* Map reads that already live in device memory: no base crosses PCIe, the batch is laid out on the device by k_ingest.
 * Sequence i is d_seq[d_off[i] .. d_off[i+1]) (n_seq + 1 int64 offsets, themselves in device memory, non-decreasing, within
 * [0, seq_bytes]), bytes in any case: they are upper-cased on the device by gmap.c:81 mg_toupper's rule (only 'a'..'z' change).
 * n_seg == NULL: n_frag single-segment reads (n_seq == n_frag); otherwise as mg_map_batch_frag() (the caller has already
 * reverse-complemented mates, as gmap.c:38-40 does).  names[] is per fragment, on the host, and may be NULL.  stream: the
 * caller's cudaStream_t (NULL: the legacy default stream); the first read of d_seq / d_off is ordered after the work already
 * queued on it, nothing is queued on it, and the call returns only once it no longer reads them.  Neither buffer is modified.
 * The results are byte for byte those of mg_map_batch_frag() / mgb_map_batch_gaf() on the same reads after mg_toupper: gcs has
 * n_seq entries filled as mg_map_batch_frag() fills them, and the text follows mgb_map_batch_gaf()'s buffer rules and refusals.
 * Returns 0, or a negative code with the reason in mgb_last_error() and no partial results, also when d_seq or d_off is not device
 * or managed memory on the index's device, the offsets decrease or fall outside [0, seq_bytes], or a read is longer than INT32_MAX.
 * The host copies the offsets back (8 bytes per read) for the batch's layout.  MGB_DEVICES works as for mg_map_batch(): a part
 * that maps on a peer device gets its span of d_seq copied device to device.  In the stats of such a call, h2d_bytes counts only
 * the per-read tables, t_pack_ms is 0, and t_h2d_ms covers the copy of the offsets, the tables and the ingest kernel. */
int mgb_map_batch_dev(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
					  const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream, mg_gchains_t **gcs);
int mgb_map_batch_dev_gaf(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
						  const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream, char **out, size_t *out_len,
						  size_t *out_cap);

/* Map reads that already live in device memory straight to result tables in device memory: the content of the mg_gchains_t that
 * mgb_map_batch_dev() would give, as dense row-major tables in one block, written on the device from the result blobs (no blob
 * crosses PCIe).  The arguments, their checks and refusals are those of mgb_map_batch_dev().  alloc(alloc_ctx, bytes) is called
 * exactly once, from the calling thread, by every call that passes those checks, and only once mapping succeeded; it returns a
 * block of at least `bytes` bytes of device memory on the index's device, which the caller owns (a NULL return fails the call).
 * The call returns once the tables are written: they may be used on any stream right away.  *out receives the rows of every table,
 * the block and the byte offset of each table in it (256-byte aligned):
 *   MGB_REC_SEQ_CSR   int64 [n_seq + 1][3]  sequence i's first record, first linear chain and first anchor; row n_seq: the totals
 *   MGB_REC_SEQ_INFO  int32 [n_seq][2]      has_result (1 where mgb_map_batch_dev() leaves gcs[i] non-NULL: not for an empty or
 *                                           over-long read, nor for the non-first segments of a fragment), rep_len
 *   MGB_REC_GC        int32 [n_rec][MGB_GC_NCOL]  the fields of mg_gchain_t in struct order but div (hash as its bits, off
 *                                           relative to the read's linear chains), then has_cigar, n_cigar and the mg_cigar_t header
 *   MGB_REC_GC_DIV    float [n_rec]         mg_gchain_t.div
 *   MGB_REC_CIGAR_CSR int64 [n_rec + 1]     record k's first CIGAR operation; row n_rec: their number
 *   MGB_REC_LC        int32 [n_lc][5]       mg_llchain_t (off relative to the read's anchors, cnt, v, score, ed)
 *   MGB_REC_A         int64 [n_a][2]        mg128_t (x, y as their bits)
 *   MGB_REC_CIGAR     int64 [n_cigar]       mg_cigar_t.cigar (len<<4 | op)
 * The ds:Z strings are not in these tables: mgb_map_batch_dev_rec_ds() below adds them.  MGB_DEVICES works as for
 * mg_map_batch(): every part is mapped and tabled on its device and the tables are joined in input order in the one block.  In the
 * stats of such a call, out_bytes counts the bytes copied back (what the div values need, 16 per record), t_d2h_ms covers the
 * table kernels, those copies and the host work between them, and t_asm_ms is 0: nothing is assembled after the kernels. */
typedef void *(*mgb_dev_alloc_fn)(void *ctx, size_t bytes);
enum { MGB_REC_SEQ_CSR, MGB_REC_SEQ_INFO, MGB_REC_GC, MGB_REC_GC_DIV, MGB_REC_CIGAR_CSR, MGB_REC_LC, MGB_REC_A, MGB_REC_CIGAR, MGB_REC_NTAB };
enum { /* the columns of MGB_REC_GC */
	MGB_GC_ID, MGB_GC_PARENT, MGB_GC_OFF, MGB_GC_CNT, MGB_GC_N_ANCHOR, MGB_GC_SCORE, MGB_GC_QS, MGB_GC_QE, MGB_GC_PLEN, MGB_GC_PS,
	MGB_GC_PE, MGB_GC_BLEN, MGB_GC_MLEN, MGB_GC_HASH, MGB_GC_SUBSC, MGB_GC_N_SUB, MGB_GC_MAPQ, MGB_GC_FLT,
	MGB_GC_HAS_CIGAR, MGB_GC_N_CIGAR, MGB_GC_C_MLEN, MGB_GC_C_BLEN, MGB_GC_C_APLEN, MGB_GC_C_SS, MGB_GC_C_EE, MGB_GC_NCOL
};
typedef struct {
	int64_t n_seq, n_rec, n_lc, n_a, n_cigar; /* rows of the tables above */
	void *block; int64_t bytes;               /* the one block alloc() returned, and its size */
	int64_t off[MGB_REC_NTAB];                /* byte offset of each table in the block, 256-byte aligned */
} mgb_records_t;
int mgb_map_batch_dev_rec(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
						  const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream,
						  mgb_dev_alloc_fn alloc, void *alloc_ctx, mgb_records_t *out);

/* mgb_map_batch_dev_rec() with the ds:Z strings too: the same arguments, checks, refusals, allocator contract, stream rules and
 * MGB_DEVICES behaviour, and in *out the same eight tables with the same rows and offsets.  The one block also holds three more
 * tables, placed after those eight; *ds_out receives their rows and byte offsets in the block (256-byte aligned), and out->bytes
 * counts them too:
 *   MGB_REC_DS_CSR  int64 [n_rec + 1][2]  record k's first byte in MGB_REC_DS and first entry in MGB_REC_DS_OFF; row n_rec: the totals
 *   MGB_REC_DS      uint8 [n_ds]          each record's mg_ds_t.ds (ds.len bytes, no terminating 0), records one after another
 *   MGB_REC_DS_OFF  int32 [n_ds_off]      each record's mg_ds_t.off[0 .. ds.n_off)
 * A record without a CIGAR (has_cigar 0: without MG_M_CIGAR, fragments with several segments, no alignment) has an empty ds.  The
 * strings are copied on the device from the result blobs; only the two totals come back.  In the stats, out_bytes is that of
 * mgb_map_batch_dev_rec() plus 16 bytes per part (the totals), t_d2h_ms also covers the ds copy, and t_asm_ms is 0. */
enum { MGB_REC_DS_CSR, MGB_REC_DS, MGB_REC_DS_OFF, MGB_REC_DS_NTAB };
typedef struct {
	int64_t n_ds, n_ds_off;        /* rows of MGB_REC_DS and MGB_REC_DS_OFF */
	int64_t off[MGB_REC_DS_NTAB];  /* byte offset of each table in out->block, 256-byte aligned */
} mgb_records_ds_t;
int mgb_map_batch_dev_rec_ds(const mg_idx_t *gi, int n_frag, const int *n_seg, int n_seq, const char *d_seq, int64_t seq_bytes,
							 const int64_t *d_off, const char *const *names, const mg_mapopt_t *opt, void *stream,
							 mgb_dev_alloc_fn alloc, void *alloc_ctx, mgb_records_t *out, mgb_records_ds_t *ds_out);

/* Parse FASTA/FASTQ text that lives in device memory into reads in device memory, on the device: d_text[0 .. text_bytes) gives the
 * records mgb_reads_load() gives for the same bytes in a file (names up to the first white space, sequences without CR/LF and
 * upper-cased, qualities skipped; malformed input alike), and SEQ / OFF feed mgb_map_batch_dev*() as they are.  Streaming: *out->used
 * is the byte where the first record not emitted starts (junk before the first header counts as used).  final == 0: a record is
 * emitted only when the start of the record after it lies in the text, so a caller that carries d_text[used ..] in front of its next
 * bytes gets the records of one whole parse, wherever its buffers end; final != 0: the last record runs to the end of the text.
 * max_bases > 0 stops after the record that reaches it (per call; used is then the start of the record after it).  The stream,
 * allocator and ownership rules are those of mgb_map_batch_dev_rec(): the first read of d_text is ordered after the work queued on
 * stream, alloc() is called once, after the parse succeeded, and the call returns once the tables are written:
 *   MGB_DR_SEQ       uint8 [n_bases]       the bases, records one after another
 *   MGB_DR_OFF       int64 [n_reads + 1]   record i is SEQ[OFF[i] .. OFF[i+1])
 *   MGB_DR_NAME      uint8 [name_bytes]    the names, no terminators
 *   MGB_DR_NAME_OFF  int64 [n_reads + 1]   record i's name is NAME[NAME_OFF[i] .. NAME_OFF[i+1])
 * Empty text, or text without a header: 0 reads, the two rows of totals written.  Returns 0, or a negative code with the reason
 * in mgb_last_error() and nothing in *out, also when d_text is not device or managed memory on the index's device, a size is
 * negative, an emitted record is longer than INT32_MAX or alloc() returns NULL.  Scratch memory (about 8 bytes per line and 25 per
 * '>' / '@' byte) is kept with the index and grown as needed; one call runs at a time per index. */
enum { MGB_DR_SEQ, MGB_DR_OFF, MGB_DR_NAME, MGB_DR_NAME_OFF, MGB_DR_NTAB };
typedef struct {
	int64_t n_reads, n_bases, name_bytes; /* rows */
	int64_t used;                         /* bytes of the text consumed: where the next call starts */
	void *block; int64_t bytes; int64_t off[MGB_DR_NTAB]; /* one block from alloc(), 256-byte aligned tables */
} mgb_dev_reads_t;
int mgb_reads_parse_dev(const mg_idx_t *gi, const char *d_text, int64_t text_bytes, int64_t max_bases, int final, void *stream,
						mgb_dev_alloc_fn alloc, void *alloc_ctx, mgb_dev_reads_t *out);

/* ------------------------------------------------------------------------------------------------------------
 * Engine controls and instrumentation (not part of the reference API)
 * ---------------------------------------------------------------------------------------------------------- */

typedef struct {
	double t_h2d_ms, t_seed_ms, t_chain_ms, t_align_ms, t_d2h_ms, t_host_ms; /* last batch, CUDA events / host clock */
	double t_wfa_ms, t_finish_ms; /* t_align_ms = graph chaining + alignment plan; t_wfa_ms = gap alignment jobs; t_finish_ms = cigar/ds/blob */
	double t_dev_span_ms;   /* device time from the first kernel start to the last kernel end over all sub-batches (they overlap) */
	int64_t skip1_len, skip2_len; /* WFA tier routing this batch ran with: gaps at or above these lengths skipped tier 1 / tier 2
	                                 (skip2_len is always INT32_MAX: every gap within tier 2's lengths is aligned there) */
	int64_t n_jobs_side;    /* gaps aligned by the tier-3 launch that runs beside tiers 1/2 */
	int64_t n_slots;        /* sub-batches the batch was cut into (each on its own stream and host thread) */
	double t_pack_ms, t_asm_ms; /* host: packing reads into the staging buffer; building mg_gchains_t objects */
	int64_t n_jobs;         /* WFA jobs of the batch */
	int64_t n_jobs_mid, n_jobs_big; /* jobs that went to tier 2 / tier 3 */
	int64_t n_reads, n_bases;
	int64_t n_seeds;        /* sum of seeds entering the chaining kernel */
	int64_t n_anchors_out;  /* sum of anchors kept in linear chains */
	int64_t n_chains_out;   /* sum of linear chains out of the DP */
	int64_t n_minimizers;
	int64_t out_bytes;      /* result bytes copied back */
	int64_t n_launches;     /* kernels launched for the batch */
	int64_t n_retry;        /* reads re-run with a larger arena */
	uint64_t arena_peak;    /* largest per-worker arena use */
	double t_kernel_ms[10]; /* CUDA-event time of each kernel of the first pass: k_seed, k_chain, k_gchain, (index), k_wfa_small, k_finish, k_wfa_mid, k_wfa_big, k_gwfa, k_gchain_gen */
	uint64_t prof[32];      /* device cycle counters per phase (see mgb_pipeline.cuh PROF_*) */
	double t_lab_ms;        /* k_gc_labels: reachability labels of source vertices seen for the first time (0 once the table is warm) */
	int64_t n_lab_new;      /* such sources in this batch */
	int64_t n_lab_big;      /* ... of which needed the second, warp-per-source pass */
	int64_t h2d_bytes;      /* bytes of reads and per-read tables copied to the device (reads travel 2 bits per base unless they hold letters other than A/C/G/T) */
	double w_gpu_wait_ms;   /* host wall clock spent waiting for the kernels of another call in flight to finish */
	double w_slot_wait_ms, w_upload_ms, w_pass_ms, w_redo_ms, w_download_ms; /* host wall clock of the call: waiting for a slot; packing + H2D; the kernels of the first pass
	                           with the host syncs between them; the large-arena pass over reads that outgrew their arena; result packing + D2H up to the assembly */
} mgb_stats_t;

/* test hook: align one gap through the tier-3 WFA path (exact up to max_iter cells, then the reference's chaining
 * heuristic, miniwfa.c:824-834, with checkpoints every `step` scores); returns n_cigar (len<<4|op) or a negative code */
int mgb_test_wfa(const char *ts, int tl, const char *qs, int ql, int64_t max_iter, int step, uint32_t *cigar, int cap, int *score);

/* test hook: n gaps through one on-chip WFA tier (1: windows of 62 diagonals, sides of 256 bases, 4096 traceback bytes in shared
 * memory; 2: 254 diagonals, 1024 bases; MGB_TEST_TIER2_CONT: tier 2 as k_wfa_mid runs it, where a gap whose window outgrows the
 * 254 diagonals before score 240 is carried on in the worker arena instead of refused), launched as the tier's kernel is.  Gap i is ts[t_off[i]..+tl[i]) against
 * qs[q_off[i]..+ql[i]).  out[4i..4i+3] = rc (0: aligned, 1: does not fit the tier, < 0: error), score, n_iter, n_cigar; the CIGAR
 * (len<<4|op) goes to cigar[i*cap..].  Returns 0, or a negative code (nothing run) when a gap has an empty side. */
#define MGB_TEST_TIER2_CONT 4
int mgb_test_wfa_tier(int tier, int n, const char *ts, const int64_t *t_off, const int32_t *tl, const char *qs, const int64_t *q_off,
					  const int32_t *ql, int64_t *out, uint32_t *cigar, int cap);

/* test hook: n bridging alignments (gchain1.c:349-381 bridge_gwfa) on the graph of gi: query q[q_off[i]..+ql[i]) from
 * (v0[i], off0[i]) to (v1[i], off1[i]), stopping at score max_ed[i].  mode 0: the warp-wide alignment of the bridging kernel;
 * mode 1: the sequential one of graph chaining.  out[6i..6i+5] = rc, s (-1: not reached), end_v, end_off, nv, n_iter; the walk
 * goes to walk[i*walk_cap..].  Returns 0, or a negative code (nothing run) when a query is empty or an end lies outside the graph. */
int mgb_test_gwfa(const mg_idx_t *gi, int mode, int n, const char *q, const int64_t *q_off, const int32_t *ql, const uint32_t *v0,
				  const int32_t *off0, const uint32_t *v1, const int32_t *off1, const int32_t *max_ed, int64_t *out, int32_t *walk, int walk_cap);

/* test hook: the exact radix sort of the seeds (klib's radix_sort_128x order, ties included) on one warp, in place (walk 0) or
 * by digit walk (walk 1), with hot_bytes of shared memory for its scratch (0: all of it in global memory); 0 or a negative code */
int mgb_test_radix128(mg128_t *a, int64_t n, int walk, int hot_bytes);

/* test hook: linear chaining of n anchor sets as the chaining kernels run it, the anchors staged into a warp's slice of shared
 * memory when they fit.  mode 0: DP (k_chain, lr); 1: RMQ with opt.bw (k_chain, asm); 2: the anchors sorted back into target
 * order, then RMQ (k_chain_rescue, which the caller gives bw_long as opt.bw).  Set i is a[off[i]..+cnt[i]) with the options opt[i]
 * (the RMQ chaining takes max_dist_x as its max_dist).  out[6i..6i+5] = rc, n_u, n_v, staged (0/1), path (0: DP, 1: RMQ, the
 * warp-wide fill; 2: RMQ, the warp-wide fill gave up on a tie of priorities; 3: RMQ, sequential because cnt[i] > cap_rmq_size;
 * -1: no anchors), worker; the chains go to u[off[i]..+n_u), the compacted anchors to a_out[off[i]..+n_v).  Returns 0, or a
 * negative code (nothing run) for a bad mode, offset or count. */
typedef struct {
	int32_t max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc;
	float pen_gap, pen_skip;
	int32_t is_cdna, n_seg, max_dist_inner, cap_rmq_size;
} mgb_lchain_opt_t;
int mgb_test_lchain(int mode, int n, const mg128_t *a, const int64_t *off, const int32_t *cnt, const mgb_lchain_opt_t *opt, int32_t *out,
					uint64_t *u, mg128_t *a_out);

/* test hook: the (w,k)-minimizers (sketch.c mg_sketch) of n sequences seq[off[i]..+len[i]) (bytes, not strings: 0..3 are bases),
 * sequence i with rid i, on a warp launched as the seeding kernel is.  mode 0: the sketch of the seeding kernel, cut into chunks
 * over the lanes where it can be, the window rings in the warp's slice of shared memory and, for a sequence that is all A/C/G/T,
 * the bases read from the 2-bit words of the batch upload; mode 1: the sequential sketch of the index build, on lane 0.
 * out[3i..3i+2] = rc, n, path (mode 0: MGB_SKETCH_PATH_*; mode 1: -1); the list goes to mz[mz_off[i]..+n) if it fits before
 * mz_off[i+1].  Returns 0, or a negative code (nothing run) for bad k, w, mode or an empty sequence. */
#define MGB_SKETCH_PATH_SMEM_PK 0 /* chunks, rings in shared memory, 2-bit words */
#define MGB_SKETCH_PATH_SMEM 1    /* chunks, rings in shared memory, ASCII */
#define MGB_SKETCH_PATH_ARENA 2   /* chunks, rings in the worker arena (w > 12) */
#define MGB_SKETCH_PATH_SEQ 3     /* the sequential scan on lane 0 */
int mgb_test_sketch(int k, int w, int n, const char *seq, const int64_t *off, const int32_t *len, int mode, int32_t *out, mg128_t *mz, const int64_t *mz_off);

/* test hook: the seeding stage itself (minimizers, index lookup with the occurrence filter, seed expansion, seed sort or the heap
 * merge of MG_M_HEAP_SORT) on n reads with the graph and index of gi and the options flag, occ_max1 and max_qlen, the batch
 * packed as mg_map_batch packs it.  seg_off == NULL: single-segment reads; otherwise read i is the concatenation of the
 * non-empty segments seg_len[seg_off[i]..seg_off[i+1]) (qlens[i] their sum).  names (may be NULL) decide MG_M_NO_DIAG.
 * out[5i..5i+4] = status (0; 1: not mapped, empty or longer than max_qlen; < 0: error), n_mz, rep_len, n_a, n_mp; the seeds of
 * the reads with status 0 follow each other in a[] in read order, as the stage leaves them, and so do their mini_pos.  Returns 0,
 * MGB_E_POOL when they do not fit a_cap / mp_cap (out[] is filled), or a negative code (nothing run) for bad reads. */
int mgb_test_seed(const mg_idx_t *gi, int n, const int *qlens, const char *const *seqs, const int32_t *seg_off, const int32_t *seg_len,
				  const char *const *names, uint64_t flag, int occ_max1, int max_qlen, int32_t *out, mg128_t *a, int64_t a_cap, int32_t *mini_pos, int64_t mp_cap);

/* test hook: graph-chain materialisation, the primary/secondary filters and mapq (map-algo.c:464-474 up to the CIGAR) as the kernels
 * k_gchain (its bridging plan), k_gwfa and k_gchain_gen run them, on n reads whose graph chaining is given, with the graph of gi
 * and the options opt (MG_M_CIGAR is ignored).  Read i is seqs[i] (qlens[i] > 0 bases); seg_off == NULL: one segment each,
 * otherwise as for mgb_test_seed.  hash[i] is its hash (map-algo.c:362-364), rep_len[i] and n_mz[i] its repeat length and
 * minimizer count; its n_u[i] chains (score<<32 | linear chains), n_lc[i] linear chains in the order mg_gchain1_dp leaves them
 * and n_a[i] anchors (minimizer index in x>>32, as after mg_update_anchors; lc[].off counts from the read's first anchor) follow
 * those of read i-1 in u, lc and a.  out[4i..4i+3] = rc (0 or a negative code), bridging jobs planned, of which aligned, pairs
 * of linear chains bridged again in place after a failed bridge; gcs[i] (NULL unless rc is 0) is freed by mg_gchain_free.
 * Returns 0, or a negative code (nothing run) for malformed input. */
int mgb_test_gchain_gen(const mg_idx_t *gi, const mg_mapopt_t *opt, int n, const int *qlens, const char *const *seqs, const int32_t *seg_off,
						const int32_t *seg_len, const uint32_t *hash, const int32_t *rep_len, const int32_t *n_mz, const int32_t *n_u, const uint64_t *u,
						const int32_t *n_lc, const mg_lchain_t *lc, const int32_t *n_a, const mg128_t *a, int32_t *out, mg_gchains_t **gcs);

/* test hook: the ingest step of reads in device memory as mgb_map_batch_dev() runs it (k_ingest on the device, its body on every
 * lane of a simulated warp in the simulators) on n sequences seq[off[i] .. off[i+1]) (host memory, copied to the device first).  Sequence i's upper-case copy goes
 * to ascii_out[off[i] .. off[i+1]); unless segmented (a batch of fragments with segments, which has no 2-bit words), its
 * (len + 31) / 32 words follow those of sequence i-1 in pk_out; raw_out[i] is 1 when it holds a byte other than A/C/G/T.
 * Returns 0, or a negative code for bad offsets or when the batch's pk_off does not mark exactly the flagged reads. */
int mgb_test_ingest(int n, const char *seq, const int64_t *off, int segmented, char *ascii_out, uint64_t *pk_out, int32_t *raw_out);

const char *mgb_last_error(void);
void mgb_get_stats(const mg_idx_t *gi, mgb_stats_t *st);
/* knobs: "arena_mb" (per worker), "workers_per_sm", "device"; returns 0 if the key is known */
int mgb_set_param(const char *key, int64_t value);
const char *mgb_version(void);

/* Convenience for callers without a gfa_t (bench, tests): parse GFA/rGFA text the way gfa-io.c:294-337 gfa_read()
 * does for S/L lines with SN/SO/SR tags and plain FASTA, and finalize arcs like gfa-base.c:421-430. */
gfa_t *mgb_gfa_read(const char *fn);
void mgb_gfa_destroy(gfa_t *g);

/* Input side for hosts without the reference's bseq.c: a whole FASTA/FASTQ file (plain or gzip, "-" = stdin) parsed by kseq.h's rules
 * (bseq.c:46-98) and upper-cased (gmap.c:81) into the arrays mg_map_batch() takes.  max_bases > 0 stops after the record that
 * reaches it (the reference's mini-batch rule, bseq.c:70-72).  NULL if the file cannot be opened. */
typedef struct { int64_t n_reads, n_bases; const char **name, **seq; int *len; char *block; } mgb_reads_t;
mgb_reads_t *mgb_reads_load(const char *fn, int64_t max_bases);
void mgb_reads_free(mgb_reads_t *r);

/* Byte-exact GAF line(s) for one read, restating format.c:121-291 mg_write_gaf() for flag bits used by -c. The text is
 * appended to *buf (realloc()ed; *len and *cap updated). */
void mgb_write_gaf(char **buf, size_t *len, size_t *cap, const gfa_t *g, const mg_gchains_t *gs, int32_t qlen, const char *qname, uint64_t flag);

/* The same for a whole batch, input order preserved, formatted by n_threads host threads (0: up to 16). The text is
 * 0-terminated and *out_len receives its length. out_cap == NULL: *out is a fresh malloc() block the caller frees.
 * out_cap != NULL: (*out, *out_cap) is a buffer owned by the caller (NULL/0 the first time) that is reused and grown
 * with realloc semantics, like mgb_write_gaf() does with (buf, cap). */
void mgb_write_gaf_batch(const gfa_t *g, int n_reads, mg_gchains_t *const *gcs, const int *qlens, const char *const *names,
						 uint64_t flag, int n_threads, char **out, size_t *out_len, size_t *out_cap);

#ifdef __cplusplus
}
#endif
#endif
