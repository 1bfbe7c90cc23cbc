"""ctypes view of include/mgb200.h -- the C ABI shared by libmgb200.so and the reference (minigraph.h).

The same structure definitions bind (a) the product library, (b) tests/hostsim and (c) oracle/_ref/libmgref.so,
because the ABI *is* the reference's (minigraph.h:41-176, gfa.h:33-106)."""
import ctypes as C
import os

MG_M_RMQ = 0x8000
MG_M_CIGAR = 0x4000000
MG_M_PRINT_2ND = 0x2000


class mg128_t(C.Structure):
    _fields_ = [("x", C.c_uint64), ("y", C.c_uint64)]


class mg_idxopt_t(C.Structure):
    _fields_ = [("w", C.c_int), ("k", C.c_int), ("bucket_bits", C.c_int)]


class mg_mapopt_t(C.Structure):  # minigraph.h:51-77
    _fields_ = [
        ("flag", C.c_uint64), ("mini_batch_size", C.c_int64), ("seed", C.c_int), ("max_qlen", C.c_int),
        ("pe_ori", C.c_int), ("occ_max1", C.c_int), ("occ_max1_cap", C.c_int), ("occ_max1_frac", C.c_float),
        ("bw", C.c_int), ("bw_long", C.c_int), ("rmq_size_cap", C.c_int), ("rmq_rescue_size", C.c_int),
        ("rmq_rescue_ratio", C.c_float), ("max_gap_pre", C.c_int), ("max_gap", C.c_int), ("max_gap_ref", C.c_int),
        ("max_frag_len", C.c_int), ("div", C.c_float), ("chn_pen_gap", C.c_float), ("chn_pen_skip", C.c_float),
        ("max_lc_skip", C.c_int), ("max_lc_iter", C.c_int), ("max_gc_skip", C.c_int), ("min_lc_cnt", C.c_int),
        ("min_lc_score", C.c_int), ("min_gc_cnt", C.c_int), ("min_gc_score", C.c_int), ("gdp_max_ed", C.c_int),
        ("lc_max_trim", C.c_int), ("lc_max_occ", C.c_int), ("mask_level", C.c_float), ("sub_diff", C.c_int),
        ("best_n", C.c_int), ("pri_ratio", C.c_float), ("ref_bonus", C.c_int), ("cap_kalloc", C.c_int64),
        ("min_cov_mapq", C.c_int), ("min_cov_blen", C.c_int),
    ]


class mg_idx_t(C.Structure):
    _fields_ = [("g", C.c_void_p), ("es", C.c_void_p), ("b", C.c_int32), ("w", C.c_int32), ("k", C.c_int32),
                ("flag", C.c_int32), ("n_seg", C.c_int32), ("B", C.c_void_p)]


class mg_lchain_t(C.Structure):  # minigraph.h:100-106
    _fields_ = [("off", C.c_int32), ("cnt", C.c_int32, 31), ("inner_pre", C.c_int32, 1), ("v", C.c_uint32), ("rs", C.c_int32),
                ("re", C.c_int32), ("qs", C.c_int32), ("qe", C.c_int32), ("score", C.c_int32), ("dist_pre", C.c_int32),
                ("hash_pre", C.c_uint32)]


class mg_llchain_t(C.Structure):
    _fields_ = [("off", C.c_int32), ("cnt", C.c_int32), ("v", C.c_uint32), ("score", C.c_int32), ("ed", C.c_int32)]


class mg_cigar_t(C.Structure):
    _fields_ = [("n_cigar", C.c_int32), ("mlen", C.c_int32), ("blen", C.c_int32), ("aplen", C.c_int32),
                ("ss", C.c_int32), ("ee", C.c_int32)]  # followed by uint64 cigar[]


class mg_ds_t(C.Structure):
    _fields_ = [("len", C.c_int32), ("n_off", C.c_int32), ("off", C.POINTER(C.c_int32)), ("ds", C.c_void_p)]


class mg_gchain_t(C.Structure):
    _fields_ = [
        ("id", C.c_int32), ("parent", C.c_int32), ("off", C.c_int32), ("cnt", C.c_int32), ("n_anchor", C.c_int32),
        ("score", C.c_int32), ("qs", C.c_int32), ("qe", C.c_int32), ("plen", C.c_int32), ("ps", C.c_int32),
        ("pe", C.c_int32), ("blen", C.c_int32), ("mlen", C.c_int32), ("div", C.c_float), ("hash", C.c_uint32),
        ("subsc", C.c_int32), ("n_sub", C.c_int32), ("mapq", C.c_uint32, 8), ("flt", C.c_uint32, 1),
        ("dummy", C.c_uint32, 23), ("p", C.POINTER(mg_cigar_t)), ("ds", mg_ds_t),
    ]


class mg_gchains_t(C.Structure):
    _fields_ = [("km", C.c_void_p), ("n_gc", C.c_int32), ("n_lc", C.c_int32), ("n_a", C.c_int32),
                ("rep_len", C.c_int32), ("gc", C.POINTER(mg_gchain_t)), ("lc", C.POINTER(mg_llchain_t)),
                ("a", C.POINTER(mg128_t))]


class gfa_seg_t(C.Structure):  # gfa.h:65-74
    _fields_ = [("len", C.c_int32), ("del_circ", C.c_uint32), ("snid", C.c_int32), ("soff", C.c_int32),
                ("rank", C.c_int32), ("name", C.c_char_p), ("seq", C.c_void_p), ("utg", C.c_void_p),
                ("aux_m", C.c_uint32), ("aux_l", C.c_uint32), ("aux", C.c_void_p)]


class gfa_sseq_t(C.Structure):
    _fields_ = [("name", C.c_char_p), ("min", C.c_int32), ("max", C.c_int32), ("rank", C.c_int32)]


class gfa_t(C.Structure):  # gfa.h:89-101
    _fields_ = [("m_seg", C.c_uint32), ("n_seg", C.c_uint32), ("max_rank", C.c_uint32), ("seg", C.POINTER(gfa_seg_t)),
                ("h_names", C.c_void_p), ("m_sseq", C.c_uint32), ("n_sseq", C.c_uint32),
                ("sseq", C.POINTER(gfa_sseq_t)), ("h_snames", C.c_void_p), ("m_arc", C.c_uint64),
                ("n_arc", C.c_uint64), ("arc", C.c_void_p), ("link_aux", C.c_void_p), ("idx", C.POINTER(C.c_uint64))]


class mgb_stats_t(C.Structure):
    _fields_ = [("t_h2d_ms", C.c_double), ("t_seed_ms", C.c_double), ("t_chain_ms", C.c_double),
                ("t_align_ms", C.c_double), ("t_d2h_ms", C.c_double), ("t_host_ms", C.c_double),
                ("t_wfa_ms", C.c_double), ("t_finish_ms", C.c_double), ("t_dev_span_ms", C.c_double), ("skip1_len", C.c_int64), ("skip2_len", C.c_int64), ("n_jobs_side", C.c_int64), ("n_slots", C.c_int64), ("t_pack_ms", C.c_double), ("t_asm_ms", C.c_double),
                ("n_jobs", C.c_int64), ("n_jobs_mid", C.c_int64), ("n_jobs_big", C.c_int64),
                ("n_reads", C.c_int64), ("n_bases", C.c_int64), ("n_seeds", C.c_int64), ("n_anchors_out", C.c_int64),
                ("n_chains_out", C.c_int64), ("n_minimizers", C.c_int64), ("out_bytes", C.c_int64),
                ("n_launches", C.c_int64), ("n_retry", C.c_int64), ("arena_peak", C.c_uint64), ("t_kernel_ms", C.c_double * 10), ("prof", C.c_uint64 * 32), ("t_lab_ms", C.c_double), ("n_lab_new", C.c_int64), ("n_lab_big", C.c_int64), ("h2d_bytes", C.c_int64),
                ("w_gpu_wait_ms", C.c_double), ("w_slot_wait_ms", C.c_double), ("w_upload_ms", C.c_double), ("w_pass_ms", C.c_double), ("w_redo_ms", C.c_double), ("w_download_ms", C.c_double)]


# mgb_map_batch_dev_rec(): the tables of mgb_records_t (mgb200.h MGB_REC_*) and the columns of its GC table (MGB_GC_*)
REC_TABLES = ("seq_csr", "seq_info", "gc", "gc_div", "cigar_csr", "lc", "a", "cigar")
GC_COLUMNS = ("id", "parent", "off", "cnt", "n_anchor", "score", "qs", "qe", "plen", "ps", "pe", "blen", "mlen", "hash", "subsc", "n_sub",
              "mapq", "flt", "has_cigar", "n_cigar", "c_mlen", "c_blen", "c_aplen", "c_ss", "c_ee")


class mgb_records_t(C.Structure):
    _fields_ = [("n_seq", C.c_int64), ("n_rec", C.c_int64), ("n_lc", C.c_int64), ("n_a", C.c_int64), ("n_cigar", C.c_int64),
                ("block", C.c_void_p), ("bytes", C.c_int64), ("off", C.c_int64 * len(REC_TABLES))]


# mgb_map_batch_dev_rec_ds(): the ds tables of mgb_records_ds_t (mgb200.h MGB_REC_DS_*), in the same block after REC_TABLES
REC_DS_TABLES = ("ds_csr", "ds", "ds_off")


class mgb_records_ds_t(C.Structure):
    _fields_ = [("n_ds", C.c_int64), ("n_ds_off", C.c_int64), ("off", C.c_int64 * len(REC_DS_TABLES))]


# void *alloc(void *ctx, size_t bytes)
mgb_dev_alloc_fn = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)


class mgb_reads_t(C.Structure):
    _fields_ = [("n_reads", C.c_int64), ("n_bases", C.c_int64), ("name", C.POINTER(C.c_char_p)), ("seq", C.POINTER(C.c_char_p)),
                ("len", C.POINTER(C.c_int)), ("block", C.c_void_p)]


KERNEL_NAMES = ["k_seed", "k_chain", "k_gchain", "k_index_sketch", "k_wfa_small", "k_finish", "k_wfa_mid", "k_wfa_big", "k_gwfa", "k_gchain_gen"]
PROF_NAMES = ["wfa_fast_cyc", "wfa_fast_n", "wfa_slow_cyc", "wfa_slow_n", "wfa_max_cyc", "wfa_cells", "wfa_tb_cyc", "gc_dp_cyc", "gc_gen_cyc",
              "gc_post_cyc", "gc_plan_cyc", "fin_cigar_cyc", "fin_ds_cyc", "seed_sketch_cyc", "seed_match_cyc", "seed_sort_cyc", "chain_dp_cyc",
              "chain_onchip_n", "chain_rmq_cyc", "chain_post_cyc", "wfa_mid_cyc", "wfa_mid_n", "gc_gwfa_cyc", "gc_bridge_shortk_cyc", "gc_extra_sort_cyc", "gwfa_max_cyc", "gc_dp_max_cyc", "wfa_handoff_cells", "wfa_handoff_n", "lab_cyc", "lab_n"]
# mgb_test_wfa_tier(): tier 2 as k_wfa_mid runs it, carrying a gap whose window outgrows the shared-memory ring on in the arena
# (mgb200.h MGB_TEST_TIER2_CONT)
WFA_TIER2_CONT = 4
# mgb_test_lchain(): modes (k_chain DP, k_chain RMQ, k_chain_rescue) and fill paths (mgb200.h)
LCHAIN_DP, LCHAIN_RMQ, LCHAIN_RESCUE = 0, 1, 2
LCHAIN_PATH_DP, LCHAIN_PATH_RMQ_W, LCHAIN_PATH_RMQ_TIE, LCHAIN_PATH_RMQ_CAP = 0, 1, 2, 3
# mgb_test_sketch(): the ways the seeding kernel's sketch makes a list (mgb200.h MGB_SKETCH_PATH_*)
SKETCH_PATH_SMEM_PK, SKETCH_PATH_SMEM, SKETCH_PATH_ARENA, SKETCH_PATH_SEQ = 0, 1, 2, 3


class mgb_lchain_opt_t(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("max_dist_x", "max_dist_y", "bw", "max_skip", "max_iter", "min_cnt", "min_sc")] + \
               [("pen_gap", C.c_float), ("pen_skip", C.c_float)] + \
               [(k, C.c_int32) for k in ("is_cdna", "n_seg", "max_dist_inner", "cap_rmq_size")]


def bind_mapping_api(lib):
    """Declare the prototypes of the symbols that exist in both the reference and libmgb200."""
    lib.mg_index.restype = C.POINTER(mg_idx_t)
    lib.mg_index.argtypes = [C.POINTER(gfa_t), C.POINTER(mg_idxopt_t), C.c_int, C.POINTER(mg_mapopt_t)]
    lib.mg_idx_destroy.restype = None
    lib.mg_idx_destroy.argtypes = [C.POINTER(mg_idx_t)]
    lib.mg_tbuf_init.restype = C.c_void_p
    lib.mg_tbuf_destroy.restype = None
    lib.mg_tbuf_destroy.argtypes = [C.c_void_p]
    lib.mg_map.restype = C.POINTER(mg_gchains_t)
    lib.mg_map.argtypes = [C.POINTER(mg_idx_t), C.c_int, C.c_char_p, C.c_void_p, C.POINTER(mg_mapopt_t), C.c_char_p]
    lib.mg_gchain_free.restype = None
    lib.mg_gchain_free.argtypes = [C.POINTER(mg_gchains_t)]
    lib.mg_idx_get.restype = C.POINTER(C.c_uint64)
    lib.mg_idx_get.argtypes = [C.POINTER(mg_idx_t), C.c_uint64, C.POINTER(C.c_int)]
    if hasattr(lib, "mgb_map_batch_gaf"):  # the engine's; the reference has no such symbol
        lib.mgb_map_batch_gaf.restype = C.c_int
        lib.mgb_map_batch_gaf.argtypes = [C.POINTER(mg_idx_t), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_char_p),
                                          C.POINTER(C.c_char_p), C.POINTER(mg_mapopt_t), C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                          C.POINTER(C.c_size_t)]
    return lib


_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def env_params():
    """engine parameters from the environment: MGB_PARAMS="lab_cache=0,arena_mb=4" (pairs for mgb_set_param)"""
    out = {}
    for kv in os.environ.get("MGB_PARAMS", "").split(","):
        if "=" in kv:
            k, v = kv.split("=", 1)
            out[k.strip()] = int(v, 0)
    return out


def apply_env_params(lib):
    for k, v in env_params().items():
        if lib.mgb_set_param(k.encode(), v) != 0:
            raise RuntimeError("MGB_PARAMS: unknown engine parameter %r" % k)
    return lib


def load_product(path=None):
    """Load libmgb200.so (the CUDA build). Fails loudly when it has not been built -- there is no fallback."""
    path = path or os.environ.get("MGB_LIB") or os.path.join(_REPO, "minigraph_b200", "libmgb200.so")  # MGB_LIB: another build of the same library (A/B runs of bench.py)
    if not os.path.exists(path):
        raise RuntimeError("libmgb200.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(path)
    return apply_env_params(bind_engine_api(bind_mapping_api(lib)))


def bind_engine_api(lib):
    lib.mg_map_batch.restype = C.c_int
    lib.mg_map_batch.argtypes = [C.POINTER(mg_idx_t), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_char_p),
                                 C.POINTER(C.c_char_p), C.POINTER(C.POINTER(mg_gchains_t)), C.POINTER(mg_mapopt_t)]
    lib.mgb_last_error.restype = C.c_char_p
    lib.mgb_get_stats.restype = None
    lib.mgb_get_stats.argtypes = [C.POINTER(mg_idx_t), C.POINTER(mgb_stats_t)]
    lib.mgb_set_param.restype = C.c_int
    lib.mgb_set_param.argtypes = [C.c_char_p, C.c_int64]
    lib.mgb_gfa_read.restype = C.POINTER(gfa_t)
    lib.mgb_gfa_read.argtypes = [C.c_char_p]
    lib.mgb_gfa_destroy.restype = None
    lib.mgb_gfa_destroy.argtypes = [C.POINTER(gfa_t)]
    lib.mgb_write_gaf.restype = None
    lib.mgb_write_gaf.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(gfa_t),
                                  C.POINTER(mg_gchains_t), C.c_int32, C.c_char_p, C.c_uint64]
    lib.mgb_test_wfa.restype = C.c_int
    lib.mgb_test_wfa.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_uint32), C.c_int, C.POINTER(C.c_int)]
    i64p, i32p, u32p = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
    lib.mgb_test_wfa_tier.restype = C.c_int
    lib.mgb_test_wfa_tier.argtypes = [C.c_int, C.c_int, C.c_char_p, i64p, i32p, C.c_char_p, i64p, i32p, i64p, u32p, C.c_int]
    lib.mgb_test_gwfa.restype = C.c_int
    lib.mgb_test_gwfa.argtypes = [C.POINTER(mg_idx_t), C.c_int, C.c_int, C.c_char_p, i64p, i32p, u32p, i32p, u32p, i32p, i32p, i64p, i32p, C.c_int]
    lib.mgb_test_radix128.restype = C.c_int
    lib.mgb_test_radix128.argtypes = [C.POINTER(mg128_t), C.c_int64, C.c_int, C.c_int]
    lib.mgb_test_lchain.restype = C.c_int
    lib.mgb_test_lchain.argtypes = [C.c_int, C.c_int, C.POINTER(mg128_t), i64p, i32p, C.POINTER(mgb_lchain_opt_t), i32p, C.POINTER(C.c_uint64), C.POINTER(mg128_t)]
    lib.mgb_test_sketch.restype = C.c_int
    lib.mgb_test_sketch.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, i64p, i32p, C.c_int, i32p, C.POINTER(mg128_t), i64p]
    lib.mgb_test_seed.restype = C.c_int
    lib.mgb_test_seed.argtypes = [C.POINTER(mg_idx_t), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_char_p), i32p, i32p, C.POINTER(C.c_char_p),
                                  C.c_uint64, C.c_int, C.c_int, i32p, C.POINTER(mg128_t), C.c_int64, i32p, C.c_int64]
    lib.mgb_test_gchain_gen.restype = C.c_int
    lib.mgb_test_gchain_gen.argtypes = [C.POINTER(mg_idx_t), C.POINTER(mg_mapopt_t), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_char_p), i32p, i32p,
                                        u32p, i32p, i32p, i32p, C.POINTER(C.c_uint64), i32p, C.POINTER(mg_lchain_t), i32p, C.POINTER(mg128_t), i32p,
                                        C.POINTER(C.POINTER(mg_gchains_t))]
    lib.mg_map_batch_frag.restype = C.c_int
    lib.mg_map_batch_frag.argtypes = [C.POINTER(mg_idx_t), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_char_p),
                                      C.POINTER(C.POINTER(mg_gchains_t)), C.POINTER(mg_mapopt_t)]
    lib.mgb_reads_load.restype = C.POINTER(mgb_reads_t)
    lib.mgb_reads_load.argtypes = [C.c_char_p, C.c_int64]
    lib.mgb_reads_free.restype = None
    lib.mgb_reads_free.argtypes = [C.POINTER(mgb_reads_t)]
    lib.mgb_free_batch.restype = None
    lib.mgb_free_batch.argtypes = [C.c_int, C.POINTER(C.POINTER(mg_gchains_t))]
    lib.mgb_write_gaf_batch.restype = None
    lib.mgb_write_gaf_batch.argtypes = [C.POINTER(gfa_t), C.c_int, C.POINTER(C.POINTER(mg_gchains_t)), C.POINTER(C.c_int),
                                        C.POINTER(C.c_char_p), C.c_uint64, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    # reads in device memory: d_seq, d_off and the stream are plain addresses (a CUDA tensor's data_ptr(), a cudaStream_t)
    dev_args = [C.POINTER(mg_idx_t), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_char_p),
                C.POINTER(mg_mapopt_t), C.c_void_p]
    lib.mgb_map_batch_dev.restype = C.c_int
    lib.mgb_map_batch_dev.argtypes = dev_args + [C.POINTER(C.POINTER(mg_gchains_t))]
    lib.mgb_map_batch_dev_gaf.restype = C.c_int
    lib.mgb_map_batch_dev_gaf.argtypes = dev_args + [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.mgb_map_batch_dev_rec.restype = C.c_int
    lib.mgb_map_batch_dev_rec.argtypes = dev_args + [mgb_dev_alloc_fn, C.c_void_p, C.POINTER(mgb_records_t)]
    lib.mgb_map_batch_dev_rec_ds.restype = C.c_int
    lib.mgb_map_batch_dev_rec_ds.argtypes = dev_args + [mgb_dev_alloc_fn, C.c_void_p, C.POINTER(mgb_records_t), C.POINTER(mgb_records_ds_t)]
    lib.mgb_test_ingest.restype = C.c_int
    lib.mgb_test_ingest.argtypes = [C.c_int, C.c_char_p, i64p, C.c_int, C.c_void_p, C.POINTER(C.c_uint64), i32p]
    return lib
