"""Reads that live in GPU memory as torch tensors, mapped without a host copy of their bases (mgb_map_batch_dev*, include/mgb200.h).

A batch is two CUDA tensors: `seq`, uint8, every read's bytes one after the other (any case: they are upper-cased on the device), and
`off`, int64, n + 1 offsets (read i is seq[off[i]:off[i+1]]).  pack_reads() builds them from host bytes for tests and tools."""
import ctypes as C

from . import capi


def pack_reads(reads, device):
    """(seq, off) on `device` for a list of bytes objects"""
    import numpy as np
    import torch
    off = np.zeros(len(reads) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(r) for r in reads], dtype=np.int64)
    seq = np.frombuffer(b"".join(reads), dtype=np.uint8)
    return torch.from_numpy(seq.copy()).to(device), torch.from_numpy(off).to(device)


def _batch_args(who, gi, seq, off, names, opt, n_seg):
    """the arguments that mgb_map_batch_dev*() share, after the checks of a (seq, off) pair"""
    import torch
    if opt is None:
        raise TypeError("%s: opt is the mg_mapopt_t that mg_index() updated" % who)
    if seq.dtype != torch.uint8 or off.dtype != torch.int64:
        raise TypeError("%s: seq must be torch.uint8 and off torch.int64, not %s and %s" % (who, seq.dtype, off.dtype))
    if not (seq.is_cuda and off.is_cuda and seq.device == off.device):
        raise ValueError("%s: seq and off must be CUDA tensors on one device (%s, %s)" % (who, seq.device, off.device))
    if not (seq.is_contiguous() and off.is_contiguous()) or seq.dim() != 1 or off.dim() != 1 or off.numel() < 1:
        raise ValueError("%s: seq and off must be contiguous 1-D tensors, off with n + 1 entries" % who)
    n_seq = off.numel() - 1
    n_frag = len(n_seg) if n_seg is not None else n_seq
    cnseg = (C.c_int * max(1, n_frag))(*n_seg) if n_seg is not None else None
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    stream = torch.cuda.current_stream(seq.device).cuda_stream
    return n_seq, (gi, n_frag, cnseg, n_seq, seq.data_ptr(), seq.numel(), off.data_ptr(), cnames, C.byref(opt), stream)


def map_cuda_reads(lib, gi, seq, off, names=None, opt=None, n_seg=None, gaf=True):
    """Map the reads of (seq, off) with the index gi and the options opt (the mg_mapopt_t that mg_index() updated), ordered after
    the work queued on the current stream.  n_seg: segments per fragment (read pairs), or None for single-segment reads; names:
    one bytes object per fragment, or None.  Returns the GAF text (bytes) or, with gaf=False, a ctypes array of one
    mg_gchains_t pointer per sequence, owned by the caller (mgb_free_batch).  Raises RuntimeError with the library's reason when
    it refuses the batch (for instance tensors on another device than the index's)."""
    n_seq, args = _batch_args("map_cuda_reads", gi, seq, off, names, opt, n_seg)
    if gaf:
        out, ln = C.c_void_p(0), C.c_size_t(0)
        rc = lib.mgb_map_batch_dev_gaf(*args, C.byref(out), C.byref(ln), None)
        if rc < 0:
            raise RuntimeError("mgb_map_batch_dev_gaf: %s" % lib.mgb_last_error().decode())
        text = C.string_at(out, ln.value)
        C.CDLL(None).free(out)
        return text
    gcs = (C.POINTER(capi.mg_gchains_t) * max(1, n_seq))()
    rc = lib.mgb_map_batch_dev(*args, gcs)
    if rc < 0:
        raise RuntimeError("mgb_map_batch_dev: %s" % lib.mgb_last_error().decode())
    return gcs


# the mg_gchain_t fields (and the mg_cigar_t header) of the columns of MappedTables.gc, in order (mgb200.h MGB_GC_*)
GC_COLUMNS = capi.GC_COLUMNS


class MappedTables:
    """The results of a batch as tensors on the index's device, all views of one uint8 tensor (`block`), row-major:

      seq_csr   int64 [n_seq + 1, 3]  sequence i's first record (row of gc), first linear chain (row of lc), first anchor (row of a);
                                      the last row holds the totals
      seq_info  int32 [n_seq, 2]      has_result (1 where map_cuda_reads(gaf=False) gives a non-NULL result), rep_len
      gc        int32 [n_rec, len(GC_COLUMNS)]  one row per graph chain (hash as its bits; off counts from the read's first lc row)
      gc_div    float32 [n_rec]       mg_gchain_t.div
      cigar_csr int64 [n_rec + 1]     record k's CIGAR operations are cigar[cigar_csr[k]:cigar_csr[k+1]]
      lc        int32 [n_lc, 5]       mg_llchain_t: off (from the read's first anchor row), cnt, v, score, ed
      a         int64 [n_a, 2]        mg128_t x, y (as their bits)
      cigar     int64 [n_cigar]       len<<4 | op

    With ds=True (map_cuda_reads_to_tensors), the ds:Z strings too (without them, map_cuda_reads gives them):

      ds_csr    int64 [n_rec + 1, 2]  record k's ds is ds[ds_csr[k,0]:ds_csr[k+1,0]] and its offsets ds_off[ds_csr[k,1]:ds_csr[k+1,1]]
      ds        uint8 [n_ds]          mg_ds_t.ds of every record, one after another, no terminating 0 (empty without a CIGAR)
      ds_off    int32 [n_ds_off]      mg_ds_t.off of every record"""

    def __init__(self, block, rec, rec_ds=None):
        import torch
        shapes = {"seq_csr": (torch.int64, (rec.n_seq + 1, 3)), "seq_info": (torch.int32, (rec.n_seq, 2)),
                  "gc": (torch.int32, (rec.n_rec, len(GC_COLUMNS))), "gc_div": (torch.float32, (rec.n_rec,)),
                  "cigar_csr": (torch.int64, (rec.n_rec + 1,)), "lc": (torch.int32, (rec.n_lc, 5)), "a": (torch.int64, (rec.n_a, 2)),
                  "cigar": (torch.int64, (rec.n_cigar,))}
        tables = [(name, rec.off[t]) for t, name in enumerate(capi.REC_TABLES)]
        if rec_ds is not None:
            shapes.update({"ds_csr": (torch.int64, (rec.n_rec + 1, 2)), "ds": (torch.uint8, (rec_ds.n_ds,)),
                           "ds_off": (torch.int32, (rec_ds.n_ds_off,))})
            tables += [(name, rec_ds.off[t]) for t, name in enumerate(capi.REC_DS_TABLES)]
        self.block = block
        for name, o in tables:
            dtype, shape = shapes[name]
            n = 1
            for x in shape:
                n *= x
            size = n * torch.empty((), dtype=dtype).element_size()
            setattr(self, name, block[o:o + size].view(dtype).view(shape))


def map_cuda_reads_to_tensors(lib, gi, seq, off, names=None, opt=None, n_seg=None, ds=False):
    """map_cuda_reads() with the results as tables written on the device into one block that torch allocates on seq's device
    (mgb_map_batch_dev_rec): returns a MappedTables.  The same arguments, checks and refusals as map_cuda_reads().  ds=True: the
    tables also hold every record's ds:Z string and its offsets (mgb_map_batch_dev_rec_ds), in the same block."""
    import torch
    who = "mgb_map_batch_dev_rec_ds" if ds else "mgb_map_batch_dev_rec"
    n_seq, args = _batch_args("map_cuda_reads_to_tensors", gi, seq, off, names, opt, n_seg)
    got, failed = [], []

    def alloc(ctx, nbytes):
        try:
            got.append(torch.empty(nbytes, dtype=torch.uint8, device=seq.device))
            return got[-1].data_ptr()
        except BaseException as e:  # a NULL block fails the call with a reason; the exception is raised from it below
            failed.append(e)
            return None

    cb = capi.mgb_dev_alloc_fn(alloc)  # referenced until the call returns
    rec = capi.mgb_records_t()
    rec_ds = capi.mgb_records_ds_t() if ds else None
    if ds:
        rc = lib.mgb_map_batch_dev_rec_ds(*args, cb, None, C.byref(rec), C.byref(rec_ds))
    else:
        rc = lib.mgb_map_batch_dev_rec(*args, cb, None, C.byref(rec))
    if rc < 0:
        raise RuntimeError("%s: %s" % (who, lib.mgb_last_error().decode())) from (failed[0] if failed else None)
    return MappedTables(got[0], rec, rec_ds)
