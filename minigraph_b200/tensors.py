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


def map_cuda_reads(lib, gi, seq, off, names=None, opt=None, n_seg=None, gaf=True):
    """Map the reads of (seq, off) with the index gi and the options opt (the mg_mapopt_t that mg_index() updated), ordered after
    the work queued on the current stream.  n_seg: segments per fragment (read pairs), or None for single-segment reads; names:
    one bytes object per fragment, or None.  Returns the GAF text (bytes) or, with gaf=False, a ctypes array of one
    mg_gchains_t pointer per sequence, owned by the caller (mgb_free_batch).  Raises RuntimeError with the library's reason when
    it refuses the batch (for instance tensors on another device than the index's)."""
    import torch
    if opt is None:
        raise TypeError("map_cuda_reads: opt is the mg_mapopt_t that mg_index() updated")
    if seq.dtype != torch.uint8 or off.dtype != torch.int64:
        raise TypeError("map_cuda_reads: seq must be torch.uint8 and off torch.int64, not %s and %s" % (seq.dtype, off.dtype))
    if not (seq.is_cuda and off.is_cuda and seq.device == off.device):
        raise ValueError("map_cuda_reads: seq and off must be CUDA tensors on one device (%s, %s)" % (seq.device, off.device))
    if not (seq.is_contiguous() and off.is_contiguous()) or seq.dim() != 1 or off.dim() != 1 or off.numel() < 1:
        raise ValueError("map_cuda_reads: seq and off must be contiguous 1-D tensors, off with n + 1 entries")
    n_seq = off.numel() - 1
    n_frag = len(n_seg) if n_seg is not None else n_seq
    cnseg = (C.c_int * max(1, n_frag))(*n_seg) if n_seg is not None else None
    cnames = (C.c_char_p * max(1, n_frag))(*names) if names is not None else None
    stream = torch.cuda.current_stream(seq.device).cuda_stream
    args = (gi, n_frag, cnseg, n_seq, seq.data_ptr(), seq.numel(), off.data_ptr(), cnames, C.byref(opt), stream)
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
