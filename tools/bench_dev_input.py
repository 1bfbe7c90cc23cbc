#!/usr/bin/env python3
"""The same reads mapped to GAF text two ways in one process, steps of the two arms alternating, one call at a time:

  host  mgb_map_batch_gaf(): host strings, packed to 2 bits per base by the host threads and copied up;
  dev   mgb_map_batch_dev_gaf(): the reads already in GPU memory as a CUDA tensor (uint8 bytes + int64 offsets), laid out there by
        k_ingest; only the offsets come back and the per-read tables go up.

    python tools/bench_dev_input.py --workload c3 --steps 3 --warmup 1

Prints one JSON line: per call of each arm the mean wall time, w_upload_ms (host wall clock of the upload step), t_h2d_ms (CUDA
events over the upload step; for the dev arm plus the host time of the offsets' copy), t_pack_ms and h2d_bytes; the md5 of each
arm's text over all calls of the last step (they must be equal); and the GPU's name, power limit and SM clock read in the same
run.  Needs a CUDA device; there is no fallback."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
import bench  # noqa: E402
from bench_gaf import gpu_info  # noqa: E402
from minigraph_b200 import capi, options  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reads", type=int, default=0, help="reads (default: the workload's own number)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--mini-batch", type=int, default=400000000, help="bases per call")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_dev_input.py: no CUDA device")
    before = gpu_info()
    lib = capi.load_product()
    tmp = tempfile.mkdtemp(prefix="mgb_bench_dev_")
    n_reads = a.reads or bench.WORKLOADS[a.workload][0]
    preset = bench.WORKLOADS[a.workload][2]
    gfa, fa = bench.make_workload(a.workload, tmp, 0, n_reads)
    rd = lib.mgb_reads_load(fa.encode(), 0)
    n, bases = int(rd.contents.n_reads), int(rd.contents.n_bases)
    qlens, cseqs, cnames = rd.contents.len, rd.contents.seq, rd.contents.name
    g = lib.mgb_gfa_read(gfa.encode())
    io, mo = options.opt_set(preset, cigar=True)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    mbs = bench.mini_batches(qlens[:n], a.mini_batch)

    # the reads on the device: every read's bytes one after the other, and n + 1 offsets
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum(np.ctypeslib.as_array(qlens, shape=(n,)), dtype=np.int64)
    blob = np.empty(max(1, int(off[n])), dtype=np.uint8)
    for i in range(n):
        C.memmove(blob.ctypes.data + int(off[i]), cseqs[i], qlens[i])
    d_seq, d_off = torch.from_numpy(blob).cuda(), torch.from_numpy(off).cuda()
    torch.cuda.synchronize()

    def sub(arr, ctype, lo):
        return C.cast(C.addressof(arr.contents) + lo * C.sizeof(ctype), C.POINTER(ctype))

    bufs = {arm: [(C.c_void_p(0), C.c_size_t(0), C.c_size_t(0)) for _ in mbs] for arm in ("host", "dev")}
    keys = ("wall_ms", "w_upload_ms", "t_h2d_ms", "t_pack_ms", "h2d_bytes")

    def run(arm, acc):
        st = capi.mgb_stats_t()
        stream = torch.cuda.current_stream().cuda_stream
        for k, (lo, hi) in enumerate(mbs):
            buf, ln, cap = bufs[arm][k]
            t0 = time.perf_counter()
            if arm == "host":
                rc = lib.mgb_map_batch_gaf(gi, hi - lo, None, sub(qlens, C.c_int, lo), sub(cseqs, C.c_char_p, lo), sub(cnames, C.c_char_p, lo),
                                           C.byref(mo), C.byref(buf), C.byref(ln), C.byref(cap))
            else:
                rc = lib.mgb_map_batch_dev_gaf(gi, hi - lo, None, hi - lo, d_seq.data_ptr(), d_seq.numel(), d_off[lo:].data_ptr(),
                                               sub(cnames, C.c_char_p, lo), C.byref(mo), stream, C.byref(buf), C.byref(ln), C.byref(cap))
            dt = (time.perf_counter() - t0) * 1e3
            assert rc == 0, lib.mgb_last_error()
            lib.mgb_get_stats(gi, C.byref(st))
            for key, v in zip(keys, (dt, st.w_upload_ms, st.t_h2d_ms, st.t_pack_ms, st.h2d_bytes)):
                acc[key] += v
            acc["calls"] += 1

    def zero():
        return dict({k: 0.0 for k in keys}, calls=0)

    for _ in range(a.warmup):
        run("host", zero()), run("dev", zero())
    acc = {"host": zero(), "dev": zero()}
    for _ in range(a.steps):
        for arm in ("host", "dev"):
            run(arm, acc[arm])
    after = gpu_info()
    md5 = {}
    for arm in ("host", "dev"):
        h = hashlib.md5()
        for buf, ln, _ in bufs[arm]:
            h.update(C.string_at(buf, ln.value))
        md5[arm] = h.hexdigest()
    per_call = {arm: {k: acc[arm][k] / max(1, acc[arm]["calls"]) for k in keys} for arm in acc}
    print(json.dumps({
        "workload": bench.workload_text(a.workload, n), "reads": n, "bases": bases, "steps": a.steps, "warmup": a.warmup,
        "calls_per_step": len(mbs), "host_cores": os.cpu_count(),
        "host_mgb_map_batch_gaf": per_call["host"], "dev_mgb_map_batch_dev_gaf": per_call["dev"],
        "identical_text": md5["host"] == md5["dev"], "md5": md5, "gpu_before": before, "gpu_after": after,
    }))
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
    lib.mgb_reads_free(rd)


if __name__ == "__main__":
    main()
