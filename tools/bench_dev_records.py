#!/usr/bin/env python3
"""The same reads, already in GPU memory, mapped four ways in one process, steps of the four arms alternating, one call at a time:

  gcs   mgb_map_batch_dev(): one host mg_gchains_t per read, assembled by the host threads from a download of every result blob;
  gaf   mgb_map_batch_dev_gaf(): GAF text formatted on the device and copied back;
  rec   mgb_map_batch_dev_rec(): dense tables written on the device into one block torch allocates there (as map_cuda_reads_to_tensors);
        only the div requests come back (16 bytes per record) and the values go up (4);
  rds   mgb_map_batch_dev_rec_ds(): the same tables and the ds:Z strings in the same block (map_cuda_reads_to_tensors(ds=True)); the
        two totals of the ds tables come back too.

    python tools/bench_dev_records.py --workload c3 --steps 3 --warmup 1

Prints one JSON line: per call of each arm the mean wall time (host clock around the call, which returns with its results in place),
w_download_ms, t_d2h_ms, t_asm_ms and out_bytes, and for the table arms the block's bytes and ds bytes per read; whether the tables
(and the ds tables) and the mg_gchains_t results of the same reads agree on every call (field by field on a sample of --check reads
per call, the CSR row counts on all of them); and the GPU's name, power limit and SM clock read in the same run.  Needs a CUDA device; there is no fallback."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
sys.path.insert(0, os.path.join(REPO, "tests"))
import bench  # noqa: E402
from bench_gaf import gpu_info  # noqa: E402
from minigraph_b200 import capi, options  # noqa: E402
from minigraph_b200.tensors import MappedTables  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reads", type=int, default=0, help="reads (default: the workload's own number)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--mini-batch", type=int, default=400000000, help="bases per call")
    ap.add_argument("--check", type=int, default=200, help="reads per call compared field by field (spread over the call)")
    a = ap.parse_args()
    import numpy as np
    import torch
    import mgtest as T
    import recdscases as RD
    import reccases as RC
    if not torch.cuda.is_available():
        sys.exit("bench_dev_records.py: no CUDA device")
    before = gpu_info()
    lib = capi.load_product()
    tmp = tempfile.mkdtemp(prefix="mgb_bench_rec_")
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

    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum(np.ctypeslib.as_array(qlens, shape=(n,)), dtype=np.int64)
    blob = np.empty(max(1, int(off[n])), dtype=np.uint8)
    for i in range(n):
        C.memmove(blob.ctypes.data + int(off[i]), cseqs[i], qlens[i])
    d_seq, d_off = torch.from_numpy(blob).cuda(), torch.from_numpy(off).cuda()
    torch.cuda.synchronize()

    def sub(arr, ctype, lo):
        return C.cast(C.addressof(arr.contents) + lo * C.sizeof(ctype), C.POINTER(ctype))

    keys = ("wall_ms", "w_download_ms", "t_d2h_ms", "t_asm_ms", "out_bytes", "block_bytes", "n_ds_per_read")
    arms = ("gcs", "gaf", "rec", "rds")
    last = {}  # call -> what the gcs arm gave (rows of every read, a sample of whole results) and the rec arm's tables

    def run(arm, acc):
        st = capi.mgb_stats_t()
        stream = torch.cuda.current_stream().cuda_stream
        for k, (lo, hi) in enumerate(mbs):
            m = hi - lo
            names = sub(cnames, C.c_char_p, lo)
            t0 = time.perf_counter()
            if arm == "gcs":
                gcs = (C.POINTER(capi.mg_gchains_t) * m)()
                rc = lib.mgb_map_batch_dev(gi, m, None, m, d_seq.data_ptr(), d_seq.numel(), d_off[lo:].data_ptr(), names, C.byref(mo), stream, gcs)
            elif arm == "gaf":
                buf, ln = C.c_void_p(0), C.c_size_t(0)
                rc = lib.mgb_map_batch_dev_gaf(gi, m, None, m, d_seq.data_ptr(), d_seq.numel(), d_off[lo:].data_ptr(), names, C.byref(mo), stream,
                                               C.byref(buf), C.byref(ln), None)
            elif arm == "rec":
                rec, rec_ds = capi.mgb_records_t(), None
                rc = lib.mgb_map_batch_dev_rec(gi, m, None, m, d_seq.data_ptr(), d_seq.numel(), d_off[lo:].data_ptr(), names, C.byref(mo), stream,
                                               alloc_cb, None, C.byref(rec))
            else:
                rec, rec_ds = capi.mgb_records_t(), capi.mgb_records_ds_t()
                rc = lib.mgb_map_batch_dev_rec_ds(gi, m, None, m, d_seq.data_ptr(), d_seq.numel(), d_off[lo:].data_ptr(), names, C.byref(mo),
                                                  stream, alloc_cb, None, C.byref(rec), C.byref(rec_ds))
            dt = (time.perf_counter() - t0) * 1e3
            assert rc == 0, lib.mgb_last_error()
            lib.mgb_get_stats(gi, C.byref(st))
            block_bytes = rec.bytes if arm in ("rec", "rds") else 0
            n_ds = rec_ds.n_ds / m if arm == "rds" else 0
            for key, v in zip(keys, (dt, st.w_download_ms, st.t_d2h_ms, st.t_asm_ms, st.out_bytes, block_bytes, n_ds)):
                acc[key] += v
            acc["calls"] += 1
            if arm == "gcs":
                rows = [None if not gcs[i] else (gcs[i].contents.n_gc, gcs[i].contents.n_lc, gcs[i].contents.n_a) for i in range(m)]
                sample = list(range(0, m, max(1, m // max(1, a.check))))
                last.setdefault(k, {})["gcs"] = (rows, sample, [T.gchains_to_py(gcs[i]) for i in sample])
                lib.mgb_free_batch(m, gcs)
            elif arm == "gaf":
                C.CDLL(None).free(buf)
            else:
                last.setdefault(k, {})[arm] = MappedTables(blocks.pop(), rec, rec_ds)

    # the rec arm's blocks, allocated by torch on the reads' device as map_cuda_reads_to_tensors() does
    blocks = []

    def alloc(ctx, nbytes):
        blocks.append(torch.empty(nbytes, dtype=torch.uint8, device=d_seq.device))
        return blocks[-1].data_ptr()
    alloc_cb = capi.mgb_dev_alloc_fn(alloc)

    def zero():
        return dict({k: 0.0 for k in keys}, calls=0)

    agree, agree_ds, checked = True, True, 0

    def compare():
        nonlocal agree, agree_ds, checked
        for k, got in sorted(last.items()):
            rows, sample, want = got["gcs"]
            for arm in ("rec", "rds"):
                t = {name: getattr(got[arm], name).cpu().numpy() for name in capi.REC_TABLES}
                csr, info = t["seq_csr"], t["seq_info"]
                for i, r in enumerate(rows):  # every read: a result or none, and its rows
                    if bool(info[i, 0]) != (r is not None) or (r is not None and (csr[i + 1] - csr[i]).tolist() != ([r[0], r[1], r[2]] if r[0] > 0 else [0, 0, 0])):
                        agree = False
                for w, g in zip(want, RC.records_to_py(t, sample)):
                    if T.diff_results(RC.comparable(w), RC.comparable(g)) is not None:
                        agree = False
            t = {name: getattr(got["rds"], name).cpu().numpy() for name in capi.REC_TABLES}
            ds = {name: getattr(got["rds"], name).cpu().numpy() for name in capi.REC_DS_TABLES}
            try:  # the sampled reads' ds against their mg_ds_t (the other reads' results as None: not compared)
                full = [None] * len(rows)
                for i, w in zip(sample, want):
                    full[i] = w
                RD.check_ds(full, t, ds)
            except AssertionError:
                agree_ds = False
            checked += len(sample)
        last.clear()

    for _ in range(a.warmup):
        for arm in arms:
            run(arm, zero())
        compare()
    acc = {arm: zero() for arm in arms}
    for _ in range(a.steps):
        for arm in arms:
            run(arm, acc[arm])
        compare()
    after = gpu_info()
    per_call = {arm: {k: acc[arm][k] / max(1, acc[arm]["calls"]) for k in keys} for arm in arms}
    print(json.dumps({
        "workload": bench.workload_text(a.workload, n), "reads": n, "bases": bases, "steps": a.steps, "warmup": a.warmup,
        "calls_per_step": len(mbs), "host_cores": os.cpu_count(),
        "gcs_mgb_map_batch_dev": per_call["gcs"], "gaf_mgb_map_batch_dev_gaf": per_call["gaf"], "rec_mgb_map_batch_dev_rec": per_call["rec"],
        "rds_mgb_map_batch_dev_rec_ds": per_call["rds"], "tables_agree_with_gchains": agree, "ds_tables_agree_with_gchains": agree_ds,
        "reads_compared_field_by_field": checked, "gpu_before": before, "gpu_after": after,
    }))
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
    lib.mgb_reads_free(rd)


if __name__ == "__main__":
    main()
