#!/usr/bin/env python3
"""GAF text end to end, two ways, on the same reads in one process (steps of the two arms alternate):

  A  `--pipe` host threads call mg_map_batch() on successive mini-batches, a writer thread turns the mg_gchains_t objects into
     GAF text in input order with mgb_write_gaf_batch() -- bench.py's end-to-end arm;
  B  `--pipe` host threads call mgb_map_batch_gaf() on the same mini-batches: the text is formatted on the device.

    python tools/bench_gaf.py --workload c3 --steps 3 --warmup 1

Prints one JSON line: Gbp/s of each arm, host ms per call, bytes copied back per read, the GAF kernels' time (CUDA events: the
GAF kernels plus the copy of the text), whether the two texts are byte-identical (md5 of the last step), and the GPU's name,
power limit and SM clock read in the same run.  Needs a CUDA device; there is no fallback."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402
from minigraph_b200 import capi, options  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], check=True, stdout=subprocess.PIPE, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.strip().split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reads", type=int, default=0, help="reads (default: the workload's own number)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--pipe", type=int, default=3, help="host threads mapping at once")
    ap.add_argument("--mini-batch", type=int, default=400000000, help="bases per call")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_gaf.py: no CUDA device")
    before = gpu_info()
    lib = capi.load_product()
    n_pipe = max(1, a.pipe)
    lib.mgb_set_param(b"slots", n_pipe)
    ncores = os.cpu_count() or 1
    host_threads = max(2, min(32, ncores // (n_pipe + 1)))  # as bench.py sizes them for one GPU
    gaf_threads = max(2, min(48, ncores - n_pipe * host_threads // 2))
    lib.mgb_set_param(b"host_threads", host_threads)
    tmp = tempfile.mkdtemp(prefix="mgb_bench_gaf_")
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

    def sub(arr, ctype, lo):
        return C.cast(C.addressof(arr.contents) + lo * C.sizeof(ctype), C.POINTER(ctype))

    bufs = {arm: [(C.c_void_p(0), C.c_size_t(0), C.c_size_t(0)) for _ in mbs] for arm in "AB"}

    def run(arm, acc):
        """one pass over the reads; acc collects host ms per call, bytes copied back and the GAF kernels' time"""
        nxt, lock, errs, done = [0], threading.Lock(), [], {}
        cv = threading.Condition()

        def mapper():
            st = capi.mgb_stats_t()
            while True:
                with lock:
                    k = nxt[0]
                    nxt[0] += 1
                if k >= len(mbs) or errs:
                    return
                lo, hi = mbs[k]
                buf, ln, cap = bufs[arm][k]
                t0 = time.perf_counter()
                if arm == "A":
                    gcs = (C.POINTER(capi.mg_gchains_t) * (hi - lo))()
                    rc = lib.mg_map_batch(gi, hi - lo, sub(qlens, C.c_int, lo), sub(cseqs, C.c_char_p, lo), sub(cnames, C.c_char_p, lo), gcs, C.byref(mo))
                else:
                    gcs = None
                    rc = lib.mgb_map_batch_gaf(gi, hi - lo, None, sub(qlens, C.c_int, lo), sub(cseqs, C.c_char_p, lo), sub(cnames, C.c_char_p, lo),
                                               C.byref(mo), C.byref(buf), C.byref(ln), C.byref(cap))
                dt = (time.perf_counter() - t0) * 1e3
                if rc != 0:
                    errs.append(lib.mgb_last_error())
                    return
                lib.mgb_get_stats(gi, C.byref(st))
                with lock:
                    acc["call_ms"] += dt
                    acc["calls"] += 1
                    acc["out_bytes"] += st.out_bytes
                    acc["d2h_ms"] += st.t_d2h_ms
                with cv:
                    done[k] = gcs
                    cv.notify_all()

        def writer():  # arm A: text in input order, as bench.py's end-to-end arm writes it
            for k, (lo, hi) in enumerate(mbs):
                with cv:
                    while k not in done and not errs:
                        cv.wait(0.1)
                    if errs:
                        return
                    gcs = done.pop(k)
                buf, ln, cap = bufs[arm][k]
                lib.mgb_write_gaf_batch(g, hi - lo, gcs, sub(qlens, C.c_int, lo), sub(cnames, C.c_char_p, lo), mo.flag, gaf_threads,
                                        C.byref(buf), C.byref(ln), C.byref(cap))
                lib.mgb_free_batch(hi - lo, gcs)

        th = [threading.Thread(target=mapper) for _ in range(n_pipe)] + ([threading.Thread(target=writer)] if arm == "A" else [])
        t0 = time.perf_counter()
        for t in th:
            t.start()
        for t in th:
            t.join()
        torch.cuda.synchronize()
        assert not errs, errs
        return time.perf_counter() - t0

    zero = {"call_ms": 0.0, "calls": 0, "out_bytes": 0, "d2h_ms": 0.0}
    scratch = {"A": dict(zero), "B": dict(zero)}
    for _ in range(a.warmup):
        run("A", scratch["A"]), run("B", scratch["B"])
    acc, wall = {"A": dict(zero), "B": dict(zero)}, {"A": 0.0, "B": 0.0}
    for _ in range(a.steps):
        for arm in "AB":
            wall[arm] += run(arm, acc[arm])
    after = gpu_info()
    md5 = {}
    for arm in "AB":
        h = hashlib.md5()
        for buf, ln, _ in bufs[arm]:
            h.update(C.string_at(buf, ln.value))
        md5[arm] = h.hexdigest()

    def arm_out(arm):
        x = acc[arm]
        return {"gbps": bases * a.steps / wall[arm] / 1e9, "host_ms_per_call": x["call_ms"] / max(1, x["calls"]),
                "out_bytes_per_read": x["out_bytes"] / (n * a.steps), "d2h_ms_per_call": x["d2h_ms"] / max(1, x["calls"])}
    print(json.dumps({
        "workload": bench.workload_text(a.workload, n), "reads": n, "bases": bases, "steps": a.steps, "warmup": a.warmup, "pipe": n_pipe,
        "mini_batches": len(mbs), "host_threads": host_threads, "gaf_threads": gaf_threads, "host_cores": ncores,
        "A_map_batch_then_write_gaf_batch": arm_out("A"), "B_map_batch_gaf": arm_out("B"),
        "B_gaf_kernels_plus_copy_ms_per_call": arm_out("B")["d2h_ms_per_call"],
        "identical_text": md5["A"] == md5["B"], "md5": md5, "gpu_before": before, "gpu_after": after,
        "note": "arm A's out_bytes are the result blobs (GChain | LLChain | anchors | CIGAR words | ds); arm B's the GAF text; "
                "d2h_ms: CUDA events over the result packing (A) or the GAF kernels (B) plus the copy",
    }))
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)
    lib.mgb_reads_free(rd)


if __name__ == "__main__":
    main()
