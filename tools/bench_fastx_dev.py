#!/usr/bin/env python3
"""The same FASTQ text mapped to GAF two ways in one process, one call at a time, the two arms alternating call by call:

  host  mgb_reads_load() on the call's FASTQ file, then mgb_map_batch_gaf() on the host strings;
  dev   the call's FASTQ text copied to the GPU in one H2D, parsed there by mgb_reads_parse_dev(), and the parsed reads mapped by
        mgb_map_batch_dev_gaf().

    python tools/bench_fastx_dev.py --workload c3 --reads 50000 --per-call 25000 --steps 2 --warmup 1

The workload's reads are written as 4-line FASTQ (qualities drawn to hold '@', '>' and '+' a third of the time), --per-call reads per
file.  Prints one JSON line: per call of each arm the mean wall time and, for the dev arm, the H2D time and the parse time (CUDA
events around each), the parse's bytes per second of text, and for the host arm the time of mgb_reads_load(); the md5 of each arm's
GAF text over all calls of the last step (they must be equal); and the GPU's name, power limit and SM clock read in the same run.
Needs a CUDA device; there is no fallback."""
import argparse
import ctypes as C
import hashlib
import json
import os
import random
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
import bench  # noqa: E402
from bench_gaf import gpu_info  # noqa: E402
from minigraph_b200 import capi, options  # noqa: E402

_QUAL = b"!\"#$%&'()*+,-./0123456789:;<=>?@ABCDEFGHIJ"


def fastq(names, seqs, rng):
    out = []
    for nm, s in zip(names, seqs):
        q = bytes(rng.choice(b"@>+") if rng.random() < 0.34 else rng.choice(_QUAL) for _ in range(256))
        out += [b"@", nm, b" rq:f:0.9\n", s, b"\n+\n", (q * (len(s) // 256 + 1))[:len(s)], b"\n"]
    return b"".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reads", type=int, default=50000)
    ap.add_argument("--per-call", type=int, default=25000, help="reads per call (per FASTQ file)")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_fastx_dev.py: no CUDA device")
    before = gpu_info()
    lib = capi.load_product()
    tmp = tempfile.mkdtemp(prefix="mgb_bench_fastx_")
    preset = bench.WORKLOADS[a.workload][2]
    gfa, fa = bench.make_workload(a.workload, tmp, 0, a.reads)
    rd = lib.mgb_reads_load(fa.encode(), 0)
    n = int(rd.contents.n_reads)
    names = [rd.contents.name[i] for i in range(n)]
    seqs = [C.string_at(rd.contents.seq[i], rd.contents.len[i]) for i in range(n)]
    lib.mgb_reads_free(rd)
    rng = random.Random(1)
    files, texts = [], []
    for k, lo in enumerate(range(0, n, a.per_call)):
        texts.append(fastq(names[lo:lo + a.per_call], seqs[lo:lo + a.per_call], rng))
        files.append(os.path.join(tmp, "call%d.fq" % k))
        with open(files[-1], "wb") as f:
            f.write(texts[-1])
    del names, seqs
    pinned = [torch.frombuffer(bytearray(t), dtype=torch.uint8).pin_memory() for t in texts]
    g = lib.mgb_gfa_read(gfa.encode())
    io, mo = options.opt_set(preset, cigar=True)
    gi = lib.mg_index(g, C.byref(io), 1, C.byref(mo))
    assert gi, lib.mgb_last_error()
    d_text = torch.empty(max(t.numel() for t in pinned), dtype=torch.uint8, device="cuda")
    blocks = []

    def alloc(_, nbytes):
        blocks.append(torch.empty(nbytes, dtype=torch.uint8, device="cuda"))
        return blocks[-1].data_ptr()

    cb = capi.mgb_dev_alloc_fn(alloc)
    bufs = {arm: [(C.c_void_p(0), C.c_size_t(0), C.c_size_t(0)) for _ in files] for arm in ("host", "dev")}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def call(arm, k, acc):
        buf, ln, cap = bufs[arm][k]
        stream = torch.cuda.current_stream()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "host":
            r = lib.mgb_reads_load(files[k].encode(), 0)
            t_load = (time.perf_counter() - t0) * 1e3
            c = r.contents
            rc = lib.mgb_map_batch_gaf(gi, c.n_reads, None, c.len, c.seq, c.name, C.byref(mo), C.byref(buf), C.byref(ln), C.byref(cap))
            lib.mgb_reads_free(r)
            acc["load_ms"] += t_load
        else:
            blocks.clear()
            nb = pinned[k].numel()
            ev[0].record(stream)
            d_text[:nb].copy_(pinned[k], non_blocking=True)
            ev[1].record(stream)
            dr = capi.mgb_dev_reads_t()
            rc = lib.mgb_reads_parse_dev(gi, d_text.data_ptr(), nb, 0, 1, stream.cuda_stream, cb, None, C.byref(dr))
            assert rc == 0, lib.mgb_last_error()
            ev[2].record(stream)
            blk = blocks[0]
            seq = blk[dr.off[0]:]
            off = blk[dr.off[1]:dr.off[1] + 8 * (dr.n_reads + 1)].view(torch.int64)
            name = bytes(blk[dr.off[2]:dr.off[2] + dr.name_bytes].cpu().numpy())
            noff = blk[dr.off[3]:dr.off[3] + 8 * (dr.n_reads + 1)].view(torch.int64).tolist()
            cn = (C.c_char_p * dr.n_reads)(*[name[noff[i]:noff[i + 1]] for i in range(dr.n_reads)])
            rc = lib.mgb_map_batch_dev_gaf(gi, dr.n_reads, None, dr.n_reads, seq.data_ptr(), dr.n_bases, off.data_ptr(), cn, C.byref(mo),
                                           stream.cuda_stream, C.byref(buf), C.byref(ln), C.byref(cap))
            ev[2].synchronize()
            acc["h2d_ms"] += ev[0].elapsed_time(ev[1])
            acc["parse_ms"] += ev[1].elapsed_time(ev[2])
            acc["text_bytes"] += nb
        assert rc == 0, lib.mgb_last_error()
        acc["wall_ms"] += (time.perf_counter() - t0) * 1e3
        acc["calls"] += 1

    def zero():
        return {"wall_ms": 0.0, "load_ms": 0.0, "h2d_ms": 0.0, "parse_ms": 0.0, "text_bytes": 0, "calls": 0}

    for _ in range(a.warmup):
        for k in range(len(files)):
            call("host", k, zero()), call("dev", k, zero())
    acc = {"host": zero(), "dev": zero()}
    for _ in range(a.steps):
        for k in range(len(files)):
            for arm in ("host", "dev"):
                call(arm, k, acc[arm])
    after = gpu_info()
    md5 = {}
    for arm in ("host", "dev"):
        h = hashlib.md5()
        for buf, ln, _ in bufs[arm]:
            h.update(C.string_at(buf, ln.value))
        md5[arm] = h.hexdigest()
    per = {arm: {k: v / max(1, acc[arm]["calls"]) for k, v in acc[arm].items() if k != "calls"} for arm in acc}
    d = per["dev"]
    d["parse_gb_per_s"] = d["text_bytes"] / (d["parse_ms"] * 1e6) if d["parse_ms"] else 0.0
    for arm in ("host", "dev"):
        per[arm] = {k: v for k, v in per[arm].items() if v or arm == "dev"}
    print(json.dumps({
        "workload": bench.workload_text(a.workload, n) + ", written as FASTQ", "reads": n, "reads_per_call": a.per_call,
        "steps": a.steps, "warmup": a.warmup, "calls_per_step": len(files), "host_cores": os.cpu_count(),
        "host_load_and_map_gaf": per["host"], "dev_h2d_parse_map_dev_gaf": per["dev"],
        "identical_text": md5["host"] == md5["dev"], "md5": md5, "gpu_before": before, "gpu_after": after,
    }))
    lib.mg_idx_destroy(gi)
    lib.mgb_gfa_destroy(g)


if __name__ == "__main__":
    main()
