#!/usr/bin/env python
"""Throughput of `bus --devices` (kb_bus_group_*) against one bus run.

Workload: the benchmark's synthetic transcriptome and reference-built k=31 index (bench.workload, --genes genes, cached
as bench.py caches it), and --sets simulated 10x v3 read sets (R1 = 16-nt barcode from 6000 cells + 12-nt UMI, R2 = 91
nt of a transcript on either strand, 0.5 % substitutions, 5 % random sequence; tools/bus_batch_bench.simulate).

  * library arm: the read sets in pinned host batches of --batch sets, fed through one kb_bus_batch handle, through a
    group of two members on device 0 ("0,0") and through a group over every distinct visible GPU; read sets / s from
    host clocks around the whole synchronised run (best of --repeats), with the member count and device list.
  * CLI arm: wall clock of `bus -x 10xv3 -t THREADS` with `--device 0` against `--devices 0,0` on the same FASTQ files
    (best of --repeats, the two alternating).

Prints one JSON line with the GPU's name and power limit.  Inputs and outputs live in a temporary directory.

    python tools/bus_devices_bench.py --genes 2000 --sets 2000000 --batch 262144 --threads 16
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import benchdata  # noqa: E402
from bus_batch_bench import CLI, gpu_info, simulate, timed, write_fastq  # noqa: E402


class Tx:
    def __init__(self, concat, lens):
        self.concat, self.lens = concat, lens
        self.starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)


def pinned_batches(r1, r2, size):
    """the read sets cut into batches, each file in page-locked memory (kb_host_alloc) -> [(ptrs, n, keep-alive)]"""
    import kallisto_b200 as K
    L = K.lib()
    out = []
    for a in range(0, len(r1), size):
        n = min(size, len(r1) - a)
        bufs = []
        for r in (r1, r2):
            blk = np.ascontiguousarray(r[a:a + n]).reshape(-1)
            p = L.kb_host_alloc(blk.nbytes + 16)
            C.memmove(p, blk.ctypes.data, blk.nbytes)
            off = np.arange(n + 1, dtype=np.uint32) * np.uint32(r.shape[1])
            q = L.kb_host_alloc(off.nbytes)
            C.memmove(q, off.ctypes.data, off.nbytes)
            bufs.append((p, q))
        out.append(((C.c_void_p * 2)(bufs[0][0], bufs[1][0]), (C.c_void_p * 2)(bufs[0][1], bufs[1][1]), n, bufs))
    return out


def free_batches(batches):
    import kallisto_b200 as K
    for _, _, _, bufs in batches:
        for p, q in bufs:
            K.lib().kb_host_free(p)
            K.lib().kb_host_free(q)


def run_plain(ix, batches, max_sets):
    import kallisto_b200 as K
    L = K.lib()
    bp = K.BUSProcessor(ix, "10xv3", max_batch_sets=max_sets)
    rec = np.zeros(max_sets, K.BUS_RECORD_DTYPE)
    nrec = C.c_uint32(0)
    t0 = time.perf_counter()
    for bb, oo, n, _ in batches:
        K._ck(L.kb_bus_batch(bp._h, bb, oo, n, K._p(rec), C.byref(nrec)))
    dt = time.perf_counter() - t0
    n_al = bp.finalize()["n_pseudoaligned"]
    bp.close()
    return dt, n_al


def run_group(ixs, batches, max_sets):
    """round-robin, one batch per member in flight, completed in submission order"""
    import kallisto_b200 as K
    L = K.lib()
    members = [K.BUSProcessor(x, "10xv3", max_batch_sets=max_sets) for x in ixs]
    g = K.BUSGroup(members)
    rec = np.zeros(max_sets, K.BUS_RECORD_DTYPE)
    nrec = C.c_uint32(0)
    pending, busy = [], [False] * len(members)
    t0 = time.perf_counter()
    for i, (bb, oo, n, _) in enumerate(batches):
        m = i % len(members)
        while busy[m]:
            t, mm = pending.pop(0)
            K._ck(L.kb_bus_group_complete(g._h, t, K._p(rec), C.byref(nrec)))
            busy[mm] = False
        t = C.c_uint64(0)
        K._ck(L.kb_bus_group_submit(g._h, m, bb, oo, n, C.byref(t)))
        pending.append((t.value, m))
        busy[m] = True
    while pending:
        K._ck(L.kb_bus_group_complete(g._h, pending.pop(0)[0], K._p(rec), C.byref(nrec)))
    dt = time.perf_counter() - t0
    n_al = g.finalize()["n_pseudoaligned"]
    g.close()
    for m in members:
        m.close()
    return dt, n_al


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--sets", type=int, default=2000000)
    ap.add_argument("--batch", type=int, default=1 << 18, help="read sets per batch of the library arm")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-cli", action="store_true")
    a = ap.parse_args()
    import torch
    import kallisto_b200 as K
    idx, concat, lens = bench.workload(a.genes)
    r1, r2 = simulate(Tx(concat, lens), a.sets, 7)
    n_gpus = torch.cuda.device_count()
    out = dict(metric="bus_devices", gpu=gpu_info(), n_gpus_visible=n_gpus, genes=a.genes, sets=a.sets, batch=a.batch)
    batches = pinned_batches(r1, r2, a.batch)
    arms = [("one_handle", [0]), ("group_0_0", [0, 0])]
    if n_gpus > 1:
        arms.append(("group_all_gpus", list(range(n_gpus))))
    lib_out = {}
    for name, devs in arms:
        ixs = [K.KmerIndex(idx, device=d, threads=8) for d in devs]
        runs, n_al = [], None
        for _ in range(a.repeats + 1):                       # the first run warms up (allocations, L2 window)
            dt, n_al = run_plain(ixs[0], batches, a.batch) if name == "one_handle" else run_group(ixs, batches, a.batch)
            runs.append(dt)
        runs = runs[1:]
        lib_out[name] = dict(members=len(devs), devices=devs, sets_per_s=round(a.sets / min(runs)),
                             runs_sets_per_s=[round(a.sets / t) for t in runs], n_pseudoaligned=n_al)
        for x in ixs:
            x.close()
    free_batches(batches)
    out["library"] = lib_out
    if not a.no_cli:
        with tempfile.TemporaryDirectory() as td:
            f1, f2 = os.path.join(td, "r_1.fq"), os.path.join(td, "r_2.fq")
            write_fastq(f1, r1, b"s")
            write_fastq(f2, r2, b"s")
            base = [CLI, "bus", "-x", "10xv3", "-t", str(a.threads), "-i", idx, "-o"]
            one, two = [], []
            for i in range(a.repeats):
                one.append(timed(base + [os.path.join(td, "a%d" % i), "--device", "0", f1, f2]))
                two.append(timed(base + [os.path.join(td, "b%d" % i), "--devices", "0,0", f1, f2]))
            same = all(open(os.path.join(td, "a0", f), "rb").read() == open(os.path.join(td, "b0", f), "rb").read()
                       for f in ("output.bus", "matrix.ec"))
            out["cli"] = dict(device_0_s=round(min(one), 3), devices_0_0_s=round(min(two), 3),
                              device_0_runs_s=[round(t, 3) for t in one], devices_0_0_runs_s=[round(t, 3) for t in two],
                              outputs_identical=same)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
