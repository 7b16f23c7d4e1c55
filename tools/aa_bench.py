#!/usr/bin/env python
"""Throughput of `kallisto_b200 bus --aa` (translated search: six comma-free frames per read set) on 10x v3 read sets.

The protein index is built with the unmodified reference (`oracle/_ref/kallisto index --aa`) from the benchmark's
synthetic transcriptome (benchdata.make_transcriptome, --genes genes), every transcript translated in frame 0 (a stop
codon becomes '*').  --sets read sets are simulated from the transcripts: R1 = 16-nt barcode from 6000 cells + 12-nt
UMI, R2 = 91 nt of a transcript on either strand, 0.5 % substitutions, 5 % random sequence.  Reports
  * cli_sets_per_s       `kallisto_b200 bus --aa -x 10xv3 -t THREADS`, FASTQ to output.bus, wall clock (best of 2)
  * library_sets_per_s   the same sets through kb_bus_batch in batches of --batch sets (host buffers in, records out)
  * kernel_ms            device time per kernel over the library run, from torch.profiler: cfc_len_kernel +
                         cfc_frames_kernel (the frames), pack / match / resolve over the 6 x sets frames, cfc_select_kernel
  * reference_sets_per_s `oracle/_ref/kallisto bus --aa -x 10xv3 -t THREADS` on the same files (--reference)
with the GPU's name and power limit.  Inputs and outputs live in a temporary directory.  Prints one JSON line.

    python tools/aa_bench.py --genes 2000 --sets 1000000 --threads 16 [--reference]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import benchdata  # noqa: E402

CLI = os.path.join(ROOT, "kallisto_b200", "kallisto_b200")
REF = os.path.join(ROOT, "oracle", "_ref", "kallisto")
CODE = {}
for _i, _a in enumerate("FFLLSSSSYY**CC*WLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG"):
    CODE["TCAG"[_i // 16] + "TCAG"[(_i // 4) % 4] + "TCAG"[_i % 4]] = _a


def write_proteins(tx, path):
    with open(path, "w") as f:
        for name, s in zip(tx.names, tx.seqs):
            t = s.tobytes().decode()
            f.write(">%s\n%s\n" % (name, "".join(CODE[t[i:i + 3]] for i in range(0, len(t) - 2, 3))))


def simulate(tx, n, seed, L=91):
    rng = np.random.default_rng(seed)
    lens = tx.lens
    t = rng.choice(len(lens), n, p=lens / lens.sum())
    start = tx.starts[t] + (rng.random(n) * np.maximum(lens[t] - L + 1, 1)).astype(np.int64)
    r2 = tx.concat[start[:, None] + np.arange(L)[None, :]]
    flip = rng.random(n) < 0.5
    r2[flip] = benchdata.COMP[r2[flip][:, ::-1]]
    err = rng.random(r2.shape) < 0.005
    r2[err] = benchdata.ACGT[rng.integers(0, 4, int(err.sum()))]
    rnd = rng.random(n) < 0.05
    r2[rnd] = benchdata.ACGT[rng.integers(0, 4, (int(rnd.sum()), L))]
    wl = benchdata.ACGT[np.random.default_rng(6000).integers(0, 4, (6000, 16))]
    r1 = np.concatenate([wl[rng.integers(0, 6000, n)], benchdata.ACGT[rng.integers(0, 4, (n, 12))]], axis=1)
    return np.ascontiguousarray(r1), np.ascontiguousarray(r2)


def write_fastq(path, reads, tag):
    n, L = reads.shape
    with open(path, "wb") as f:
        for c in range(0, n, 1 << 16):
            blk = reads[c:c + (1 << 16)]
            f.write(b"".join(b"@%s%d\n%s\n+\n%s\n" % (tag, c + i, r.tobytes(), b"I" * L) for i, r in enumerate(blk)))


def timed(args, cwd=None):
    t0 = time.perf_counter()
    r = subprocess.run(args, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True, cwd=cwd)
    dt = time.perf_counter() - t0
    if r.returncode != 0:
        sys.exit("%s failed (exit %d): %s" % (args[0], r.returncode, r.stderr[-800:]))
    return dt


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def library_run(idx, r1, r2, batch, profile):
    import torch
    import kallisto_b200 as K
    ix = K.KmerIndex(idx, device=0)
    n = len(r1)
    off = np.arange(n + 1, dtype=np.uint32)

    def one():
        bp = K.BUSProcessor(ix, "10xv3", aa=True, max_batch_sets=batch)
        nrec = 0
        for a in range(0, n, batch):
            b = min(n, a + batch)
            o1 = (off[:b - a + 1] * r1.shape[1]).astype(np.uint32)
            o2 = (off[:b - a + 1] * r2.shape[1]).astype(np.uint32)
            nrec += len(bp.process_sets([(r1[a:b].reshape(-1), o1), (r2[a:b].reshape(-1), o2)]))
        torch.cuda.synchronize()
        clashes = bp.frame_clashes()
        bp.close()
        return nrec, clashes

    one()                                          # warm-up: module load, allocations
    t0 = time.perf_counter()
    nrec, clashes = one()
    dt = time.perf_counter() - t0
    kernels = {}
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            one()
        for e in p.key_averages():
            for k in ("cfc_len_kernel", "cfc_frames_kernel", "pack_kernel", "match_kernel", "resolve_kernel", "cfc_select_kernel"):
                if k in e.key:
                    kernels[k] = kernels.get(k, 0.0) + e.device_time_total / 1000.0
    ix.close()
    return dict(library_seconds=round(dt, 3), library_sets_per_s=round(n / dt), records=nrec, frame_clashes=clashes,
                kernel_ms={k: round(v, 2) for k, v in kernels.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--sets", type=int, default=1000000)
    ap.add_argument("--batch", type=int, default=1 << 18)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--reference", action="store_true")
    a = ap.parse_args()
    if not os.path.exists(REF):
        sys.exit("needs oracle/_ref/kallisto to build the protein index")
    tx = benchdata.make_transcriptome(a.genes, seed=44)
    out = dict(metric="bus_aa", gpu=gpu_info(), genes=a.genes, transcripts=len(tx.seqs), sets=a.sets, threads=a.threads)
    with tempfile.TemporaryDirectory() as td:
        fa = os.path.join(td, "proteins.fa")
        idx = os.path.join(td, "proteins.kidx")
        write_proteins(tx, fa)
        t0 = time.perf_counter()
        timed([REF, "index", "--aa", "-i", idx, "-k", "31", "-t", str(a.threads), "-T", os.path.join(td, "tmp"), fa])
        out["index_seconds"] = round(time.perf_counter() - t0, 2)
        r1, r2 = simulate(tx, a.sets, a.seed)
        f1, f2 = os.path.join(td, "r1.fq"), os.path.join(td, "r2.fq")
        write_fastq(f1, r1, b"s")
        write_fastq(f2, r2, b"s")
        runs = [timed([CLI, "bus", "--aa", "-x", "10xv3", "-t", str(a.threads), "-i", idx, "-o", os.path.join(td, "o%d" % i),
                       f1, f2]) for i in range(2)]
        out["cli_seconds"] = round(min(runs), 3)
        out["cli_sets_per_s"] = round(a.sets / min(runs))
        info = json.load(open(os.path.join(td, "o0", "run_info.json")))
        for k in ("n_processed", "n_pseudoaligned", "n_unique", "n_frame_clashes"):
            out[k] = info[k]
        out.update(library_run(idx, r1, r2, a.batch, profile=True))
        if a.reference:
            dt = timed([REF, "bus", "--aa", "-x", "10xv3", "-t", str(a.threads), "-i", idx, "-o", os.path.join(td, "ref"), f1, f2])
            out["reference_seconds"] = round(dt, 3)
            out["reference_sets_per_s"] = round(a.sets / dt)
            rinfo = json.load(open(os.path.join(td, "ref", "run_info.json")))
            for k in ("n_processed", "n_pseudoaligned", "n_unique", "n_frame_clashes"):
                out["reference_" + k] = rinfo[k]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
