#!/usr/bin/env python
"""Throughput of `kallisto_b200 bus --batch FILE --batch-barcodes` against one sample over the same files.

A nucleotide index is built with the unmodified reference (`oracle/_ref/kallisto index`) from the benchmark's synthetic
transcriptome (benchdata.make_transcriptome, --genes genes).  --samples samples of --sets 10x v3 read sets each are
simulated: R1 = 16-nt barcode from 6000 cells + 12-nt UMI, R2 = 91 nt of a transcript on either strand, 0.5 %
substitutions, 5 % random sequence.  Reports
  * batch_sets_per_s    `bus -x 10xv3 --batch FILE --batch-barcodes -t THREADS`, one line per sample, FASTQ to output.bus
  * single_sets_per_s   `bus -x 10xv3 -t THREADS` over the same files as one sample
    (each the best of --repeats runs, the two alternating; every run's rate is listed too)
  * bus_fields_ms       device time of bus_fields_kernel over the sets through the library with batch barcodes on,
                        from torch.profiler, and the same with them off
with the GPU's name and power limit.  Inputs and outputs live in a temporary directory.  Prints one JSON line.

    python tools/bus_batch_bench.py --genes 2000 --samples 8 --sets 250000 --threads 16
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


def timed(args):
    t0 = time.perf_counter()
    r = subprocess.run(args, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
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


def fields_ms(idx, samples, batch_barcodes):
    """bus_fields_kernel device time over every sample through the library, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import kallisto_b200 as K
    ix = K.KmerIndex(idx, device=0)

    def one():
        bp = K.BUSProcessor(ix, "10xv3", batch_barcodes=batch_barcodes)
        for j, (r1, r2) in enumerate(samples):
            bp.begin_sample(j)
            off = np.arange(len(r1) + 1, dtype=np.uint32)
            bp.process_sets([(r1.reshape(-1), off * r1.shape[1]), (r2.reshape(-1), off * r2.shape[1])])
        torch.cuda.synchronize()
        bp.close()

    one()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        one()
    ix.close()
    return round(sum(e.device_time_total for e in p.key_averages() if "bus_fields_kernel" in e.key) / 1000.0, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--sets", type=int, default=250000, help="read sets per sample")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not os.path.exists(REF):
        sys.exit("needs oracle/_ref/kallisto to build the index")
    tx = benchdata.make_transcriptome(a.genes, seed=44)
    n = a.samples * a.sets
    out = dict(metric="bus_batch", gpu=gpu_info(), genes=a.genes, samples=a.samples, sets=n, threads=a.threads)
    with tempfile.TemporaryDirectory() as td:
        fa, idx = os.path.join(td, "tx.fa"), os.path.join(td, "tx.kidx")
        with open(fa, "w") as f:
            for name, s in zip(tx.names, tx.seqs):
                f.write(">%s\n%s\n" % (name, s.tobytes().decode()))
        timed([REF, "index", "-i", idx, "-k", "31", "-t", str(a.threads), "-T", os.path.join(td, "tmp"), fa])
        samples, files = [], []
        with open(os.path.join(td, "batch.txt"), "w") as bf:
            for j in range(a.samples):
                r1, r2 = simulate(tx, a.sets, 100 + j)
                samples.append((r1, r2))
                f1, f2 = os.path.join(td, "s%d_1.fq" % j), os.path.join(td, "s%d_2.fq" % j)
                write_fastq(f1, r1, b"s")
                write_fastq(f2, r2, b"s")
                files += [f1, f2]
                bf.write("sample%d %s %s\n" % (j, f1, f2))
        base = [CLI, "bus", "-x", "10xv3", "-t", str(a.threads), "-i", idx, "-o"]
        batch_runs, single_runs = [], []
        for i in range(a.repeats):
            batch_runs.append(timed(base + [os.path.join(td, "b%d" % i), "--batch-barcodes", "--batch", os.path.join(td, "batch.txt")]))
            single_runs.append(timed(base + [os.path.join(td, "s%d" % i)] + files))
        out["batch_sets_per_s"] = round(n / min(batch_runs))
        out["single_sets_per_s"] = round(n / min(single_runs))
        out["batch_runs_sets_per_s"] = [round(n / t) for t in batch_runs]
        out["single_runs_sets_per_s"] = [round(n / t) for t in single_runs]
        for tag in ("b0", "s0"):
            info = json.load(open(os.path.join(td, tag, "run_info.json")))
            out[tag + "_n_pseudoaligned"] = info["n_pseudoaligned"]
        out["bus_fields_ms_batch_barcodes"] = fields_ms(idx, samples, True)
        out["bus_fields_ms_plain"] = fields_ms(idx, samples, False)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
