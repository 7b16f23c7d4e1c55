#!/usr/bin/env python
"""Throughput of `kallisto_b200 quant-tcc -b B` on a bulk-like TCC matrix: R samples over the EC table of the stored
2 400-target index (tests/golden/abundant), each sample its own multinomial draw of --reads fragments from the fixture's
EC counts.  Runs the CLI with --matrix-to-files --plaintext and reports the wall clock and the (sample, bootstrap) EMs
per second, and the same bootstraps through the library with a callback that writes nothing (`library_seconds`: device
work and transfers, no text); with --reference (and oracle/_ref/kallisto built) the unmodified `kallisto quant-tcc` on
the same files.  With --genes, a transcript-to-gene map over the index's targets (genes of 1 to 7 consecutive
transcripts, every 10th transcript in none) is written too, and the library (main EMs and bootstraps, alternately
with and without the map, best of three each) and the CLI (alternately without and with `-g`, with and without
`-b`, best of three each) are also timed with gene-level output; `gene_kernels_ms` is the device time of the gene
kernels in one library call, from torch.profiler.  Inputs and
outputs live in a temporary directory.  Prints one JSON line.

    python tools/tcc_bootstrap_bench.py --samples 96 --bootstraps 100 --threads 16 [--reference] [--genes]
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
DATA = os.path.join(ROOT, "tests", "golden", "abundant")
CLI = os.path.join(ROOT, "kallisto_b200", "kallisto_b200")
REF = os.path.join(ROOT, "oracle", "_ref", "kallisto")


def write_inputs(td, R, reads, seed):
    g = np.load(os.path.join(DATA, "ecs_paired.npz"))
    off, tids, frag = g["ec_off"], g["ec_tids"], g["frag_ec"]
    n_ec = len(off) - 1
    with open(os.path.join(td, "matrix.ec"), "w") as f:
        for e in range(n_ec):
            f.write("%d\t%s\n" % (e, ",".join(str(int(x)) for x in tids[int(off[e]):int(off[e + 1])])))
    p = np.bincount(frag[frag >= 0], minlength=n_ec).astype(np.float64)
    p /= p.sum()
    rng = np.random.default_rng(seed)
    rows = [rng.multinomial(reads, p) for _ in range(R)]
    nnz = sum(int((r > 0).sum()) for r in rows)
    with open(os.path.join(td, "tcc.mtx"), "w") as f:
        f.write("%%%%MatrixMarket matrix coordinate real general\n%d\t%d\t%d\n" % (R, n_ec, nnz))
        for i, r in enumerate(rows):
            for e in np.flatnonzero(r):
                f.write("%d\t%d\t%d\n" % (i + 1, e + 1, r[e]))
    return off, tids, rows


def run(exe, td, out, B, threads, extra=()):
    args = [exe, "quant-tcc", "-i", os.path.join(DATA, "transcripts.kidx"), "-e", os.path.join(td, "matrix.ec"),
            "-o", os.path.join(td, out), "-l", "180", "-s", "20", "--matrix-to-files", "--plaintext", "-b", str(B),
            "-t", str(threads)] + list(extra) + [os.path.join(td, "tcc.mtx")]
    t0 = time.perf_counter()
    r = subprocess.run(args, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
    dt = time.perf_counter() - t0
    if r.returncode != 0:
        sys.exit("%s failed (exit %d): %s" % (exe, r.returncode, r.stderr[-800:]))
    return dt


def write_t2g(td, names, seed):
    """-> (gene of every target, n_genes); writes t2g.txt."""
    rng = np.random.default_rng(seed)
    gene_of = np.full(len(names), -1, np.int32)
    lines, t, G = [], 0, 0
    while t < len(names):
        for i in range(t, min(len(names), t + int(rng.integers(1, 8)))):
            if i % 10 != 9:
                gene_of[i] = G
                lines.append("%s\tG%05d\tname%d\n" % (names[i], G, G))
            t = i + 1
        G += 1
    with open(os.path.join(td, "t2g.txt"), "w") as f:
        f.writelines(lines)
    return gene_of, G


def gene_kernel_ms(fn):
    """Device time of the gene pass (tcc_gene_*_kernel) in one call of fn, from torch.profiler's CUDA activity trace."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return round(sum(e.device_time_total for e in prof.key_averages() if "tcc_gene" in e.key) / 1000.0, 3)


def library_seconds(off, tids, rows, B, res, td, genes):
    sys.path.insert(0, ROOT)
    import kallisto_b200 as K
    ix = K.KmerIndex(os.path.join(DATA, "transcripts.kidx"), device=0)
    eff, _, _ = K.eff_lens(ix, fld_mean=180.0, fld_sd=20.0)
    ids = [np.flatnonzero(r) for r in rows]
    ro = np.concatenate([[0], np.cumsum([len(i) for i in ids])]).astype(np.uint64)
    ec_ids = np.concatenate(ids).astype(np.uint32)
    vals = np.concatenate([r[i] for r, i in zip(rows, ids)]).astype(np.uint32)
    n = [0]

    def on_chunk(first, est, rounds, samples):
        n[0] += len(rounds)
    K.tcc_bootstrap(ix, off, tids, ro, ec_ids, vals, eff, 42, 1, on_chunk)      # warm-up
    t0 = time.perf_counter()
    K.tcc_bootstrap(ix, off, tids, ro, ec_ids, vals, eff, 42, B, on_chunk)
    res["library_seconds"] = round(time.perf_counter() - t0, 3)
    assert n[0] == len(rows) * (B + 1)
    T = ix.num_trans
    if genes:
        gmap = write_t2g(td, ix.target_names_, 2)
        res["n_genes"] = gmap[1]
        sets = [tuple(int(x) for x in tids[int(off[e]):int(off[e + 1])]) for e in range(len(off) - 1)]
        sparse = [[(int(e), int(r[e])) for e in i] for r, i in zip(rows, ids)]
        best = {}

        def timed(key, fn):
            t0 = time.perf_counter()
            fn()
            best[key] = min(best.get(key, 1e9), time.perf_counter() - t0)
        K.tcc_run(ix, sets, sparse, eff, genes=gmap)                                 # warm-up
        for _ in range(3):
            timed("run", lambda: K.tcc_run(ix, sets, sparse, eff))
            timed("run_genes", lambda: K.tcc_run(ix, sets, sparse, eff, genes=gmap))
            timed("bs", lambda: K.tcc_bootstrap(ix, off, tids, ro, ec_ids, vals, eff, 42, B, on_chunk))
            timed("bs_genes", lambda: K.tcc_bootstrap(ix, off, tids, ro, ec_ids, vals, eff, 42, B,
                                                      lambda *a: None, genes=gmap))
        res.update({"library_%s_seconds" % k: round(v, 4) for k, v in best.items()})
        res["gene_kernels_ms"] = {
            "run": gene_kernel_ms(lambda: K.tcc_run(ix, sets, sparse, eff, genes=gmap)),
            "bootstrap": gene_kernel_ms(lambda: K.tcc_bootstrap(ix, off, tids, ro, ec_ids, vals, eff, 42, B,
                                                                lambda *a: None, genes=gmap))}
    ix.close()
    return T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=96)
    ap.add_argument("--bootstraps", type=int, default=100)
    ap.add_argument("--reads", type=int, default=2_000_000, help="fragments per sample")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--reference", action="store_true", help="also time the reference (oracle/_ref/kallisto)")
    ap.add_argument("--genes", action="store_true", help="also time gene-level output (-g)")
    a = ap.parse_args()
    R, B = a.samples, a.bootstraps
    res = dict(tool="tcc_bootstrap_bench", samples=R, bootstraps=B, reads_per_sample=a.reads, threads=a.threads)
    with tempfile.TemporaryDirectory() as td:
        off, tids, rows = write_inputs(td, R, a.reads, 1)
        res["n_ecs"] = len(off) - 1
        res["n_targets"] = library_seconds(off, tids, rows, B, res, td, a.genes)
        run(CLI, td, "warm", 0, a.threads)                  # the same run without bootstraps: index load + main EMs
        t_main = run(CLI, td, "main", 0, a.threads)
        t = run(CLI, td, "kb", B, a.threads)
        res.update(seconds_without_bootstrap=round(t_main, 3), seconds=round(t, 3),
                   bootstrap_ems_per_s=round(R * B / max(1e-9, t - t_main), 1))
        if a.genes:
            # alternately without and with -g, best of three each
            g = ["-g", os.path.join(td, "t2g.txt")]
            best = {}
            for i in range(3):
                for key, b, extra in (("main", 0, []), ("main_g", 0, g), ("kb", B, []), ("kb_g", B, g)):
                    best[key] = min(best.get(key, 1e9), run(CLI, td, "%s%d" % (key, i), b, a.threads, extra))
            res.update(cli_best_of_3={k: round(v, 3) for k, v in best.items()})
        if a.reference and os.path.exists(REF):
            tr = run(REF, td, "ref", B, a.threads)
            res.update(reference_seconds=round(tr, 3), speedup=round(tr / t, 2))
            for fn in ("bs_abundance_1_0.tsv", "bs_abundance_%d_%d.tsv" % (R, B - 1), "matrix.abundance.mtx"):
                res.setdefault("identical_to_reference", True)
                if open(os.path.join(td, "kb", fn), "rb").read() != open(os.path.join(td, "ref", fn), "rb").read():
                    res["identical_to_reference"] = False
    print(json.dumps(res))


if __name__ == "__main__":
    main()
