#!/usr/bin/env python
"""Generates tests/golden/priors.json.gz from the UNMODIFIED reference (oracle/_ref/kallisto, `make -C oracle`):
`kallisto quant` and `kallisto quant-tcc` with -p/--priors (EMAlgorithm::read_priors / set_priors, src/EMAlgorithm.h:52-93)
on the reads of synth_small, manyecs and dlist and on the inputs of tests/golden/quanttcc, which are read, not
regenerated.  The priors files are written here from a fixed seed over the targets of each index.

    python tests/golden/make_golden_priors.py

The fixture is one gzip-compressed JSON object:
  {"inputs": {file name: text}, "quant": {name: [data set, arguments]}, "tcc": {name: [arguments, TCC file]},
   "outputs": {name: {relative path: text}}, "stderr": {name: [the priors lines of stderr]},
   "aborts": {name: {"priors": text, "exit": code}}}
Priors files are named <index>_<kind>.txt (kinds: prob, counts, half, short, long, odd, uniform, empty).  The reference
runs in a directory that holds them, with their plain names on the command line, so that messages carry no temporary
path.  quant reads and quanttcc/ files are given by absolute path.  Every output file except run_info.json is stored.
"aborts" records what the reference does with priors lines std::stod rejects (it dies on the uncaught exception).
"""
import gzip
import json
import os
import random
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

G = os.path.join(ROOT, "tests", "golden")
SRC = os.path.join(G, "quanttcc")
OUT = os.path.join(G, "priors.json.gz")
SETS = ("synth_small", "manyecs", "dlist")
KINDS = ("prob", "counts", "half", "short", "long", "odd", "uniform", "empty")

BASE = ["--plaintext", "-b", "2", "-t", "1"]
QUANT = {"q_%s" % k: ("synth_small", BASE + ["--priors", "synth_small_%s.txt" % k]) for k in KINDS if k != "counts"}
QUANT.update({
    "q_counts_p": ("synth_small", BASE + ["-p", "synth_small_counts.txt"]),
    "q_single_counts": ("synth_small", ["--plaintext", "-t", "1", "--single", "-l", "200", "-s", "20", "--priors",
                                        "synth_small_counts.txt"]),
    "q_fr_prob": ("synth_small", ["--plaintext", "-t", "1", "--fr-stranded", "--priors", "synth_small_prob.txt"]),
    "q_manyecs_prob": ("manyecs", BASE + ["--priors", "manyecs_prob.txt"]),
    "q_dlist_prob": ("dlist", BASE + ["--priors", "dlist_prob.txt"]),
    "q_dlist_long": ("dlist", BASE + ["--priors", "dlist_long.txt"]),
})
TCC = {
    "t_mtx_prob": (["--priors", "synth_small_prob.txt"], "tcc.mtx"),
    "t_files_ls_counts": (["--matrix-to-files", "-l", "180", "-s", "25", "--priors", "synth_small_counts.txt"], "tcc.mtx"),
    "t_dirs_b3_prob": (["--matrix-to-directories", "--plaintext", "-b", "3", "-f", "fld_rows.txt", "--priors",
                        "synth_small_prob.txt"], "tcc.mtx"),
    "t_single_b2_counts": (["-b", "2", "-p", "synth_small_counts.txt"], "tcc_single.txt"),
    "t_mtx_short": (["--priors", "synth_small_short.txt"], "tcc.mtx"),
    "t_mtx_g_prob": (["-g", "t2g.txt", "--priors", "synth_small_prob.txt"], "tcc.mtx"),
}
ABORTS = {"blank_line": "0.5\n\n0.5\n", "abc": "0.5\nabc\n", "huge": "1e999\n"}


def priors_files(name, T):
    rng = random.Random(1000 + T)
    raw = [0.0 if rng.random() < 0.2 else rng.random() for _ in range(T + 1)]
    tot = sum(raw[:T])
    prob = [x / tot for x in raw]
    cnt = [0 if rng.random() < 0.25 else rng.randrange(1, 2000) for _ in range(T)]
    odd = []
    for i in range(T):
        c = cnt[i]
        form = i % 6
        odd.append(["  %d" % c, "%d\r" % c, "%d reads" % c, "%.6e" % (c * 1e-3) if c else "1e-3", "%s" % float(c).hex(),
                    "\t%d" % c][form])
    lines = lambda v: "".join("%.17g\n" % x for x in v)
    return {
        "%s_prob.txt" % name: lines(prob[:T]),
        "%s_counts.txt" % name: "".join("%d\n" % c for c in cnt),
        "%s_half.txt" % name: lines([x * 0.5 for x in prob[:T]]),
        "%s_short.txt" % name: lines(prob[:T - 1]),
        "%s_long.txt" % name: lines(prob[:T + 1]),
        "%s_odd.txt" % name: "\r\n".join(odd[:-1]) + "\r\n" + odd[-1],     # CRLF endings, no final newline
        "%s_uniform.txt" % name: lines([1.0 / T] * T),
        "%s_empty.txt" % name: "",
    }


def inputs():
    files = {}
    for s in SETS:
        files.update(priors_files(s, O.OracleIndex(os.path.join(G, s, "transcripts.kidx")).n_targets))
    files["t2g.txt"] = json.loads(gzip.open(os.path.join(G, "quanttcc_genes.json.gz")).read())["inputs"]["t2g.txt"]
    return files


def quant_command(ds, out, args):
    d = os.path.join(G, ds)
    reads = [os.path.join(d, "reads_1.fastq.gz")]
    if "--single" not in args:
        reads.append(os.path.join(d, "reads_2.fastq.gz"))
    return ["quant", "-i", os.path.join(d, "transcripts.kidx"), "-o", out] + list(args) + reads


def tcc_command(out, args, tcc):
    args = [os.path.join(SRC, a) if a.startswith("fld_") else a for a in args]
    idx = os.path.join(G, "synth_small", "transcripts.kidx")
    return ["quant-tcc", "-i", idx, "-e", os.path.join(SRC, "matrix.ec"), "-o", out] + args + [os.path.join(SRC, tcc)]


def priors_lines(stderr):
    return [l for l in stderr.splitlines() if l.startswith("[   em] reading priors") or l.startswith("[   em] number of priors")
            or l.startswith("        defaulting")]


def collect(out):
    got = {}
    for d, _, fns in os.walk(out):
        for fn in fns:
            if fn != "run_info.json":
                p = os.path.join(d, fn)
                got[os.path.relpath(p, out)] = open(p).read()
    return dict(sorted(got.items()))


def main():
    O.build()
    assert O.have_ref(), "build the reference first: make -C oracle"
    files = inputs()
    outputs, stderr, aborts = {}, {}, {}
    with tempfile.TemporaryDirectory() as td:
        for fn, text in files.items():
            with open(os.path.join(td, fn), "w", newline="") as f:
                f.write(text)
        runs = [(n, quant_command(ds, os.path.join(td, "o"), a)) for n, (ds, a) in QUANT.items()]
        runs += [(n, tcc_command(os.path.join(td, "o"), a, t)) for n, (a, t) in TCC.items()]
        for name, cmd in runs:
            r = O.ref_run(cmd, cwd=td)
            outputs[name] = collect(os.path.join(td, "o"))
            stderr[name] = priors_lines(r.stderr.decode())
            shutil.rmtree(os.path.join(td, "o"))
        for name, text in ABORTS.items():
            with open(os.path.join(td, "bad.txt"), "w") as f:
                f.write(text)
            r = O.ref_run(tcc_command(os.path.join(td, "e"), ["--priors", "bad.txt"], "tcc.mtx"), cwd=td, check=False)
            aborts[name] = {"priors": text, "exit": r.returncode}
            assert r.returncode != 0, (name, r.stderr.decode())
            shutil.rmtree(os.path.join(td, "e"), ignore_errors=True)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(json.dumps({"inputs": files, "quant": QUANT, "tcc": TCC, "outputs": outputs, "stderr": stderr,
                            "aborts": aborts}, sort_keys=True).encode())
    print("priors:", {k: len(v) for k, v in outputs.items()}, aborts, os.path.getsize(OUT), "bytes")
    for k, v in stderr.items():
        print(k, v)


if __name__ == "__main__":
    main()
