#!/usr/bin/env python
"""Generates tests/golden/quanttcc_bs.json.gz from the UNMODIFIED reference (oracle/_ref/kallisto, `make -C oracle`):
`kallisto quant-tcc` with bootstraps (-b, --seed) and --matrix-to-directories on the inputs of tests/golden/quanttcc
(matrix.ec; tcc.mtx, whose rows are all reads / first half / a sparse row / an empty row; tcc_single.txt; fld_*.txt),
which are read, not regenerated.

    python tests/golden/make_golden_quanttcc_bs.py

The fixture is one gzip-compressed JSON object: {"cases": {name: [arguments, TCC file]}, "outputs": {name: {relative
path: text}}} with every file of each run except run_info.json.  File names in the arguments are relative to quanttcc/.
"""
import gzip
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

G = os.path.join(ROOT, "tests", "golden")
SRC = os.path.join(G, "quanttcc")
OUT = os.path.join(G, "quanttcc_bs.json.gz")

CASES = {
    "single_b3": (["-b", "3"], "tcc_single.txt"),
    "single_b3_plaintext": (["-b", "3", "--plaintext"], "tcc_single.txt"),
    "single_ls_b4_seed7": (["-l", "200", "-s", "20", "-b", "4", "--seed", "7"], "tcc_single.txt"),
    "files_b3": (["-l", "180", "-s", "25", "--matrix-to-files", "--plaintext", "-b", "3", "-t", "2"], "tcc.mtx"),
    "dirs_fld_rows_b3": (["-f", "fld_rows.txt", "--matrix-to-directories", "--plaintext", "-b", "3"], "tcc.mtx"),
    "dirs": (["--matrix-to-directories"], "tcc.mtx"),
}


def main():
    O.build()
    assert O.have_ref(), "build the reference first: make -C oracle"
    idx = os.path.join(G, "synth_small", "transcripts.kidx")
    outputs = {}
    for name, (extra, tcc) in CASES.items():
        extra = [os.path.join(SRC, a) if a.endswith(".txt") else a for a in extra]
        with tempfile.TemporaryDirectory() as td:
            out = os.path.join(td, "o")
            O.ref_run(["quant-tcc", "-i", idx, "-e", os.path.join(SRC, "matrix.ec"), "-o", out] + extra + [os.path.join(SRC, tcc)])
            files = {}
            for d, _, fns in os.walk(out):
                for fn in fns:
                    if fn != "run_info.json":
                        p = os.path.join(d, fn)
                        files[os.path.relpath(p, out)] = open(p).read()
            outputs[name] = dict(sorted(files.items()))
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(json.dumps({"cases": CASES, "outputs": outputs}, sort_keys=True).encode())
    print("quanttcc_bs:", {k: len(v) for k, v in outputs.items()}, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
