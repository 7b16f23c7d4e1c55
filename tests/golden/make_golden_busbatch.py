#!/usr/bin/env python
"""Generates tests/golden/busbatch/ from the UNMODIFIED reference (oracle/_ref/kallisto, `make -C oracle`):
`kallisto bus --batch FILE` with a technology, with and without --batch-barcodes.

    python tests/golden/make_golden_busbatch.py

The inputs are cut from existing golden reads, a few hundred read sets per batch-file line:
  v3_{a,b,c}_{1,2}   bus10xv3's 10x v3 reads 0-399, 400-699, 700-999 (batch_v3.txt: three lines, a and c share an id)
  v2_{a,b}_{1,2}     bus10x's 10x v2 reads 0-499, 500-999
  ss3_{a,b}_{1..4}   the SMARTSEQ3 layout of buspaired (index reads with N and short ones, tag reads, second mates),
                     read sets 0-299 and 300-599
  aa_{a,b}_{1,2}     aa's 10x v3 reads 0-149, 150-299 (protein index)
Runs (each keeps output.bus, matrix.ec, run_info.json and, where written, flens.txt, matrix.cells and
matrix.sample.barcodes; manifest.json lists every file each run wrote, index.saved included):
  ref_v3          -x 10xv3 --batch batch_v3.txt
  ref_v3_bb       the same with --batch-barcodes
  ref_v2_bb_num   -x 10xv2 --batch-barcodes --num --unstranded --batch batch_v2.txt
  ref_ss3_paired_bb  -x smartseq3 --paired --batch --batch-barcodes (header barcode length 0, flens.txt per line)
  ref_ss3         -x smartseq3 --batch (no flens.txt)
  ref_nobc_bb     -x -1,-1,-1:0,16,28:1,0,0 --batch-barcodes (no barcode read: the sample number is the barcode)
  ref_bc32_bb     -x 0,0,16,1,0,16:0,16,28:1,0,0 --batch-barcodes (a two-piece barcode of exactly 32 letters)
  ref_aa_bb       --aa -x 10xv3 --batch --batch-barcodes
The reference runs inside tests/golden/busbatch under the name `kallisto` with -t 1 and relative file names, so the
call recorded in run_info.json holds no path of the machine that made it.  cli_errors.json holds the exit codes and
`Error:` lines of invocations the reference rejects, keyed as in cli_args.json (arguments after the program name,
run from tests/golden/busbatch).
"""
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests import util  # noqa: E402

G = os.path.join(ROOT, "tests", "golden")
OUT = os.path.join(G, "busbatch")
SS = os.path.join("..", "synth_small", "transcripts.kidx")
C1 = os.path.join("..", "config1", "transcripts.kidx")
AA = os.path.join("..", "aa", "proteins.kidx")

RUNS = {
    "ref_v3": (SS, ["-x", "10xv3", "--batch", "batch_v3.txt"]),
    "ref_v3_bb": (SS, ["-x", "10xv3", "--batch-barcodes", "--batch", "batch_v3.txt"]),
    "ref_v2_bb_num": (C1, ["-x", "10xv2", "--batch-barcodes", "--num", "--unstranded", "--batch", "batch_v2.txt"]),
    "ref_ss3_paired_bb": (SS, ["-x", "smartseq3", "--paired", "--batch-barcodes", "--batch", "batch_ss3.txt"]),
    "ref_ss3": (SS, ["-x", "smartseq3", "--batch", "batch_ss3.txt"]),
    "ref_nobc_bb": (SS, ["-x", "-1,-1,-1:0,16,28:1,0,0", "--batch-barcodes", "--batch", "batch_v3.txt"]),
    "ref_bc32_bb": (SS, ["-x", "0,0,16,1,0,16:0,16,28:1,0,0", "--batch-barcodes", "--batch", "batch_v3.txt"]),
    "ref_aa_bb": (AA, ["--aa", "-x", "10xv3", "--batch-barcodes", "--batch", "batch_aa.txt"]),
}
KEEP = ("output.bus", "matrix.ec", "run_info.json", "flens.txt", "matrix.cells", "matrix.sample.barcodes")
# rejected before any work; run from tests/golden/busbatch
ERRORS = [
    ["bus", "-i", SS, "-o", "o", "-x", "10xv3", "--batch", "batch_v3.txt", "v3_a_1.fastq.gz", "v3_a_2.fastq.gz"],
    ["bus", "-i", SS, "-o", "o", "-x", "10xv3", "--batch", "batch_malformed.txt"],
    ["bus", "-i", SS, "-o", "o", "-x", "10xv3", "--batch", "batch_missing.txt"],
    ["bus", "-i", SS, "-o", "o", "-x", "10xv3", "--batch-barcodes", "--batch", "nope.txt"],
]


def write_fastq(path, seqs):
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        for i, s in enumerate(seqs):
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)))


def cut(prefix, files, ranges):
    """files: one list of sequences per file of the technology; writes prefix_{a,b,..}_{1..} -> batch-file lines"""
    lines = []
    for j, (lo, hi) in enumerate(ranges):
        names = []
        for f, seqs in enumerate(files):
            name = "%s_%s_%d.fastq.gz" % (prefix, "abc"[j], f + 1)
            write_fastq(os.path.join(OUT, name), seqs[lo:hi])
            names.append(name)
        lines.append(names)
    return lines


def write_batch(name, ids, lines, comment=True):
    with open(os.path.join(OUT, name), "w") as f:
        if comment:
            f.write("# id files\n")
        for i, names in zip(ids, lines):
            f.write(" ".join([i] + names) + "\n")


def main():
    if not O.have_ref():
        sys.exit("needs oracle/_ref/kallisto (make -C oracle)")
    if os.path.isdir(OUT):
        shutil.rmtree(OUT)
    os.makedirs(OUT)
    v3 = [O.read_fastq(os.path.join(G, "bus10xv3", "sc_reads_%d.fastq.gz" % k)) for k in (1, 2)]
    write_batch("batch_v3.txt", ["s1", "s2", "s1"], cut("v3", v3, [(0, 400), (400, 700), (700, 1000)]))
    v2 = [O.read_fastq(os.path.join(G, "bus10x", "sc_reads_%d.fastq.gz" % k)) for k in (1, 2)]
    write_batch("batch_v2.txt", ["lib1", "lib2"], cut("v2", v2, [(0, 500), (500, 1000)]), comment=False)
    with tempfile.TemporaryDirectory() as tin:
        inp = util.buspaired_inputs(tin)
        ss3 = [O.read_fastq(inp[k]) for k in ("i_1", "i_2", "t_1", "s_2")]
    write_batch("batch_ss3.txt", ["plateA", "plateB"], cut("ss3", ss3, [(0, 300), (300, 600)]))
    aa = [O.read_fastq(os.path.join(G, "aa", "sc_%d.fastq.gz" % k)) for k in (1, 2)]
    write_batch("batch_aa.txt", ["x", "y"], cut("aa", aa, [(0, 150), (150, 300)]))
    with open(os.path.join(OUT, "batch_malformed.txt"), "w") as f:
        f.write("s1 v3_a_1.fastq.gz v3_a_2.fastq.gz\ns2 v3_b_1.fastq.gz\n")
    with open(os.path.join(OUT, "batch_missing.txt"), "w") as f:
        f.write("s1 v3_a_1.fastq.gz v3_a_2.fastq.gz\ns2 v3_b_1.fastq.gz missing_2.fastq.gz\n")
    manifest = {}
    for name, (idx, args) in RUNS.items():
        call = ["bus", "-t", "1", "-i", idx, "-o", name] + args
        r = subprocess.run(["kallisto"] + call, executable=O.REF_BIN, cwd=OUT, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE)
        if r.returncode != 0:
            sys.exit("%s failed (exit %d): %s" % (name, r.returncode, r.stderr.decode(errors="replace")[-600:]))
        d = os.path.join(OUT, name)
        manifest[name] = dict(args=call, files=sorted(os.listdir(d)))
        for f in os.listdir(d):
            if f not in KEEP:
                os.remove(os.path.join(d, f))
        info = json.load(open(os.path.join(d, "run_info.json")))
        print(name, manifest[name]["files"], "processed", info["n_processed"], "pseudoaligned", info["n_pseudoaligned"])
    with open(os.path.join(OUT, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=1, sort_keys=True)
        f.write("\n")
    errors = {}
    for args in ERRORS:
        r = subprocess.run(["kallisto"] + args, executable=O.REF_BIN, cwd=OUT, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
        assert r.returncode != 0, args
        shutil.rmtree(os.path.join(OUT, "o"), ignore_errors=True)      # the reference makes -o before it checks
        errors[" ".join(args)] = [r.returncode, [l.strip() for l in r.stderr.splitlines() if l.startswith("Error")]]
    with open(os.path.join(OUT, "cli_errors.json"), "w") as f:
        json.dump(errors, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
