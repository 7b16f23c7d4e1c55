#!/usr/bin/env python
"""Generates tests/golden/aa/ from the UNMODIFIED reference (oracle/_ref/kallisto, `make -C oracle`): a protein index
built with `kallisto index --aa`, and `kallisto bus --aa` runs over reads simulated from the nucleotide sequences the
proteins were translated from.

    python tests/golden/make_golden_aa.py

Everything is drawn from a fixed seed:
  * 16 nucleotide "transcripts" of stop-free codons.  Some share an in-frame segment (multi-protein equivalence
    classes), some carry the reverse complement of another's segment, in frame on both strands (a read over it
    translates to a protein in a forward AND a reverse frame: a frame clash), and some carry a stop codon.
  * proteins.fa: each transcript translated in frame 0 (a stop becomes '*'), plus X / B / J / Z letters and a lower
    case protein, and one protein that repeats another's sequence under a new name.
  * reads: substrings of the transcripts on both strands, lengths 30-101 (every length mod 3, k, k + 1, k + 2), with
    N, lower-case letters and foreign letters in some, and random reads that hit nothing.
Runs (each keeps output.bus, matrix.ec, transcripts.txt, run_info.json):
  ref_bulk_num      bus --aa -x bulk --num reads.fastq.gz
  ref_10xv3         bus --aa -x 10xv3 sc_1.fastq.gz sc_2.fastq.gz       (default --fr-stranded)
  ref_10xv3_rf      the same with --rf-stranded
  ref_10xv3_unstr   the same with --unstranded
  ref_batch         bus --aa --batch batch.txt                          (two samples)
The reference runs inside tests/golden/aa with relative file names, writing each run into its own directory.
"""
import gzip
import os
import random
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "aa")
BASES = "ACGT"
CODE = {}
for i, a in enumerate("FFLLSSSSYY**CC*WLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG"):
    CODE["TCAG"[i // 16] + "TCAG"[(i // 4) % 4] + "TCAG"[i % 4]] = a
STOPS = [c for c, a in CODE.items() if a == "*"]
COMP = {"A": "T", "C": "G", "G": "C", "T": "A"}

RUNS = {
    "ref_bulk_num": ["-x", "bulk", "--num", "reads.fastq.gz"],
    "ref_10xv3": ["-x", "10xv3", "sc_1.fastq.gz", "sc_2.fastq.gz"],
    "ref_10xv3_rf": ["-x", "10xv3", "--rf-stranded", "sc_1.fastq.gz", "sc_2.fastq.gz"],
    "ref_10xv3_unstr": ["-x", "10xv3", "--unstranded", "sc_1.fastq.gz", "sc_2.fastq.gz"],
    "ref_batch": ["--batch", "batch.txt"],
}
KEEP = ("output.bus", "matrix.ec", "transcripts.txt", "run_info.json")


def revcomp(s):
    return "".join(COMP[c] for c in reversed(s))


def translate(s):
    return "".join(CODE[s[i:i + 3]] for i in range(0, len(s) - 2, 3))


def codon(rng, both_strands=False):
    while True:
        c = "".join(rng.choice(BASES) for _ in range(3))
        if CODE[c] != "*" and (not both_strands or CODE[revcomp(c)] != "*"):
            return c


def orf(rng, n, both_strands=False):
    return "".join(codon(rng, both_strands) for _ in range(n))


def transcripts(rng):
    tx = [orf(rng, rng.randint(120, 260)) for _ in range(12)]
    shared = orf(rng, 40)
    for i in (1, 2, 3):                     # one segment in three transcripts: an EC of three proteins
        p = 3 * rng.randint(5, 30)
        tx[i] = tx[i][:p] + shared + tx[i][p:]
    pair = orf(rng, 40)
    tx[4] = tx[4][:60] + pair + tx[4][60:]  # in two: an EC of two
    tx[5] = tx[5][:90] + pair + tx[5][90:]
    for a, b in ((6, 7), (8, 9)):           # segments in frame on both strands: clashes between a forward and a reverse frame
        s = orf(rng, 45, both_strands=True)
        tx[a] = tx[a][:120] + s + tx[a][120:]
        tx[b] = tx[b][:150] + revcomp(s) + tx[b][150:]
    tx[10] = tx[10][:200] + STOPS[0] + tx[10][200:]   # an internal stop: '*' in the protein
    tx[11] = tx[11][:99] + STOPS[2] + tx[11][99:]
    tx += [orf(rng, 15), orf(rng, 9)]       # short proteins: 15 aa (45 cfc letters) and 9 aa (27 < k: no k-mer)
    tx += [orf(rng, 150), orf(rng, 150)]
    return tx


def proteins(tx, rng):
    out = []
    for i, t in enumerate(tx):
        p = translate(t)
        if i == 12:
            p = p[:5] + "X" + p[6:]
        if i == 14:                         # ambiguity codes and an unknown letter
            p = p[:20] + "B" + p[21:40] + "J" + p[41:60] + "Z" + p[61:80] + "U" + p[81:]
        if i == 15:
            p = p.lower()
        out.append(("prot%d description %d" % (i, i), p))
    out.append(("prot_dup", out[3][1]))     # the same sequence under a second name
    return out


def mutate(s, rng, kind):
    s = list(s)
    if kind == "N":
        for _ in range(rng.randint(1, 2)):
            s[rng.randrange(len(s))] = "N"
    elif kind == "lower":
        a = rng.randrange(len(s))
        for j in range(a, min(len(s), a + rng.randint(3, 40))):
            s[j] = s[j].lower()
    elif kind == "foreign":
        s[rng.randrange(len(s))] = rng.choice("RYKMX.")
    elif kind == "snp":
        j = rng.randrange(len(s))
        s[j] = rng.choice([b for b in BASES if b != s[j]])
    return "".join(s)


LENGTHS = [30, 31, 32, 33, 34, 35, 36, 40, 47, 51, 60, 61, 62, 63, 75, 89, 90, 91, 100, 101]


def reads(tx, rng, n):
    out = []
    for _ in range(n):
        L = rng.choice(LENGTHS)
        r = rng.random()
        if r < 0.08:
            s = "".join(rng.choice(BASES) for _ in range(L))        # hits nothing
        else:
            t = tx[rng.randrange(len(tx))]
            if len(t) < L:
                t = tx[0]
            a = rng.randrange(len(t) - L + 1)
            s = t[a:a + L]
            if rng.random() < 0.5:
                s = revcomp(s)
            x = rng.random()
            kind = "N" if x < 0.06 else ("lower" if x < 0.12 else ("foreign" if x < 0.15 else ("snp" if x < 0.25 else "")))
            if kind:
                s = mutate(s, rng, kind)
        out.append(s)
    return out


def write_fastq(path, seqs, name):
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        for i, s in enumerate(seqs):
            f.write(("@%s%d\n%s\n+\n%s\n" % (name, i, s, "I" * len(s))).encode())


def main():
    if not O.have_ref():
        sys.exit("needs oracle/_ref/kallisto (make -C oracle)")
    rng = random.Random(20261017)
    if os.path.isdir(OUT):
        shutil.rmtree(OUT)
    os.makedirs(OUT)
    tx = transcripts(rng)
    prots = proteins(tx, rng)
    with open(os.path.join(OUT, "proteins.fa"), "w") as f:
        for name, p in prots:
            f.write(">%s\n%s\n" % (name, p))
    with tempfile.TemporaryDirectory() as td:
        O.ref_run(["index", "--aa", "-i", os.path.join(OUT, "proteins.kidx"), "-k", "31", "-t", "1", "-T",
                   os.path.join(td, "tmp"), os.path.join(OUT, "proteins.fa")])
    write_fastq(os.path.join(OUT, "reads.fastq.gz"), reads(tx, rng, 400), "r")
    # 10x v3: R1 = 16 barcode + 12 UMI letters (a few short ones: the read set is skipped), R2 = the cDNA read
    n = 300
    r1 = []
    for i in range(n):
        bc = "".join(rng.choice(BASES) for _ in range(16)) if rng.random() < 0.7 else "ACGTACGTACGTACAA"
        umi = "".join(rng.choice(BASES) for _ in range(12))
        s = bc + umi
        if rng.random() < 0.03:
            s = s[:rng.randint(10, 27)]
        r1.append(s)
    write_fastq(os.path.join(OUT, "sc_1.fastq.gz"), r1, "s")
    write_fastq(os.path.join(OUT, "sc_2.fastq.gz"), reads(tx, rng, n), "s")
    write_fastq(os.path.join(OUT, "batch_a.fastq.gz"), reads(tx, rng, 150), "a")
    write_fastq(os.path.join(OUT, "batch_b.fastq.gz"), reads(tx, rng, 120), "b")
    with open(os.path.join(OUT, "batch.txt"), "w") as f:
        f.write("sampleA batch_a.fastq.gz\nsampleB batch_b.fastq.gz\n")
    for name, args in RUNS.items():
        # the call recorded in run_info.json names the program "kallisto" and the run's own directory, so that the
        # fixture holds no path of the machine that made it
        r = subprocess.run(["kallisto", "bus", "--aa", "-t", "1", "-i", "proteins.kidx", "-o", name] + args,
                           executable=O.REF_BIN, cwd=OUT, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        if r.returncode != 0:
            sys.exit("kallisto bus --aa failed (exit %d): %s" % (r.returncode, r.stderr.decode(errors="replace")[-600:]))
        for f in os.listdir(os.path.join(OUT, name)):
            if f not in KEEP:
                os.remove(os.path.join(OUT, name, f))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
