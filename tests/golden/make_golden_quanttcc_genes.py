#!/usr/bin/env python
"""Generates tests/golden/quanttcc_genes.json.gz from the UNMODIFIED reference (oracle/_ref/kallisto, `make -C oracle`):
`kallisto quant-tcc` with gene-level output (-g/--genemap, -G/--gtf) on the inputs of tests/golden/quanttcc (matrix.ec;
tcc.mtx, whose rows are all reads / first half / a sparse row / an empty row; tcc_single.txt; fld_*.txt), which are read,
not regenerated, plus transcript-to-gene maps and GTFs that this script writes over synth_small's transcript names
(SYNTnnnnnn.N, 491 of them).

    python tests/golden/make_golden_quanttcc_genes.py

The fixture is one gzip-compressed JSON object:
  {"inputs": {file name: text}, "cases": {name: [arguments, TCC file]}, "error_cases": {name: [arguments, TCC file]},
   "outputs": {name: {relative path: text}}, "errors": {name: {"exit": code, "errors": [the "Error:" lines of stderr]}}}
The reference runs in a directory that holds the inputs (genes.gtf.gz is genes.gtf, gzip-compressed), with their plain
names on the command line, so that messages carry no temporary path.  quanttcc/ files in the arguments are relative to
quanttcc/.  Every output file except run_info.json is stored.
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
OUT = os.path.join(G, "quanttcc_genes.json.gz")

CASES = {
    "mtx_g": (["-g", "t2g.txt"], "tcc.mtx"),
    "files_ls_g": (["-l", "180", "-s", "25", "--matrix-to-files", "-g", "t2g.txt"], "tcc.mtx"),
    "dirs_fld_rows_b3_g": (["-f", "fld_rows.txt", "--matrix-to-directories", "--plaintext", "-b", "3", "-g", "t2g.txt"],
                           "tcc.mtx"),
    "files_b2_gtfgz": (["--matrix-to-files", "--plaintext", "-b", "2", "-G", "genes.gtf.gz"], "tcc.mtx"),
    "single_g_b2": (["-g", "t2g.txt", "-b", "2"], "tcc_single.txt"),
    "mtx_gtf": (["-G", "genes.gtf"], "tcc.mtx"),
    "single_ls_gtf": (["-l", "200", "-s", "20", "-G", "genes.gtf"], "tcc_single.txt"),
}
ERRORS = {
    "err_unknown_transcript": (["-g", "t2g_unknown.txt"], "tcc.mtx"),
    "err_no_gene": (["-g", "t2g_nogene.txt"], "tcc.mtx"),
    "err_both": (["-g", "t2g.txt", "-G", "genes.gtf"], "tcc.mtx"),
    "err_missing_map": (["-g", "t2g_missing.txt"], "tcc.mtx"),
    "err_missing_gtf": (["-G", "genes_missing.gtf"], "tcc.mtx"),
}


def make_t2g(names):
    """Genes follow the SYNTnnnnnn prefix, listed in a shuffled order (so gene ids are not in transcript order).  Every
    7th transcript is in no line; every 3rd gene has no common name, every 5th has extra columns (kb-python's t2g has
    more).  GLONE's only transcript is reassigned by a later line, so GLONE ends up with no members.  One blank line."""
    rng = random.Random(7)
    lines = []
    for i, n in enumerate(names):
        if i % 7 == 3:
            continue
        gi = int(n[4:10])
        g = "ENSG%011d.%d" % (gi * 13, 1 + gi % 3)
        if gi % 3 == 0:
            lines.append("%s\t%s" % (n, g))
        elif gi % 5 == 0:
            lines.append("%s\t%s\tGene%d\t%s\tchr1\t+" % (n, g, gi, n))
        else:
            lines.append("%s %s  Gene%d" % (n, g, gi))
    rng.shuffle(lines)
    moved = names[10]
    lines.insert(0, "%s\tGLONE\tLonely" % moved)
    lines.insert(len(lines) // 2, "")
    lines.append("%s\tENSG99999999999.1\tLate" % moved)
    return "\n".join(lines) + "\n"


def make_gtf(names):
    """Genes GENEnnnn (gene_version 2, from the SYNTnnnnnn prefix), transcripts with transcript_version split out, and:
    exon / CDS / UTR lines; comments; a duplicate `gene` line; a transcript whose gene has no `gene` line; a transcript
    line before its gene's `gene` line; transcripts that are not in the index; a transcript listed twice (the first
    line decides); versioned transcript ids without transcript_version; genes without gene_name; and the gene-id quirk
    of transcript lines (gene_id "GQ.1" gene_version "5" is looked up as "GQ.1.5" first, which names another gene)."""
    out = ["#!genome-build synthetic", "#!genome-version 1"]
    attrs = lambda **kw: " ".join('%s "%s";' % kv for kv in kw.items())

    def line(typ, start, stop, a, strand="+", chrom="chr1"):
        out.append("\t".join([chrom, "synth", typ, str(start), str(stop), ".", strand, ".", a]))
    by_gene = {}
    for n in names:
        by_gene.setdefault(int(n[4:10]), []).append(n)
    pos = 1
    for gi in sorted(by_gene, key=lambda g: (g * 37) % 120):
        gid = "GENE%04d" % gi
        chrom = "chr%d" % (1 + gi % 4)
        if gi == 11:
            continue                                          # in no line at all (one is the quirk's transcript below)
        if gi == 9:                                           # transcript line before the gene line
            t = by_gene[gi][0]
            line("transcript", pos, pos + 900, attrs(gene_id=gid, gene_version="2", transcript_id=t[:10],
                                                     transcript_version=t[11:]), chrom=chrom)
        if gi == 5:
            pass                                              # no `gene` line: its transcripts get no gene
        elif gi % 4 == 0:
            line("gene", pos, pos + 1000, attrs(gene_id=gid, gene_version="2", gene_biotype="protein_coding"), chrom=chrom)
        else:
            line("gene", pos, pos + 1000, attrs(gene_id=gid, gene_version="2", gene_name="Syn%d" % gi,
                                                gene_source="synth"), chrom=chrom)
        if gi == 17:                                          # duplicate gene line: a second list entry, same name
            line("gene", pos, pos + 1200, attrs(gene_id=gid, gene_version="2", gene_name="Syn17dup"), chrom=chrom)
        for k, t in enumerate(by_gene[gi]):
            if gi % 6 == 1:                                   # versioned id, no transcript_version
                a = attrs(gene_id=gid, gene_version="2", transcript_id=t, gene_name="Syn%d" % gi)
            else:
                a = attrs(gene_id=gid, gene_version="2", transcript_id=t[:10], transcript_version=t[11:],
                          transcript_biotype="protein_coding")
            line("transcript", pos + k, pos + 800, a, strand="-" if gi % 2 else "+", chrom=chrom)
            line("exon", pos + k, pos + 300, a + ' exon_number "1";', chrom=chrom)
            line("CDS", pos + k + 10, pos + 250, a, chrom=chrom)
            line("five_prime_utr", pos + k, pos + k + 9, a, chrom=chrom)
        pos += 2000
    # a transcript listed a second time under another gene: the first line stays
    t = by_gene[2][0]
    line("transcript", 5, 900, attrs(gene_id="GENE0003", gene_version="2", transcript_id=t[:10], transcript_version=t[11:]))
    # transcripts the index does not hold
    for k in range(3):
        line("transcript", 10 + k, 500, attrs(gene_id="GENE0001", gene_version="2", transcript_id="SYNTX%05d" % k,
                                              transcript_version="1"))
    # the gene-id quirk: GQ.1 (version not appended, it has a '.') and GQ.1.5; the transcript line looks up GQ.1.5 first
    line("gene", 1, 100, attrs(gene_id="GQ.1", gene_version="5", gene_name="Quirk"))
    line("gene", 1, 100, attrs(gene_id="GQ.1.5", gene_name="QuirkTarget"))
    t = by_gene[11][0]
    line("transcript", 1, 100, attrs(gene_id="GQ.1", gene_version="5", transcript_id=t[:10], transcript_version=t[11:]))
    return "\n".join(out) + "\n"


def inputs():
    names = O.OracleIndex(os.path.join(G, "synth_small", "transcripts.kidx")).target_names
    t2g = make_t2g(names)
    return {
        "t2g.txt": t2g,
        "t2g_unknown.txt": t2g.replace(names[20] + "\t", "SYNT999999.1\t", 1).replace(names[20] + " ", "SYNT999999.1 ", 1),
        "t2g_nogene.txt": "%s\tENSG1\n%s\n%s\tENSG2\n" % (names[0], names[1], names[2]),
        "genes.gtf": make_gtf(names),
    }


def write_inputs(d, files):
    """Writes the inputs into d; genes.gtf.gz = genes.gtf compressed."""
    for fn, text in files.items():
        with open(os.path.join(d, fn), "w") as f:
            f.write(text)
    with gzip.open(os.path.join(d, "genes.gtf.gz"), "wt") as f:
        f.write(files["genes.gtf"])


def command(idx, out, args, tcc):
    args = [os.path.join(SRC, a) if a.startswith("fld_") else a for a in args]
    return ["quant-tcc", "-i", idx, "-e", os.path.join(SRC, "matrix.ec"), "-o", out] + args + [os.path.join(SRC, tcc)]


def main():
    O.build()
    assert O.have_ref(), "build the reference first: make -C oracle"
    idx = os.path.join(G, "synth_small", "transcripts.kidx")
    files = inputs()
    assert files["t2g_unknown.txt"] != files["t2g.txt"]
    outputs, errors = {}, {}
    with tempfile.TemporaryDirectory() as td:
        write_inputs(td, files)
        for name, (extra, tcc) in CASES.items():
            out = os.path.join(td, "o")
            O.ref_run(command(idx, out, extra, tcc), cwd=td)
            got = {}
            for d, _, fns in os.walk(out):
                for fn in fns:
                    if fn != "run_info.json":
                        p = os.path.join(d, fn)
                        got[os.path.relpath(p, out)] = open(p).read()
            outputs[name] = dict(sorted(got.items()))
            shutil.rmtree(out)
        for name, (extra, tcc) in ERRORS.items():
            r = O.ref_run(command(idx, os.path.join(td, "e"), extra, tcc), cwd=td, check=False)
            errors[name] = {"exit": r.returncode,
                            "errors": [l for l in r.stderr.decode().splitlines() if l.startswith("Error:")]}
            assert r.returncode != 0 and errors[name]["errors"], (name, r.stderr.decode())
            shutil.rmtree(os.path.join(td, "e"), ignore_errors=True)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(json.dumps({"inputs": files, "cases": CASES, "error_cases": ERRORS, "outputs": outputs, "errors": errors}, sort_keys=True).encode())
    print("quanttcc_genes:", {k: len(v) for k, v in outputs.items()}, errors, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
