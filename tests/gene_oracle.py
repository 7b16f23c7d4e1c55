"""CPU restatement of quant-tcc's gene-level output: the gene model (Transcriptome::parseGeneMap / parseGTF,
src/GeneModel.cpp:268-632, as quant-tcc calls them) and the gene sums (src/main.cpp:3026-3058, plaintext_writer_gene
src/PlaintextWriter.cpp:67-112).  The device gene pass of kb_tcc_run_genes / kb_tcc_bootstrap_run_genes is held to it.

The sums keep the reference's order: counts_to_tpm's total is a sequential sum in target order, and every gene adds its
transcripts in increasing id.  numpy's sum is pairwise, so the loops below run over targets, one IEEE operation per
step, vectorised across problems only."""
import gzip

import numpy as np


class GeneModelError(Exception):
    """An input the reference rejects; the message is the reference's "Error: ..." line."""


def parse_genemap(text, targets, fn):
    """-> (gene names, common names, gene of every target (-1: none)).  fn is the file name the messages carry."""
    tr = {}
    for i, n in enumerate(targets):
        tr.setdefault(n, i)
    names, common, ids = [], [], {}
    gene_of = np.full(len(targets), -1, np.int32)
    for line in text.split("\n"):
        if not line:
            continue
        f = line.split()
        txp, gene, com = (f + ["", "", ""])[:3]
        if not gene:
            raise GeneModelError("Error: No gene associated with transcript %s in %s" % (txp, fn))
        if txp not in tr:
            raise GeneModelError("Error: Invalid transcript: %s in %s" % (txp, fn))
        if gene not in ids:
            ids[gene] = len(names)
            names.append(gene)
            common.append(com)
        gene_of[tr[txp]] = ids[gene]
    return names, common, gene_of


def read_gtf(path):
    data = open(path, "rb").read()
    return (gzip.decompress(data) if data[:2] == b"\x1f\x8b" else data).decode()


def parse_gtf(text, targets):
    """-> (gene names, common names, gene of every target).  addGTFLine with every chromosome accepted: only `gene` and
    `transcript` lines matter.  A gene line appends .<gene_version> to an id without '.'; a duplicate gene line is a new
    list entry whose name keeps the first id.  A transcript line looks up transcript_id.<transcript_version> (id without
    '.') then the bare id, and gene_id.<gene_version> (always appended: src/GeneModel.cpp:450 tests the line's empty gene
    model) then the bare gene id; the first transcript line of a target decides its gene."""
    tr = {}
    for i, n in enumerate(targets):
        tr.setdefault(n, i)
    names, common, ids = [], [], {}
    seen = set()
    gene_of = np.full(len(targets), -1, np.int32)
    for line in text.split("\n"):
        if not line or line[0] == "#":
            continue
        f = line.split("\t")
        if len(f) < 3 or f[2] not in ("gene", "transcript"):
            continue
        is_gene = f[2] == "gene"
        attr = "\t".join(f[8:])
        gene = gver = txp = tver = com = ""
        keycount = 0
        p = 0
        while True:
            q = attr.find('"', p)
            if q < 0:
                break
            s = attr.find('"', q + 1)
            if s < 0:
                break
            key, value = (attr[p:q - 1] if q > p else attr[p:]), attr[q + 1:s]
            if key == "gene_id":
                keycount += 1
                gene = value
            elif key == "gene_version":
                keycount += 1
                gver = value
            if is_gene:
                if key == "gene_name":
                    keycount += 1
                    com = value
                elif key == "gene_id" and keycount == 3:
                    break
            else:
                if key == "transcript_id":
                    keycount += 1
                    txp = value
                elif key == "transcript_version":
                    keycount += 1
                    tver = value
                if keycount == 4:
                    break
            p = attr.find(" ", s)
            if p < 0:
                break
            p += 1
            if p >= len(attr):
                break
        if is_gene:
            if gver and "." not in gene:
                gene += "." + gver
            ids.setdefault(gene, len(names))
            names.append(gene)
            common.append(com)
            continue
        t = tr.get(txp + "." + tver) if tver and "." not in txp else None
        if t is None:
            t = tr.get(txp)
        if t is None:
            continue
        g = ids.get(gene + "." + gver) if gver else None
        if g is None:
            g = ids.get(gene, -1)
        if t not in seen:
            seen.add(t)
            gene_of[t] = g
    return names, common, gene_of


def gene_sums(alpha, eff, gene_of, n_genes):
    """alpha (P, T) estimates, eff (T,) or (P, T) -> gene counts and gene TPM, (P, n_genes) each."""
    alpha = np.atleast_2d(np.asarray(alpha, np.float64))
    P, T = alpha.shape
    eff = np.broadcast_to(np.asarray(eff, np.float64), (P, T))
    total = np.zeros(P)
    for t in range(T):
        total = total + alpha[:, t] / eff[:, t]
    gc, gt = np.zeros((P, n_genes)), np.zeros((P, n_genes))
    for t in range(T):
        g = gene_of[t]
        if g < 0:
            continue
        pos = alpha[:, t] > 0.0
        if pos.any():
            a = alpha[pos, t]
            gc[pos, g] = gc[pos, g] + a
            gt[pos, g] = gt[pos, g] + (a / eff[pos, t] / total[pos]) * 1e6
    return gc, gt


def gene_tsv(names, common, gc, gt):
    lines = ["gene_id\tgene_name\test_counts\ttpm"]
    lines += ["%s\t%s\t%g\t%g" % (n, c, x, y) for n, c, x, y in zip(names, common, gc, gt)]
    return "\n".join(lines) + "\n"


def sparse_mtx(rows, n_cols):
    """writeSparseBatchMatrix (src/PlaintextWriter.h): rows = per row a list of (column, value); zeros are left out."""
    ent = [(r + 1, c + 1, v) for r, row in enumerate(rows) for c, v in row if v != 0.0]
    out = "%%%%MatrixMarket matrix coordinate real general\n%d\t%d\t%d\n" % (len(rows), n_cols, len(ent))
    return out + "".join("%d\t%d\t%g\n" % e for e in ent)
