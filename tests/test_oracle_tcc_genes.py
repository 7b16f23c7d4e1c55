"""CPU: the CPU restatement of quant-tcc's gene-level output (tests/gene_oracle.py) against every file and error of the
unmodified reference (tests/golden/quanttcc_genes.json.gz, from make_golden_quanttcc_genes.py).

- The gene model reproduces every genes.txt and the gene list of every gene file.
- Its gene sums of the transcript estimates (oracle.em, and oracle.bootstrap_sample + oracle.em for bootstraps, which
  test_oracle_tcc_bootstrap.py holds to the reference) reproduce every *.gene*.tsv and *.gene*.mtx byte for byte.
- The error cases give the stored "Error:" lines."""
import gzip
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import gene_oracle as GO
from tests import util
from tests.test_oracle_tcc_bootstrap import eff_of, opt, read_tcc

SRC = os.path.join(util.GOLDEN, "quanttcc")
IDX = os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx")
GOLD = json.loads(gzip.open(os.path.join(util.GOLDEN, "quanttcc_genes.json.gz")).read())
CASES, INPUTS = GOLD["cases"], GOLD["inputs"]


def gene_model(args, targets):
    if "-g" in args:
        fn = opt(args, "-g")
        return GO.parse_genemap(INPUTS[fn], targets, fn)
    return GO.parse_gtf(INPUTS[opt(args, "-G").replace(".gz", "")], targets)


def expected_gene_files(args, tcc):
    """-> {relative path: text} of every gene file the case writes."""
    ix = O.OracleIndex(IDX)
    sets = O.read_matrix_ec(os.path.join(SRC, "matrix.ec"))
    off = np.zeros(len(sets) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in sets])
    tids = np.array([t for s in sets for t in s], np.uint32)
    rows, is_matrix = read_tcc(os.path.join(SRC, tcc), len(sets))
    B, seed = int(opt(args, "-b", 0)), int(opt(args, "--seed", 42))
    effs = eff_of(args, ix.target_lens, len(rows))
    names, common, gene_of = gene_model(args, ix.target_names)
    G = len(names)
    dirs = "--matrix-to-directories" in args
    files = "--matrix-to-files" in args or dirs
    out, mtx_c, mtx_t = {}, [], []
    for r, counts in enumerate(rows):
        est, _ = O.em(off, tids, counts, effs[r], ix.n_targets)
        gc, gt = GO.gene_sums(est, effs[r], gene_of, G)
        if not is_matrix:
            out["abundance.gene.tsv"] = GO.gene_tsv(names, common, gc[0], gt[0])
            continue
        mtx_c.append([(g, gc[0, g]) for g in range(G) if gc[0, g] > 0])
        mtx_t.append([(g, gt[0, g]) for g in range(G) if gc[0, g] > 0])
        if not files:
            continue
        out["abundance_%d/abundance.gene.tsv" % (r + 1) if dirs else "abundance.gene_%d.tsv" % (r + 1)] = \
            GO.gene_tsv(names, common, gc[0], gt[0])
        if B and "--plaintext" in args:
            alphas = ([est] * B if not (est > 0).any() else
                      [O.em(off, tids, O.bootstrap_sample(counts, seed, b), effs[r], ix.n_targets, counts_w=counts)[0]
                       for b in range(B)])
            bgc, bgt = GO.gene_sums(np.stack(alphas), effs[r], gene_of, G)
            for b in range(B):
                fn = ("abundance_%d/bs_abundance.gene_%d.tsv" % (r + 1, b) if dirs
                      else "bs_abundance.gene_%d_%d.tsv" % (r + 1, b))
                out[fn] = GO.gene_tsv(names, common, bgc[b], bgt[b])
    if is_matrix:
        out["matrix.abundance.gene.mtx"] = GO.sparse_mtx(mtx_c, G)
        out["matrix.abundance.gene.tpm.mtx"] = GO.sparse_mtx(mtx_t, G)
        out["genes.txt"] = "".join(n + "\n" for n in names)
    return out


def golden_gene_files(name):
    return {fn: t for fn, t in GOLD["outputs"][name].items() if ".gene" in fn or fn == "genes.txt"}


@pytest.mark.parametrize("name", list(CASES))
def test_gene_files_identical_to_reference(name):
    args, tcc = CASES[name]
    exp, ref = expected_gene_files(args, tcc), golden_gene_files(name)
    assert sorted(exp) == sorted(ref)
    for fn in ref:
        assert exp[fn] == ref[fn], fn


@pytest.mark.parametrize("name", list(CASES))
def test_gene_model_reproduces_gene_list(name):
    args, _ = CASES[name]
    names, common, _ = gene_model(args, O.OracleIndex(IDX).target_names)
    out = GOLD["outputs"][name]
    if "genes.txt" in out:
        assert out["genes.txt"] == "".join(n + "\n" for n in names)
    for fn, text in out.items():
        if ".gene" in fn and fn.endswith(".tsv"):
            rows = [l.split("\t")[:2] for l in text.splitlines()[1:]]
            assert rows == [[n, c] for n, c in zip(names, common)], fn


@pytest.mark.parametrize("name", list(GOLD["errors"]))
def test_error_cases(name):
    """Errors of the gene model itself; the option checks (-g with -G, missing files) come from the CLI (GPU tests)."""
    err = GOLD["errors"][name]
    assert err["exit"] == 1 and len(err["errors"]) == 1
    args, _ = GOLD["error_cases"][name]
    fn = opt(args, "-g")
    if "-G" in args or fn not in INPUTS:
        return
    with pytest.raises(GO.GeneModelError) as e:
        GO.parse_genemap(INPUTS[fn], O.OracleIndex(IDX).target_names, fn)
    assert [str(e.value)] == err["errors"]


def test_fixture_covers_the_gene_model_rules():
    """The map leaves transcripts out, has genes without a common name, a gene emptied by a reassignment and gene ids
    out of transcript order; the GTF has a duplicate gene line, a transcript whose gene has no gene line, transcripts
    not in the index and the gene-id quirk of transcript lines."""
    targets = O.OracleIndex(IDX).target_names
    names, common, gene_of = GO.parse_genemap(INPUTS["t2g.txt"], targets, "t2g.txt")
    members = np.bincount(gene_of[gene_of >= 0], minlength=len(names))
    assert (gene_of == -1).any() and "" in common and "Gene5" in common and (members == 0).sum() == 1
    first = [gene_of[t] for t in range(len(targets)) if gene_of[t] >= 0]
    assert first != sorted(first)
    names, common, gene_of = GO.parse_gtf(INPUTS["genes.gtf"], targets)
    assert len(names) > len(set(names)) and "" in common
    assert names[gene_of[[t for t, n in enumerate(targets) if n.startswith("SYNT000011")][0]]] == "GQ.1.5"
    assert all(gene_of[t] == -1 for t, n in enumerate(targets) if n.startswith("SYNT000005"))
    assert "SYNTX00000" in INPUTS["genes.gtf"] and "\texon\t" in INPUTS["genes.gtf"] and "\tCDS\t" in INPUTS["genes.gtf"]
