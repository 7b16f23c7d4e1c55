"""GPU: gene-level output of `kallisto_b200 quant-tcc` (-g / -G; kb_tcc_run_genes and kb_tcc_bootstrap_run_genes, whose
gene sums run on the device).

- The CLI against every file and every error of the unmodified reference (tests/golden/quanttcc_genes.json.gz), byte for
  byte, with the automatic chunks, with one sample per launch (KB_TCC_CHUNK=1) and with one and five bootstrap problems
  per launch (KB_TCC_BS_CHUNK).
- The library against the CPU restatement (tests/gene_oracle.py) on tables generated from seeds over stored indices
  (T = 14, 491, 2 400; the tables of test_gpu_em_shapes.py): gene maps with genes without members, every transcript in
  one gene and transcripts without a gene; an all-zero row; per-row and shared effective lengths; and 8 199 bootstrap
  problems, so that chunks split rows.  Estimates equal oracle.em, and the gene sums of those estimates equal the
  device's bit for bit.
- genes=None gives the same arrays as the calls without genes."""
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import gene_oracle as GO
from tests import util
from tests.test_gpu_em_shapes import KNOB_VARS, _case
from tests.test_gpu_tcc_bootstrap import _csr_rows, _effs

pytestmark = pytest.mark.gpu

SRC = os.path.join(util.GOLDEN, "quanttcc")
IDX = os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx")
CLI = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")
GOLD = json.loads(gzip.open(os.path.join(util.GOLDEN, "quanttcc_genes.json.gz")).read())
CASES = GOLD["cases"]
SEED = 23
CHUNKS = {"auto": {}, "tcc1": {"KB_TCC_CHUNK": "1"}, "bs1": {"KB_TCC_BS_CHUNK": "1"}, "bs5": {"KB_TCC_BS_CHUNK": "5"}}


def _inputs(d):
    for fn, text in GOLD["inputs"].items():
        (d / fn).write_text(text)
    with gzip.open(d / "genes.gtf.gz", "wt") as f:
        f.write(GOLD["inputs"]["genes.gtf"])


def _cli(d, args, tcc, env_extra):
    args = [os.path.join(SRC, a) if a.startswith("fld_") else a for a in args]
    env = {k: v for k, v in os.environ.items() if k not in ("KB_TCC_CHUNK", "KB_TCC_BS_CHUNK")}
    env.update(env_extra)
    return subprocess.run([CLI, "quant-tcc", "-i", IDX, "-e", os.path.join(SRC, "matrix.ec"), "-o", str(d / "out")] + args +
                          [os.path.join(SRC, tcc)], capture_output=True, text=True, env=env, cwd=str(d))


def _tree(root):
    return {os.path.relpath(os.path.join(d, fn), root): os.path.join(d, fn) for d, _, fns in os.walk(root) for fn in fns}


@pytest.mark.parametrize("chunk", list(CHUNKS))
@pytest.mark.parametrize("name", list(CASES))
def test_quant_tcc_gene_files_identical_to_reference(tmp_path, name, chunk):
    _inputs(tmp_path)
    args, tcc = CASES[name]
    r = _cli(tmp_path, args, tcc, CHUNKS[chunk])
    assert r.returncode == 0, r.stderr[-1000:]
    ref, got = GOLD["outputs"][name], _tree(tmp_path / "out")
    got.pop("run_info.json", None)
    assert sorted(got) == sorted(ref)
    for fn in ref:
        assert open(got[fn], "rb").read() == ref[fn].encode(), fn


@pytest.mark.parametrize("name", list(GOLD["errors"]))
def test_quant_tcc_gene_errors_as_reference(tmp_path, name):
    _inputs(tmp_path)
    args, tcc = GOLD["error_cases"][name]
    r = _cli(tmp_path, args, tcc, {})
    exp = GOLD["errors"][name]
    assert r.returncode == exp["exit"], r.stderr[-1000:]
    assert [l for l in r.stderr.splitlines() if l.startswith("Error:")] == exp["errors"]


# ---------------------------------------------------------------------------------------------------------------------
# library level
# ---------------------------------------------------------------------------------------------------------------------
def _gene_map(kind, T, rng):
    """-> (gene of every target, n_genes).  random: ~T/4 genes in a shuffled numbering, ~1/6 of the targets in none,
    and genes without members (in the middle and at the end); one: every target in gene 0; none: no target in any of 3
    genes."""
    if kind == "one":
        return np.zeros(T, np.int32), 1
    if kind == "none":
        return np.full(T, -1, np.int32), 3
    G = max(3, T // 4) + 2
    g = rng.integers(0, G - 2, T).astype(np.int32)
    g[g == (G - 2) // 2] = (G - 2) // 2 + 1                 # gene (G-2)//2 has no members, nor have the last two
    g[rng.random(T) < 1 / 6] = -1
    return g, G


def _rows(c, rng):
    """An all-zero row, the table's counts, two random subsets of them and one row of a single EC."""
    own = np.minimum(c.counts, 5000).astype(np.uint32)
    rows = [np.zeros(c.n, np.uint32), own]
    rows += [np.where(rng.random(c.n) < p, own, 0).astype(np.uint32) for p in (0.5, 0.2)]
    one = np.zeros(c.n, np.uint32)
    one[rng.integers(0, c.n)] = 1000
    return rows + [one]


@pytest.fixture(scope="module")
def cases():
    return {}


@pytest.fixture(scope="module")
def indices():
    out = {name: K.KmerIndex(util.dataset(name)["index"], device=0) for name in ("synth_small", "config1", "abundant")}
    yield out
    for ix in out.values():
        ix.close()


def _knobs(monkeypatch, env):
    for k in KNOB_VARS + ("KB_TCC_BS_CHUNK",):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("per_row_eff", [False, True])
@pytest.mark.parametrize("chunk", ["", "1", "2"])
@pytest.mark.parametrize("kind", ["random", "one", "none"])
@pytest.mark.parametrize("table", ["golden_synth", "golden_config1", "hub"])
def test_tcc_run_genes_equal_oracle(cases, indices, monkeypatch, table, kind, chunk, per_row_eff):
    c = _case(cases, table)
    _knobs(monkeypatch, {"KB_TCC_CHUNK": chunk} if chunk else {})
    rng = np.random.default_rng([len(table), len(kind)])
    rows = _rows(c, rng)
    gene_of, G = _gene_map(kind, c.T, rng)
    eff = _effs(c, len(rows)) if per_row_eff else _effs(c, 1)[0]
    sets = c.sets()
    sparse = [[(int(e), int(r[e])) for e in np.flatnonzero(r)] for r in rows]
    est, rounds, gc, gt = K.tcc_run(indices[c.index], sets, sparse, eff, genes=(gene_of, G))
    assert gc.shape == gt.shape == (len(rows), G)
    est0, rounds0 = K.tcc_run(indices[c.index], sets, sparse, eff)          # genes=None: the arrays of today's calls
    np.testing.assert_array_equal(est, est0)
    np.testing.assert_array_equal(rounds, rounds0)
    for r, row in enumerate(rows):
        e = eff[r] if per_row_eff else eff
        alpha, n = O.em(c.off, c.tids, row, e, c.T)
        np.testing.assert_array_equal(est[r], alpha, err_msg="row %d" % r)
        assert rounds[r] == n
        xc, xt = GO.gene_sums(alpha, e, gene_of, G)
        np.testing.assert_array_equal(gc[r], xc[0], err_msg="gene counts, row %d" % r)
        np.testing.assert_array_equal(gt[r], xt[0], err_msg="gene TPM, row %d" % r)
    assert not gc[0].any() and not gt[0].any()                              # the all-zero row
    if kind == "one":
        assert (gc[1:, 0] > 0).all()
    if kind == "none":
        assert not gc.any()


def _bootstrap(ix, c, rows, eff, B, genes):
    ro, ids, vals = _csr_rows(rows)
    got = []

    def on_chunk(first, est, rounds, samples, *g):
        assert first == sum(len(x[0]) for x in got)
        got.append((est, rounds) + tuple(g))
    K.tcc_bootstrap(ix, c.off, c.tids, ro, ids, vals, eff, SEED, B, on_chunk, genes=genes)
    return [np.concatenate([x[i] for x in got]) for i in range(len(got[0]))], len(got)


@pytest.mark.parametrize("chunk", ["", "1", "5"])
@pytest.mark.parametrize("table", ["golden_synth", "golden_config1", "hub"])
def test_tcc_bootstrap_genes_equal_oracle(cases, indices, monkeypatch, table, chunk):
    """Five rows (one all-zero) x 3 bootstraps with per-row effective lengths, every problem against the oracle."""
    c = _case(cases, table)
    _knobs(monkeypatch, {"KB_TCC_BS_CHUNK": chunk} if chunk else {})
    rng = np.random.default_rng(len(table) + 100)
    rows = _rows(c, rng)
    gene_of, G = _gene_map("random", c.T, rng)
    eff = _effs(c, len(rows))
    B = 3
    (est, rounds, gc, gt), _ = _bootstrap(indices[c.index], c, rows, eff, B, (gene_of, G))
    (est0, rounds0), _ = _bootstrap(indices[c.index], c, rows, eff, B, None)
    np.testing.assert_array_equal(est, est0)
    np.testing.assert_array_equal(rounds, rounds0)
    for g in range(len(rows) * B):
        r, b = divmod(g, B)
        if rows[r].any():
            alpha, _ = O.em(c.off, c.tids, O.bootstrap_sample(rows[r], SEED, b), eff[r], c.T, counts_w=rows[r])
            np.testing.assert_array_equal(est[g], alpha, err_msg="problem %d" % g)
        xc, xt = GO.gene_sums(est[g], eff[r], gene_of, G)
        np.testing.assert_array_equal(gc[g], xc[0], err_msg="gene counts, problem %d" % g)
        np.testing.assert_array_equal(gt[g], xt[0], err_msg="gene TPM, problem %d" % g)


@pytest.mark.parametrize("chunk", ["", "3000"])
def test_tcc_bootstrap_genes_past_one_launch(cases, indices, monkeypatch, chunk):
    """9 rows x 911 bootstraps = 8 199 problems, more than one launch holds (8 192), so chunks split rows; the gene sums
    of every problem are checked against the restatement, the estimates of some against oracle.em."""
    c = _case(cases, "golden_synth")
    _knobs(monkeypatch, {"KB_TCC_BS_CHUNK": chunk} if chunk else {})
    rng = np.random.default_rng(8199)
    rows = _rows(c, rng)
    rows += [np.where(rng.random(c.n) < 0.3, np.minimum(c.counts, 50), 0).astype(np.uint32) for _ in range(9 - len(rows))]
    gene_of, G = _gene_map("random", c.T, rng)
    eff = _effs(c, len(rows))
    B = 911
    (est, rounds, gc, gt), n_chunks = _bootstrap(indices[c.index], c, rows, eff, B, (gene_of, G))
    assert n_chunks == (2 if not chunk else 3) and len(gc) == len(rows) * B
    effp = np.repeat(eff, B, axis=0)
    xc, xt = GO.gene_sums(est, effp, gene_of, G)
    np.testing.assert_array_equal(gc, xc)
    np.testing.assert_array_equal(gt, xt)
    for g in sorted({B, 3000, 6000, 8191, 8192, 8198} | {r * B + B - 1 for r in range(1, len(rows))}):
        r, b = divmod(g, B)
        alpha, _ = O.em(c.off, c.tids, O.bootstrap_sample(rows[r], SEED, b), eff[r], c.T, counts_w=rows[r])
        np.testing.assert_array_equal(est[g], alpha, err_msg="problem %d" % g)
