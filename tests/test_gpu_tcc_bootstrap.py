"""GPU: bootstraps of `kallisto_b200 quant-tcc` (kb_tcc_bootstrap_run: per-row sparse resampling + the batched EM with
each row's weights shared by its B problems).

- The CLI against every file the unmodified reference wrote (tests/golden/quanttcc_bs.json.gz), byte for byte, with the
  automatic chunking and with one and five problems per launch (KB_TCC_BS_CHUNK).
- The library against the CPU oracle on tables generated from seeds over stored indices (the tables of
  test_gpu_em_shapes.py): every resampled count equals oracle.bootstrap_sample and every estimate and round count equals
  oracle.em with the row's counts as weights.  The rows cover N = 0, 1 and more than 10^6 draws, a single non-zero EC,
  the last EC zero and non-zero (the sentinel of the sparse table), per-row effective lengths, and more (row, bootstrap)
  problems than one launch holds.
- One row through kb_tcc_bootstrap_run equals kb_bootstrap_run on the same imported table (sparse tables against the
  dense one)."""
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import util
from tests.test_gpu_em_shapes import KNOB_VARS, _case, _fld, _imported

pytestmark = pytest.mark.gpu

SRC = os.path.join(util.GOLDEN, "quanttcc")
IDX = os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx")
CLI = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")
GOLD = json.loads(gzip.open(os.path.join(util.GOLDEN, "quanttcc_bs.json.gz")).read())
CASES = GOLD["cases"]
SEED = 11


def _tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for fn in files:
            out[os.path.relpath(os.path.join(d, fn), root)] = os.path.join(d, fn)
    return out


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("chunk", ["", "1", "5"])
def test_quant_tcc_bootstrap_files_identical_to_reference(tmp_path, name, chunk):
    args, tcc = CASES[name]
    args = [os.path.join(SRC, a) if a.endswith(".txt") else a for a in args]
    out = tmp_path / "out"
    env = dict(os.environ)
    env.pop("KB_TCC_BS_CHUNK", None)
    if chunk:
        env["KB_TCC_BS_CHUNK"] = chunk
    r = subprocess.run([CLI, "quant-tcc", "-i", IDX, "-e", os.path.join(SRC, "matrix.ec"), "-o", str(out)] + args +
                       [os.path.join(SRC, tcc)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-1000:]
    ref, got = GOLD["outputs"][name], _tree(out)
    assert sorted(got) == sorted(ref)
    for fn in ref:
        assert open(got[fn], "rb").read() == ref[fn].encode(), fn


def test_quant_tcc_bootstrap_refusals(tmp_path):
    """-b on a matrix needs --matrix-to-files / --matrix-to-directories AND --plaintext; a non-matrix file without any
    count cannot be bootstrapped; --matrix-to-directories fails where abundance_<row> is a file."""
    base = [CLI, "quant-tcc", "-i", IDX, "-e", os.path.join(SRC, "matrix.ec")]
    for extra in (["--matrix-to-files", "-b", "2"], ["--matrix-to-directories", "-b", "2"], ["--plaintext", "-b", "2"]):
        r = subprocess.run(base + ["-o", str(tmp_path / "o1")] + extra + [os.path.join(SRC, "tcc.mtx")], capture_output=True, text=True)
        assert r.returncode == 1 and "not supported" in r.stderr, extra
    zero = tmp_path / "zero.txt"
    zero.write_text("3\t0\n")
    r = subprocess.run(base + ["-o", str(tmp_path / "o2"), "-b", "2", str(zero)], capture_output=True, text=True)
    assert r.returncode == 1 and "Error" in r.stderr
    (tmp_path / "o3").mkdir()
    (tmp_path / "o3" / "abundance_2").write_text("")
    r = subprocess.run(base + ["-o", str(tmp_path / "o3"), "--matrix-to-directories", os.path.join(SRC, "tcc.mtx")],
                       capture_output=True, text=True)
    assert r.returncode == 1 and "Error: file %s exists and is not a directory" % (tmp_path / "o3" / "abundance_2") in r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# library level
# ---------------------------------------------------------------------------------------------------------------------
def _rows(c, rng, big):
    """Dense rows over the table's ECs: empty, one draw, one non-zero EC, a random subset with the last EC zero and one
    with it non-zero, and the table's own counts (big: with more than 10^6 in all; else capped at 50)."""
    n = c.n
    own = c.counts.copy() if big else np.minimum(c.counts, 50)
    if big and own.sum() <= 10 ** 6:
        own[rng.integers(0, n)] += 1_000_000
    rows = [np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)]
    rows[1][rng.integers(0, max(1, n - 1))] = 1
    rows[2][rng.integers(0, max(1, n - 1))] = 777
    for last in (0, 1):
        r = np.where(rng.random(n) < 0.5, own, 0).astype(np.uint32)
        r[-1] = own[-1] if last else 0
        rows.append(r)
    rows.append(own)
    return rows


def _csr_rows(rows):
    ids = [np.flatnonzero(r).astype(np.uint32) for r in rows]
    ro = np.zeros(len(rows) + 1, np.uint64)
    ro[1:] = np.cumsum([len(i) for i in ids])
    return ro, np.concatenate(ids), np.concatenate([r[i] for r, i in zip(rows, ids)]).astype(np.uint32)


def _effs(c, R):
    return np.stack([O.eff_lens(c.lens, O.mean_fl_trunc(np.zeros(1000, np.uint32), 120.0 + 15 * r, 20.0)) for r in range(R)])


def _run(ix, c, rows, eff, B, want_samples):
    ro, ids, vals = _csr_rows(rows)
    got = {}

    def on_chunk(first, est, rounds, samples):
        assert first == sum(len(v[1]) for v in got.values())          # chunks come in order
        got[first] = (est, rounds, samples)
    K.tcc_bootstrap(ix, c.off, c.tids, ro, ids, vals, eff, SEED, B, on_chunk, want_samples)
    est = np.concatenate([v[0] for v in got.values()])
    rounds = np.concatenate([v[1] for v in got.values()])
    samples = np.concatenate([v[2] for v in got.values()]) if want_samples else None
    assert len(rounds) == len(rows) * B
    return est, rounds, samples, len(got)


def _check(c, rows, eff, B, est, rounds, samples, problems):
    for g in problems:
        r, b = divmod(g, B)
        s = O.bootstrap_sample(rows[r], SEED, b)
        if samples is not None:
            np.testing.assert_array_equal(samples[g], s, err_msg="problem %d (row %d)" % (g, r))
        alpha, n = O.em(c.off, c.tids, s, eff[r], c.T, counts_w=rows[r])
        assert rounds[g] == n, g
        np.testing.assert_array_equal(est[g], alpha, err_msg="problem %d (row %d)" % (g, r))


def _knobs(monkeypatch, chunk):
    for k in KNOB_VARS + ("KB_TCC_BS_CHUNK",):
        monkeypatch.delenv(k, raising=False)
    if chunk:
        monkeypatch.setenv("KB_TCC_BS_CHUNK", chunk)


@pytest.fixture(scope="module")
def cases():
    return {}


@pytest.fixture(scope="module")
def indices():
    out = {name: K.KmerIndex(util.dataset(name)["index"], device=0) for name in ("synth_small", "config1", "abundant")}
    yield out
    for ix in out.values():
        ix.close()


@pytest.mark.parametrize("chunk", ["", "5", "1"])
@pytest.mark.parametrize("table", ["golden_synth", "golden_config1", "wide", "singletons", "one_ec", "hub"])
def test_tcc_bootstrap_every_problem(cases, indices, monkeypatch, table, chunk):
    """Six rows x 4 bootstraps, every problem checked; the last row draws more than 10^6 times."""
    c = _case(cases, table)
    _knobs(monkeypatch, chunk)
    rows = _rows(c, np.random.default_rng(len(table)), big=True)
    eff = _effs(c, len(rows))
    B = 4
    est, rounds, samples, n_chunks = _run(indices[c.index], c, rows, eff, B, True)
    if chunk:
        assert n_chunks == -(-len(rows) * B // int(chunk))
    assert rows[-1].sum() > 10 ** 6
    _check(c, rows, eff, B, est, rounds, samples, range(len(rows) * B))


@pytest.mark.parametrize("chunk", ["", "3000"])
def test_tcc_bootstrap_past_one_launch(cases, indices, monkeypatch, chunk):
    """9 rows x 911 bootstraps = 8 199 problems: more than KB_EM_MAX_BATCH (8 192), so chunks split rows."""
    c = _case(cases, "golden_synth")
    _knobs(monkeypatch, chunk)
    rng = np.random.default_rng(8199)
    rows = _rows(c, rng, big=False)
    rows += [np.where(rng.random(c.n) < 0.3, np.minimum(c.counts, 50), 0).astype(np.uint32) for _ in range(9 - len(rows))]
    eff = _effs(c, len(rows))
    B = 911
    est, rounds, samples, n_chunks = _run(indices[c.index], c, rows, eff, B, False)
    assert n_chunks == (2 if not chunk else 3)
    spots = {0, B - 1, B, 3000, 6000, 8191, 8192, 8198} | {r * B + b for r in range(len(rows)) for b in (0, 1, B - 1)}
    spots |= set(int(x) for x in rng.choice(len(rows) * B, 10, replace=False))
    _check(c, rows, eff, B, est, rounds, None, sorted(spots))


@pytest.mark.parametrize("table", ["golden_synth", "wide", "hub"])
def test_one_row_equals_quant_bootstrap(cases, indices, monkeypatch, table):
    """kb_tcc_bootstrap_run on one row = kb_bootstrap_run on the same table imported into a run: same draws (sparse
    against dense cumulative table), same EMs."""
    c = _case(cases, table)
    _knobs(monkeypatch, "")
    ix = indices[c.index]
    B, mode = 6, "flens"
    mc = _imported(ix, c, mode)
    r = mc.run_bootstrap(B, seed=SEED, want_samples=True, **_fld(mode))
    mc.close()
    eff, _, _ = K.eff_lens(ix, flens=c.flens)
    est, rounds, samples, _ = _run(ix, c, [c.counts], eff, B, True)
    for b in range(B):
        np.testing.assert_array_equal(samples[b], r["samples"][b][:c.n], err_msg="sample %d" % b)
        np.testing.assert_array_equal(est[b], r["est_counts"][b], err_msg="sample %d" % b)
        assert rounds[b] == r["rounds"][b]

