"""GPU: -p/--priors.  quant and quant-tcc through the command line against the reference's bytes in
tests/golden/priors.json.gz (make_golden_priors.py) at every EM kernel and chunk size; kb_em_set_priors / kb_tcc_run_priors
against the oracle's EM started from the same priors (tests/priors_oracle.py); and the invariants of the start path."""
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from tests import priors_oracle as P
from tests import util
from tests.test_gpu_em_shapes import KNOB_VARS, _case, _collector, _fld, _set_knobs, cases, indices  # noqa: F401

pytestmark = pytest.mark.gpu

GOLD = json.loads(gzip.open(os.path.join(util.GOLDEN, "priors.json.gz")).read())
CLI = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")
SRC = os.path.join(util.GOLDEN, "quanttcc")
EM_MODES = {"components": {}, "streamed": {"KB_EM_COMP_SMEM": "0"}, "grid": {"KB_EM_SHAPE": "1"}}
TCC_MODES = {"auto": {}, "chunk1": {"KB_TCC_CHUNK": "1"}, "bs_chunk1": {"KB_TCC_BS_CHUNK": "1"}}
PRIORS_LINES = ("[   em] reading priors", "[   em] number of priors", "        defaulting")


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("priors_in")
    for fn, text in GOLD["inputs"].items():
        with open(d / fn, "w", newline="") as f:
            f.write(text)
    return d


def run(args, cwd, env_extra):
    env = {k: v for k, v in os.environ.items() if k not in KNOB_VARS + ("KB_EM_COMP_SMEM", "KB_TCC_BS_CHUNK")}
    env.update(env_extra)
    r = subprocess.run([CLI] + args, cwd=str(cwd), capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return r


def outputs(out):
    got = {}
    for d, _, fns in os.walk(out):
        for fn in fns:
            if fn != "run_info.json":
                p = os.path.join(d, fn)
                got[os.path.relpath(p, out)] = open(p).read()
    return got


def quant_args(name, out):
    ds, args = GOLD["quant"][name]
    d = os.path.join(util.GOLDEN, ds)
    reads = [os.path.join(d, "reads_1.fastq.gz")] + ([] if "--single" in args else [os.path.join(d, "reads_2.fastq.gz")])
    return ["quant", "-i", os.path.join(d, "transcripts.kidx"), "-o", str(out)] + list(args) + reads


def priors_lines(stderr):
    return [l for l in stderr.splitlines() if l.startswith(PRIORS_LINES)]


@pytest.mark.parametrize("mode", list(EM_MODES))
@pytest.mark.parametrize("name", sorted(GOLD["quant"]))
def test_quant_identical_to_reference(inputs, tmp_path, name, mode):
    r = run(quant_args(name, tmp_path / "o"), inputs, EM_MODES[mode])
    assert outputs(tmp_path / "o") == GOLD["outputs"][name]
    assert priors_lines(r.stderr) == GOLD["stderr"][name]


@pytest.mark.parametrize("name", ["q_prob", "q_counts_p"])
def test_quant_h5_and_two_devices(inputs, tmp_path, name):
    """Without --plaintext, h5dump of abundance.h5 gives the reference's text; --devices 0,0 gives the same bytes."""
    args = [a for a in quant_args(name, tmp_path / "h") if a != "--plaintext"]
    run(args, inputs, {})
    run(["h5dump", "-o", str(tmp_path / "d"), str(tmp_path / "h" / "abundance.h5")], inputs, {})
    got = outputs(tmp_path / "d")
    for fn, text in GOLD["outputs"][name].items():
        assert got[fn] == text, fn
    run(quant_args(name, tmp_path / "m") + ["--devices", "0,0"], inputs, {})
    assert outputs(tmp_path / "m") == GOLD["outputs"][name]


@pytest.mark.parametrize("mode", list(TCC_MODES))
@pytest.mark.parametrize("name", sorted(GOLD["tcc"]))
def test_tcc_identical_to_reference(inputs, tmp_path, name, mode):
    args, tcc = GOLD["tcc"][name]
    args = [os.path.join(SRC, a) if a.startswith("fld_") else a for a in args]
    cmd = ["quant-tcc", "-i", os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx"), "-e",
           os.path.join(SRC, "matrix.ec"), "-o", str(tmp_path / "o")] + args + [os.path.join(SRC, tcc)]
    r = run(cmd, inputs, TCC_MODES[mode])
    assert outputs(tmp_path / "o") == GOLD["outputs"][name]
    assert priors_lines(r.stderr) == GOLD["stderr"][name]


# ---- the library against the oracle ------------------------------------------------------------------------------
TABLES = ["golden_synth", "golden_config1", "wide", "hub", "many"]
LIB_MODES = {"components": {}, "streamed": {"KB_EM_COMP_SMEM": "0"}, "shape1": {"KB_EM_SHAPE": "1"},
             "batched": {"KB_EM_SHAPE": "-1", "KB_EM_TPB": "256"}}


def random_priors(T, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "prob":
        v = rng.random(T)
        v[rng.random(T) < 0.2] = 0.0
        return v / v.sum()
    c = rng.integers(0, 3000, T).astype(np.float64)
    c[rng.random(T) < 0.3] = 0.0
    s = 0.0
    for x in c:
        s += x
    return (c + 1.0) / (s + T)           # read_priors' pseudocount arithmetic, in file order


_oracle = {}


def oracle_em(c, mode, kind):
    key = (c.name, mode, kind)
    if key not in _oracle:
        pri = random_priors(c.T, kind, len(c.name))
        _oracle[key] = (pri,) + P.em(c.off, c.tids, c.counts, c.eff(mode), c.T, alpha0=pri)
    return _oracle[key]


@pytest.mark.parametrize("knob", list(LIB_MODES))
@pytest.mark.parametrize("kind", ["prob", "counts"])
@pytest.mark.parametrize("table", TABLES)
def test_em_run_table_with_priors_equals_oracle(cases, indices, monkeypatch, table, kind, knob):
    monkeypatch.delenv("KB_EM_COMP_SMEM", raising=False)
    _set_knobs(monkeypatch, LIB_MODES[knob])
    c = _case(cases, table)
    pri, alpha, rounds = oracle_em(c, "flens", kind)
    mc = _collector(indices[c.index], c, "flens")
    mc.set_priors(pri)
    r = mc.run_em(table=(c.off, c.tids, c.counts), **_fld("flens"))
    assert r["rounds"] == rounds
    np.testing.assert_array_equal(r["est_counts"], alpha)
    mc.close()


def test_priors_invariants(indices, monkeypatch):
    """On a pseudoaligned run (kb_em_run): 1 / T as priors is the uniform start bit for bit; bootstraps ignore priors;
    None restores the uniform start; a wrong count is refused and changes nothing."""
    _set_knobs(monkeypatch, {})
    ds = util.dataset("synth_small")
    mc = K.MinCollector(indices["synth_small"], paired=True)
    mc.process_buffer(*util.batch(ds, True), want_handles=False)
    T = indices["synth_small"].num_trans
    base = mc.run_em()
    bs0 = mc.run_bootstrap(3, seed=7)
    assert bs0["rounds"].min() > 0
    mc.set_priors(np.full(T, 1.0 / T))
    same = mc.run_em()
    assert same["rounds"] == base["rounds"] and np.array_equal(same["est_counts"], base["est_counts"])
    pri = random_priors(T, "prob", 3)
    mc.set_priors(pri)
    moved = mc.run_em()
    assert not np.array_equal(moved["est_counts"], base["est_counts"])
    assert np.array_equal(mc.run_bootstrap(3, seed=7)["est_counts"], bs0["est_counts"])
    with pytest.raises(K.KallistoB200Error) as e:
        mc.set_priors(pri[:-1])
    assert e.value.code == -1            # KB_ERR_INVALID
    again = mc.run_em()
    assert np.array_equal(again["est_counts"], moved["est_counts"])
    mc.set_priors(None)
    back = mc.run_em()
    assert back["rounds"] == base["rounds"] and np.array_equal(back["est_counts"], base["est_counts"])
    mc.close()


@pytest.mark.parametrize("chunk", [None, "1", "3"])
@pytest.mark.parametrize("table", ["golden_synth", "wide", "hub"])
def test_tcc_run_priors_equals_oracle(cases, indices, monkeypatch, table, chunk):
    """Many samples (the table's counts scaled, shuffled, thinned, and one all-zero row), every one started from the
    priors, equal the oracle per sample; priors of 1 / T equal no priors bit for bit."""
    _set_knobs(monkeypatch, {} if chunk is None else {"KB_TCC_CHUNK": chunk})
    c = _case(cases, table)
    rng = np.random.default_rng(11)
    dense = [c.counts, np.zeros(c.n, np.uint32)]
    for k in range(5):
        x = rng.permutation(c.counts) // (k + 1)
        x[rng.random(c.n) < 0.3] = 0
        dense.append(x.astype(np.uint32))
    rows = [[(int(e), int(v)) for e in np.flatnonzero(d) for v in (d[e],)] for d in dense]
    eff = c.eff("flens")
    pri = random_priors(c.T, "counts", 5)
    ix = indices[c.index]
    est, rounds = K.tcc_run(ix, c.sets(), rows, eff, priors=pri)
    for s, d in enumerate(dense):
        a, r = P.em(c.off, c.tids, d, eff, c.T, alpha0=pri)
        assert rounds[s] == r, s
        np.testing.assert_array_equal(est[s], a)
    uni, ru = K.tcc_run(ix, c.sets(), rows, eff, priors=np.full(c.T, 1.0 / c.T))
    none, rn = K.tcc_run(ix, c.sets(), rows, eff)
    assert np.array_equal(uni, none) and np.array_equal(ru, rn)
