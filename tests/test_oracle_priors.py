"""CPU: -p/--priors.  The oracle's EM started from the priors (tests/priors_oracle.py) against the reference's outputs in
tests/golden/priors.json.gz (make_golden_priors.py); kb_read_priors (host only) against the reference's arithmetic; the
command line's handling of the option on the stand-in library of tests/stub."""
import gzip
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import priors_oracle as P
from tests import util
from tests.test_oracle_tcc_bootstrap import eff_of, opt, read_tcc

GOLD = json.loads(gzip.open(os.path.join(util.GOLDEN, "priors.json.gz")).read())
SRC = os.path.join(util.GOLDEN, "quanttcc")


def priors_for(name, T):
    """The start the reference's EM takes: the file's priors when their count is T, else None (uniform)."""
    v = P.read_priors_text(GOLD["inputs"][name])
    return v if len(v) == T else None


def tsv(ix, eff, est):
    return O.abundance_tsv(ix.target_names, ix.target_lens, eff, est, O.tpm(est, eff))


def test_uniform_start_is_oracle_em():
    """priors_oracle.em from 1 / T is oracle.em bit for bit: the restatement shares the oracle's model."""
    ix = O.OracleIndex(os.path.join(util.GOLDEN, "manyecs", "transcripts.kidx"))
    run = O.OracleRun(ix, True, 0, True)
    s1 = O.read_fastq(os.path.join(util.GOLDEN, "manyecs", "reads_1.fastq.gz"))
    s2 = O.read_fastq(os.path.join(util.GOLDEN, "manyecs", "reads_2.fastq.gz"))
    run.pseudoalign(*O.to_batch(s1, s2))
    off, tids, counts = run.ec_table()
    eff = O.eff_lens(ix.target_lens, O.mean_fl_trunc(run.flens()))
    a, r = O.em(off, tids, counts, eff, ix.n_targets)
    b, s = P.em(off, tids, counts, eff, ix.n_targets, alpha0=np.full(ix.n_targets, 1.0 / ix.n_targets))
    assert r == s and np.array_equal(a, b)


@pytest.mark.parametrize("name", sorted(GOLD["quant"]))
def test_quant_estimates_identical_to_reference(name):
    ds, args = GOLD["quant"][name]
    d = os.path.join(util.GOLDEN, ds)
    ix = O.OracleIndex(os.path.join(d, "transcripts.kidx"))
    single = "--single" in args
    strand = 1 if "--fr-stranded" in args else 0
    s1 = O.read_fastq(os.path.join(d, "reads_1.fastq.gz"))
    if single:
        run = O.OracleRun(ix, False, strand, False, fp_fl=int(float(opt(args, "-l"))))
        run.pseudoalign(*O.to_batch(s1))
        fl = O.mean_fl_trunc(np.zeros(1000, np.uint32), float(opt(args, "-l")), float(opt(args, "-s")))
    else:
        run = O.OracleRun(ix, True, strand, True)
        run.pseudoalign(*O.to_batch(s1, O.read_fastq(os.path.join(d, "reads_2.fastq.gz"))))
        fl = O.mean_fl_trunc(run.flens())
    off, tids, counts = run.ec_table()
    eff = O.eff_lens(ix.target_lens, fl)
    pf = opt(args, "--priors") or opt(args, "-p")
    est, _ = P.em(off, tids, counts, eff, ix.n_targets, alpha0=priors_for(pf, ix.n_targets))
    assert tsv(ix, eff, est) == GOLD["outputs"][name]["abundance.tsv"]
    # bootstraps start uniform whatever the priors (Bootstrap::run_em)
    for b in range(int(opt(args, "-b", 0))):
        alpha, _ = O.em(off, tids, O.bootstrap_sample(counts, 42, b), eff, ix.n_targets, counts_w=counts)
        assert tsv(ix, eff, alpha) == GOLD["outputs"][name]["bs_abundance_%d.tsv" % b]


@pytest.mark.parametrize("name", ["t_files_ls_counts", "t_dirs_b3_prob", "t_single_b2_counts"])
def test_tcc_estimates_identical_to_reference(name):
    args, tcc = GOLD["tcc"][name]
    ix = O.OracleIndex(os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx"))
    sets = O.read_matrix_ec(os.path.join(SRC, "matrix.ec"))
    off = np.zeros(len(sets) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in sets])
    tids = np.array([t for s in sets for t in s], np.uint32)
    rows, is_matrix = read_tcc(os.path.join(SRC, tcc), len(sets))
    effs = eff_of(args, ix.target_lens, len(rows))
    alpha0 = priors_for(opt(args, "--priors") or opt(args, "-p"), ix.n_targets)
    assert alpha0 is not None
    out = GOLD["outputs"][name]
    for r, counts in enumerate(rows):
        est, _ = P.em(off, tids, counts, effs[r], ix.n_targets, alpha0=alpha0)
        if not is_matrix:
            fn = "abundance.tsv"
        elif "--matrix-to-directories" in args:
            fn = "abundance_%d/abundance.tsv" % (r + 1)
        else:
            fn = "abundance_%d.tsv" % (r + 1)
        if not (est > 0).any():
            continue                  # the empty row: its TPM column is 0 / 0 (test_oracle_tcc_bootstrap writes that)
        assert tsv(ix, effs[r], est) == out[fn], fn


def test_fixture_priors_change_the_estimates():
    """The priors that apply move the estimates away from the uniform start's; a wrong count and an empty file do not."""
    o = GOLD["outputs"]
    assert o["q_prob"]["abundance.tsv"] != o["q_empty"]["abundance.tsv"]
    assert o["q_short"]["abundance.tsv"] == o["q_empty"]["abundance.tsv"] == o["q_long"]["abundance.tsv"]
    assert o["q_prob"]["bs_abundance_1.tsv"] == o["q_empty"]["bs_abundance_1.tsv"]
    assert all(e["exit"] != 0 for e in GOLD["aborts"].values())


# ---- kb_read_priors (host only) ---------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", sorted(f for f in GOLD["inputs"] if f.endswith(".txt") and f != "t2g.txt"))
def test_read_priors_matches_the_reference_arithmetic(fn, tmp_path):
    p = tmp_path / fn
    p.write_bytes(GOLD["inputs"][fn].encode())
    got = K.read_priors(str(p))
    exp = P.read_priors_text(GOLD["inputs"][fn])
    assert got.dtype == np.float64 and np.array_equal(got, exp)


def test_read_priors_two_calls(tmp_path):
    import ctypes as C
    p = tmp_path / "p.txt"
    p.write_text("3\n4\n5\n")
    n = C.c_uint64(0)
    out = np.zeros(2, np.float64)
    assert K.lib().kb_read_priors(str(p).encode(), out.ctypes.data_as(C.c_void_p), 2, C.byref(n)) == K.KB_OK
    assert n.value == 3 and not out.any()                       # cap too small: only the count
    assert np.array_equal(K.read_priors(str(p)), np.array([4.0, 5.0, 6.0]) / 15.0)


@pytest.mark.parametrize("text,code,line", [(None, -5, None), ("0.5\n\n0.5\n", -1, 2), ("0.5\nabc\n", -1, 2),
                                            ("1e999\n", -1, 1)])
def test_read_priors_errors(text, code, line, tmp_path):
    p = tmp_path / "p.txt"
    if text is not None:
        p.write_text(text)
    with pytest.raises(K.KallistoB200Error) as e:
        K.read_priors(str(p))
    assert e.value.code == code
    if line:
        assert ("line %d of priors file" % line) in str(e.value)
    else:
        assert "could not open priors file" in str(e.value)


# ---- the command line on the stand-in library -------------------------------------------------------------------
@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    from tests.test_cli_host_pipeline import CSRC, INC
    if not shutil.which("g++"):
        pytest.skip("no g++")
    d = str(tmp_path_factory.mktemp("stubpriors"))
    lib = os.path.join(d, "libkallisto_b200.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I" + INC, "-I" + CSRC, "-o", lib,
                           os.path.join(util.ROOT, "tests", "stub", "stub_priors.cpp")])
    exe = os.path.join(d, "cli")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + INC, "-I" + CSRC, "-o", exe, os.path.join(CSRC, "cli_main.cpp"),
                           "-L" + d, "-lkallisto_b200", "-Wl,-rpath," + d, "-lz", "-lpthread"])
    ds = os.path.join(util.GOLDEN, "synth_small")
    return dict(exe=exe, idx=os.path.join(ds, "transcripts.kidx"), reads=[os.path.join(ds, "reads_%d.fastq.gz" % m) for m in (1, 2)])


def run_quant(s, out, args):
    return subprocess.run([s["exe"], "quant", "-i", s["idx"], "-o", str(out), "--plaintext"] + args + s["reads"],
                          capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("flag", ["--priors", "-p"])
@pytest.mark.parametrize("lines", [3, 2])
def test_cli_accepts_priors(stub, tmp_path, flag, lines):
    """The stand-in index has 3 targets: 3 lines apply (kb_em_set_priors), 2 fall back to uniform with the two lines."""
    p = tmp_path / "p.txt"
    p.write_text("0.2\n0.3\n0.5\n"[: 4 * lines])
    r = run_quant(stub, tmp_path / "o", [flag, str(p)])
    assert r.returncode == 0, r.stderr
    assert "[   em] reading priors from file %s\n" % p in r.stderr
    mismatch = "[   em] number of priors does not match number of transcripts.\n        defaulting to uniform priors.\n"
    assert (mismatch in r.stderr) == (lines != 3)
    assert r.stderr.index("reading priors") < r.stderr.index("[   em] quantifying the abundances")
    assert (tmp_path / "o" / "abundance.tsv").exists()


@pytest.mark.parametrize("text,msg", [(None, "Error: could not open priors file {p}\n"),
                                      ("0.5\nabc\n", "Error: line 2 of priors file {p} is not a number\n")])
def test_cli_priors_errors_stop_before_any_read(stub, tmp_path, text, msg):
    p = tmp_path / "p.txt"
    if text is not None:
        p.write_text(text)
    r = run_quant(stub, tmp_path / "o", ["--priors", str(p)])
    assert r.returncode == 1 and msg.format(p=p) in r.stderr
    assert "finding pseudoalignments" not in r.stderr and "[index]" not in r.stderr
    ec = os.path.join(SRC, "matrix.ec")
    r = subprocess.run([stub["exe"], "quant-tcc", "-i", stub["idx"], "-e", ec, "-o", str(tmp_path / "t"), "-p", str(p),
                        os.path.join(SRC, "tcc.mtx")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 1 and msg.format(p=p) in r.stderr
    assert "[index]" not in r.stderr and "Running EM" not in r.stderr


@pytest.mark.parametrize("cmd", ["quant", "quant-tcc"])
def test_usage_lists_priors(stub, cmd):
    r = subprocess.run([stub["exe"], cmd], capture_output=True, text=True)
    assert "-p, --priors                  Priors for the EM algorithm, either as raw counts or as" in r.stdout
