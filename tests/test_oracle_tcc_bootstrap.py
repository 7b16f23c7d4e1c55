"""CPU: the oracle's model of a quant-tcc bootstrap (oracle.bootstrap_sample over the row's dense counts, then oracle.em on
the resampled counts with the row's ORIGINAL counts / eff_len as weights, written with the row's eff_lens) against every
bs_abundance*.tsv the unmodified reference wrote (tests/golden/quanttcc_bs.json.gz, from make_golden_quanttcc_bs.py).
This pins the model the device bootstrap of quant-tcc is held to."""
import gzip
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import util

SRC = os.path.join(util.GOLDEN, "quanttcc")
IDX = os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx")
GOLD = json.loads(gzip.open(os.path.join(util.GOLDEN, "quanttcc_bs.json.gz")).read())
CASES = GOLD["cases"]


def opt(args, name, default=None):
    return args[args.index(name) + 1] if name in args else default


def read_tcc(path, n_ec):
    """-> dense counts, one row per sample (matrix file) or a single row (two-column file), and whether it is a matrix."""
    lines = open(path).read().splitlines()
    if lines[0].startswith("%%MatrixMarket"):
        body = [l for l in lines[1:] if not l.startswith("%")]
        nrow = int(body[0].split()[0])
        rows = np.zeros((nrow, n_ec), np.uint32)
        for l in body[1:]:
            r, c, v = (int(x) for x in l.split())
            rows[r - 1, c - 1] = v
        return rows, True
    rows = np.zeros((1, n_ec), np.uint32)
    for l in lines:
        c, v = (int(x) for x in l.split())
        rows[0, c] = v
    return rows, False


def eff_of(args, lens, nrow):
    """The effective lengths of every row (src/main.cpp:2998-3028): 1 without fragment-length information."""
    if opt(args, "-l"):
        fl = O.mean_fl_trunc(np.zeros(1000, np.uint32), float(opt(args, "-l")), float(opt(args, "-s")))
        return [O.eff_lens(lens, fl)] * nrow
    if opt(args, "-f"):
        flds = [np.array(l.split(), np.uint32) for l in open(os.path.join(SRC, opt(args, "-f")))
                if l.strip() and not l.startswith("#")]
        return [O.eff_lens(lens, O.mean_fl_trunc(flds[r if len(flds) > 1 else 0])) for r in range(nrow)]
    return [np.ones(len(lens))] * nrow


def expected_bootstraps(args, tcc):
    """-> {relative path: text} of every bootstrap file the case writes."""
    ix = O.OracleIndex(IDX)
    sets = O.read_matrix_ec(os.path.join(SRC, "matrix.ec"))
    off = np.zeros(len(sets) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in sets])
    tids = np.array([t for s in sets for t in s], np.uint32)
    rows, is_matrix = read_tcc(os.path.join(SRC, tcc), len(sets))
    B, seed = int(opt(args, "-b", 0)), int(opt(args, "--seed", 42))
    effs = eff_of(args, ix.target_lens, len(rows))
    out = {}

    def text(eff, est):
        # an empty row's TPM is 0 / 0: the C++ stream writes the sign of that NaN ("-nan"), Python's %g does not
        tpm = O.tpm(est, eff)
        t = O.abundance_tsv(ix.target_names, ix.target_lens, eff, est, np.where(np.isnan(tpm), 0.0, tpm))
        if not np.isnan(tpm).any():
            return t
        lines = t.split("\n")
        for i in np.flatnonzero(np.isnan(tpm)):
            a = lines[i + 1].split("\t")
            a[4] = "-nan" if np.signbit(tpm[i]) else "nan"
            lines[i + 1] = "\t".join(a)
        return "\n".join(lines)
    for r, counts in enumerate(rows):
        if is_matrix:
            name = ("abundance_%d/bs_abundance_%%d.tsv" % (r + 1) if "--matrix-to-directories" in args
                    else "bs_abundance_%d_%%d.tsv" % (r + 1))
        else:
            name = "bs_abundance_%d.tsv"
        est, _ = O.em(off, tids, counts, effs[r], ix.n_targets)
        for b in range(B):
            if is_matrix and not (est > 0).any():         # a row without any estimate: B copies of it (main.cpp:3110-3124)
                out[name % b] = text(effs[r], est)
                continue
            alpha, _ = O.em(off, tids, O.bootstrap_sample(counts, seed, b), effs[r], ix.n_targets, counts_w=counts)
            out[name % b] = text(effs[r], alpha)
    return out


def golden_bootstraps(name):
    return {fn: t for fn, t in GOLD["outputs"][name].items() if os.path.basename(fn).startswith("bs_abundance")}


@pytest.mark.parametrize("name", list(CASES))
def test_bootstrap_files_identical_to_reference(name):
    args, tcc = CASES[name]
    exp, ref = expected_bootstraps(args, tcc), golden_bootstraps(name)
    assert sorted(exp) == sorted(ref)
    for fn in ref:
        assert exp[fn] == ref[fn], fn
    if "-b" in args:
        assert ref


def test_fixture_covers_the_sparse_and_the_empty_row():
    """tcc.mtx: row 3 holds 40 of the ECs, row 4 none -- the ECs the sparse resampling table skips, and a row whose
    bootstraps are copies of its (zero) estimate; the last EC is zero in some rows and not in others."""
    n_ec = len(O.read_matrix_ec(os.path.join(SRC, "matrix.ec")))
    rows, _ = read_tcc(os.path.join(SRC, "tcc.mtx"), n_ec)
    assert (rows[2] > 0).sum() == 40 and not rows[3].any()
    assert {bool(r[-1]) for r in rows} == {False, True}
