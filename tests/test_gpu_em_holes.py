"""GPU: equivalence classes without a transcript in a table given from the host (kb_em_run_table, kb_tcc_run).

Such an EC takes an id and a count and adds to no sum: the CPU oracle (oracle.em) skips it, and the host-side builder of
the EM structure gives it no row.  The table is tests/test_gpu_em_shapes.py's golden table of synth_small (T = 491)
with four empty ECs put in -- the first, two in a row, the last -- and goes through the same launch knobs and chunk sizes,
bit for bit and round count included.  (A run never records an empty set, so the imported entry point has no such
case.)"""
import numpy as np
import pytest

import kallisto_b200 as K
from tests import test_gpu_em_shapes as S
from tests import util

pytestmark = pytest.mark.gpu

HOLES_AT = (0, 7, 8)       # ids of the empty ECs, besides the last one


@pytest.fixture(scope="module")
def case():
    c = S.Case("golden_synth")
    lens = list(np.diff(c.off.astype(np.int64)))
    counts = list(c.counts)
    for at in HOLES_AT:
        lens.insert(at, 0)
        counts.insert(at, 11 + at)
    lens.append(0)
    counts.append(1000)
    c.off = np.zeros(len(lens) + 1, np.uint64)
    c.off[1:] = np.cumsum(lens)
    c.counts = np.asarray(counts, np.uint32)
    c.n = len(counts)
    assert c.off[-1] == len(c.tids) and (np.diff(c.off.astype(np.int64)) == 0).sum() == len(HOLES_AT) + 1
    return c


@pytest.fixture(scope="module")
def index():
    ix = K.KmerIndex(util.dataset("synth_small")["index"], device=0)
    yield ix
    ix.close()


@pytest.mark.parametrize("knob", list(S.ALL_KNOBS))
def test_em_table_with_empty_ecs(case, index, monkeypatch, knob):
    S._set_knobs(monkeypatch, S.ALL_KNOBS[knob])
    mode = "flens" if knob != "shape2" else "ls"
    mc = S._collector(index, case, mode)
    S._check_em(mc.run_em(table=(case.off, case.tids, case.counts), **S._fld(mode)), case, mode)
    mc.close()


@pytest.mark.parametrize("tc", list(S.TCC_CASES))
def test_tcc_with_empty_ecs(case, index, monkeypatch, tc):
    chunk, knob, per_sample = S.TCC_CASES[tc]
    env = dict(S.ALL_KNOBS[knob])
    if chunk:
        env["KB_TCC_CHUNK"] = chunk
    S._set_knobs(monkeypatch, env)
    n_rows = 5
    ids, vals, ro = S._tcc_rows(case, n_rows, np.random.default_rng(11), empty_at=2)
    empty = np.flatnonzero(np.diff(case.off.astype(np.int64)) == 0)
    assert np.isin(empty, ids).all()            # every empty EC has a count in some row
    eff = case.eff("flens")
    if per_sample:
        eff = np.stack([S.O.eff_lens(case.lens, S.O.mean_fl_trunc(np.zeros(1000, np.uint32), 120.0 + 15 * s, 20.0))
                        for s in range(n_rows)])
    est, rounds = S._tcc_call(index, case, ids, vals, ro, eff)
    for s in range(n_rows):
        alpha, n = S.O.em(case.off, case.tids, S._dense(case, ids, vals, ro, s), eff[s] if per_sample else eff, case.T)
        assert rounds[s] == n, s
        np.testing.assert_array_equal(est[s], alpha, err_msg="sample %d" % s)
