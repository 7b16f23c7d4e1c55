"""GPU: the single-problem EM with each slice's entries resident in shared memory (em_component_kernel rebuilding the
weights from the row counts and the effective lengths) against the CPU oracle, bit for bit and round count included.

The tables are the gene-like, late-converging and singleton-only tables of tests/test_gpu_em_components.py and the
golden synth_small table with empty ECs of tests/test_gpu_em_holes.py.  Each runs through kb_em_run_table and (except
the one with empty ECs, which a run never records) through an imported run, with the shared-memory budget of the
resident layout (KB_EM_COMP_SMEM) unset, exactly at the largest slice's resident bytes, and one byte below, where the
streamed kernel runs on the same slices.  The reported kernel and number of blocks are checked in every case, so that
a silent fall-back cannot pass."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components
import torch

import kallisto_b200 as K
from tests import test_gpu_em_components as CC
from tests import test_gpu_em_holes as H
from tests import test_gpu_em_shapes as S
from tests import util

pytestmark = pytest.mark.gpu

SMEM_VAR = "KB_EM_COMP_SMEM"
TABLES = ["genes", "genes_small", "late", "singletons", "holes"]
BUDGETS = ["default", "max", "max-1"]


def _slices(off, tids, T, sms):
    """The layout's slices: components sorted by their smallest transcript id, sizes transcripts + rows + entries,
    target ceil(total / SMs), component -> floor(start / target).  -> (slices, largest slice's resident bytes)."""
    ln = np.diff(off.astype(np.int64))
    multi = np.flatnonzero(ln > 1)
    rows = np.repeat(np.arange(len(multi)), ln[multi])
    ent = tids[np.repeat(ln > 1, ln)].astype(np.int64)
    first = tids[off[:-1].astype(np.int64)[multi]].astype(np.int64)
    g = sp.coo_matrix((np.ones(len(ent)), (first[rows], ent)), shape=(T, T))
    n_comp, comp = connected_components(g, directed=False)
    root = np.full(n_comp, T, np.int64)
    np.minimum.at(root, comp, np.arange(T))
    size = 1 + np.bincount(ent, minlength=T) + np.bincount(first, minlength=T)
    order = np.lexsort((np.arange(T), root[comp]))
    scan = np.concatenate([[0], np.cumsum(size[order])])
    pos = np.empty(T, np.int64)
    pos[order] = np.arange(T)
    total = int(scan[-1])
    target = -(-total // sms)
    n = (total - 1) // target + 1
    sl = scan[pos[root]][comp] // target            # slice of every transcript
    nt = np.bincount(sl, minlength=n)
    nr = np.bincount(sl[first], minlength=n)
    ne = np.bincount(sl[ent], minlength=n)
    return n, int((36 * nt + 16 * nr + 4 * ne + 8).max())


def _holes():
    """tests/test_gpu_em_holes.py's table: the golden synth_small table with empty ECs put in."""
    c = S.Case("golden_synth")
    lens = list(np.diff(c.off.astype(np.int64)))
    counts = list(c.counts)
    for at in H.HOLES_AT:
        lens.insert(at, 0)
        counts.insert(at, 11 + at)
    lens.append(0)
    counts.append(1000)
    c.off = np.zeros(len(lens) + 1, np.uint64)
    c.off[1:] = np.cumsum(lens)
    c.counts = np.asarray(counts, np.uint32)
    c.n = len(counts)
    return c


@pytest.fixture(scope="module")
def cases():
    return {}


@pytest.fixture(scope="module")
def indices():
    names = set(CC.INDEX_OF.values()) | {"synth_small"}
    out = {name: K.KmerIndex(util.dataset(name)["index"], device=0) for name in names}
    yield out
    for ix in out.values():
        ix.close()


def _case(cases, name):
    if name not in cases:
        c = _holes() if name == "holes" else CC.Case(name)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        c.slices, c.resident_bytes = _slices(c.off, c.tids, c.T, sms)
        if name != "holes":
            assert c.slices == c.expected_blocks(None)
        cases[name] = c
    return cases[name]


def _run(cases, indices, monkeypatch, table, budget, imported):
    c = _case(cases, table)
    S._set_knobs(monkeypatch, {})
    monkeypatch.delenv(CC.CAP_VAR, raising=False)
    monkeypatch.delenv(SMEM_VAR, raising=False)
    v = {"default": None, "max": c.resident_bytes, "max-1": c.resident_bytes - 1}[budget]
    if v is not None:
        monkeypatch.setenv(SMEM_VAR, str(v))
    mode = "ls" if imported else "flens"
    ix = indices[c.index]
    if imported:
        mc = S._imported(ix, c, mode)
        r = mc.run_em(**S._fld(mode))
    else:
        mc = S._collector(ix, c, mode)
        r = mc.run_em(table=(c.off, c.tids, c.counts), **S._fld(mode))
    alpha, rounds = c.em(mode)
    assert r["rounds"] == rounds
    np.testing.assert_array_equal(r["est_counts"], alpha)
    tm = mc.timings()
    assert tm["em_comp_blocks"] == c.slices
    assert tm["em_comp_resident"] == (0 if budget == "max-1" else 1)
    mc.close()


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("table", TABLES)
def test_resident_table(cases, indices, monkeypatch, table, budget):
    _run(cases, indices, monkeypatch, table, budget, imported=False)


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("table", [t for t in TABLES if t != "holes"])
def test_resident_imported(cases, indices, monkeypatch, table, budget):
    _run(cases, indices, monkeypatch, table, budget, imported=True)
