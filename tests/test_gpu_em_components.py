"""GPU: the single-problem EM solved one connected component per block (em_component_kernel) against the CPU oracle,
bit for bit and round count included, and the fall-back to the grid-wide kernel when a component does not fit.

The tables are generated from seeds over the targets of stored indices, gene-like: every EC lies inside one gene of 1 to
15 transcripts, gene membership is a random permutation of the transcript ids (a component's ids interleave with
other components'), EC ids are shuffled.  One table adds a gene whose counts are near 10^6 and converges long after the
rest (blocks without a change wait for it every round), one has no multi-transcript EC at all.  Every table runs
through kb_em_run_table and through an imported run (device EC numbering, kb_em_run) at the default component cap,
at caps of 1, 7 and 64, and at caps exactly at and one below the largest component.  The reported number of component
blocks is checked in every case, so that a silent fall-back cannot pass."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components
import torch

import kallisto_b200 as K
from oracle import oracle as O
from tests import util
from tests.test_gpu_em_shapes import _collector, _counts, _csr, _fld, _imported, _set_knobs

pytestmark = pytest.mark.gpu

INDEX_OF = {"genes": "abundant", "genes_small": "synth_small", "late": "abundant", "singletons": "config1"}
TABLES = list(INDEX_OF)
CAP_VAR = "KB_EM_COMP_CAP"


def _genes(rng, T):
    """Transcript ids in a random order, cut into genes of 1 + Poisson(3) transcripts (at most 15)."""
    perm = rng.permutation(T)
    genes, i = [], 0
    while i < T:
        n = min(15, 1 + int(rng.poisson(3.0)), T - i)
        genes.append(np.sort(perm[i:i + n]))
        i += n
    return genes


def _gene_sets(rng, g, n_max):
    """Distinct multi-transcript subsets of one gene, plus a singleton now and then."""
    sets = set()
    if len(g) >= 2:
        for _ in range(int(rng.integers(1, n_max + 1))):
            k = int(rng.integers(2, len(g) + 1))
            sets.add(tuple(int(x) for x in np.sort(rng.choice(g, k, replace=False))))
    if rng.random() < 0.5:
        sets.add((int(rng.choice(g)),))
    return list(sets)


def _table(name, T, rng):
    if name == "singletons":
        sets = [(int(t),) for t in rng.choice(T, T // 2, replace=False)]
        counts = _counts(rng, len(sets))
    else:
        genes = _genes(rng, T)
        sets = [s for g in genes for s in _gene_sets(rng, g, 12)]
        counts = _counts(rng, len(sets))
        if name == "late":
            # the largest gene: every pair of its transcripts an EC with a count near 10^6
            g = max(genes, key=len)
            late = {tuple(int(x) for x in np.sort(p)) for p in [(a, b) for i, a in enumerate(g) for b in g[i + 1:]]}
            sets = [s for s in sets if not set(s) <= set(int(x) for x in g)] + sorted(late)
            counts = np.concatenate([_counts(rng, len(sets) - len(late)),
                                     rng.integers(900_000, 1_100_000, len(late)).astype(np.uint32)])
    order = rng.permutation(len(sets))                 # EC ids in no particular order
    sets = [sets[i] for i in order]
    off, tids = _csr(sets)
    return off, tids, np.asarray(counts, np.uint32)[order]


class Case:
    def __init__(self, name):
        rng = np.random.default_rng([ord(ch) for ch in name])
        self.name, self.index = name, INDEX_OF[name]
        ds = util.dataset(self.index)
        self.flens = np.asarray(util.golden_ecs(ds, "paired")["flens"], np.uint32)
        self.lens = O.OracleIndex(ds["index"]).target_lens
        self.T = len(self.lens)
        self.off, self.tids, self.counts = _table(name, self.T, rng)
        self.n = len(self.counts)
        self.imp = rng.permutation(self.n)
        self.first = np.arange(self.n, dtype=np.int64) * 3 + 5
        self._em, self._eff = {}, {}
        # component sizes (transcripts + rows + entries) and the slices of the layout
        ln = np.diff(self.off.astype(np.int64))
        multi = np.flatnonzero(ln > 1)
        rows = np.repeat(np.arange(len(multi)), ln[multi])
        ent = np.concatenate([self.tids[int(self.off[e]):int(self.off[e + 1])] for e in multi]) if len(multi) else \
            np.zeros(0, np.uint32)
        first = self.tids[self.off[multi].astype(np.int64)] if len(multi) else np.zeros(0, np.uint32)
        g = sp.coo_matrix((np.ones(len(ent)), (first[rows], ent)), shape=(self.T, self.T))
        _, comp = connected_components(g, directed=False)
        size = np.ones(self.T, np.int64) + np.bincount(ent, minlength=self.T) + np.bincount(first, minlength=self.T)
        self.max_comp = int(np.bincount(comp, weights=size).max())
        self.total = int(size.sum())

    def eff(self, mode):
        if mode not in self._eff:
            m, s = {"flens": (0.0, 0.0), "ls": (200.0, 20.0)}[mode]
            fl = self.flens if mode == "flens" else np.zeros(1000, np.uint32)
            self._eff[mode] = O.eff_lens(self.lens, O.mean_fl_trunc(fl, m, s))
        return self._eff[mode]

    def em(self, mode):
        if mode not in self._em:
            self._em[mode] = O.em(self.off, self.tids, self.counts, self.eff(mode), self.T)
        return self._em[mode]

    def expected_blocks(self, cap):
        """Slices of the layout: target ceil(total / SMs), component -> floor(start / target); 0 = fall-back."""
        if cap is not None and self.max_comp > cap:
            return 0
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        target = -(-self.total // sms)
        return (self.total - 1) // target + 1


@pytest.fixture(scope="module")
def cases():
    return {}


@pytest.fixture(scope="module")
def indices():
    out = {name: K.KmerIndex(util.dataset(name)["index"], device=0) for name in set(INDEX_OF.values())}
    yield out
    for ix in out.values():
        ix.close()


def _case(cases, name):
    if name not in cases:
        cases[name] = Case(name)
    return cases[name]


CAPS = ["default", "1", "7", "64", "max", "max-1"]


def _cap(c, cap):
    if cap.isdigit():
        return int(cap)
    return {"default": None, "max": c.max_comp, "max-1": c.max_comp - 1}[cap]


def _check(mc, r, c, mode, cap):
    alpha, rounds = c.em(mode)
    assert r["rounds"] == rounds
    np.testing.assert_array_equal(r["est_counts"], alpha)
    blocks = c.expected_blocks(cap)
    assert mc.timings()["em_comp_blocks"] == blocks
    return blocks


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("table", TABLES)
def test_components_table(cases, indices, monkeypatch, table, cap):
    c = _case(cases, table)
    _set_knobs(monkeypatch, {})
    v = _cap(c, cap)
    if v is not None:
        monkeypatch.setenv(CAP_VAR, str(v))
    mc = _collector(indices[c.index], c, "flens")
    _check(mc, mc.run_em(table=(c.off, c.tids, c.counts), **_fld("flens")), c, "flens", v)
    mc.close()


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("table", TABLES)
def test_components_imported(cases, indices, monkeypatch, table, cap):
    c = _case(cases, table)
    _set_knobs(monkeypatch, {})
    v = _cap(c, cap)
    if v is not None:
        monkeypatch.setenv(CAP_VAR, str(v))
    mc = _imported(indices[c.index], c, "ls")
    blocks = _check(mc, mc.run_em(**_fld("ls")), c, "ls", v)
    if cap == "default" and table != "singletons":
        assert blocks > 1      # the gene tables are cut into several slices
    mc.close()


def test_explicit_shape_keeps_grid_kernel(cases, indices, monkeypatch):
    """KB_EM_SHAPE selects the grid-wide kernels, as before the component kernel existed."""
    c = _case(cases, "genes")
    _set_knobs(monkeypatch, {"KB_EM_SHAPE": "0"})
    mc = _collector(indices[c.index], c, "flens")
    r = mc.run_em(table=(c.off, c.tids, c.counts), **_fld("flens"))
    alpha, rounds = c.em("flens")
    assert r["rounds"] == rounds
    np.testing.assert_array_equal(r["est_counts"], alpha)
    assert mc.timings()["em_comp_blocks"] == 0
    mc.close()
