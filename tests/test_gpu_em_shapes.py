"""GPU: the EM, the bootstrap and quant-tcc against the CPU oracle (oracle.em / oracle.bootstrap_sample), bit for bit
and round count included, at the launch shapes the fixture EMs never reach.

The fixture tables fit in one block of the EM kernels (at most ~1 000 rows and ~500 transcripts), so the grid barrier,
the grid-stride loops, the batch dimension and the chunking of samples hardly run there.  The tables here are
generated from seeds over the targets of stored indices (T = 14, 491 and 2 400 -- the first two not multiples of 32,
so that warps of the batched kernel straddle two problems) and reach every part of that machinery: a 300 000-row
table larger than the widest grid, one transcript in 20 000 ECs, an EC of every transcript, no multi-transcript EC at
all, one EC only.  Each table goes through the three entry points -- kb_em_run_table, an imported run
(kb_quant_import_device -> kb_em_run / kb_bootstrap_run) and kb_tcc_run -- under every launch knob, and the batch
paths run past the sample counts a single launch can hold (shared-memory state of em_kernel, gridDim.y of the
resample and quant-tcc fill kernels)."""
import os

import numpy as np
import pytest
import torch

import kallisto_b200 as K
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu

INDEX_OF = {"golden_synth": "synth_small", "golden_config1": "config1", "wide": "synth_small", "singletons": "synth_small",
            "one_ec": "config1", "hub": "abundant", "many": "abundant"}        # T = 491, 14, 2 400
SEED = 42
BIG_COUNT = (900_000, 1_000_000)   # a few counts this large; the total stays far below 2^31 (Multinomial::n_ is an int)


# ---------------------------------------------------------------------------------------------------------------------
# tables: (off uint64, tids uint32, counts uint32) in EC-id order; sets are sorted transcript lists, all distinct
# ---------------------------------------------------------------------------------------------------------------------
def _csr(sets):
    off = np.zeros(len(sets) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in sets])
    tids = np.fromiter((t for s in sets for t in s), np.uint32, int(off[-1]))
    return off, tids


def _counts(rng, n):
    c = rng.integers(1, 51, n).astype(np.uint32)
    if n >= 10:
        c[rng.choice(n, 3, replace=False)] = rng.integers(*BIG_COUNT, 3)
    return c


def _random_sets(rng, pool, k, n):
    """n distinct sorted k-subsets of `pool` (fewer if duplicates or repeated members are drawn)."""
    pool = np.asarray(pool, np.int64)
    a = np.sort(pool[rng.integers(0, len(pool), (n, k))], axis=1)
    a = a[np.all(np.diff(a, axis=1) > 0, axis=1)]
    return np.unique(a, axis=0)


def _table(name, T, rng):
    if name.startswith("golden"):
        g = util.golden_ecs(util.dataset(INDEX_OF[name]), "paired")
        frag = g["frag_ec"]
        counts = np.bincount(frag[frag >= 0], minlength=len(g["ec_off"]) - 1).astype(np.uint32)
        return np.asarray(g["ec_off"], np.uint64), np.asarray(g["ec_tids"], np.uint32), counts
    if name == "wide":            # one EC holding every transcript, random pairs, some singletons
        sets = [tuple(range(T))] + [tuple(r) for r in _random_sets(rng, range(T), 2, 1600)]
        sets += [(int(t),) for t in rng.choice(T, 100, replace=False)]
    elif name == "singletons":    # n_multi = 0
        sets = [(int(t),) for t in rng.choice(T, 400, replace=False)]
    elif name == "one_ec":        # a single multi-transcript EC
        sets = [(1, 4, 9, 13)]
    elif name == "hub":           # transcript 7 in ~20 000 ECs; transcripts 2 000..2 399 in none
        others = [t for t in range(2000) if t != 7]
        sets = []
        for k in (1, 2, 3):       # 1 999 pairs with transcript 7, ~9 000 triples and quadruples each
            sets += [tuple(sorted((7,) + tuple(int(x) for x in r))) for r in _random_sets(rng, others, k, 9000)]
        sets += [tuple(r) for r in _random_sets(rng, others, 2, 1500)] + [(int(t),) for t in range(0, 2000, 3)]
    elif name == "many":          # ~300 000 rows: more than the 270 k threads of the widest single-problem shape
        sets = []
        for k in range(2, 9):
            sets += [tuple(int(x) for x in r) for r in _random_sets(rng, range(T), k, 43_500)]
    else:
        raise KeyError(name)
    sets = list(dict.fromkeys(sets))
    order = rng.permutation(len(sets))            # EC ids are not in smallest-transcript order
    sets = [sets[i] for i in order]
    off, tids = _csr(sets)
    return off, tids, _counts(rng, len(sets))


TABLES = ["golden_synth", "golden_config1", "wide", "singletons", "one_ec", "hub", "many"]
EFF_MODES = {"flens": (0.0, 0.0), "ls": (200.0, 20.0)}    # golden fragment-length histogram / -l 200 -s 20


class Case:
    def __init__(self, name):
        rng = np.random.default_rng([ord(ch) for ch in name])
        self.name = name
        self.index = INDEX_OF[name]
        ds = util.dataset(self.index)
        self.flens = np.asarray(util.golden_ecs(ds, "paired")["flens"], np.uint32)
        self.lens = O.OracleIndex(ds["index"]).target_lens
        self.T = len(self.lens)
        self.off, self.tids, self.counts = _table(name, self.T, rng)
        self.n = len(self.counts)
        # the sets are imported in a random order (EC id imp[j] at position j) with first-occurrence indices that
        # number them back in EC-id order
        self.imp = rng.permutation(self.n)
        self.first = np.arange(self.n, dtype=np.int64) * 3 + 5
        self._em, self._eff, self._samp, self._bs = {}, {}, {}, {}

    def sets(self):
        return util.ec_sets(self.off, self.tids)

    def eff(self, mode):
        if mode not in self._eff:
            m, s = EFF_MODES[mode]
            fl = self.flens if mode == "flens" else np.zeros(1000, np.uint32)
            self._eff[mode] = O.eff_lens(self.lens, O.mean_fl_trunc(fl, m, s))
        return self._eff[mode]

    def em(self, mode):
        if mode not in self._em:
            self._em[mode] = O.em(self.off, self.tids, self.counts, self.eff(mode), self.T)
        return self._em[mode]

    def sample(self, seed, b):
        if (seed, b) not in self._samp:
            self._samp[(seed, b)] = O.bootstrap_sample(self.counts, seed, b)
        return self._samp[(seed, b)]

    def bootstrap_em(self, mode, seed, b):
        if (mode, seed, b) not in self._bs:
            self._bs[(mode, seed, b)] = O.em(self.off, self.tids, self.sample(seed, b), self.eff(mode), self.T,
                                             counts_w=self.counts)
        return self._bs[(mode, seed, b)]


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


# launch knobs: none of them may change a bit of the result
SINGLE_KNOBS = {                  # single-problem EM (kb_em_run_table, kb_em_run)
    "default": {},
    "shape1": {"KB_EM_SHAPE": "1"},
    "shape2": {"KB_EM_SHAPE": "2"},
    "shape3": {"KB_EM_SHAPE": "3"},
}
BATCHED_KNOBS = {                 # em_kernel (KB_EM_SHAPE=-1 sends the single-problem EM there too)
    "tpb%d_occ%d" % (tpb, occ): {"KB_EM_SHAPE": "-1", "KB_EM_TPB": str(tpb), "KB_EM_OCC": str(occ)}
    for tpb in (256, 512, 1024) for occ in (1, 2)
}
BATCHED_KNOBS["blocks1"] = {"KB_EM_SHAPE": "-1", "KB_EM_BLOCKS": "1"}
BATCHED_KNOBS["blocks3"] = {"KB_EM_SHAPE": "-1", "KB_EM_BLOCKS": "3"}
ALL_KNOBS = dict(SINGLE_KNOBS, **BATCHED_KNOBS)
KNOB_VARS = ("KB_EM_SHAPE", "KB_EM_TPB", "KB_EM_OCC", "KB_EM_BLOCKS", "KB_BS_CHUNK", "KB_TCC_CHUNK")


def _set_knobs(monkeypatch, env):
    for k in KNOB_VARS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _collector(ix, c, mode):
    mc = K.MinCollector(ix, paired=True)
    if mode == "flens":
        mc.set_flens(c.flens)
    return mc


def _imported(ix, c, mode):
    """An empty run that receives the table through kb_quant_import_device, in import order, as multigpu.export_table
    hands tables over (device int32 / int64 tensors)."""
    mc = _collector(ix, c, mode)
    dev = torch.device("cuda", 0)
    lens = np.diff(c.off.astype(np.int64))[c.imp]
    off = np.zeros(c.n + 1, np.int64)
    off[1:] = np.cumsum(lens)
    tids = np.concatenate([c.tids[int(c.off[e]):int(c.off[e + 1])] for e in c.imp]).astype(np.int32)
    t_off = torch.from_numpy(off.astype(np.int32)).to(dev)
    t_tids = torch.from_numpy(tids).to(dev)
    t_counts = torch.from_numpy(c.counts[c.imp].astype(np.int32)).to(dev)
    t_first = torch.from_numpy(c.first[c.imp]).to(dev)
    mc.import_device(c.n, t_off.data_ptr(), t_tids.data_ptr(), t_counts.data_ptr(), t_first.data_ptr(), 0,
                     int(c.counts.sum()))
    torch.cuda.synchronize()
    return mc


def _fld(mode):
    return dict(zip(("fld_mean", "fld_sd"), EFF_MODES[mode]))


def _check_em(r, c, mode):
    alpha, rounds = c.em(mode)
    np.testing.assert_array_equal(r["eff_lens"], c.eff(mode))
    assert r["rounds"] == rounds
    np.testing.assert_array_equal(r["est_counts"], alpha)


# ---------------------------------------------------------------------------------------------------------------------
# 1. kb_em_run_table: host set-up, launch_em(p, 256)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob", list(ALL_KNOBS))
@pytest.mark.parametrize("table", TABLES)
def test_em_table(cases, indices, monkeypatch, table, knob):
    c = _case(cases, table)
    _set_knobs(monkeypatch, ALL_KNOBS[knob])
    mode = "flens" if knob != "shape2" else "ls"
    mc = _collector(indices[c.index], c, mode)
    _check_em(mc.run_em(table=(c.off, c.tids, c.counts), **_fld(mode)), c, mode)
    mc.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. an imported run: device EC numbering by first occurrence, emprep, kb_em_run; kb_bootstrap_run on top of it
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob", list(ALL_KNOBS))
@pytest.mark.parametrize("table", TABLES)
def test_imported_em(cases, indices, monkeypatch, table, knob):
    c = _case(cases, table)
    _set_knobs(monkeypatch, ALL_KNOBS[knob])
    mode = "ls" if knob in ("default", "tpb256_occ2") else "flens"
    mc = _imported(indices[c.index], c, mode)
    if knob == "default":
        eo, et, ec, _ = mc.ec_table()              # the table comes back in EC-id (= first occurrence) order
        np.testing.assert_array_equal(eo, c.off)
        np.testing.assert_array_equal(et, c.tids)
        np.testing.assert_array_equal(ec, c.counts)
    _check_em(mc.run_em(**_fld(mode)), c, mode)
    mc.close()


BS_B = 8
BS_CASES = {                       # name: (KB_BS_CHUNK, launch knobs)
    "chunk_auto": (None, "default"),
    "chunk1": ("1", "default"),    # nb == 1: the single-problem kernel, default shape and KB_EM_SHAPE=3
    "chunk1_shape3": ("1", "shape3"),
    "chunk3": ("3", "default"),    # 3 + 3 + 2: a partial last chunk
    "chunk3_tpb256_occ2": ("3", "tpb256_occ2"),
    "tpb256_occ1": (None, "tpb256_occ1"),
    "tpb512_occ2": (None, "tpb512_occ2"),
    "tpb1024_occ2": (None, "tpb1024_occ2"),
    "blocks1": (None, "blocks1"),
    "blocks3": (None, "blocks3"),
}


@pytest.mark.parametrize("bs", list(BS_CASES))
@pytest.mark.parametrize("table", TABLES)
def test_imported_bootstrap(cases, indices, monkeypatch, table, bs):
    c = _case(cases, table)
    chunk, knob = BS_CASES[bs]
    env = dict(ALL_KNOBS[knob])
    if chunk:
        env["KB_BS_CHUNK"] = chunk
    _set_knobs(monkeypatch, env)
    mode = "ls" if bs == "chunk3" else "flens"
    mc = _imported(indices[c.index], c, mode)
    r = mc.run_bootstrap(BS_B, seed=SEED, want_samples=True, **_fld(mode))
    for b in range(BS_B):
        np.testing.assert_array_equal(r["samples"][b][:c.n], c.sample(SEED, b), err_msg="sample %d" % b)
        alpha, rounds = c.bootstrap_em(mode, SEED, b)
        assert r["rounds"][b] == rounds, b
        np.testing.assert_array_equal(r["est_counts"][b], alpha, err_msg="sample %d" % b)
    mc.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. kb_tcc_run: every row is its own EM over the same ECs, weighted by its own counts
# ---------------------------------------------------------------------------------------------------------------------
def _tcc_rows(c, S, rng, empty_at=None):
    """S rows of random subsets of the ECs (a quarter to all of them), counts drawn around the table's; row `empty_at`
    is empty -> (ec ids, counts, row offsets) in CSR."""
    ids, vals, ro = [], [], [0]
    for s in range(S):
        keep = np.zeros(0, np.int64) if s == empty_at else np.flatnonzero(rng.random(c.n) < rng.uniform(0.25, 1.0))
        ids.append(keep.astype(np.uint32))
        vals.append(np.maximum(1, c.counts[keep] * rng.uniform(0.2, 1.5, len(keep))).astype(np.uint32))
        ro.append(ro[-1] + len(keep))
    return np.concatenate(ids), np.concatenate(vals), np.asarray(ro, np.uint64)


def _tcc_call(ix, c, ids, vals, ro, eff):
    """kb_tcc_run on CSR rows (K.tcc_run builds the same arrays from Python lists, too slowly for 70 000 rows)."""
    S = len(ro) - 1
    eff = np.ascontiguousarray(eff, np.float64)
    est = np.zeros((S, c.T), np.float64)
    rounds = np.zeros(S, np.int32)
    K._ck(K.lib().kb_tcc_run(ix._h, c.n, K._p(c.off), K._p(c.tids), S, K._p(ro), K._p(ids), K._p(vals), K._p(eff),
                             int(eff.ndim == 2), K._p(est), K._p(rounds)))
    return est, rounds


def _dense(c, ids, vals, ro, s):
    out = np.zeros(c.n, np.uint32)
    a, b = int(ro[s]), int(ro[s + 1])
    out[ids[a:b]] = vals[a:b]
    return out


TCC_CASES = {                      # name: (KB_TCC_CHUNK, launch knobs, per-sample effective lengths)
    "chunk_auto": (None, "default", False),
    "chunk1": ("1", "default", False),
    "chunk5": ("5", "default", False),           # 5 + 5 + 2
    "chunk5_per_sample_eff": ("5", "default", True),
    "per_sample_eff": (None, "default", True),
    "tpb256_occ2": (None, "tpb256_occ2", False),
    "tpb512_occ1": (None, "tpb512_occ1", False),
    "blocks1": (None, "blocks1", False),
    "blocks3": ("5", "blocks3", False),
}
TCC_S = 12


@pytest.fixture(scope="module")
def tcc_rows(cases):
    out = {}

    def get(table):
        if table not in out:
            c = _case(cases, table)
            rng = np.random.default_rng(7 + len(table))
            ids, vals, ro = _tcc_rows(c, TCC_S, rng, empty_at=4)
            # per-sample effective lengths: each sample its own fragment-length mean (-l m -s 20)
            eff2 = np.stack([O.eff_lens(c.lens, O.mean_fl_trunc(np.zeros(1000, np.uint32), 120.0 + 15 * s, 20.0))
                             for s in range(TCC_S)])
            ref, ref2 = [], []
            for s in range(TCC_S):
                d = _dense(c, ids, vals, ro, s)
                ref.append(O.em(c.off, c.tids, d, c.eff("flens"), c.T))
                ref2.append(O.em(c.off, c.tids, d, eff2[s], c.T))
            out[table] = (ids, vals, ro, eff2, ref, ref2)
        return out[table]
    return get


@pytest.mark.parametrize("tc", list(TCC_CASES))
@pytest.mark.parametrize("table", TABLES)
def test_tcc(cases, indices, tcc_rows, monkeypatch, table, tc):
    c = _case(cases, table)
    chunk, knob, per_sample = TCC_CASES[tc]
    env = dict(ALL_KNOBS[knob])
    if chunk:
        env["KB_TCC_CHUNK"] = chunk
    _set_knobs(monkeypatch, env)
    ids, vals, ro, eff2, ref, ref2 = tcc_rows(table)
    est, rounds = _tcc_call(indices[c.index], c, ids, vals, ro, eff2 if per_sample else c.eff("flens"))
    for s, (alpha, n) in enumerate(ref2 if per_sample else ref):
        assert rounds[s] == n, s
        np.testing.assert_array_equal(est[s], alpha, err_msg="sample %d" % s)


def test_tcc_python_binding_matches_csr_call(cases, indices):
    """K.tcc_run (a list of (ec, count) pairs per row) hands kb_tcc_run the same arrays as the CSR call above."""
    c = _case(cases, "golden_synth")
    ids, vals, ro = _tcc_rows(c, 3, np.random.default_rng(3), empty_at=1)
    rows = [[(int(e), int(v)) for e, v in zip(ids[ro[s]:ro[s + 1]], vals[ro[s]:ro[s + 1]])] for s in range(3)]
    est, rounds = K.tcc_run(indices[c.index], c.sets(), rows, c.eff("flens"))
    est2, rounds2 = _tcc_call(indices[c.index], c, ids, vals, ro, c.eff("flens"))
    np.testing.assert_array_equal(est, est2)
    np.testing.assert_array_equal(rounds, rounds2)


# ---------------------------------------------------------------------------------------------------------------------
# sample counts past what one launch can hold: 12 288 problems fill em_kernel's 48 KB of default shared memory, 65 535
# is the largest gridDim.y of the resample and quant-tcc fill kernels; a chunk of 8 192 problems (32 KB of state) in
# 256-thread blocks fits fewer blocks per SM than the same kernel with little shared memory
# ---------------------------------------------------------------------------------------------------------------------
def _spot(n, rng):
    pick = {0, 1, 8191, 8192, 12287, 12288, n - 1} | set(int(x) for x in rng.choice(n, 20, replace=False))
    return sorted(p for p in pick if p < n)


@pytest.mark.parametrize("table,B,knobs", [
    ("golden_config1", 13000, {}),
    ("golden_config1", 65537, {}),
    ("golden_synth", 8200, dict(BATCHED_KNOBS["tpb256_occ2"], KB_BS_CHUNK="8192")),
], ids=["13000", "65537", "8200_chunk8192_tpb256_occ2"])
def test_bootstrap_past_launch_limits(cases, indices, monkeypatch, table, B, knobs):
    c = _case(cases, table)
    _set_knobs(monkeypatch, knobs)
    mc = _imported(indices[c.index], c, "flens")
    r = mc.run_bootstrap(B, seed=SEED, want_samples=True)
    assert (r["rounds"] > 0).all()
    for b in _spot(B, np.random.default_rng(B)):
        np.testing.assert_array_equal(r["samples"][b][:c.n], c.sample(SEED, b), err_msg="sample %d" % b)
        alpha, rounds = c.bootstrap_em("flens", SEED, b)
        assert r["rounds"][b] == rounds, b
        np.testing.assert_array_equal(r["est_counts"][b], alpha, err_msg="sample %d" % b)
    mc.close()


@pytest.mark.parametrize("table,S", [("golden_synth", 20000), ("golden_config1", 70000)])
def test_tcc_past_launch_limits(cases, indices, monkeypatch, table, S):
    c = _case(cases, table)
    _set_knobs(monkeypatch, {})
    if table == "golden_synth":     # the golden table is quant-tcc's own EC file for synth_small's index
        assert O.read_matrix_ec(os.path.join(util.GOLDEN, "quanttcc", "matrix.ec")) == c.sets()
    rng = np.random.default_rng(S)
    ids, vals, ro = _tcc_rows(c, S, rng, empty_at=S // 2)
    est, rounds = _tcc_call(indices[c.index], c, ids, vals, ro, c.eff("flens"))
    assert (rounds > 0).all()
    for s in _spot(S, rng):
        alpha, n = O.em(c.off, c.tids, _dense(c, ids, vals, ro, s), c.eff("flens"), c.T)
        assert rounds[s] == n, s
        np.testing.assert_array_equal(est[s], alpha, err_msg="sample %d" % s)
