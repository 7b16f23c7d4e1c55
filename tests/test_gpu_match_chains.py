"""GPU: match_kernel runs the lookup chains of both mates of a pair side by side in one lane.  Cases where the two
chains end at different times, or push the same EC sets in the same iteration, against the oracle: per-fragment ECs,
the EC table and counts, fragment lengths and the exact number of k-mer lookups."""
import zlib

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu

N_FRAG = 4000
_COMP = bytes.maketrans(b"ACGTNacgtn", b"TGCANtgcan")


def revcomp(s):
    return bytes(s).translate(_COMP)[::-1]


def spoil(s, kind, rng):
    if kind == "empty":
        return b""
    if kind == "short":                       # shorter than k = 31
        return bytes(s[: int(rng.integers(1, 31))])
    if kind == "allN":
        return b"N" * len(s)
    if kind == "random":                      # unmappable: every k-mer is looked up
        return bytes(rng.choice(list(b"ACGT"), size=len(s)).astype(np.uint8))
    return bytes(s)


def make_case(ds, case, rng):
    s1, s2 = [bytes(x) for x in ds["s1"][:N_FRAG]], [bytes(x) for x in ds["s2"][:N_FRAG]]
    if case == "one_mate_spoilt":
        # fragment i: mate (i // 4) % 2 is empty / shorter than k / all N / intact, the other mate is left alone
        kinds = ["empty", "short", "allN", "none"]
        for i in range(len(s1)):
            kind = kinds[i % 4]
            if (i // 4) % 2 == 0:
                s1[i] = spoil(s1[i], kind, rng)
            else:
                s2[i] = spoil(s2[i], kind, rng)
    elif case == "random_mate":
        for i in range(len(s1)):
            if rng.random() < 0.5:
                if rng.random() < 0.5:
                    s1[i] = spoil(s1[i], "random", rng)
                else:
                    s2[i] = spoil(s2[i], "random", rng)
    elif case == "same_read":
        s2 = list(s1)
    elif case == "revcomp_read":
        s2 = [revcomp(x) for x in s1]
    return s1, s2


def check(ds, s1, s2, strand=0, fp=False):
    paired = s2 is not None
    bases, off = O.to_batch(s1, s2)
    ix = K.KmerIndex(ds["index"], device=0, load_positions=fp)
    o_ix = O.OracleIndex(ds["index"])
    kw = dict(collect_fld=False, single_overhang=False, fld_mean=200.0) if fp else dict(collect_fld=paired)
    mc = K.MinCollector(ix, paired=paired, strand=strand, **kw)
    h = mc.process_buffer(bases, off)
    eo, et, ec, eh = mc.ec_table()
    o_run = O.OracleRun(o_ix, paired, strand, paired and not fp, **(dict(fp_fl=200) if fp else {}))
    ofrag = o_run.pseudoalign(bases, off)
    oo, ot, oc = o_run.ec_table()
    np.testing.assert_array_equal(util.handles_to_ids(h, eh), ofrag)
    assert util.ec_sets(eo, et) == util.ec_sets(oo, ot)
    np.testing.assert_array_equal(ec, oc)
    if paired and not fp:
        np.testing.assert_array_equal(mc.flens, o_run.flens())
    mc.close()
    if paired:
        # without fragment-length sampling the oracle counts exactly the lookups of KmerIndex::match
        mc = K.MinCollector(ix, paired=True, strand=strand, collect_fld=False)
        mc.process_buffer(bases, off, want_handles=False)
        st = mc.finalize()
        o_run = O.OracleRun(o_ix, True, strand, False)
        o_run.pseudoalign(bases, off)
        assert st["n_probes"] == o_run.n_find()
        mc.close()
    ix.close()


@pytest.mark.parametrize("name", ["synth_small", "manyecs", "abundant"])
@pytest.mark.parametrize("case", ["one_mate_spoilt", "random_mate", "same_read", "revcomp_read", "intact"])
def test_two_chains_match_oracle(name, case):
    ds = util.dataset(name)
    rng = np.random.default_rng(zlib.crc32((name + case).encode()))
    s1, s2 = make_case(ds, case, rng)
    check(ds, s1, s2)


@pytest.mark.parametrize("strand", [1, 2])
@pytest.mark.parametrize("case", ["one_mate_spoilt", "random_mate", "revcomp_read"])
def test_two_chains_stranded(strand, case):
    ds = util.dataset("synth_small")
    rng = np.random.default_rng(31 * strand + len(case))
    s1, s2 = make_case(ds, case, rng)
    check(ds, s1, s2, strand=strand)


def test_two_chains_many_ec_sets_both_mates():
    """manyecs reads cross more than KB_MAX_E distinct EC sets; as both mates of one fragment, both chains write into
    the lane's spill tail."""
    ds = util.dataset("manyecs")
    s1 = [bytes(x) for x in ds["s1"][:N_FRAG]]
    s2 = [bytes(x) for x in ds["s2"][:N_FRAG]]
    s2 = [revcomp(a) if i % 2 else b for i, (a, b) in enumerate(zip(s1, s2))]
    check(ds, s1, s2)


@pytest.mark.parametrize("case", ["random_mate", "one_mate_spoilt"])
def test_two_chains_position_filter_one_mate_mapped(case):
    ds = util.dataset("synth_small")
    rng = np.random.default_rng(5 + len(case))
    s1, s2 = make_case(ds, case, rng)
    check(ds, s1, s2, fp=True)


@pytest.mark.parametrize("name,strand,fp", [("synth_small", 0, False), ("manyecs", 0, False), ("abundant", 0, False),
                                           ("synth_small", 1, False), ("synth_small", 2, False), ("synth_small", 0, True)])
def test_single_end_one_chain(name, strand, fp):
    ds = util.dataset(name)
    rng = np.random.default_rng(11 + strand)
    s1, _ = make_case(ds, "one_mate_spoilt", rng)
    check(ds, s1, None, strand=strand, fp=fp)
