"""GPU: every host batch reaches the device through one staging copy (Quant::stage).  The paths no other test drives from
Python: per-mate buffers with offsets that are positions in the whole bases buffer and do not start at 0 (what the
command line's LockStep hands over), per-mate buffers without offsets, BUS batches cut the same way, and a quant run on
the staging buffers a closed BUS run left in the index's shared work space."""
import os

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import util
from tests.test_gpu_batch_overlap import N_FRAG, cuts, oracle, table

pytestmark = pytest.mark.gpu


def check(mc, handles, want):
    """handles (None: not downloaded), the run's EC table, counts and fragment lengths against the oracle's"""
    ofrag, osets, ocounts, oflens = want
    sets, counts, eh = table(mc)
    if handles is not None:
        np.testing.assert_array_equal(util.handles_to_ids(handles, eh), ofrag)
    assert sets == osets
    np.testing.assert_array_equal(counts, ocounts)
    np.testing.assert_array_equal(mc.flens, oflens)


def bus10x():
    d = os.path.join(util.GOLDEN, "bus10x")
    s1 = O.read_fastq(os.path.join(d, "sc_reads_1.fastq.gz"))
    s2 = O.read_fastq(os.path.join(d, "sc_reads_2.fastq.gz"))
    _, ref = O.read_bus(os.path.join(d, "ref_10xv2", "output.bus"))
    return O.to_batch(s1), O.to_batch(s2), ref


@pytest.mark.parametrize("name", ["synth_small", "dlist"])
def test_process_buffer_pe_offset_slices(name):
    ds = util.dataset(name)
    rng = np.random.default_rng(11)
    # ragged first mates: a batch's longest read may be a second mate's
    s1 = [bytes(x)[: int(rng.integers(20, len(x) + 1))] for x in ds["s1"][:N_FRAG]]
    s2 = [bytes(x) for x in ds["s2"][:N_FRAG]]
    want = oracle(ds, s1, s2, 0)
    ix = K.KmerIndex(ds["index"], device=0)
    one = K.MinCollector(ix, paired=True)
    check(one, one.process_buffer(*O.to_batch(s1, s2)), want)
    one.close()
    (b1, o1), (b2, o2) = O.to_batch(s1), O.to_batch(s2)
    for want_handles in (True, False):
        mc = K.MinCollector(ix, paired=True)
        hs = [mc.process_buffer_pe(b1, o1[a:b + 1], b2, o2[a:b + 1], want_handles=want_handles) for a, b in cuts(len(s1))]
        check(mc, np.concatenate(hs) if want_handles else None, want)
        mc.close()
    ix.close()


@pytest.mark.parametrize("name", ["synth_small", "dlist"])
def test_batch_pe_fixed_len_without_offsets(name):
    ds = util.dataset(name)
    s1 = [bytes(x) for x in ds["s1"][:N_FRAG]]
    s2 = [bytes(x) for x in ds["s2"][:N_FRAG]]
    n = len(s1[0])
    assert all(len(x) == n for x in s1 + s2)
    want = oracle(ds, s1, s2, 0)
    b1 = np.frombuffer(b"".join(s1), np.uint8)
    b2 = np.frombuffer(b"".join(s2), np.uint8)
    ix = K.KmerIndex(ds["index"], device=0)
    mc = K.MinCollector(ix, paired=True)
    hs = []
    for a, b in cuts(len(s1)):
        out = np.full(b - a, -1, np.int32)
        K._ck(K.lib().kb_pseudoalign_batch_pe(mc._h, b1.ctypes.data + a * n, None, b2.ctypes.data + a * n, None, b - a, n,
                                              K._p(out)))
        hs.append(out)
    check(mc, np.concatenate(hs), want)
    mc.close()
    ix.close()


def test_bus_offset_slices():
    (b1, o1), (b2, o2), ref = bus10x()
    ix = K.KmerIndex(os.path.join(util.GOLDEN, "config1", "transcripts.kidx"), device=0)
    bp = K.BUSProcessor(ix, "10xv2")
    parts = [bp.process_sets([(b1, o1[a:b + 1]), (b2, o2[a:b + 1])]) for a, b in cuts(len(o1) - 1)]
    assert np.concatenate(parts).tobytes() == ref.tobytes()
    bp.close()
    ix.close()


def test_quant_after_bus_on_shared_staging():
    (b1, o1), (b2, o2), ref = bus10x()
    ds = util.dataset("config1")
    ix = K.KmerIndex(ds["index"], device=0)
    # a BUS run stages its batches into the index's work space (up to 1000 offsets per file), and is closed
    bp = K.BUSProcessor(ix, "10xv2", max_batch_sets=1000)
    n = len(o1) - 1
    parts = [bp.process_sets([(b1, o1[a:a + 1001]), (b2, o2[a:a + 1001])]) for a in range(0, n, 1000)]
    assert np.concatenate(parts).tobytes() == ref.tobytes()
    bp.close()
    # quant runs borrow the same buffers: a single buffer of every read, then one buffer per mate
    s1, s2 = ds["s1"], ds["s2"]
    want = oracle(ds, s1, s2, 0)
    mc = K.MinCollector(ix, paired=True)
    check(mc, mc.process_buffer(*O.to_batch(s1, s2)), want)
    mc.close()
    (q1, p1), (q2, p2) = O.to_batch(s1), O.to_batch(s2)
    mc = K.MinCollector(ix, paired=True)
    check(mc, mc.process_buffer_pe(q1, p1, q2, p2), want)
    mc.close()
    ix.close()
