"""GPU: consecutive batches of one run overlap on the device.  Batch i runs on one of two work spaces and internal
streams while batch i + 1 is packed and matched, and match_kernel hands fragments to its warps from one counter.  Many
small and odd-sized batches (1 fragment, fewer than one block, sizes that are not multiples of 32), a caller that
overwrites its device input right after each call, and two runs fed with interleaved global fragment indices must give
the per-fragment ECs, the EC table and the counts of a one-batch run and of the oracle."""
import os

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu

N_FRAG = 3000
SIZES = [1, 31, 33, 100, 7, 257, 1, 64, 999, 5, 250]


def cuts(n):
    out, a, i = [], 0, 0
    while a < n:
        b = min(n, a + SIZES[i % len(SIZES)])
        out.append((a, b))
        a, i = b, i + 1
    return out


def reads(name, paired, n=N_FRAG):
    ds = util.dataset(name)
    s1 = [bytes(x) for x in ds["s1"][:n]]
    s2 = [bytes(x) for x in ds["s2"][:n]] if paired else None
    return ds, s1, s2


def table(mc):
    eo, et, ec, eh = mc.ec_table()
    return util.ec_sets(eo, et), np.asarray(ec), eh


def oracle(ds, s1, s2, strand):
    paired = s2 is not None
    bases, off = O.to_batch(s1, s2)
    run = O.OracleRun(O.OracleIndex(ds["index"]), paired, strand, paired)
    frag = run.pseudoalign(bases, off)
    oo, ot, oc = run.ec_table()
    return frag, util.ec_sets(oo, ot), np.asarray(oc), run.flens()


@pytest.mark.parametrize("name", ["synth_small", "dlist"])
@pytest.mark.parametrize("strand", [0, 1, 2])
@pytest.mark.parametrize("paired", [True, False])
def test_small_batches_match_one_batch_and_oracle(name, strand, paired):
    ds, s1, s2 = reads(name, paired)
    ofrag, osets, ocounts, oflens = oracle(ds, s1, s2, strand)
    ix = K.KmerIndex(ds["index"], device=0)
    # one batch
    one = K.MinCollector(ix, paired=paired, strand=strand, collect_fld=paired)
    bases, off = O.to_batch(s1, s2)
    h = one.process_buffer(bases, off)
    sets, counts, eh = table(one)
    np.testing.assert_array_equal(util.handles_to_ids(h, eh), ofrag)
    assert sets == osets
    np.testing.assert_array_equal(counts, ocounts)
    one.close()
    # many small batches, handles downloaded after each, and the same batches left to overlap (no download)
    for want_handles in (True, False):
        mc = K.MinCollector(ix, paired=paired, strand=strand, collect_fld=paired)
        hs = []
        for a, b in cuts(len(s1)):
            bb, oo = O.to_batch(s1[a:b], s2[a:b] if paired else None)
            hs.append(mc.process_buffer(bb, oo, want_handles=want_handles))
        sets, counts, eh = table(mc)
        if want_handles:
            np.testing.assert_array_equal(util.handles_to_ids(np.concatenate(hs), eh), ofrag)
        assert sets == osets
        np.testing.assert_array_equal(counts, ocounts)
        if paired:
            np.testing.assert_array_equal(mc.flens, oflens)
        mc.close()
    ix.close()


@pytest.mark.parametrize("paired", [True, False])
def test_caller_overwrites_device_input_after_each_call(paired):
    torch = pytest.importorskip("torch")
    ds, s1, s2 = reads("synth_small", paired)
    # ragged reads: the lengths come from the caller's offsets, which are overwritten too
    rng = np.random.default_rng(7)
    s1 = [x[: int(rng.integers(20, len(x) + 1))] for x in s1]
    _, osets, ocounts, _ = oracle(ds, s1, s2, 0)
    ix = K.KmerIndex(ds["index"], device=0)
    mc = K.MinCollector(ix, paired=paired, collect_fld=False)
    stream = torch.cuda.current_stream()
    mc.set_stream(stream.cuda_stream)
    dev = torch.device("cuda", 0)
    d_bases = torch.empty(400 * 1000 * 2, dtype=torch.uint8, device=dev)
    d_off = torch.empty(2 * 1000 + 1, dtype=torch.int32, device=dev)
    for a, b in cuts(len(s1)):
        bb, oo = O.to_batch(s1[a:b], s2[a:b] if paired else None)
        n_reads = len(oo) - 1
        maxlen = int(np.diff(oo.astype(np.int64)).max())
        d_bases[: len(bb)].copy_(torch.from_numpy(np.ascontiguousarray(bb, np.uint8)))
        d_off[: len(oo)].copy_(torch.from_numpy(oo.astype(np.int32)))
        mc.process_buffer_device(d_bases.data_ptr(), d_off.data_ptr(), n_reads, 0, maxlen)
        # the next use of the buffers, in stream order: other bases, and offsets that would give every read no length
        d_bases.fill_(ord("A"))
        d_off.zero_()
    sets, counts, _ = table(mc)
    assert sets == osets
    np.testing.assert_array_equal(counts, ocounts)
    mc.close()
    ix.close()


def test_two_runs_with_interleaved_frag_base():
    ds, s1, s2 = reads("synth_small", True)
    _, osets, ocounts, _ = oracle(ds, s1, s2, 0)
    ix = K.KmerIndex(ds["index"], device=0)
    runs = [K.MinCollector(ix, paired=True, collect_fld=False) for _ in range(2)]
    for i, (a, b) in enumerate(cuts(len(s1))):
        r = runs[i % 2]
        r.set_frag_base(a)
        bb, oo = O.to_batch(s1[a:b], s2[a:b])
        r.process_buffer(bb, oo, want_handles=False)
    runs[0].merge_local([runs[1]])
    sets, counts, _ = table(runs[0])
    assert sets == osets
    np.testing.assert_array_equal(counts, ocounts)
    for r in runs:
        r.close()
    ix.close()


def test_bus_small_batches_concatenate():
    d = os.path.join(util.GOLDEN, "bus10x")
    s1 = O.read_fastq(os.path.join(d, "sc_reads_1.fastq.gz"))
    s2 = O.read_fastq(os.path.join(d, "sc_reads_2.fastq.gz"))
    _, ref = O.read_bus(os.path.join(d, "ref_10xv2", "output.bus"))
    ix = K.KmerIndex(os.path.join(util.GOLDEN, "config1", "transcripts.kidx"), device=0)
    bp = K.BUSProcessor(ix, "10xv2")
    parts = [bp.process_sets([O.to_batch(s1[a:b]), O.to_batch(s2[a:b])]) for a, b in cuts(len(s1))]
    assert np.concatenate(parts).tobytes() == ref.tobytes()
    bp.close()
    ix.close()
