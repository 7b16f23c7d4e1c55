"""GPU (one device is enough): the export / import kernels of the multi-GPU path.  Two runs over the
two halves of the reads, the second exported and folded into the first, must equal one run over
everything -- EC table (sets, counts, order of first occurrence) and EM bit for bit."""
import numpy as np
import pytest
import torch

import kallisto_b200 as K
from kallisto_b200 import multigpu
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["config1", "synth_small"])
def test_export_import_equals_single_run(name):
    ds = util.dataset(name)
    ix = K.KmerIndex(ds["index"], device=0)
    n = len(ds["s1"])
    h = n // 2
    whole = K.MinCollector(ix, paired=True)
    whole.process_buffer(*util.batch(ds, True), want_handles=False)
    a = K.MinCollector(ix, paired=True)
    b = K.MinCollector(ix, paired=True, collect_fld=False)
    a.process_buffer(*O.to_batch(ds["s1"][:h], ds["s2"][:h]), want_handles=False)
    b.process_buffer(*O.to_batch(ds["s1"][h:], ds["s2"][h:]), want_handles=False)
    dev = torch.device("cuda", 0)
    off, tids, counts, first = multigpu.export_table(b, dev)
    # the exported table is b's own EC table
    bo, bt, bc, _ = b.ec_table()
    np.testing.assert_array_equal(off.cpu().numpy().astype(np.uint64), bo)
    np.testing.assert_array_equal(tids.cpu().numpy().astype(np.uint32), bt)
    np.testing.assert_array_equal(counts.cpu().numpy().astype(np.uint32), bc)
    assert np.all(np.diff(first.cpu().numpy()) > 0)
    a.import_device(len(counts), off.data_ptr(), tids.data_ptr(), counts.data_ptr(), first.data_ptr(),
                    multigpu.RANK_STRIDE, n - h)
    wo, wt, wc, _ = whole.ec_table()
    ao, at, ac, _ = a.ec_table()
    assert util.ec_sets(ao, at) == util.ec_sets(wo, wt)      # same sets in the same (first-occurrence) order
    np.testing.assert_array_equal(ac, wc)
    # fragment-length distribution comes from the first slice only; here both see the first 10000 unique pairs
    # only if they fall in the first half, so compare the EM on an explicit common distribution
    a.set_flens(whole.flens)
    ra, rw = a.run_em(), whole.run_em()
    assert ra["rounds"] == rw["rounds"]
    np.testing.assert_array_equal(ra["est_counts"], rw["est_counts"])
    st = a.finalize()
    assert st["n_processed"] == n
    for m in (whole, a, b):
        m.close()
    ix.close()


def test_nccl_merge_with_one_rank_is_the_identity():
    """kb_comm_create / kb_quant_merge_nccl on a one-rank communicator (what a one-GPU machine can run; the
    N-rank exchange is checked by tools/multi_check.py under torchrun)."""
    ds = util.dataset("synth_small")
    ix = K.KmerIndex(ds["index"], device=0)
    a = K.MinCollector(ix, paired=True)
    a.process_buffer(*util.batch(ds, True), want_handles=False)
    before = a.ec_table()
    comm = K.Comm(1, 0, K.Comm.unique_id(), 0)
    assert a.merge_nccl(comm) == len(ds["s1"])
    after = a.ec_table()
    for x, y in zip(before, after):
        np.testing.assert_array_equal(x, y)
    comm.close(); a.close(); ix.close()


def test_global_fragment_indices_give_stream_order():
    """Two runs fed alternating batches of one stream with kb_quant_set_frag_base, merged by content, number their
    ECs like one run over the whole stream (what `kallisto_b200 quant --devices` relies on)."""
    ds = util.dataset("synth_small")
    ix = K.KmerIndex(ds["index"], device=0)
    n = len(ds["s1"])
    whole = K.MinCollector(ix, paired=True)
    whole.process_buffer(*util.batch(ds, True), want_handles=False)
    a = K.MinCollector(ix, paired=True)
    b = K.MinCollector(ix, paired=True, collect_fld=False)
    cuts = list(range(0, n, 3000)) + [n]
    for i, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
        mc = a if i % 2 == 0 else b
        mc.set_frag_base(lo)
        mc.process_buffer(*O.to_batch(ds["s1"][lo:hi], ds["s2"][lo:hi]), want_handles=False)
    dev = torch.device("cuda", 0)
    off, tids, counts, first = multigpu.export_table(b, dev)
    a.import_device(len(counts), off.data_ptr(), tids.data_ptr(), counts.data_ptr(), first.data_ptr(), 0, 0)
    wo, wt, wc, _ = whole.ec_table()
    ao, at, ac, _ = a.ec_table()
    assert util.ec_sets(ao, at) == util.ec_sets(wo, wt)
    np.testing.assert_array_equal(ac, wc)
    for m in (whole, a, b):
        m.close()
    ix.close()
