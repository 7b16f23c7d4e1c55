#!/usr/bin/env python
"""Connected components of the benchmark's EM problem (the bipartite graph of multi-transcript ECs and transcripts;
em_component_kernel solves one slice of whole components per block): an EC table of 15 x 2 M benchmark pairs, built as
tools/em_sweep.py builds it, then the number of components and the largest by transcripts, rows and entries (size =
transcripts + rows + entries, the unit of KB_EM_COMP_CAP).  Transcripts in no multi-transcript EC are components of their own.  Also
the slices of the layout (one per SM) and their shared memory in the resident layout (emcomp_resident_bytes, the unit of
KB_EM_COMP_SMEM): max and mean over slices.  Prints one JSON line; KB_COMP_STEPS sets the number of 2 M-pair batches."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
from scipy.sparse.csgraph import connected_components  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import benchdata  # noqa: E402
import kallisto_b200 as K  # noqa: E402


def components(off, tids, T, sms):
    ln = np.diff(off.astype(np.int64))
    multi = np.flatnonzero(ln > 1)
    rows = np.repeat(np.arange(len(multi)), ln[multi])
    ent = tids[np.repeat(ln > 1, ln)]
    first = tids[off[:-1].astype(np.int64)[multi]]
    g = sp.coo_matrix((np.ones(len(ent)), (first[rows], ent)), shape=(T, T))
    n_comp, comp = connected_components(g, directed=False)
    n_t = np.bincount(comp, minlength=n_comp)
    n_r = np.bincount(comp[first], minlength=n_comp)
    n_e = np.bincount(comp[ent], minlength=n_comp)
    size = n_t + n_r + n_e
    multi_comp = n_r > 0
    # slices: components in order of their smallest transcript id, target ceil(total / SMs), component -> start // target
    root = np.full(n_comp, T, np.int64)
    np.minimum.at(root, comp, np.arange(T))
    t_size = 1 + np.bincount(ent, minlength=T) + np.bincount(first, minlength=T)
    order = np.lexsort((np.arange(T), root[comp]))
    scan = np.concatenate([[0], np.cumsum(t_size[order])])
    pos = np.empty(T, np.int64)
    pos[order] = np.arange(T)
    total = int(scan[-1])
    target = -(-total // sms)
    n_sl = (total - 1) // target + 1
    sl = scan[pos[root]][comp] // target
    res = (36 * np.bincount(sl, minlength=n_sl) + 16 * np.bincount(sl[first], minlength=n_sl)
           + 4 * np.bincount(sl[ent], minlength=n_sl) + 8)
    return {"n_targets": int(T), "n_multi_ecs": int(len(multi)), "nnz_multi": int(len(ent)),
            "components": int(n_comp), "components_with_rows": int(multi_comp.sum()),
            "max_transcripts": int(n_t.max()), "max_rows": int(n_r.max()), "max_entries": int(n_e.max()),
            "max_size": int(size.max()), "mean_size_with_rows": float(size[multi_comp].mean()) if multi_comp.any() else 0.0,
            "total_size": int(size.sum()), "slices": int(n_sl), "max_slice_resident_bytes": int(res.max()),
            "mean_slice_resident_bytes": float(res.mean())}


def main():
    steps = int(os.environ.get("KB_COMP_STEPS", "15"))
    P = 2000000
    idx, concat, lens = bench.workload(62000)
    dev = torch.device("cuda", 0)
    ix = K.KmerIndex(idx, device=0, threads=16)
    sim = benchdata.TorchSimulator(concat, lens, dev, read_len=100)
    mc = K.MinCollector(ix, paired=True, max_batch_reads=P, max_batch_bases=P * 200 + 64)
    for sd in bench.job_seeds(0, 3, steps):
        b = sim.pairs(P, seed=sd)
        mc.process_buffer_device(b.data_ptr(), None, 2 * P, 100)
        mc.sync()
        del b
    mc.run_em()
    eo, et, _, _ = mc.ec_table()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps(components(np.asarray(eo), np.asarray(et).astype(np.int64), ix.num_trans, sms)), flush=True)
    mc.close()
    ix.close()


if __name__ == "__main__":
    main()
