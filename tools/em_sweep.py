#!/usr/bin/env python
"""EM kernel sweep on the benchmark's EC table (20 x 2 M pairs): em_ms / us per round of the default path
(em_component_kernel with the entries resident in shared memory), of the same kernel streaming its entries
(KB_EM_COMP_SMEM=0) and of the launch shapes of the grid-wide kernels, KB_EM_SHAPE x KB_EM_TPB x KB_EM_BLOCKS (the
library reads them at every launch).  Prints one JSON line per configuration."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import benchdata  # noqa: E402
import kallisto_b200 as K  # noqa: E402


def main():
    steps = int(os.environ.get("KB_SWEEP_STEPS", "20"))
    P = 2000000
    idx, concat, lens = bench.workload(62000)
    dev = torch.device("cuda", 0)
    ix = K.KmerIndex(idx, device=0, threads=16)
    sim = benchdata.TorchSimulator(concat, lens, dev, read_len=100)
    mc = K.MinCollector(ix, paired=True, max_batch_reads=P, max_batch_bases=P * 200 + 64)
    for sd in bench.job_seeds(0, 5, steps):
        b = sim.pairs(P, seed=sd)
        mc.process_buffer_device(b.data_ptr(), None, 2 * P, 100)
        mc.sync()
        del b
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ref = None
    # KB_EM_SHAPE: launch shape of the single-problem kernel (-1: the batched kernel with one problem, KB_EM_TPB x KB_EM_BLOCKS);
    # unset: the default path, em_component_kernel when every component fits a block
    for shape, smem, name in [(None, None, "em_component_kernel (default)"),
                              (None, "0", "em_component_kernel, entries streamed (KB_EM_COMP_SMEM=0)"),
                              (-1, None, "em_kernel<1024,1> (batched kernel, nb = 1)"),
                              (0, None, "em_single 1024 x 1"), (1, None, "em_single 512 x 3"), (2, None, "em_single 768 x 2"),
                              (3, None, "em_single 1024 x 2")]:
        if shape is None:
            os.environ.pop("KB_EM_SHAPE", None)
        else:
            os.environ["KB_EM_SHAPE"] = str(shape)
        if smem is None:
            os.environ.pop("KB_EM_COMP_SMEM", None)
        else:
            os.environ["KB_EM_COMP_SMEM"] = smem
        os.environ["KB_EM_TPB"] = "1024"
        os.environ.pop("KB_EM_BLOCKS", None)
        os.environ["KB_EM_OCC"] = "1"
        best = None
        for _ in range(3):
            r = mc.run_em()
            tm = mc.timings()
            if best is None or tm["em_ms"] < best[0]:
                best = (tm["em_ms"], r["rounds"], tm["em_prep_ms"], tm["em_comp_blocks"], tm["em_comp_resident"])
        if ref is None:
            ref = r["est_counts"].copy()
        same = bool((r["est_counts"] == ref).all())
        print(json.dumps({"shape": shape, "kernel": name, "em_ms": best[0], "rounds": best[1], "us_per_round": best[0] * 1e3 / best[1],
                          "prep_ms": best[2], "component_blocks": best[3], "component_resident": best[4],
                          "bit_identical_to_first": same}), flush=True)
    mc.close()
    ix.close()


if __name__ == "__main__":
    main()
