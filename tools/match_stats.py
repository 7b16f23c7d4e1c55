#!/usr/bin/env python
"""Where match_kernel's iterations go, on the benchmark workload: builds the library with -DKB_MATCH_STATS into a
temporary directory (the in-tree build is untouched), runs the benchmark batches once and prints one JSON line with
the summed per-launch counters and their shares.  The counters slow the kernel, so its times are not reported; the counts themselves do not depend on that.
Of the chain iterations (a live chain's probes, collisions included), the share settled on the straight-line path
(collisions, MAIN misses on mates without N) is reported, and the passes of the general transition per warp-iteration
(a warp runs as many as its busiest lane needs).
The clock split of a lookup iteration (keys and hashes / the wait for the filter and slot loads / the state transitions)
is given in cycles per lane-iteration.  KB_NVCC_DEFS adds defines to the build (e.g. -DKB_MATCH_MIN_BLOCKS=4); a
library built beforehand with -DKB_MATCH_STATS (and those defines) can be named by KB_LIB_PATH instead."""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build(out_dir):
    lib = os.path.join(out_dir, "libkallisto_b200.so")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "kallisto_b200", "csrc"), "-j8", lib, "OUT=" + lib,
                           "OBJDIR=" + os.path.join(out_dir, "obj"), "NVCC=nvcc -DKB_MATCH_STATS " + os.environ.get("KB_NVCC_DEFS", "")], stdout=subprocess.DEVNULL)
    return lib


def main():
    with tempfile.TemporaryDirectory(prefix="kb_match_stats_") as tmp:
        run(tmp)


def run(tmp):
    if not os.environ.get("KB_LIB_PATH"):
        os.environ["KB_LIB_PATH"] = build(tmp)
    import torch
    import bench
    import benchdata
    import kallisto_b200 as K

    P, steps = 2000000, int(os.environ.get("KB_SWEEP_STEPS", "8"))
    idx, concat, lens = bench.workload(62000)
    dev = torch.device("cuda", 0)
    sim = benchdata.TorchSimulator(concat, lens, dev, read_len=100)
    batches = [sim.pairs(P, seed=sd) for sd in bench.job_seeds(0, 5, steps)]
    ix = K.KmerIndex(idx, device=0, threads=16)
    log = os.path.join(tmp, "stats.txt")
    saved = os.dup(2)
    with open(log, "w") as f:
        os.dup2(f.fileno(), 2)       # the library prints one line per launch to stderr
        try:
            mc = K.MinCollector(ix, paired=True, max_batch_reads=P, max_batch_bases=P * 200 + 64)
            for b in batches:
                mc.process_buffer_device(b.data_ptr(), None, 2 * P, 100)
            st = mc.finalize()
            mc.close()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
    tot = {}
    for line in open(log):
        if line.startswith("kb_match_stats "):
            for k, v in json.loads(line[len("kb_match_stats "):]).items():
                tot[k] = tot.get(k, 0) + v
    lane = max(1, tot["chain_iters"])
    main_miss = tot["main_miss_filter"] + tot["main_miss_slot"]
    runs = {k: v for k, v in tot.items() if k.startswith("run_")}
    out = {"defs": os.environ.get("KB_NVCC_DEFS", ""), "launches": steps, "pairs": steps * P, **tot,
           "n_probes": st["n_probes"], "n_slot_visits": st["n_slot_visits"],
           "main_miss_lookups": main_miss,
           "share_main_miss_of_lookups": main_miss / max(1, st["n_probes"]),
           "share_main_miss_of_chain_iters": main_miss / lane,
           "live_chains_per_warp_iter": tot["chain_iters"] / max(1, tot["warp_iters"]),
           "share_straight_of_chain_iters": tot["straight"] / lane,
           "general_passes_per_warp_iter": tot["gen_passes"] / max(1, tot["warp_iters"]),
           "service_share_of_cycles": tot["cycles_service"] / max(1, tot["cycles_service"] + tot["cycles_lookup"]),
           "cycles_per_warp_iter": tot["cycles_lookup"] / max(1, tot["warp_iters"]),
           "cycles_per_lane_iter": {p: tot["cycles_" + p] / max(1, tot["lane_iters"]) for p in ("key", "wait", "step")},
           "miss_runs": sum(runs.values())}
    print(json.dumps(out), flush=True)
    ix.close()


if __name__ == "__main__":
    main()
