#!/usr/bin/env python
"""match_kernel A/B on the benchmark workload: presence-filter size (KB_FILTER_LOG2; 32 = off), table load factor
(KB_TABLE_FACTOR), persisting-L2 carve-out (KB_L2_PERSIST_MB) and lanes per fragment of resolve_kernel (KB_RESOLVE_G).  One JSON line per configuration: ms per launch of
2 M pairs, slot visits per pair (HBM sectors), probes per pair, and a digest of the EC counts (must not change).
A configuration with "KB_NVCC_DEFS" (e.g. "-DKB_MATCH_MIN_BLOCKS=4") runs on a library built
with those defines into a temporary directory (the in-tree build is untouched), in a process of its own; with
KB_SWEEP_CHILD=1 the configurations run on the library KB_LIB_PATH names instead (built beforehand with those defines)."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import benchdata  # noqa: E402
import kallisto_b200 as K  # noqa: E402


def run_built(cfg):
    with tempfile.TemporaryDirectory(prefix="kb_match_sweep_") as tmp:
        lib = os.path.join(tmp, "libkallisto_b200.so")
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "kallisto_b200", "csrc"), "-j8", lib, "OUT=" + lib,
                               "OBJDIR=" + os.path.join(tmp, "obj"), "NVCC=nvcc " + cfg["KB_NVCC_DEFS"]], stdout=subprocess.DEVNULL)
        ptxas = open(os.path.join(tmp, "obj", "kernels_align.ptxas.log")).read().split("\n")
        i = next(j for j, ln in enumerate(ptxas) if "Compiling entry function" in ln and "match_kernel" in ln)
        print("# %s ptxas: %s / %s" % (cfg["KB_NVCC_DEFS"], ptxas[i + 2].strip(), ptxas[i + 3].strip()), flush=True)
        env = dict(os.environ, KB_LIB_PATH=lib, KB_SWEEP_CHILD="1")
        subprocess.check_call([sys.executable, os.path.abspath(__file__), json.dumps(cfg)], env=env)


def main():
    P, steps = 2000000, int(os.environ.get("KB_SWEEP_STEPS", "8"))
    idx, concat, lens = bench.workload(62000)
    dev = torch.device("cuda", 0)
    sim = benchdata.TorchSimulator(concat, lens, dev, read_len=100)
    batches = [sim.pairs(P, seed=sd) for sd in bench.job_seeds(0, 5, steps)]
    configs = [dict(KB_FILTER_LOG2="32"), dict(KB_FILTER_LOG2="29"), dict(KB_FILTER_LOG2="28"), dict(KB_FILTER_LOG2="30"),
               dict(KB_FILTER_LOG2="29", KB_L2_PERSIST_MB="0"), dict(KB_FILTER_LOG2="29", KB_TABLE_FACTOR="2"),
               dict(KB_FILTER_LOG2="32", KB_TABLE_FACTOR="2")]
    if len(sys.argv) > 1:
        configs = [json.loads(a) for a in sys.argv[1:]]
    for cfg in configs:
        if "KB_NVCC_DEFS" in cfg and not os.environ.get("KB_SWEEP_CHILD"):
            run_built(cfg)
            continue
        for k in ("KB_FILTER_LOG2", "KB_L2_PERSIST_MB", "KB_TABLE_FACTOR", "KB_RESOLVE_G", "KB_REFILL_MIN"):
            os.environ.pop(k, None)
        os.environ.update({k: v for k, v in cfg.items() if k != "KB_NVCC_DEFS"})
        ix = K.KmerIndex(idx, device=0, threads=16)
        best = None
        for rep in range(2):
            mc = K.MinCollector(ix, paired=True, max_batch_reads=P, max_batch_bases=P * 200 + 64)
            mc.enable_timing(True)
            for b in batches:
                mc.process_buffer_device(b.data_ptr(), None, 2 * P, 100)
            st = mc.finalize()
            tm = mc.timings()
            eo, et, ec, _ = mc.ec_table()
            dig = hashlib.md5(eo.tobytes() + et.tobytes() + ec.tobytes()).hexdigest()[:12]
            mc.close()
            ms = tm["match_ms"] / tm["match_launches"]
            if best is None or ms < best["match_ms_per_launch"]:
                best = {"pack_ms_per_launch": tm["pack_ms"] / tm["match_launches"], "match_ms_per_launch": ms, "resolve_ms_per_launch": tm["resolve_ms"] / tm["resolve_launches"],
                        "slot_visits_per_pair": st["n_slot_visits"] / (steps * P), "probes_per_pair": st["n_probes"] / (steps * P),
                        "ec_digest": dig, "table_slots": ix.info["table_slots"]}
        print(json.dumps({**cfg, **best}), flush=True)
        ix.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
