"""bench.py --workload bus10xv3 | bootstrap: BASELINE configs 3 and 4 (SURVEY.md 8d).  Same JSON contract as the
quant workload (bench.py); run by hand; the default run of bench.py is `quant`.

  bus10xv3   `kallisto bus -x 10xv3` record path: R1 = 16-nt barcode + 12-nt UMI, R2 = 91-nt cDNA, synthetic
             (benchdata.TorchSimulator10x), human-like index.  step = one batch of read sets through kb_bus_batch_device
             (barcode/UMI slicing + pseudoalignment with the technology's strand filter + EC ids + 32-byte records).
             value = read sets/s with the batch files resident in HBM; e2e = `kallisto_b200 bus` FASTQ -> output.bus,
             process wall clock; --impl reference = `kallisto bus -x 10xv3 -t T` on the same FASTQ files.
  bootstrap  `quant -b 100`: the bootstrap phase (multinomial resampling of the EC counts + one EM per sample) on the EC
             table of the K x P pair job.  value = bootstrap samples/s (kb_bootstrap_run, B = 100, resample + batched EM);
             --impl reference = the reference's sequential loop (src/main.cpp:2769-2782; it only runs with -t 1) timed on a
             2 M-pair sample for 3 samples, from the timestamps of its own "[bstrp]" progress lines, with our arm's time
             on the SAME sample next to it.
"""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

import bench
import benchdata
from bench import CACHE_ROOT, READ_LEN, ROOT, ClockSampler, log, measured_peak, workload

CDNA = 91


def main(args, rank, world, local_rank, workload_name):
    if world > 1 and rank != 0:
        return 0        # these two workloads are single-GPU lines
    if args.workload == "bus10xv3":
        return bus_main(args, local_rank, workload_name)
    return bootstrap_main(args, local_rank, workload_name)


# ---------------------------------------------------------------------------------------------------------------
def _bus_files(genes, P, K, W, sim_factory):
    import fcntl
    d = os.path.join(CACHE_ROOT, "bus_g%d_p%d_k%d_w%d" % (genes, P, K, W))
    os.makedirs(d, exist_ok=True)
    f1, f2 = os.path.join(d, "r_1.fq"), os.path.join(d, "r_2.fq")
    done = os.path.join(d, "complete")
    with open(os.path.join(d, ".lock"), "w") as lockf:
        fcntl.flock(lockf, fcntl.LOCK_EX)
        try:
            if not os.path.exists(done):
                t0 = time.time()
                sim = sim_factory()
                for f in (f1, f2):
                    open(f, "wb").close()
                for j in range(K):
                    r1, r2 = sim.sets(P, seed=7000 + W + j)
                    for f, r, tag in ((f1, r1, 1), (f2, r2, 2)):
                        with open(f, "ab") as fh:
                            benchdata.fastq_image(r, tag, j * P).cpu().numpy().tofile(fh)
                open(done, "w").write("%d sets\n" % (K * P))
                log("bus FASTQ (%d read sets, %.1f GB) written in %.0f s" % (K * P, (os.path.getsize(f1) + os.path.getsize(f2)) / 1e9,
                                                                           time.time() - t0))
        finally:
            fcntl.flock(lockf, fcntl.LOCK_UN)
    return d, f1, f2


def bus_main(args, local_rank, workload_name):
    import torch
    import kallisto_b200 as K200
    from oracle import oracle as O
    K, W = args.steps, max(args.warmup, 0)
    P = args.pairs_per_step if args.pairs_per_step != 2000000 else int(os.environ.get("KB_BENCH_SETS", "8000000"))
    idx, concat, lens = workload(args.genes)
    dev = torch.device("cuda", local_rank) if torch.cuda.is_available() else torch.device("cpu")
    name = workload_name.replace("synthetic 2x100bp pairs", "synthetic 10x v3 read sets (28-nt R1, %d-nt cDNA R2)" % CDNA)

    def sim_factory():
        return benchdata.TorchSimulator10x(concat, lens, dev, cdna_len=CDNA)

    d, f1, f2 = _bus_files(args.genes, P, K, W, sim_factory)
    cores = os.cpu_count() or 1
    if args.impl == "reference":
        out = os.path.join(d, "ref_out")
        with open(idx, "rb") as f:
            while f.read(1 << 26):
                pass
        threads = min(cores, 32)
        t0 = time.perf_counter()
        r = O.ref_run(["bus", "-x", "10xv3", "-i", idx, "-o", out, "-t", str(threads), f1, f2], check=False)
        dt = time.perf_counter() - t0
        if r.returncode != 0:
            raise RuntimeError(r.stderr.decode(errors="replace")[-300:])
        v = K * P / dt
        line = {"metric": "read sets/sec bus 10xv3", "value": v, "unit": "reads/s", "n_gpus": args.gpus, "steps": K, "warmup": W,
                "ms_per_step": dt * 1e3 / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u64",
                "data": "synthetic", "impl": "reference",
                "config": {"workload": name, "sets_per_step": P, "reference": "oracle/_ref/kallisto bus -x 10xv3 -t %d, plain FASTQ in "
                           "/dev/shm -> output.bus; process wall clock incl. index load" % threads, "seconds_process_wall": round(dt, 2),
                           "threads": threads, "host_cores": cores},
                "cpu_baseline": {"value": v, "unit": "reads/s", "cores": threads, "kind": "reference", "sample": "all %d read sets" % (K * P)},
                "e2e": {"value": v, "unit": "reads/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        json.dump(line, open(os.path.join(d, "reference_line.json"), "w"))
        print(json.dumps(line), flush=True)
        return 0

    torch.cuda.set_device(local_rank)
    index = K200.KmerIndex(idx, device=local_rank, threads=min(16, cores))
    sim = sim_factory()
    batches = []
    for j in range(W + K):
        r1, r2 = sim.sets(P, seed=7000 + j)
        batches.append((r1, r2))
    o1 = (torch.arange(P + 1, device=dev, dtype=torch.int64) * 28).to(torch.int32)
    o2 = (torch.arange(P + 1, device=dev, dtype=torch.int64) * CDNA).to(torch.int32)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()

    def job(bs, timed):
        bp = K200.BUSProcessor(index, "10xv3", max_batch_sets=P)
        bp.set_stream(stream.cuda_stream)
        if timed:
            bp.enable_timing(True)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        n_rec = 0
        for r1, r2 in bs:
            n, _ = bp.process_sets_device([r1.data_ptr(), r2.data_ptr()], [o1.data_ptr(), o2.data_ptr()], P, CDNA)
            n_rec += n
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1), n_rec, bp

    ms, _, bp = job(batches[:max(1, W)], False)
    bp.close()
    ms, _, bp = job(batches[W:], False)
    bp.close()
    runs = []
    ms, _, bp = job(batches[W:], True)
    bp.close()
    runs.append(ms)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ms, n_rec, bp = job(batches[W:], True)
    clocks = sampler.stop()
    runs.append(ms)
    st = bp.finalize()
    tm = bp.timings()
    bp.close()
    value = K * P / (ms * 1e-3)
    probes = st["n_probes"] / max(1, K * P)
    visits = st["n_slot_visits"] / max(1, K * P)
    bytes_per_set = 28 + CDNA + probes * 32 + 16 + 32.0 * n_rec / (K * P)
    peak, peak_src = measured_peak()
    mml = tm["match_ms"] / max(1, tm["match_launches"])
    ach = (CDNA + probes * 32 + 16) * P / (mml * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": "match_kernel", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                "peak_source": peak_src, "traffic": None, "bytes_per_read": CDNA + probes * 32 + 16, "probes_per_read": probes,
                "slot_visits_per_read": visits, "ms_per_launch": mml, "bytes_per_set_whole_step": bytes_per_set,
                "record_bytes_per_step": 32.0 * n_rec / K}
    del batches, sim
    index.close()
    torch.cuda.empty_cache()
    # e2e: the command line, FASTQ -> output.bus
    exe = os.path.join(ROOT, "kallisto_b200", "kallisto_b200")
    out = os.path.join(d, "cli_out")
    threads = min(cores, 64)
    walls = []
    for _ in range(2):
        t0 = time.perf_counter()
        r = subprocess.run([exe, "bus", "-x", "10xv3", "-i", idx, "-o", out, "-t", str(threads), "--device", str(local_rank), f1, f2],
                           stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True, env=dict(os.environ, KB_CLI_TIMING="1"))
        walls.append(time.perf_counter() - t0)
        if r.returncode != 0:
            raise RuntimeError(r.stderr[-400:])
    ph = {m.group(1): float(m.group(2)) for m in re.finditer(r"\[timing\] ([^:\n]+): ([0-9.eE+-]+) s \(at", r.stderr)}
    e2e = {"value": K * P / walls[-1], "unit": "reads/s", "h2d_bytes_per_step": P * (28 + CDNA) + 8 * (P + 1), "d2h_bytes_per_step": int(32 * n_rec / K),
           "api": "kallisto_b200 bus -x 10xv3 -t %d (plain FASTQ in /dev/shm -> output.bus, matrix.ec): read sets / process wall clock, "
                  "index load included" % threads, "seconds_process_wall_runs": [round(x, 3) for x in walls], "phases_s": ph,
           "output_bus_bytes": os.path.getsize(os.path.join(out, "output.bus"))}
    cpu = None
    rl = os.path.join(d, "reference_line.json")
    if os.path.exists(rl):
        cpu = json.load(open(rl))["cpu_baseline"]
    line = {"metric": "read sets/sec bus 10xv3", "value": value, "unit": "reads/s", "n_gpus": 1, "steps": K, "warmup": W,
            "ms_per_step": ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u64", "data": "synthetic",
            "config": {"workload": name, "sets_per_step": P, "l2": "every step reads a different %d MB batch (> 50 MB L2)" % (P * (28 + CDNA) // 1000000),
                       "total_ms_runs": [round(x, 3) for x in runs], "reported_run": "second of two timed runs", "records": n_rec,
                       "p_pseudoaligned": st["n_pseudoaligned"] / max(1, st["n_processed"]), "n_ecs": st["n_ecs"],
                       "resolve_ms_per_launch": tm["resolve_ms"] / max(1, tm["resolve_launches"])},
            "clocks": clocks, "e2e": e2e, "gpu_launches": int(tm["kernel_launches"]), "roofline": roofline}
    if cpu:
        line["cpu_baseline"] = cpu
    print(json.dumps(line), flush=True)
    return 0


# ---------------------------------------------------------------------------------------------------------------
def _ref_bootstrap_phase(idx, f1, f2, n_samples, outdir):
    """Runs `kallisto quant --plaintext -t 1 -b n` and timestamps its progress lines.  -> (seconds per bootstrap sample,
    seconds of the main EM, whole wall)."""
    from oracle import oracle as O
    p = subprocess.Popen([O.REF_BIN, "quant", "-i", idx, "-o", outdir, "--plaintext", "-t", "1", "-b", str(n_samples), "--seed", "42", f1, f2],
                         stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    t0 = time.perf_counter()
    marks = {}
    buf = b""
    while True:
        c = p.stderr.read(1)
        if not c:
            break
        buf += c
        for key in ([b"quantifying the abundances ...", b"Expectation-Maximization algorithm ran for"] +
                    [b"running EM for the bootstrap: %d" % (k + 1) for k in range(n_samples)]):
            if key not in marks and key in buf:
                marks[key] = time.perf_counter() - t0
    p.wait()
    t_end = time.perf_counter() - t0
    bs = [marks.get(b"running EM for the bootstrap: %d" % (k + 1)) for k in range(n_samples)] + [t_end]
    per = [b - a for a, b in zip(bs[:-1], bs[1:]) if a is not None and b is not None]
    em = None
    if b"quantifying the abundances ..." in marks and b"Expectation-Maximization algorithm ran for" in marks:
        em = marks[b"Expectation-Maximization algorithm ran for"] - marks[b"quantifying the abundances ..."]
    return (float(np.mean(per)) if per else None), em, t_end


def bootstrap_main(args, local_rank, workload_name):
    import torch
    import kallisto_b200 as K200
    K, W, P = args.steps, max(args.warmup, 0), args.pairs_per_step
    B = int(os.environ.get("KB_BENCH_BOOTSTRAPS", "100"))
    idx, concat, lens = workload(args.genes)
    dev = torch.device("cuda", local_rank) if torch.cuda.is_available() else torch.device("cpu")
    cores = os.cpu_count() or 1

    def sim_factory(dv=None):
        return benchdata.TorchSimulator(concat, lens, dv if dv is not None else dev, read_len=READ_LEN)

    files = bench.fastq_job_files(args.genes, P, K, W, sim_factory)
    d, f1, f2, s1, s2, t1, t2 = files
    n_s = sum(1 for _ in open(s1, "rb")) // 4
    if args.impl == "reference":
        per, em, wall = _ref_bootstrap_phase(idx, s1, s2, 3, os.path.join(d, "ref_bs_out"))
        v = 1.0 / per
        line = {"metric": "bootstrap samples/sec quant -b", "value": v, "unit": "samples/s", "n_gpus": args.gpus, "steps": K, "warmup": W,
                "ms_per_step": per * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
                "impl": "reference",
                "config": {"workload": workload_name + " -- bootstrap phase", "reference": "oracle/_ref/kallisto quant --plaintext -t 1 -b 3 on the "
                           "%d-pair sample of the job (the sequential loop of src/main.cpp:2769-2782 only runs with -t 1, and -t 1 on the whole "
                           "%d-pair job would take ~20 min of pseudoalignment first): seconds per sample from the timestamps of its own [bstrp] "
                           "lines" % (n_s, K * P), "seconds_per_sample": per, "seconds_main_em": em, "seconds_process_wall": wall,
                           "sample_pairs": n_s},
                "cpu_baseline": {"value": v, "unit": "samples/s", "cores": 1, "kind": "reference", "sample": "%d-pair sample, 3 bootstrap samples" % n_s},
                "e2e": {"value": v, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        json.dump(line, open(os.path.join(d, "reference_bs_line.json"), "w"))
        print(json.dumps(line), flush=True)
        return 0

    torch.cuda.set_device(local_rank)
    index = K200.KmerIndex(idx, device=local_rank, threads=min(16, cores))
    sim = sim_factory(dev)
    stream = torch.cuda.current_stream()

    def quant_run(seeds, n_pairs):
        mc = K200.MinCollector(index, paired=True, max_batch_reads=n_pairs, max_batch_bases=n_pairs * 2 * READ_LEN + 64)
        mc.set_stream(stream.cuda_stream)
        for sd in seeds:
            b = sim.pairs(n_pairs, seed=sd)
            mc.process_buffer_device(b.data_ptr(), None, 2 * n_pairs, READ_LEN)
            mc.sync()
            del b
        em = mc.run_em()
        return mc, em

    def timed_bootstrap(mc, nb):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = mc.run_bootstrap(nb, seed=42)
        dt = time.perf_counter() - t0
        tm = mc.timings()
        return dt, tm["bs_resample_ms"], tm["bs_em_ms"], r

    # the job's own EC table (K x P pairs)
    mc, em = quant_run(bench.job_seeds(0, W, K), P)
    st = mc.finalize()
    sampler = ClockSampler(local_rank)
    runs = []
    dt, _, _, _ = timed_bootstrap(mc, B)
    runs.append(dt)
    sampler.start()
    dt, rs_ms, em_ms, r = timed_bootstrap(mc, B)
    clocks = sampler.stop()
    runs.append(dt)
    kl = mc.timings()["kernel_launches"]
    mc.close()
    rounds = r["rounds"]
    eo_n = st["n_ecs"]
    # like for like with the reference arm: the same sample (first min(P, 2 M) pairs of the job's first batch), 3 samples
    mc2 = K200.MinCollector(index, paired=True, max_batch_reads=n_s, max_batch_bases=n_s * 2 * READ_LEN + 64)
    mc2.set_stream(stream.cuda_stream)
    b = sim.pairs(P, seed=bench.job_seeds(0, W, K)[0])[:n_s].contiguous()
    mc2.process_buffer_device(b.data_ptr(), None, 2 * n_s, READ_LEN)
    mc2.sync()
    mc2.run_em()
    timed_bootstrap(mc2, 3)
    dt3, rs3, em3, r3 = timed_bootstrap(mc2, 3)
    mc2.close()
    index.close()
    value = B / dt
    peak, peak_src = measured_peak()
    line = {"metric": "bootstrap samples/sec quant -b", "value": value, "unit": "samples/s", "n_gpus": 1, "steps": K, "warmup": W,
            "ms_per_step": dt * 1e3 / B, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": workload_name + " -- bootstrap phase of quant -b %d on the EC table of %d pairs" % (B, K * P),
                       "n_bootstraps": B, "seconds_runs": [round(x, 4) for x in runs], "reported_run": "second of two",
                       "resample_ms": rs_ms, "em_ms": em_ms, "rounds_mean": float(np.mean(rounds)), "rounds_max": int(np.max(rounds)),
                       "n_ecs": eo_n, "n_draws_per_sample": st["n_pseudoaligned"], "main_em_rounds": em["rounds"],
                       "same_sample_as_reference_arm": {"pairs": n_s, "n_bootstraps": 3, "seconds": dt3, "seconds_per_sample": dt3 / 3,
                                                        "resample_ms": rs3, "em_ms": em3, "rounds": [int(x) for x in r3["rounds"]]}},
            "clocks": clocks,
            "e2e": {"value": value, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": int(index.num_trans * 8),
                    "api": "kb_bootstrap_run (host wall clock: resample kernel, batched EM in L2-sized chunks, est_counts of every sample copied "
                           "back to the host)"},
            "gpu_launches": int(kl),
            "roofline": {"bound": "hbm", "kernel": "em_kernel (batched)", "achieved": None, "peak": peak, "unit": "GB/s", "frac": None,
                         "peak_source": peak_src, "traffic": None,
                         "note": "the batched EM works out of L2 (chunks of samples whose alpha/norm/counts take at most half of the L2); see roofline_em of the quant line"}}
    rl = os.path.join(d, "reference_bs_line.json")
    if os.path.exists(rl):
        ref = json.load(open(rl))
        line["cpu_baseline"] = ref["cpu_baseline"]
        line["config"]["reference_seconds_per_sample_on_same_sample"] = ref["config"]["seconds_per_sample"]
    print(json.dumps(line), flush=True)
    return 0
