"""GPU: parity at BASELINE config-2 scale -- the 62 000-gene / 147 M-k-mer index the benchmark uses (711 k index
EC sets, 45 k short unitigs; a 2^29-slot = 17 GB k-mer table on an 80 GB H100), >= 2 M synthetic 2x100 bp pairs, against
the UNMODIFIED reference (oracle/_ref/kallisto) run on the same FASTQ files on the host cores:

  * per-fragment equivalence classes: `kallisto bus -x bulk --paired --num -t 1` (main.cpp:1050-1107,
    ProcessReads.cpp:1643-1701) on 8 consecutive slices of the input in parallel processes; every fragment's
    transcript SET must be identical, and so must the EC count multiset, n_processed / n_pseudoaligned / n_unique,
    the fragment-length histogram (first slice = first 10 000 unique pairs of the run) and the order in which ECs
    are first seen (ids of the first slice; the first slice is 30 % of the input so that it contains the 10 000
    fragment-length samples of the run);
  * quantification: `kallisto quant --plaintext -t 1 -b 2 --seed 42` on the whole input; abundance.tsv and
    bs_abundance_{0,1}.tsv must be TEXT-identical, both through the library and through the kallisto_b200 CLI.

Everything is generated here (index by the reference's `kallisto index`, reads by benchdata.TorchSimulator), nothing
is read from /root/reference.  KB_SCALE_PAIRS / KB_SCALE_GENES shrink the case for quick local runs."""
import json
import os
import shutil
import subprocess
import tempfile
import time

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu

N_PAIRS = int(os.environ.get("KB_SCALE_PAIRS", "2000000"))
GENES = int(os.environ.get("KB_SCALE_GENES", "62000"))
N_SLICES = 8
CLI = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")


def _log(*a):
    print("[scale]", *a, flush=True)


@pytest.fixture(scope="module")
def scale():
    import torch
    import bench
    import benchdata
    t0 = time.time()
    idx, concat, lens = bench.workload(GENES)
    _log("workload ready in %.0f s" % (time.time() - t0))
    dev = torch.device("cuda", 0)
    sim = benchdata.TorchSimulator(concat, lens, dev, read_len=100)
    parts = []
    for c0 in range(0, N_PAIRS, 1 << 20):
        parts.append(sim.pairs(min(1 << 20, N_PAIRS - c0), seed=424242 + c0).cpu().numpy())
    reads = np.concatenate(parts)            # (N, 2, 100) ASCII
    del sim, parts
    torch.cuda.empty_cache()
    shm = "/dev/shm" if os.path.isdir("/dev/shm") else None
    td = tempfile.mkdtemp(prefix="kb_scale_", dir=shm)
    try:
        f1, f2 = os.path.join(td, "all_1.fq"), os.path.join(td, "all_2.fq")
        benchdata.write_fastq_fast(f1, reads[:, 0], 1)
        benchdata.write_fastq_fast(f2, reads[:, 1], 2)
        # the first slice is large enough to hold the first 10 000 fragment-length samples of the run (only ~2.5 % of the
        # pairs qualify: unique transcript and both mates on one unitig, ProcessReads.cpp:1174-1181), so that its
        # flens.txt is the histogram of the whole run; the others share the rest
        n0 = N_PAIRS * 3 // 10
        bounds = [0] + [n0 + (N_PAIRS - n0) * i // (N_SLICES - 1) for i in range(N_SLICES)]
        procs = []
        env = dict(os.environ)
        qdir = os.path.join(td, "ref_quant")
        procs.append(("quant", subprocess.Popen(
            [O.REF_BIN, "quant", "-i", idx, "-o", qdir, "--plaintext", "-t", "1", "-b", "2", "--seed", "42", f1, f2],
            stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=env)))
        for s in range(N_SLICES):
            a, b = bounds[s], bounds[s + 1]
            s1, s2 = os.path.join(td, "s%d_1.fq" % s), os.path.join(td, "s%d_2.fq" % s)
            benchdata.write_fastq_fast(s1, reads[a:b, 0], 1)
            benchdata.write_fastq_fast(s2, reads[a:b, 1], 2)
            procs.append(("bus%d" % s, subprocess.Popen(
                [O.REF_BIN, "bus", "-x", "bulk", "--paired", "--num", "-t", "1", "-i", idx, "-o", os.path.join(td, "ref_bus%d" % s),
                 s1, s2], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=env)))
        t_ref = time.time()

        # ---- the CUDA path while the reference works on the host cores ----
        ix = K.KmerIndex(idx, device=0, threads=16)
        mc = K.MinCollector(ix, paired=True, max_batch_reads=1 << 20, max_batch_bases=(1 << 20) * 100 + 64)
        hs = []
        B = 1 << 19
        for a in range(0, N_PAIRS, B):
            blk = np.ascontiguousarray(reads[a:a + B]).reshape(-1)
            hs.append(mc.process_buffer(blk, None, fixed_len=100))
        handles = np.concatenate(hs)
        st = mc.finalize()
        eo, et, ec, eh = mc.ec_table()
        flens = mc.flens.copy()
        em = mc.run_em()
        bs = mc.run_bootstrap(2, seed=42)
        mc.close()
        ix.close()
        cdir = os.path.join(td, "cli_quant")
        r = subprocess.run([CLI, "quant", "-i", idx, "-o", cdir, "--plaintext", "-b", "2", "--seed", "42", "-t", "16", f1, f2],
                           stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        _log("CUDA path done %.0f s after the reference started" % (time.time() - t_ref))
        for name, p in procs:
            _, err = p.communicate()
            assert p.returncode == 0, (name, err[-2000:])
        _log("reference done after %.0f s" % (time.time() - t_ref))
        del reads
        yield dict(td=td, idx=idx, bounds=bounds, handles=handles, st=st, ec=(eo, et, ec, eh), flens=flens, em=em, bs=bs,
                   qdir=qdir, cdir=cdir, names=ix.target_names_, lens=ix.target_lens_)
    finally:
        shutil.rmtree(td, ignore_errors=True)


def _canon(sets, table):
    """EC sets (tuples of transcript ids) -> canonical ids shared by every table of the test."""
    out = np.empty(len(sets), np.int64)
    for i, s in enumerate(sets):
        out[i] = table.setdefault(s, len(table))
    return out


def test_index_is_config2_sized(scale):
    info = K.inspect_index(scale["idx"])
    if GENES >= 62000:
        assert info["n_kmers"] > 100_000_000 and info["n_targets"] > 200_000
    n_long, n_short, n_abund = O.index_unitig_kinds(scale["idx"])
    assert n_short > 0


def test_per_fragment_sets_counts_and_order(scale):
    eo, et, ec, eh = scale["ec"]
    table = {}
    mine_sets = util.ec_sets(eo, et)
    mine_c = _canon(mine_sets, table)
    assert len(set(mine_c.tolist())) == len(mine_c)          # our ECs are distinct sets
    # our per-fragment result as canonical set ids
    lut = np.full(int(eh.max()) + 2, -1, np.int64)
    lut[eh] = mine_c
    h = scale["handles"]
    mine_frag = np.where(h >= 0, lut[np.maximum(h, 0)], -1)
    ref_counts = {}
    n_proc = n_pa = n_uniq = 0
    bounds = scale["bounds"]
    for s in range(N_SLICES):
        d = os.path.join(scale["td"], "ref_bus%d" % s)
        _, rec = O.read_bus(os.path.join(d, "output.bus"))
        sets = O.read_matrix_ec(os.path.join(d, "matrix.ec"))
        info = json.load(open(os.path.join(d, "run_info.json")))
        canon = _canon(sets, table)
        n = bounds[s + 1] - bounds[s]
        assert info["n_processed"] == n
        frag = np.full(n, -1, np.int64)
        frag[rec["flags"]] = canon[rec["ec"]]
        np.testing.assert_array_equal(mine_frag[bounds[s]:bounds[s + 1]], frag, err_msg="slice %d" % s)
        ids, cnt = np.unique(frag[frag >= 0], return_counts=True)
        for i, c in zip(ids.tolist(), cnt.tolist()):
            ref_counts[i] = ref_counts.get(i, 0) + c
        n_proc += info["n_processed"]; n_pa += info["n_pseudoaligned"]; n_uniq += info["n_unique"]
        if s == 0:
            # EC ids = order of first occurrence: the first slice's ECs are the first ECs of the whole run, in order
            assert mine_sets[:len(sets)] == sets
            fl = np.array([int(x) for x in open(os.path.join(d, "flens.txt")).read().split()], np.uint32)
            if N_PAIRS >= 2000000:
                assert int(fl.sum()) == 10000      # premise: the quota is filled inside the first slice
            if int(fl.sum()) == 10000:
                np.testing.assert_array_equal(scale["flens"], fl)
    st = scale["st"]
    assert (st["n_processed"], st["n_pseudoaligned"], st["n_unique"]) == (n_proc, n_pa, n_uniq)
    assert {int(c): int(n) for c, n in zip(mine_c, ec)} == ref_counts     # EC multiset, bit-exact


def _tsv(sc, est):
    tpm = K.counts_to_tpm(est, sc["em"]["eff_lens"])
    return O.abundance_tsv(sc["names"], sc["lens"], sc["em"]["eff_lens"], est, tpm)


def test_abundance_text_identical(scale):
    ref = open(os.path.join(scale["qdir"], "abundance.tsv")).read()
    assert _tsv(scale, scale["em"]["est_counts"]) == ref
    assert open(os.path.join(scale["cdir"], "abundance.tsv")).read() == ref
    a = json.load(open(os.path.join(scale["qdir"], "run_info.json")))
    b = json.load(open(os.path.join(scale["cdir"], "run_info.json")))
    for key in ("n_targets", "n_bootstraps", "n_processed", "n_pseudoaligned", "n_unique", "p_pseudoaligned", "p_unique"):
        assert a[key] == b[key], key
    # and the north_star tolerance on the numbers themselves
    _, _, eff, est, tpm = util.read_abundance(os.path.join(scale["qdir"], "abundance.tsv"))
    big = est > 1e-8 * est.sum()
    np.testing.assert_allclose(scale["em"]["est_counts"][big], est[big], rtol=1e-4)
    np.testing.assert_allclose(scale["em"]["eff_lens"], eff, rtol=1e-4)


@pytest.mark.parametrize("b", [0, 1])
def test_bootstrap_text_identical(scale, b):
    ref = open(os.path.join(scale["qdir"], "bs_abundance_%d.tsv" % b)).read()
    assert _tsv(scale, scale["bs"]["est_counts"][b]) == ref
    assert open(os.path.join(scale["cdir"], "bs_abundance_%d.tsv" % b)).read() == ref
