"""GPU: `kallisto bus --batch FILE` with a technology, with and without --batch-barcodes (the barcode prefix is formed
in bus_fields_kernel), through the library (kb_bus_begin_sample at every line, kb_bus_set_batch_barcodes) and through
the command line, against the files the unmodified reference wrote (tests/golden/busbatch), and against the CPU
restatement (tests/busbatch_oracle.py) on seeded random layouts.  Records are compared as sorted multisets (the
reference writes the records of a batch whose ECs are already known first, src/ProcessReads.cpp:1798-1812)."""
import os
import random
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import busbatch_oracle as BB
from tests import util
from tests.test_oracle_bus_batch import D, IDX, RUNS, read_ref

pytestmark = pytest.mark.gpu

BIN = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")
# BUSProcessor technology of each BB.TECH entry: (nfiles, bc, umi, seq, default strand[, seq2])
LIB_TECH = {
    "10XV3": "10XV3",
    "10XV2": "10XV2",
    "SMARTSEQ3": "SMARTSEQ3",
    "-1,-1,-1:0,16,28:1,0,0": (2, [], [(0, 16, 28)], (1, 0, 0), 0),
    "0,0,16,1,0,16:0,16,28:1,0,0": (2, [(0, 0, 16), (1, 0, 16)], [(0, 16, 28)], (1, 0, 0), 0),
}
STRAND = {"default": "default", 0: "unstranded", 1: "fr", 2: "rf"}
_IX = {}


def kindex(key):
    if key not in _IX:
        _IX[key] = K.KmerIndex(IDX[key], device=0)
    return _IX[key]


def run_library(ix, lines, tech, cut, strand="default", num=False, bb=False, aa=False):
    """Every line a sample, in batches of at most `cut` read sets -> (records, EC sets, flens per line)"""
    bp = K.BUSProcessor(ix, LIB_TECH[tech], strand=STRAND[strand], num=num, aa=aa, batch_barcodes=bb,
                        tag=BB.TECH[tech][5])
    nums = BB.batch_numbers([i for i, _ in lines])
    parts, flens = [], []
    for j, (_, fl) in enumerate(lines):
        bp.begin_sample(0 if (not BB.TECH[tech][0] and not bb) else nums[j])
        n = len(fl[0])
        for a in range(0, n, cut):
            b = min(n, a + cut)
            parts.append(bp.process_sets([O.to_batch(f[a:b]) for f in fl]))
        if bp.paired:
            flens.append(bp.flens.copy())
    bp.finalize()
    eo, et, _, _ = bp.ec_table()
    bp.close()
    return np.concatenate(parts), util.ec_sets(eo, et), flens


@pytest.mark.parametrize("name", sorted(RUNS))
@pytest.mark.parametrize("cut", ["sample", 37, 1])
def test_library_identical_to_reference(name, cut):
    ix, bf, tech, strand, num, bb, aa, paired = RUNS[name]
    lines = BB.read_lines(os.path.join(D, bf), tech)
    c = max(len(fl[0]) for _, fl in lines) if cut == "sample" else cut
    rec, ecs, flens = run_library(kindex(ix), lines, tech, c, strand=strand, num=num, bb=bb, aa=aa)
    ref = read_ref(name)
    assert ecs == ref["ecs"]
    assert BB.sorted_records(rec).tobytes() == BB.sorted_records(ref["records"]).tobytes()
    if ref["flens"] is not None:
        assert len(flens) == len(ref["flens"]) and all(np.array_equal(a, b) for a, b in zip(flens, ref["flens"]))


@pytest.mark.parametrize("name", sorted(RUNS))
@pytest.mark.parametrize("threads,cuts", [(1, None), (8, None), (8, "5,3,7,2")])
def test_cli_identical_to_reference(name, threads, cuts, tmp_path):
    import json
    args = json.load(open(os.path.join(D, "manifest.json")))["ref_" + name]["args"]
    args = list(args)
    args[args.index("-o") + 1] = str(tmp_path / "o")
    args[args.index("-t") + 1] = str(threads)
    env = dict(os.environ, **({"KB_CLI_BATCH_READS": cuts} if cuts else {}))
    r = subprocess.run([BIN] + args, cwd=D, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-800:]
    ref = read_ref(name)
    out = tmp_path / "o"
    hdr, rec = O.read_bus(str(out / "output.bus"))
    assert (hdr["bclen"], hdr["umilen"]) == ref["header"]
    assert O.read_matrix_ec(str(out / "matrix.ec")) == ref["ecs"]
    assert BB.sorted_records(rec).tobytes() == BB.sorted_records(ref["records"]).tobytes()
    info = json.load(open(out / "run_info.json"))
    for k in ("n_processed", "n_pseudoaligned", "n_unique"):
        assert info[k] == ref["info"][k], k
    for fn in ("matrix.cells", "matrix.sample.barcodes", "flens.txt"):
        p = os.path.join(D, "ref_" + name, fn)
        assert (out / fn).exists() == os.path.exists(p), fn
        if os.path.exists(p):
            assert (out / fn).read_bytes() == open(p, "rb").read(), fn


def random_lines(rng, seqs, n_lines, per_line, max_bc):
    """10x-like sets: file 0 = barcode of 1..max_bc letters (some with N) + a 10-letter UMI, file 1 = a cDNA read."""
    lines, k = [], 0
    for j in range(n_lines):
        f0, f1 = [], []
        for _ in range(rng.randint(1, per_line)):
            L = rng.randint(1, max_bc)
            bc = bytearray(rng.choice(b"ACGT") for _ in range(L))
            if rng.random() < 0.2:
                bc[rng.randrange(L)] = ord("N")
            f0.append(bytes(bc) + bytes(rng.choice(b"ACGT") for _ in range(10)))
            f1.append(seqs[k % len(seqs)])
            k += 1
        lines.append((rng.choice(["a", "b", "c", "d"]), [f0, f1]))
    return lines


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_layouts_against_the_model(seed):
    """Barcodes of 1 to 32 letters, read from the end of the UMI backwards: bc = file 0 from 10 to the end."""
    rng = random.Random(seed)
    seqs = O.read_fastq(os.path.join(util.GOLDEN, "synth_small", "reads_1.fastq.gz"))[:3000]
    lines = random_lines(rng, seqs, rng.randint(2, 6), 300, 32)
    lines = [(i, [[s[-10:] + s[:-10] for s in fl[0]], fl[1]]) for i, fl in lines]      # UMI first, then the barcode
    tech = "RANDOM"
    BB.TECH[tech] = ([(0, 10, 0)], [(0, 0, 10)], (1, 0), None, 0, None)
    LIB_TECH[tech] = (2, [(0, 10, 0)], [(0, 0, 10)], (1, 0, 0), 0)
    try:
        oix = O.OracleIndex(IDX["ss"])
        for bb in (False, True):
            m = BB.batch_model(oix, lines, tech, batch_barcodes=bb, strand=0)
            rec, ecs, _ = run_library(kindex("ss"), lines, tech, rng.randint(1, 200), strand=0, bb=bb)
            assert ecs == m["ecs"]
            assert BB.sorted_records(rec).tobytes() == BB.sorted_records(m["records"]).tobytes()
    finally:
        del BB.TECH[tech], LIB_TECH[tech]


def test_a_33_letter_barcode_stops_the_run(tmp_path):
    rng = random.Random(7)
    seqs = O.read_fastq(os.path.join(util.GOLDEN, "synth_small", "reads_1.fastq.gz"))[:50]
    f0 = [bytes(rng.choice(b"ACGT") for _ in range(10)) + bytes(rng.choice(b"ACGT") for _ in range(33 if i == 17 else 20))
          for i in range(50)]
    bp = K.BUSProcessor(kindex("ss"), (2, [(0, 10, 0)], [(0, 0, 10)], (1, 0, 0), 0), batch_barcodes=True)
    bp.begin_sample(3)
    bp.process_sets([O.to_batch(f0[:10]), O.to_batch(seqs[:10])])
    with pytest.raises(Exception, match="more than 32 letters"):
        bp.process_sets([O.to_batch(f0[10:]), O.to_batch(seqs[10:])])
    bp.close()
    # the command line stops with the error and a non-zero exit code
    d = tmp_path
    with open(d / "r1.fq", "wb") as f:
        for i, s in enumerate(f0):
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)))
    with open(d / "r2.fq", "wb") as f:
        for i, s in enumerate(seqs):
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)))
    (d / "b.txt").write_text("x %s %s\n" % (d / "r1.fq", d / "r2.fq"))
    r = subprocess.run([BIN, "bus", "-i", IDX["ss"], "-o", str(d / "o"), "-x", "0,10,0:0,0,10:1,0,0", "--batch-barcodes",
                        "--batch", str(d / "b.txt")], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "more than 32 letters" in r.stderr
