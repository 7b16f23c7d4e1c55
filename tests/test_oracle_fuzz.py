"""CPU: the oracle (oracle/kb_oracle.cpp) against the UNMODIFIED reference (oracle/_ref/kallisto) on small random
transcriptomes -- other k, shared exons, short transcripts, Ns, read lengths around k.  Strengthens the pin of the
oracle beyond the committed fixtures.  The transcriptomes and reads are generated here from their seeds; the index the
reference built for each one and the reference's per-fragment ECs, matrix.ec and flens.txt for each case are stored
under tests/golden/fuzz (written by `python tests/golden/make_golden.py fuzz`)."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import util

FUZZ = os.path.join(util.GOLDEN, "fuzz")
COMP = bytes.maketrans(b"ACGT", b"TGCA")


def case_index(seed, k):
    """The reference's index of the transcriptome of make_case(seed, k)."""
    return os.path.join(FUZZ, "s%d_k%d.kidx" % (seed, k))


def make_case(tmp, seed, k, read_len, n_reads, build_index=None):
    """Transcriptome (written to tmp/t.fa) and reads of one case; build_index(fasta, out, k) re-creates the stored
    index with the reference (tests/golden/make_golden.py)."""
    rng = np.random.default_rng(seed)
    lut = np.frombuffer(b"ACGT", np.uint8)
    exons = [bytes(lut[rng.integers(0, 4, int(rng.integers(k + 3, 220)))]) for _ in range(24)]
    txs = []
    for g in range(8):
        pool = list(rng.choice(len(exons), size=int(rng.integers(2, 6)), replace=False))
        for _ in range(int(rng.integers(1, 5))):
            sub = sorted(rng.choice(pool, size=int(rng.integers(1, len(pool) + 1)), replace=False))
            t = b"".join(exons[i] for i in sub)
            if len(t) >= k + 5:
                txs.append(t)
    txs = list(dict.fromkeys(txs))            # the reference refuses duplicate sequences only by name, keep it simple
    fa = os.path.join(tmp, "t.fa")
    with open(fa, "wb") as f:
        for i, t in enumerate(txs):
            f.write(b">tx%d\n%s\n" % (i, t))
    idx = case_index(seed, k)
    if build_index:
        build_index(fa, idx, k=k)
    r1, r2 = [], []
    for _ in range(n_reads):
        t = txs[int(rng.integers(0, len(txs)))]
        fl = int(min(len(t), rng.integers(read_len, read_len + 120)))
        s = int(rng.integers(0, len(t) - fl + 1))
        frag = t[s:s + fl]
        a = bytearray(frag[:read_len])
        b = bytearray(frag[-read_len:].translate(COMP)[::-1])
        for r in (a, b):
            for p in range(len(r)):
                x = rng.random()
                if x < 0.01:
                    r[p] = b"ACGT"[int(rng.integers(0, 4))]
                elif x < 0.013:
                    r[p] = ord("N")
        if rng.random() < 0.5:
            a, b = b, a
        if rng.random() < 0.03:               # unrelated sequence
            a = bytearray(bytes(lut[rng.integers(0, 4, read_len)]))
        r1.append(bytes(a))
        r2.append(bytes(b))
    paths = []
    for m, rs in ((1, r1), (2, r2)):
        p = os.path.join(tmp, "r_%d.fq" % m)
        with open(p, "wb") as f:
            for i, r in enumerate(rs):
                f.write(b"@r%d/%d\n%s\n+\n%s\n" % (i, m, r, b"I" * len(r)))
        paths.append(p)
    return idx, r1, r2, paths


def reference_ecs(seed, mode):
    """-> (per-fragment EC id or -1, EC sets, flens or None) of `kallisto bus -x bulk --num -t 1` on the case."""
    z = np.load(os.path.join(FUZZ, "s%d_%s.npz" % (seed, mode)))
    flens = z["flens"] if "flens" in z.files else None
    return z["frag_ec"].astype(np.int64), util.ec_sets(z["ec_off"], z["ec_tids"]), flens


def mode_args(mode):
    """-> (paired, strand code of the oracle, strand option of the reference)"""
    strand = {"fr": 1, "rf": 2}.get(mode.split("_")[-1], 0)
    return mode.startswith("paired"), strand, {0: [], 1: ["--fr-stranded"], 2: ["--rf-stranded"]}[strand]


CASES = [(1, 31, 75), (2, 21, 50), (3, 15, 36), (4, 31, 33), (5, 27, 150)]
MODES = ["paired", "single", "paired_fr", "single_rf"]


@pytest.mark.parametrize("seed,k,read_len", CASES)
@pytest.mark.parametrize("mode", MODES)
def test_random_transcriptome(seed, k, read_len, mode, tmp_path):
    paired, strand, _ = mode_args(mode)
    idx, r1, r2, paths = make_case(str(tmp_path), seed, k, read_len, 1500)
    want, ecs, flens = reference_ecs(seed, mode)

    ix = O.OracleIndex(idx)
    run = O.OracleRun(ix, paired, strand, True)
    bases, off = O.to_batch(r1, r2 if paired else None)
    got = run.pseudoalign(bases, off)
    eo, et, ec = run.ec_table()
    np.testing.assert_array_equal(got, want)
    assert util.ec_sets(eo, et) == ecs
    if paired and flens is not None:
        np.testing.assert_array_equal(run.flens(), flens)
