"""CPU: the BUS record model (oracle/oracle.py:bus_model -- the rules the CUDA path is held to) against the UNMODIFIED
reference (oracle/_ref/kallisto) on random small transcriptomes with random technology layouts: barcode / UMI pieces
anywhere in the files, with and without a UMI, one sequence read or a pair with random start offsets, tag sequences of
several lengths (short ones must match exactly, src/ProcessReads.cpp:1517), strand modes, --num, reads that are too
short for their slices, Ns in barcodes, UMIs and tags.  The cases are generated here from their seeds; the reference's
index of each transcriptome and its output.bus records, matrix.ec and flens.txt for each case are stored under
tests/golden/fuzz (written by `python tests/golden/make_golden.py fuzz`)."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import util
from tests.test_oracle_bus_paired import sorted_records
from tests.test_oracle_fuzz import FUZZ, make_case

SEEDS = range(16)


def layout(rng, paired, tag, no_umi):
    """Random technology: file 0 = barcode/UMI read (+ optionally the first sequence read), files 1.. = sequence reads."""
    a = int(rng.integers(0, 4))
    blen = int(rng.integers(4, 13))
    bc = [(0, a, a + blen)]
    if rng.random() < 0.4:                       # a second barcode piece further along
        b2 = a + blen + int(rng.integers(0, 5))
        bc.append((0, b2, b2 + int(rng.integers(2, 7))))
    end = bc[-1][2]
    taglen = len(tag) if tag else 0
    ulen = int(rng.integers(4, 11))
    u0 = end + int(rng.integers(0, 4))
    umi_user = None if no_umi else [(0, u0, u0 + taglen + ulen)]          # as the user writes it: tag + UMI
    pre = (umi_user[0][2] if umi_user else end) + int(rng.integers(0, 4))
    seq_in_0 = rng.random() < 0.5                # sequence read shares the barcode file (starts after the UMI)
    if paired:
        seq = (0, pre) if seq_in_0 else (1, int(rng.integers(0, 6)))
        seq2 = (2 if not seq_in_0 else 1, int(rng.integers(0, 9)))
    else:
        seq = (0, pre) if seq_in_0 else (1, int(rng.integers(0, 6)))
        seq2 = None
    nfiles = 1 + max(seq[0], seq2[0] if seq2 else 0)
    return bc, umi_user, seq, seq2, nfiles, pre


def tech_string(bc, umi_user, seq, seq2):
    t = lambda v: ",".join("%d,%d,%d" % x for x in v)
    s = [(seq[0], seq[1], 0)] + ([(seq2[0], seq2[1], 0)] if seq2 else [])
    return "%s:%s:%s" % (t(bc), t(umi_user) if umi_user else "-1,-1,-1", t(s))


def build_case(seed, tmp_path, build_index=None):
    """Index, read files and reference arguments of case `seed` -> dict"""
    rng = np.random.default_rng(1000 + seed)
    paired = bool(seed & 1)
    tag = [None, None, b"ACGTTGCA", b"TTGCA", b"ATTGCGCAATG"][seed % 5]
    no_umi = tag is None and seed % 3 == 0
    strand = int(rng.integers(0, 3))
    num = bool(rng.random() < 0.3)
    k = [31, 21, 15, 27][seed % 4]
    idx, r1, r2, _ = make_case(str(tmp_path), 50 + seed, k, int(rng.integers(k + 2, 90)), 1200, build_index)
    bc, umi_user, seq, seq2, nfiles, pre = layout(rng, paired, tag, no_umi)
    lut = np.frombuffer(b"ACGT", np.uint8)
    n = len(r1)
    cells = lut[rng.integers(0, 4, (5, pre))]
    head = []
    for i in range(n):
        h = bytearray(bytes(cells[int(rng.integers(0, 5))]))
        if umi_user:                              # a fresh UMI (and, for most reads, the tag in front of it)
            u0, u1 = umi_user[0][1], umi_user[0][2]
            h[u0:u1] = bytes(lut[rng.integers(0, 4, u1 - u0)])
            if tag and rng.random() < 0.6:
                tg = bytearray(tag)
                x = rng.random()
                if x < 0.15:
                    tg[int(rng.integers(0, len(tg)))] = ord("ACGT"[int(rng.integers(0, 4))])
                elif x < 0.2:
                    tg[int(rng.integers(0, len(tg)))] = ord("N")
                h[u0:u0 + len(tag)] = tg
        if rng.random() < 0.03:
            h[int(rng.integers(0, len(h)))] = ord("N")
        if rng.random() < 0.02:
            h = h[:int(rng.integers(0, len(h)))]     # too short for some slice: the set is skipped
        head.append(bytes(h))
    files = [None] * nfiles
    seqs = [r1, r2]
    si = 0
    for f in range(nfiles):
        if f == 0:
            if seq[0] == 0:
                files[0] = [head[i] + seqs[0][i] for i in range(n)]
                si = 1
            else:
                files[0] = head
        else:
            off = seq[1] if (seq[0] == f) else (seq2[1] if seq2 and seq2[0] == f else 0)
            files[f] = [bytes(lut[rng.integers(0, 4, off)]) + seqs[si][i] for i in range(n)]
            si += 1
    paths = []
    for f in range(nfiles):
        p = str(tmp_path / ("f%d.fq" % f))
        with open(p, "wb") as fo:
            for i, s in enumerate(files[f]):
                fo.write(b"@r%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)))
        paths.append(p)
    args = ["bus", "-i", idx, "-o", str(tmp_path / "o"), "-t", "1", "-x", tech_string(bc, umi_user, seq, seq2)]
    args += [["--unstranded"], ["--fr-stranded"], ["--rf-stranded"]][strand]
    if paired:
        args.append("--paired")
    if num:
        args.append("--num")
    if tag:
        args += ["--tag", tag.decode()]
    return dict(idx=idx, files=files, paths=paths, args=args, bc=bc, umi_user=umi_user, seq=seq, seq2=seq2, strand=strand,
                num=num, tag=tag, paired=paired)


def reference_bus(seed):
    """-> (output.bus records, matrix.ec sets, flens.txt or None) of the reference on case `seed`"""
    z = np.load(os.path.join(FUZZ, "bus%d.npz" % seed))
    return z["records"].copy(), util.ec_sets(z["ec_off"], z["ec_tids"]), (z["flens"] if "flens" in z.files else None)


@pytest.mark.parametrize("seed", SEEDS)
def test_random_layout(seed, tmp_path):
    c = build_case(seed, tmp_path)
    idx, files, args, bc, umi_user, seq, seq2 = c["idx"], c["files"], c["args"], c["bc"], c["umi_user"], c["seq"], c["seq2"]
    strand, num, tag, paired = c["strand"], c["num"], c["tag"], c["paired"]
    ref, ref_ecs, ref_flens = reference_bus(seed)
    taglen = len(tag) if tag else 0
    umi = None if umi_user is None else [(umi_user[0][0], umi_user[0][1] + taglen, umi_user[0][2])]
    ix = O.OracleIndex(idx)
    m = O.bus_model(ix, files, bc, umi, seq, seq2, strand=strand, num=num, tag=tag)
    assert len(m["records"]) == len(ref), (args, len(m["records"]), len(ref))
    assert sorted_records(m["records"]).tobytes() == sorted_records(ref.copy()).tobytes(), args
    assert m["ecs"] == (ref_ecs if len(ref) else [])
    if paired:
        np.testing.assert_array_equal(m["flens"][0], ref_flens)
