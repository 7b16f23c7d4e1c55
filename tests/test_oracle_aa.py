"""CPU: `kallisto bus --aa` restated in tests/aa_oracle.py (six comma-free frames per read set, the oracle's single-end
pseudoalignment of each, the smallest non-empty frame set, the frame clashes and the frame-0 strand filter) against the
outputs of the unmodified reference (tests/golden/aa, made by tests/golden/make_golden_aa.py).  Pins what the GPU
tests (tests/test_gpu_aa.py) then demand of the CUDA path."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import aa_oracle as A
from tests import util

D = os.path.join(util.GOLDEN, "aa")
IDX = os.path.join(D, "proteins.kidx")

# fixture run -> (files, bc, umi, seq, strand, num, samples as lists of files, sample barcodes)
RUNS = {
    "bulk_num": (["reads.fastq.gz"], [], None, (0, 0), 0, True, True),
    "10xv3": (["sc_1.fastq.gz", "sc_2.fastq.gz"], [(0, 0, 16)], [(0, 16, 28)], (1, 0), 1, False, False),
    "10xv3_rf": (["sc_1.fastq.gz", "sc_2.fastq.gz"], [(0, 0, 16)], [(0, 16, 28)], (1, 0), 2, False, False),
    "10xv3_unstr": (["sc_1.fastq.gz", "sc_2.fastq.gz"], [(0, 0, 16)], [(0, 16, 28)], (1, 0), 0, False, False),
    "batch": (["batch_a.fastq.gz", "batch_b.fastq.gz"], [], None, (0, 0), 0, False, True),
}
STRAND_NAME = {0: "unstranded", 1: "fr", 2: "rf"}


def case(name):
    """-> (files: one list of sequences per file of the technology, sample ranges or None)"""
    names, bc, umi, seq, strand, num, per_file = RUNS[name]
    reads = [O.read_fastq(os.path.join(D, f)) for f in names]
    if not per_file:
        return reads, None
    files, samples = [[]], []
    for r in reads:
        samples.append((len(files[0]), len(files[0]) + len(r)))
        files[0].extend(r)
    return files, samples


def read_ref(name):
    d = os.path.join(D, "ref_" + name)
    hdr, rec = O.read_bus(os.path.join(d, "output.bus"))
    info = json.load(open(os.path.join(d, "run_info.json")))
    return d, hdr, rec.copy(), info, O.read_matrix_ec(os.path.join(d, "matrix.ec"))


def sorted_records(r):
    return np.sort(r, order=["barcode", "umi", "ec", "flags", "count"])


@pytest.fixture(scope="module")
def oix():
    return O.OracleIndex(IDX)


def model(oix, name):
    names, bc, umi, seq, strand, num, per_file = RUNS[name]
    files, samples = case(name)
    return A.aa_bus_model(oix, files, bc, umi, seq, strand=strand, num=num, samples=samples)


@pytest.mark.parametrize("name", sorted(RUNS))
def test_aa_model_reproduces_the_reference(oix, name):
    d, hdr, ref, info, ref_ecs = read_ref(name)
    m = model(oix, name)
    assert m["n_processed"] == info["n_processed"]
    assert len(m["records"]) == info["n_pseudoaligned"] == len(ref)
    assert m["ecs"] == ref_ecs
    assert sorted_records(m["records"]).tobytes() == sorted_records(ref).tobytes()
    assert m["clashes"] == info["n_frame_clashes"]
    assert list(info)[-1] == "n_frame_clashes"


def test_fixtures_cover_the_cases_that_matter(oix):
    """Every length mod 3, lengths k and k + 2, clashes, unmapped sets, and a strand filter that drops sets."""
    files, _ = case("bulk_num")
    lens = {len(s) for s in files[0]}
    assert {l % 3 for l in lens} == {0, 1, 2} and {31, 33} <= lens
    m = model(oix, "bulk_num")
    assert m["clashes"] > 5
    assert 0 < sum(s is None for s in m["sets"]) < len(m["sets"])
    assert any(s is not None and len(s) > 1 for s in m["sets"])
    fr, rf = read_ref("10xv3")[3], read_ref("10xv3_rf")[3]
    assert rf["n_pseudoaligned"] < fr["n_pseudoaligned"]


def test_frames_translate_as_the_reference():
    """nn_to_cfc on a triplet with a lower-case letter, an N, a stop codon, and the partial triplet padded with N."""
    s = b"ATGtttTAANNAGC" + b"GA"
    f = A.frames(s)
    assert f[0] == b"ATC" + b"ACC" + b"NNN" + b"NNN" + b"AGA" + b"N"
    assert [len(x) for x in f] == [16, 15, 14, 16, 15, 14]
    assert A.revcomp(b"acgtN*") == b"NNACGT"
