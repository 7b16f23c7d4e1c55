"""CPU: `kallisto bus --batch FILE` with a technology, with and without --batch-barcodes, restated in
tests/busbatch_oracle.py, against the outputs of the unmodified reference (tests/golden/busbatch, made by
tests/golden/make_golden_busbatch.py): sorted records, matrix.ec, the header, flens.txt, matrix.cells,
matrix.sample.barcodes, whether index.saved is written, and the counts of run_info.json.  Pins what the GPU tests
(tests/test_gpu_bus_batch.py) then demand of the CUDA path."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import busbatch_oracle as BB
from tests import util

D = os.path.join(util.GOLDEN, "busbatch")
IDX = {"ss": os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx"),
       "c1": os.path.join(util.GOLDEN, "config1", "transcripts.kidx"),
       "aa": os.path.join(util.GOLDEN, "aa", "proteins.kidx")}
# run -> (index, batch file, technology, strand, --num, --batch-barcodes, --aa, --paired)
RUNS = {
    "v3": ("ss", "batch_v3.txt", "10XV3", "default", False, False, False, False),
    "v3_bb": ("ss", "batch_v3.txt", "10XV3", "default", False, True, False, False),
    "v2_bb_num": ("c1", "batch_v2.txt", "10XV2", 0, True, True, False, False),
    "ss3_paired_bb": ("ss", "batch_ss3.txt", "SMARTSEQ3", "default", False, True, False, True),
    "ss3": ("ss", "batch_ss3.txt", "SMARTSEQ3", "default", False, False, False, False),
    "nobc_bb": ("ss", "batch_v3.txt", "-1,-1,-1:0,16,28:1,0,0", "default", False, True, False, False),
    "bc32_bb": ("ss", "batch_v3.txt", "0,0,16,1,0,16:0,16,28:1,0,0", "default", False, True, False, False),
    "aa_bb": ("aa", "batch_aa.txt", "10XV3", "default", False, True, True, False),
}
_IX = {}


def index(key):
    if key not in _IX:
        _IX[key] = O.OracleIndex(IDX[key])
    return _IX[key]


def model(name):
    ix, bf, tech, strand, num, bb, aa, paired = RUNS[name]
    lines = BB.read_lines(os.path.join(D, bf), tech)
    return BB.batch_model(index(ix), lines, tech, strand=strand, num=num, batch_barcodes=bb, aa=aa, paired_flag=paired)


def read_ref(name):
    """-> dict of the reference run's outputs"""
    d = os.path.join(D, "ref_" + name)
    hdr, rec = O.read_bus(os.path.join(d, "output.bus"))
    out = dict(header=(hdr["bclen"], hdr["umilen"]), records=rec.copy(), ecs=O.read_matrix_ec(os.path.join(d, "matrix.ec")),
               info=json.load(open(os.path.join(d, "run_info.json"))),
               files=json.load(open(os.path.join(D, "manifest.json")))["ref_" + name]["files"])
    out["cells"] = open(os.path.join(d, "matrix.cells")).read().split("\n")[:-1]
    p = os.path.join(d, "matrix.sample.barcodes")
    out["sample_barcodes"] = open(p).read().split("\n")[:-1] if os.path.exists(p) else None
    p = os.path.join(d, "flens.txt")
    out["flens"] = [np.array(l.split(), np.uint32) for l in open(p).read().split("\n")[:-1]] if os.path.exists(p) else None
    return out


@pytest.mark.parametrize("name", sorted(RUNS))
def test_batch_model_reproduces_the_reference(name):
    ref = read_ref(name)
    m = model(name)
    assert m["n_processed"] == ref["info"]["n_processed"]
    assert len(m["records"]) == ref["info"]["n_pseudoaligned"] == len(ref["records"])
    assert m["ecs"] == ref["ecs"]
    assert BB.n_unique(m["records"], m["ecs"]) == ref["info"]["n_unique"]
    assert BB.sorted_records(m["records"]).tobytes() == BB.sorted_records(ref["records"]).tobytes()
    assert m["header"] == ref["header"]
    assert m["cells"] == ref["cells"]
    assert m["sample_barcodes"] == ref["sample_barcodes"]
    assert m["index_saved"] == ("index.saved" in ref["files"])
    if ref["flens"] is None:
        assert m["flens"] is None
    else:
        assert len(m["flens"]) == len(ref["flens"]) and all(np.array_equal(a, b) for a, b in zip(m["flens"], ref["flens"]))
    if RUNS[name][6]:
        assert m["clashes"] == ref["info"]["n_frame_clashes"]


def test_fixtures_cover_the_rules():
    """Lines sharing an id, Ns in barcodes, barcodes of several lengths, tag and internal reads, and flens per line."""
    v3 = read_ref("v3_bb")
    assert v3["cells"] == ["s1", "s2", "s1"] and v3["sample_barcodes"] == ["A" * 16, "A" * 15 + "C", "A" * 16]
    assert set(int(b) >> 32 for b in v3["records"]["barcode"]) == {0, 1}
    assert read_ref("v3")["sample_barcodes"] is None
    ss3 = read_ref("ss3_paired_bb")
    assert ss3["header"][0] == 0 and len(ss3["flens"]) == 2
    assert read_ref("ss3")["flens"] is None
    lines = BB.read_lines(os.path.join(D, "batch_ss3.txt"), "SMARTSEQ3")
    bcs = [a + b for _, fl in lines for a, b in zip(fl[0], fl[1])]
    assert any(b"N" in b for b in bcs) and len({len(b) for b in bcs}) == 2
    assert ss3["info"]["n_pseudoaligned"] > 0 and (ss3["records"]["umi"] == 0xFFFFFFFFFFFFFFFF).any()
    nobc = read_ref("nobc_bb")
    assert nobc["header"][0] == 16 and set(nobc["records"]["barcode"].tolist()) == {0, 1}
    bc32 = read_ref("bc32_bb")
    assert bc32["header"][0] == 32 and (bc32["records"]["flags"] == 0).all()


def test_prefix_rule():
    assert BB.prefixed(b"ACGN", 5) == b"A" * 26 + b"CC" + b"ACGG"
    assert BB.prefixed(b"T" * 32, 7) == b"T" * 32
    assert BB.binary_to_string(1, 16) == b"A" * 15 + b"C"
