"""GPU: `kallisto bus --aa` (cfc_frames_kernel -> the six frames through pack / match / resolve -> cfc_select_kernel)
through the library (kb_bus_set_aa, kb_bus_batch, kb_bus_batch_device) and through the command line, against the files
the unmodified reference wrote (tests/golden/aa), and against the CPU restatement (tests/aa_oracle.py) on seeded reads.
Records are compared as sorted multisets (the reference writes the records of a batch whose ECs are already known
first, src/ProcessReads.cpp:1798-1812, 603-612)."""
import json
import os
import random
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import aa_oracle as A
from tests import util
from tests.test_oracle_aa import D, IDX, RUNS, STRAND_NAME, case, read_ref, sorted_records

pytestmark = pytest.mark.gpu

BIN = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")
TECH = {"bulk_num": "BULK", "10xv3": "10XV3", "10xv3_rf": "10XV3", "10xv3_unstr": "10XV3", "batch": "BULK"}
CLI_ARGS = {
    "bulk_num": ["-x", "bulk", "--num", "reads.fastq.gz"],
    "10xv3": ["-x", "10xv3", "sc_1.fastq.gz", "sc_2.fastq.gz"],
    "10xv3_rf": ["-x", "10xv3", "--rf-stranded", "sc_1.fastq.gz", "sc_2.fastq.gz"],
    "10xv3_unstr": ["-x", "10xv3", "--unstranded", "sc_1.fastq.gz", "sc_2.fastq.gz"],
    "batch": ["--batch", "batch.txt"],
}


@pytest.fixture(scope="module")
def ix():
    x = K.KmerIndex(IDX, device=0)
    yield x
    x.close()


def processor(ix, name, **kw):
    names, bc, umi, seq, strand, num, per_file = RUNS[name]
    return K.BUSProcessor(ix, TECH[name], strand=STRAND_NAME[strand], num=num, aa=True, **kw)


def run_library(ix, name, cut, device=False):
    """Every sample in batches of at most `cut` read sets -> (records, clashes, stats, EC sets)."""
    files, samples = case(name)
    bp = processor(ix, name)
    parts = []
    for si, (lo, hi) in enumerate(samples or [(0, len(files[0]))]):
        if samples:
            bp.begin_sample(si)
        for a in range(lo, hi, cut):
            b = min(hi, a + cut)
            batch = [O.to_batch(f[a:b]) for f in files]
            if device:
                import torch
                tb = [torch.from_numpy(x).cuda() for x, _ in batch]
                to = [torch.from_numpy(o.view(np.int32)).cuda() for _, o in batch]
                maxlen = max(int(np.diff(o).max()) for _, o in batch)
                n, dptr = bp.process_sets_device([t.data_ptr() for t in tb], [t.data_ptr() for t in to], b - a, maxlen)
                rec = np.zeros(0, K.BUS_RECORD_DTYPE)
                if n:
                    view = type("DeviceRecords", (), {"__cuda_array_interface__": {
                        "shape": (n * rec.itemsize,), "typestr": "|u1", "data": (dptr, False), "version": 2}})()
                    rec = np.frombuffer(torch.as_tensor(view, device="cuda").cpu().numpy().tobytes(), K.BUS_RECORD_DTYPE)
                parts.append(rec)
            else:
                parts.append(bp.process_sets(batch))
    clashes = bp.frame_clashes()
    st = bp.finalize()
    eo, et, _, _ = bp.ec_table()
    bp.close()
    return np.concatenate(parts), clashes, st, util.ec_sets(eo, et)


@pytest.mark.parametrize("name", sorted(RUNS))
@pytest.mark.parametrize("cut", [100000, 37, 1])
def test_library_identical_to_reference(ix, name, cut):
    """One batch, batches of 37 read sets and batches of one: the six frames of a set always travel together."""
    d, hdr, ref, info, ref_ecs = read_ref(name)
    rec, clashes, st, ecs = run_library(ix, name, cut)
    assert sorted_records(rec).tobytes() == sorted_records(ref).tobytes()
    assert clashes == info["n_frame_clashes"]
    assert st["n_processed"] == info["n_processed"]
    assert st["n_pseudoaligned"] == info["n_pseudoaligned"]
    assert st["n_unique"] == info["n_unique"]
    assert ecs == ref_ecs


@pytest.mark.parametrize("name", ["10xv3", "bulk_num"])
def test_device_entry_point_identical_to_reference(ix, name):
    d, hdr, ref, info, ref_ecs = read_ref(name)
    rec, clashes, st, ecs = run_library(ix, name, 64, device=True)
    assert sorted_records(rec).tobytes() == sorted_records(ref).tobytes()
    assert clashes == info["n_frame_clashes"] and ecs == ref_ecs


@pytest.mark.parametrize("name", sorted(RUNS))
def test_cli_identical_to_reference(tmp_path, name):
    d, hdr, ref, info, ref_ecs = read_ref(name)
    out = tmp_path / "o"
    r = subprocess.run([BIN, "bus", "--aa", "-t", "1", "-i", "proteins.kidx", "-o", str(out)] + CLI_ARGS[name], cwd=D,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-800:]
    h2, rec = O.read_bus(str(out / "output.bus"))
    assert h2 == hdr
    assert sorted_records(rec).tobytes() == sorted_records(ref).tobytes()
    for f in ("matrix.ec", "transcripts.txt"):
        assert (out / f).read_bytes() == open(os.path.join(d, f), "rb").read(), f
    mine = json.loads((out / "run_info.json").read_text())
    for k in ("start_time", "call"):
        mine.pop(k), info.pop(k)
    assert mine == info and list(mine)[-1] == "n_frame_clashes"


def test_cli_refuses_an_index_with_a_dlist(tmp_path):
    reads = os.path.join(D, "reads.fastq.gz")
    r = subprocess.run([BIN, "bus", "--aa", "-x", "bulk", "-i", os.path.join(util.GOLDEN, "dlist", "transcripts.kidx"), "-o",
                        str(tmp_path / "o"), reads], capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "D-list" in r.stderr, r.stderr[-500:]


def random_reads(seed, n):
    """Back-translated pieces of the fixture's proteins on both strands (stops and unknown letters as TAA or NNN), pieces
    of the fixture's reads, random sequence; every length from 25 to 150, some with an N or a lower-case letter."""
    rng = random.Random(seed)
    prot = [l.strip() for l in open(os.path.join(D, "proteins.fa")) if not l.startswith(">")]
    back = {}
    for i in range(64):
        cod = "ACGT"[i >> 4] + "ACGT"[(i >> 2) & 3] + "ACGT"[i & 3]
        back.setdefault(A.CFC[3 * i:3 * i + 3].decode(), []).append(cod)
    aa = dict(zip("FLIMVSPTAYHQNKDECWRG", ["ACC", "ACA", "ATA", "ATC", "ATT", "CTA", "CTC", "CTT", "AGA", "AGC", "AGT",
                                           "AGG", "CGA", "CGC", "CGT", "CGG", "TGA", "TGC", "TGT", "TGG"]))
    fixture = [x.decode() for x in O.read_fastq(os.path.join(D, "reads.fastq.gz")) if len(x) >= 40]
    out = []
    for _ in range(n):
        L = rng.randint(25, 150)
        x = rng.random()
        if x < 0.1:
            s = "".join(rng.choice("ACGT") for _ in range(L))
        elif x < 0.4:                       # pieces of the fixture's reads: frame clashes among them
            r = rng.choice(fixture)
            a = rng.randrange(len(r) - 25)
            s = r[a:a + L]
        else:
            p = rng.choice(prot).upper()
            nt = "".join(rng.choice(back[aa[c]]) if c in aa else rng.choice(["TAA", "NNN"]) for c in p)
            if len(nt) < L:
                nt = nt * (L // len(nt) + 1)
            a = rng.randrange(len(nt) - L + 1)
            s = nt[a:a + L]
            if rng.random() < 0.5:
                s = A.revcomp(s.encode()).decode()
            if rng.random() < 0.1:
                j = rng.randrange(L)
                s = s[:j] + rng.choice("Nacgt") + s[j + 1:]
        out.append(s.encode())
    return out


@pytest.mark.parametrize("seed,strand", [(1, 0), (2, 1), (3, 2)])
def test_library_matches_the_restatement_on_random_reads(ix, seed, strand):
    reads = random_reads(seed, 3000)
    oix = O.OracleIndex(IDX)
    m = A.aa_bus_model(oix, [reads], [], None, (0, 0), strand=strand, num=True, samples=[(0, len(reads))])
    bp = K.BUSProcessor(ix, "BULK", strand=STRAND_NAME[strand], num=True, aa=True)
    bp.begin_sample(0)
    parts = [bp.process_sets([O.to_batch(reads[a:a + 700])]) for a in range(0, len(reads), 700)]
    rec = np.concatenate(parts)
    assert sorted_records(rec).tobytes() == sorted_records(m["records"]).tobytes()
    assert bp.frame_clashes() == m["clashes"]
    eo, et, _, _ = bp.ec_table()
    assert util.ec_sets(eo, et) == m["ecs"]
    assert len(rec) > 1000 and m["clashes"] > 0
    bp.close()
