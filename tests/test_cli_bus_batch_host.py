"""CPU: the command line's handling of `bus --batch FILE` with a technology and of --batch-barcodes, on the stand-in
library (tests/stub/stub_batch.cpp, whose records carry the sample of kb_bus_begin_sample as their UMI): a sample switch
at every line of the batch file, the files the command line writes itself (the header of output.bus, matrix.cells,
matrix.sample.barcodes, flens.txt and index.saved) against the reference runs of tests/golden/busbatch, and the
rejected invocations against the reference's exit codes and `Error:` lines (tests/golden/busbatch/cli_errors.json).
The records themselves are held by tests/test_gpu_bus_batch.py."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests import busbatch_oracle as BB
from tests import util
from tests.test_cli_host_pipeline import CSRC, INC

pytestmark = pytest.mark.skipif(not shutil.which("g++"), reason="no g++")
D = os.path.join(util.GOLDEN, "busbatch")
MANIFEST = json.load(open(os.path.join(D, "manifest.json")))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("stubbatch"))
    lib = os.path.join(d, "libkallisto_b200.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I" + INC, "-I" + os.path.join(util.ROOT, "tests", "stub"),
                           "-o", lib, os.path.join(util.ROOT, "tests", "stub", "stub_batch.cpp")])
    exe = os.path.join(d, "cli")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + INC, "-I" + CSRC, "-o", exe, os.path.join(CSRC, "cli_main.cpp"),
                           "-L" + d, "-lkallisto_b200", "-Wl,-rpath," + d, "-lz", "-lpthread"])
    return exe


def run(exe, args, out, env=None):
    """The reference's call of a fixture run, from the fixture directory, writing to `out`"""
    args = list(args)
    args[args.index("-o") + 1] = str(out)
    return subprocess.run([exe] + args, cwd=D, capture_output=True, text=True, timeout=600,
                          env=dict(os.environ, KB_CLI_CLEANUP="1", **(env or {})))


def line_sizes(batch):
    return [len(O.read_fastq(os.path.join(D, fl[0]))) for _, fl in BB.read_batch_file(os.path.join(D, batch))]


@pytest.mark.parametrize("name", sorted(MANIFEST))
@pytest.mark.parametrize("cuts", [None, "7,3,5,11"])
def test_host_outputs_match_the_reference(exe, tmp_path, name, cuts):
    if "--aa" in MANIFEST[name]["args"] and cuts:
        pytest.skip("one cut is enough for the --aa run")
    args = MANIFEST[name]["args"]
    r = run(exe, args, tmp_path / "o", env={"KB_CLI_BATCH_READS": cuts} if cuts else None)
    assert r.returncode == 0, r.stderr[-800:]
    out, ref = tmp_path / "o", os.path.join(D, name)
    with open(os.path.join(ref, "output.bus"), "rb") as f:
        want_hdr = f.read(20 + 29)
    with open(out / "output.bus", "rb") as f:
        assert f.read(20 + 29) == want_hdr
    for fn in ("matrix.cells", "matrix.sample.barcodes"):
        assert (out / fn).exists() == os.path.exists(os.path.join(ref, fn)), fn
        if (out / fn).exists():
            assert (out / fn).read_bytes() == open(os.path.join(ref, fn), "rb").read(), fn
    for fn in ("flens.txt", "index.saved"):
        assert (out / fn).exists() == (fn in MANIFEST[name]["files"]), fn
    # a sample switch at every line: the stand-in's records carry the sample it was last given
    ids = BB.batch_numbers([i for i, _ in BB.read_batch_file(os.path.join(D, args[args.index("--batch") + 1]))])
    bb = "--batch-barcodes" in args
    no_bc = args[args.index("-x") + 1].startswith("-1,")
    want = np.concatenate([np.full(n, 0 if (no_bc and not bb) else ids[j], np.uint64)
                           for j, n in enumerate(line_sizes(args[args.index("--batch") + 1]))])
    _, rec = O.read_bus(str(out / "output.bus"))
    assert np.array_equal(rec["umi"], want)
    assert ("stub: batch barcodes 1" in r.stderr) == (bb and not no_bc)
    if (out / "flens.txt").exists():      # the stand-in reports the sample in bin 1 of every histogram
        rows = [l.split() for l in (out / "flens.txt").read_text().splitlines()]
        assert [int(x[1]) for x in rows] == ids


def test_usage_lists_batch_barcodes(exe):
    r = subprocess.run([exe, "bus"], capture_output=True, text=True, timeout=60)
    assert "--batch-barcodes" in r.stdout and "--batch=FILE" in r.stdout


@pytest.mark.parametrize("key", sorted(json.load(open(os.path.join(D, "cli_errors.json")))))
def test_rejected_like_the_reference(exe, key):
    want = json.load(open(os.path.join(D, "cli_errors.json")))[key]
    r = subprocess.run([exe] + key.split(), cwd=D, capture_output=True, text=True, timeout=120)
    assert [r.returncode, [l.strip() for l in r.stderr.splitlines() if l.startswith("Error")]] == want
    assert not os.path.exists(os.path.join(D, "o"))


def test_deliberate_refusals(exe, tmp_path):
    """Where the reference only warns or would build a wrong barcode, this build refuses before any work."""
    idx = os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx")
    one = tmp_path / "one.txt"
    one.write_text("s1 %s\n" % os.path.join(D, "v3_a_1.fastq.gz"))
    r = subprocess.run([exe, "bus", "-i", idx, "-o", str(tmp_path / "o"), "-x", "10xv3", "--batch", str(one)],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "have 1 files, technology 10XV3 reads 2" in r.stderr
    r = subprocess.run([exe, "bus", "-i", idx, "-o", str(tmp_path / "o"), "-x", "0,0,16,1,0,17:0,16,28:1,0,0", "--batch-barcodes",
                        "--batch", os.path.join(D, "batch_v3.txt")], cwd=D, capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "--batch-barcodes needs a barcode of at most 32 letters" in r.stderr
    assert not (tmp_path / "o").exists()
