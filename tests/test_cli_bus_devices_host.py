"""CPU: the command line's handling of `bus --devices` on a stand-in library (tests/stub/stub_bus_group.cpp) whose group
hands every batch to member 0's kb_bus_batch when it completes: the output files equal the one-device run's only when
the command line completes the batches in submission order.  Also the parsing of the device list, a one-entry list
taking the plain path, and a library without the group entry points."""
import os
import re
import shutil
import subprocess

import pytest

from tests import util
from tests.test_cli_host_pipeline import CSRC, INC

pytestmark = pytest.mark.skipif(not shutil.which("g++"), reason="no g++")
STUB = os.path.join(util.ROOT, "tests", "stub")
IDX = os.path.join(util.GOLDEN, "synth_small", "transcripts.kidx")
V3 = os.path.join(util.GOLDEN, "bus10xv3")
BB = os.path.join(util.GOLDEN, "busbatch")


def build(d, src):
    lib = os.path.join(d, "libkallisto_b200.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I" + INC, "-I" + STUB, "-o", lib, os.path.join(STUB, src)])
    exe = os.path.join(d, "cli")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + INC, "-I" + CSRC, "-o", exe, os.path.join(CSRC, "cli_main.cpp"),
                           "-L" + d, "-lkallisto_b200", "-Wl,-rpath," + d, "-lz", "-lpthread"])
    return exe


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("stubgroup")), "stub_bus_group.cpp")


@pytest.fixture(scope="module")
def exe_no_group(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("stubnogroup")), "stub_batch.cpp")


def run(exe, args, cwd=None, cuts=None):
    env = dict(os.environ, KB_CLI_CLEANUP="1")
    env.pop("CUDA_VISIBLE_DEVICES", None)
    if cuts:
        env["KB_CLI_BATCH_READS"] = cuts
    return subprocess.run([exe] + args, cwd=cwd, capture_output=True, text=True, timeout=600, env=env)


def outputs(d):
    got = {}
    for fn in sorted(os.listdir(d)):
        data = open(os.path.join(d, fn), "rb").read()
        if fn == "run_info.json":
            import json
            j = json.loads(data)
            j.pop("start_time"), j.pop("call")
            data = j
        got[fn] = data
    return got


CASES = {
    "10xv3": (["-x", "10xv3", os.path.join(V3, "sc_reads_1.fastq.gz"), os.path.join(V3, "sc_reads_2.fastq.gz")], None),
    "10xv3_num": (["-x", "10xv3", "--num", os.path.join(V3, "sc_reads_1.fastq.gz"), os.path.join(V3, "sc_reads_2.fastq.gz")], None),
    "batch_bb": (["-x", "10xv3", "--batch-barcodes", "--batch", "batch_v3.txt"], BB),
    "batch_aa": (["--aa", "-x", "10xv3", "--batch", "batch_aa.txt"], BB),
    "bulk": (["-x", "bulk", os.path.join(V3, "sc_reads_2.fastq.gz"), os.path.join(V3, "sc_reads_1.fastq.gz")], None),
}


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("cuts", ["7", "64,97", "1700"])
def test_devices_outputs_equal_one_device(exe, tmp_path, name, cuts):
    args, cwd = CASES[name]
    got = {}
    for tag, dv in (("one", ["--device", "0"]), ("two", ["--devices", "0,0"]), ("three", ["--devices", "0,1,0"]),
                    ("list1", ["--devices", "0"])):
        out = tmp_path / tag
        r = run(exe, ["bus", "-i", IDX, "-o", str(out), "-t", "2"] + dv + args, cwd=cwd, cuts=cuts)
        assert r.returncode == 0, r.stderr[-800:]
        got[tag] = outputs(out)
        groups = re.findall(r"stub: group of (\d+)", r.stderr)
        if tag in ("one", "list1"):
            assert not groups                                # zero or one entries: the plain path
        else:
            assert groups == [str(len(dv[1].split(",")))]
            per = [int(x) for x in r.stderr.split("stub: batches per member")[1].split("\n")[0].split()]
            if cuts == "7":                                   # many batches: every member is dealt some
                assert all(c > 0 for c in per), per
    assert got["two"] == got["one"]
    assert got["three"] == got["one"]
    assert got["list1"] == got["one"]


@pytest.mark.parametrize("bad", ["0,x", "-1", ",", "0,,1", "1.5"])
def test_bad_device_list(exe, tmp_path, bad):
    r = run(exe, ["bus", "-i", IDX, "-o", str(tmp_path / "o"), "--devices", bad, "-x", "10xv3",
                  os.path.join(V3, "sc_reads_1.fastq.gz"), os.path.join(V3, "sc_reads_2.fastq.gz")])
    assert r.returncode == 1
    assert "Error: --devices needs a comma-separated list of device ordinals" in r.stderr
    assert "--devices=LIST" in r.stdout                     # the usage text lists the option
    assert not (tmp_path / "o").exists()


def test_library_without_group_entry_points(exe_no_group, tmp_path):
    args = ["-x", "10xv3", os.path.join(V3, "sc_reads_1.fastq.gz"), os.path.join(V3, "sc_reads_2.fastq.gz")]
    r = run(exe_no_group, ["bus", "-i", IDX, "-o", str(tmp_path / "o"), "--devices", "0,0"] + args)
    assert r.returncode == 1 and "has no kb_bus_group_create" in r.stderr
    r = run(exe_no_group, ["bus", "-i", IDX, "-o", str(tmp_path / "p"), "--devices", "0"] + args)
    assert r.returncode == 0, r.stderr[-800:]
