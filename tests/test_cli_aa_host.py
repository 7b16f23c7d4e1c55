"""CPU: the command line's handling of `bus --aa` on the stand-in library (tests/stub/stub_aa.cpp): the option is taken
and listed in the usage, run_info.json gains "n_frame_clashes" as its last field only with --aa, and what this build does
not translate is refused with the reason: --paired and technologies with two sequence reads, tag sequences, --union and
--no-jump (refused by the reference too).  The D-list refusal comes from the library (tests/test_gpu_aa.py)."""
import json
import os
import shutil
import subprocess

import pytest

from tests import util
from tests.test_cli_host_pipeline import CSRC, INC

pytestmark = pytest.mark.skipif(not shutil.which("g++"), reason="no g++")
D = os.path.join(util.GOLDEN, "aa")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("stubaa"))
    lib = os.path.join(d, "libkallisto_b200.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I" + INC, "-o", lib,
                           os.path.join(util.ROOT, "tests", "stub", "stub_aa.cpp")])
    exe = os.path.join(d, "cli")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + INC, "-I" + CSRC, "-o", exe, os.path.join(CSRC, "cli_main.cpp"),
                           "-L" + d, "-lkallisto_b200", "-Wl,-rpath," + d, "-lz", "-lpthread"])
    return exe


def bus(exe, out, args):
    return subprocess.run([exe, "bus", "-i", os.path.join(D, "proteins.kidx"), "-o", str(out)] + args, capture_output=True,
                          text=True, timeout=600, env=dict(os.environ, KB_CLI_CLEANUP="1"))


def test_aa_adds_the_frame_clashes_to_run_info(exe, tmp_path):
    reads = os.path.join(D, "reads.fastq.gz")
    r = bus(exe, tmp_path / "aa", ["--aa", "-x", "bulk", reads])
    assert r.returncode == 0, r.stderr
    text = (tmp_path / "aa" / "run_info.json").read_text()
    info = json.loads(text)
    assert list(info)[-2:] == ["call", "n_frame_clashes"] and info["n_frame_clashes"] == 400   # the stand-in's count
    assert text.endswith('",\n\t"n_frame_clashes": 400\n}\n')
    r = bus(exe, tmp_path / "nt", ["-x", "bulk", reads])
    assert r.returncode == 0, r.stderr
    text = (tmp_path / "nt" / "run_info.json").read_text()
    assert list(json.loads(text))[-1] == "call" and text.endswith('"\n}\n')


def test_usage_lists_aa(exe, tmp_path):
    r = subprocess.run([exe, "bus"], capture_output=True, text=True, timeout=60)
    assert "--aa" in r.stdout


@pytest.mark.parametrize("args,msg", [
    (["-x", "bulk", "--paired", "reads.fastq.gz", "reads.fastq.gz"], "--aa supports single-end reads only"),
    (["-x", "smartseq2", "--paired", "reads.fastq.gz", "reads.fastq.gz", "reads.fastq.gz", "reads.fastq.gz"],
     "--aa supports single-end reads only"),
    (["-x", "10xv3", "--tag", "ACGT", "sc_1.fastq.gz", "sc_2.fastq.gz"], "--aa with a UMI tag sequence (--tag) is not supported"),
    (["-x", "bulk", "--union", "reads.fastq.gz"], "--union is not compatible with this mode"),
    (["-x", "bulk", "--no-jump", "reads.fastq.gz"], "--no-jump is not compatible with this mode"),
])
def test_aa_refusals(exe, tmp_path, args, msg):
    args = [os.path.join(D, a) if a.endswith(".gz") else a for a in args]
    r = bus(exe, tmp_path / "o", ["--aa"] + args)
    assert r.returncode != 0 and msg in r.stderr, r.stderr[-600:]
    assert not (tmp_path / "o" / "output.bus").exists()
