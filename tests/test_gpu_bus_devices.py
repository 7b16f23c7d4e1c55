"""GPU: `bus --devices` and the group API under it (kb_bus_group_*): batches of one read stream dealt to several bus runs,
here two or three runs on device 0, with every output byte as with one run.  The command line runs every stored
reference run of tests/golden/bus10x, bus10xv3, buspaired, busbatch and aa with small batch cuts (KB_CLI_BATCH_READS), so
that every member gets batches and new equivalence classes first appear on members other than 0; the library tests feed
a BUSGroup and one BUSProcessor the same cuts, and check the ordering rule and the refusals."""
import gc
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

import kallisto_b200 as K
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu

BIN = os.path.join(util.ROOT, "kallisto_b200", "kallisto_b200")
G = util.GOLDEN
CUTS = ["7", "64", "1700"]


def _call_args(d, name):
    """the arguments after `bus` of a stored reference run (its run_info.json "call"), index and inputs as stored"""
    call = json.load(open(os.path.join(G, d, name, "run_info.json")))["call"].split()
    args = call[call.index("bus") + 1:]
    i = args.index("-o")
    del args[i:i + 2]
    i = args.index("-t")
    del args[i:i + 2]
    return [os.path.join(G, a.split("/golden/")[1]) if "/golden/" in a else a for a in args]


def _cases():
    out = []
    for d in ("bus10x", "bus10xv3"):
        for name in sorted(os.listdir(os.path.join(G, d))):
            if name.startswith("ref_"):
                out.append((d, name))
    for name in sorted(util.BUSPAIRED_CASES):
        out.append(("buspaired", "ref_" + name))
    out.append(("buspaired", "ref_batchfile"))
    for name in sorted(json.load(open(os.path.join(G, "busbatch", "manifest.json")))):
        out.append(("busbatch", name))
    for name in sorted(os.listdir(os.path.join(G, "aa"))):
        if name.startswith("ref_"):
            out.append(("aa", name))
    return out


CASES = _cases()


@pytest.fixture(scope="module")
def paired_inputs(tmp_path_factory):
    return util.buspaired_inputs(str(tmp_path_factory.mktemp("buspaired_in")))


def command(d, name, paired_inputs, tmp):
    """-> (arguments after `bus -o OUT -t T`, working directory)"""
    if d in ("bus10x", "bus10xv3"):
        return _call_args(d, name), None
    if d == "buspaired":
        idx = ["-i", os.path.join(G, "synth_small", "transcripts.kidx")]
        if name == "ref_batchfile":
            return idx + ["--batch", util.write_batch_file(str(tmp / "batch.txt"), paired_inputs)], None
        args, keys = util.BUSPAIRED_CASES[name[4:]]
        return idx + args + [paired_inputs[k] for k in keys], None
    if d == "busbatch":
        args = list(json.load(open(os.path.join(G, d, "manifest.json")))[name]["args"])[1:]
        i = args.index("-o")
        del args[i:i + 2]
        i = args.index("-t")
        del args[i:i + 2]
        return args, os.path.join(G, d)
    call = json.load(open(os.path.join(G, d, name, "run_info.json")))["call"].split()
    args = call[call.index("bus") + 1:]
    for opt in ("-o", "-t"):
        i = args.index(opt)
        del args[i:i + 2]
    return args, os.path.join(G, d)


def sorted_records(rec):
    return np.sort(rec, order=list(rec.dtype.names))


def files_of(out):
    got = {}
    for fn in sorted(os.listdir(out)):
        data = (out / fn).read_bytes()
        if fn == "run_info.json":
            j = json.loads(data)
            j.pop("start_time"), j.pop("call")
            data = j
        got[fn] = data
    return got


@pytest.mark.parametrize("d,name", CASES, ids=["%s/%s" % c for c in CASES])
def test_cli_devices_identical_to_one_device(d, name, paired_inputs, tmp_path):
    args, cwd = command(d, name, paired_inputs, tmp_path)
    cut = CUTS[CASES.index((d, name)) % len(CUTS)]
    env = dict(os.environ, KB_CLI_BATCH_READS=cut)
    got, codes = {}, {}
    for tag, dv in (("one", ["--device", "0"]), ("two", ["--devices", "0,0"]), ("three", ["--devices", "0,0,0"])):
        out = tmp_path / tag
        r = subprocess.run([BIN, "bus", "-o", str(out), "-t", "4"] + dv + args, cwd=cwd, capture_output=True, text=True,
                           timeout=900, env=env)
        codes[tag] = r.returncode
        assert r.returncode in (0, 1) and (out / "output.bus").exists(), r.stderr[-800:]
        got[tag] = files_of(out)
    assert codes["two"] == codes["one"] and codes["three"] == codes["one"]
    assert got["two"] == got["one"]
    assert got["three"] == got["one"]
    # and the reference's: bytes where the one-device tests compare bytes, records as sorted multisets elsewhere
    ref = os.path.join(G, d, name)
    mine = tmp_path / "three"
    if os.path.exists(os.path.join(ref, "output.bus.gz")):
        rb = gzip.open(os.path.join(ref, "output.bus.gz")).read()
        (tmp_path / "ref.bus").write_bytes(rb)
        ref_bus = str(tmp_path / "ref.bus")
    else:
        ref_bus = os.path.join(ref, "output.bus")
    if d == "bus10x":
        assert (mine / "output.bus").read_bytes() == open(ref_bus, "rb").read()
    else:
        h1, r1 = O.read_bus(str(mine / "output.bus"))
        h2, r2 = O.read_bus(ref_bus)
        assert sorted_records(r1).tobytes() == sorted_records(r2).tobytes()
    assert O.read_matrix_ec(str(mine / "matrix.ec")) == O.read_matrix_ec(os.path.join(ref, "matrix.ec"))
    for fn in ("flens.txt", "matrix.cells", "matrix.sample.barcodes"):
        if os.path.exists(os.path.join(ref, fn)):
            assert (mine / fn).read_bytes() == open(os.path.join(ref, fn), "rb").read(), fn
    info = json.load(open(os.path.join(ref, "run_info.json")))
    for k in ("n_processed", "n_pseudoaligned", "n_unique"):
        assert got["three"]["run_info.json"][k] == info[k], k


# ---- library ----------------------------------------------------------------------------------------------------------
V3 = os.path.join(G, "bus10xv3")
IDX = os.path.join(G, "synth_small", "transcripts.kidx")


@pytest.fixture(scope="module")
def reads():
    return [O.read_fastq(os.path.join(V3, "sc_reads_%d.fastq.gz" % m)) for m in (1, 2)]


@pytest.fixture(scope="module")
def indices():
    xs = [K.KmerIndex(IDX, device=0) for _ in range(4)]
    yield xs
    gc.collect()          # a run must be freed before its index: runs still held by reference cycles go first
    for x in xs:
        x.close()


def batch(reads, a, b):
    return [O.to_batch(f[a:b]) for f in reads]


def junk(n, seed):
    """read sets whose cDNA read maps nowhere"""
    rng = np.random.default_rng(seed)
    bc = [b"A" * 28] * n
    cdna = [bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), 90)) for _ in range(n)]
    return [O.to_batch(bc), O.to_batch(cdna)]


def seeded_batches(reads, seed):
    rng = np.random.default_rng(seed)
    n = len(reads[0])
    out, a = [], 0
    while a < n:
        r = rng.random()
        if r < 0.08:
            out.append(batch(reads, a, a))                  # empty
        elif r < 0.16:
            out.append(junk(int(rng.integers(1, 40)), int(rng.integers(1 << 30))))   # nothing maps
        else:
            b = min(n, a + int(rng.integers(1, 900)))
            out.append(batch(reads, a, b))
            a = b
    return out


def plain(ix, batches, samples=None, **kw):
    bp = K.BUSProcessor(ix, "10xv3", **kw)
    recs = []
    for i, b in enumerate(batches):
        if samples and i in samples:
            bp.begin_sample(samples[i])
        recs.append(bp.process_sets(b))
    return bp, np.concatenate(recs)


def grouped(ixs, batches, samples=None, **kw):
    """round-robin, one batch per member in flight, completed in submission order; a sample switch drains first"""
    members = [K.BUSProcessor(x, "10xv3", **kw) for x in ixs]
    g = K.BUSGroup(members)
    recs, pending = [], []
    busy = [False] * len(members)
    for i, b in enumerate(batches):
        if samples and i in samples:
            while pending:
                recs.append(g.complete(pending.pop(0)[0]))
            busy = [False] * len(members)
            g.begin_sample(samples[i])
        m = i % len(members)
        while busy[m]:
            t, mm = pending.pop(0)
            recs.append(g.complete(t))
            busy[mm] = False
        pending.append((g.submit(m, b), m))
        busy[m] = True
    while pending:
        recs.append(g.complete(pending.pop(0)[0]))
    return g, members, np.concatenate(recs)


def same_run(bp, rec_plain, g, rec_group):
    assert rec_group.tobytes() == rec_plain.tobytes()
    s1, s2 = bp.finalize(), g.finalize()
    for k in ("n_processed", "n_pseudoaligned", "n_unique", "n_ecs", "n_ec_entries"):
        assert s1[k] == s2[k], k
    o1, t1, c1, _ = bp.ec_table()
    o2, t2, c2 = g.ec_table()
    assert np.array_equal(o1, o2) and np.array_equal(t1, t2) and np.array_equal(c1, c2)
    b1, u1 = bp.lengths()
    b2, u2 = g.lengths()
    assert np.array_equal(b1, b2) and np.array_equal(u1, u2)


@pytest.mark.parametrize("n_members", [1, 2, 3])
@pytest.mark.parametrize("seed", [1, 2])
def test_group_equals_one_run(reads, indices, n_members, seed):
    batches = seeded_batches(reads, seed)
    bp, rp = plain(indices[0], batches)
    g, _, rg = grouped(indices[1:1 + n_members], batches)
    same_run(bp, rp, g, rg)
    assert len(rp) > 0


def test_ids_follow_ticket_order(reads, indices):
    """A set first seen by member 1 in an earlier batch and then by member 0 keeps member 1's id; member 0's batch, though
    submitted later and smaller (done on the device first), completes after it and takes later ids."""
    a, b = batch(reads, 0, 3000), batch(reads, 3000, 3040)
    again = batch(reads, 100, 160)
    batches = [a, b, again]
    bp, rp = plain(indices[0], batches)
    members = [K.BUSProcessor(x, "10xv3") for x in indices[1:3]]
    g = K.BUSGroup(members)
    t0 = g.submit(1, a)
    t1 = g.submit(0, b)
    with pytest.raises(K.KallistoB200Error) as e:
        g.complete(t1)                                  # not the oldest
    assert e.value.code == K.KB_ERR_INVALID
    r0 = g.complete(t0)
    r1 = g.complete(t1)
    t2 = g.submit(0, again)                             # sets member 1 committed, now new on member 0
    r2 = g.complete(t2)
    same_run(bp, rp, g, np.concatenate([r0, r1, r2]))


def test_num_across_a_sample_switch(reads, indices):
    batches = [batch(reads, a, min(a + 500, 4000)) for a in range(0, 4000, 500)]
    samples = {0: 0, 3: 1, 6: 2}
    bp, rp = plain(indices[0], batches, samples, num=True)
    g, _, rg = grouped(indices[1:4], batches, samples, num=True)
    same_run(bp, rp, g, rg)
    assert rg["flags"].max() < 1500                     # read numbers restart with every sample


def test_refusals(reads, indices):
    def refused(f):
        with pytest.raises(K.KallistoB200Error) as e:
            f()
        assert e.value.code == K.KB_ERR_INVALID
    m0, m1 = K.BUSProcessor(indices[0], "10xv3"), K.BUSProcessor(indices[1], "10xv3", num=True)
    refused(lambda: K.BUSGroup([m0, m1]))              # other options
    m2 = K.BUSProcessor(indices[2], "10xv3", strand="rf")
    refused(lambda: K.BUSGroup([m0, m2]))
    refused(lambda: K.BUSGroup([m0, m0]))              # one member twice
    used = K.BUSProcessor(indices[3], "10xv3")
    used.process_sets(batch(reads, 0, 50))
    refused(lambda: K.BUSGroup([m0, used]))            # not fresh
    m3 = K.BUSProcessor(indices[3], "10xv3")
    g = K.BUSGroup([m0, m3])
    t0 = g.submit(0, batch(reads, 0, 100))
    refused(lambda: g.submit(0, batch(reads, 100, 200)))   # member busy
    t1 = g.submit(1, batch(reads, 100, 200))
    refused(lambda: g.begin_sample(1))                 # batches outstanding
    refused(lambda: g.complete(t1))                    # out of order
    refused(lambda: g.complete(t0 + 7))
    g.complete(t0)
    g.complete(t1)
    refused(lambda: g.complete(t1 + 1))                # nothing outstanding
    g.begin_sample(1)
    g.close()
    for m in (m0, m1, m2, used, m3):
        m.close()
