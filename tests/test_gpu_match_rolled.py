"""GPU: match_kernel rolls a chain's k-mer one base forward when its next lookup starts one position later, and settles
collisions and MAIN misses of mates without N on a straight-line path before the general transition.  Read lengths
around the 16-base words of the packed read and longer than 100 bp, N bases next to runs of misses, and pairs where one
mate only misses while the other jumps, against the oracle: per-fragment ECs, the EC table and counts, fragment lengths
and, for pairs, the exact number of k-mer lookups (single-end reads are compared on their ECs only: the reference's
single-end early exit, `partial`, is not modelled on the device, which may look up a few more k-mers there)."""
import zlib

import numpy as np
import pytest

from tests import util
from tests.test_gpu_match_chains import check, revcomp

pytestmark = pytest.mark.gpu

N_FRAG = 3000
LENGTHS = [31, 32, 33, 47, 48, 150, 250]


def random_bases(rng, n):
    return bytes(rng.choice(list(b"ACGT"), size=n).astype(np.uint8))


def with_n(s, pos):
    return s[:pos] + b"N" + s[pos + 1:]


def make_case(ds, case, rng):
    n = min(N_FRAG, len(ds["s1"]))
    s1, s2 = [bytes(x) for x in ds["s1"][:n]], [bytes(x) for x in ds["s2"][:n]]
    if case == "lengths":
        # both ends of the fragment joined (a junction the index does not know), cut to lengths on either side of the
        # 16- and 32-base words and past 100 bp; the two mates of a fragment get different lengths
        o1, o2 = [], []
        for i, (a, b) in enumerate(zip(s1, s2)):
            long1 = (a + revcomp(b)) * 2
            long2 = (b + revcomp(a)) * 2
            o1.append(long1[: LENGTHS[i % len(LENGTHS)]])
            o2.append(long2[: LENGTHS[(i // len(LENGTHS) + 3) % len(LENGTHS)]])
        assert {len(x) for x in o1} == set(LENGTHS) and {len(x) for x in o2} == set(LENGTHS)
        return o1, o2
    if case == "n_after_misses":
        # a run of absent k-mers, then an N, then the read: the lookup after the N is rebuilt, the ones after it rolled
        o1, o2 = [], []
        for a, b in zip(s1, s2):
            r = int(rng.integers(5, 60))
            o1.append(random_bases(rng, r) + b"N" + a[r + 1:])
            o2.append(with_n(b, int(rng.integers(0, len(b)))) if rng.random() < 0.5 else b)
        return o1, o2
    if case == "n_inside_misses":
        # unmappable second mates with N bases at random places: every lookup of chain 1 is a miss on a mate with an N
        o2 = []
        for b in s2:
            x = random_bases(rng, len(b))
            for _ in range(int(rng.integers(1, 4))):
                x = with_n(x, int(rng.integers(0, len(x))))
            o2.append(x)
        return s1, o2
    if case == "miss_beside_jump":
        # one mate only misses (the straight-line path at every lookup) while the other hits and jumps
        o1, o2 = [], []
        for i, (a, b) in enumerate(zip(s1, s2)):
            x = random_bases(rng, len(b))
            o1.append(a if i % 2 else x)
            o2.append(x if i % 2 else b)
        return o1, o2
    raise ValueError(case)


@pytest.mark.parametrize("name", ["synth_small", "manyecs", "abundant"])
@pytest.mark.parametrize("case", ["lengths", "n_after_misses", "n_inside_misses", "miss_beside_jump"])
def test_rolled_kmers_match_oracle(name, case):
    ds = util.dataset(name)
    rng = np.random.default_rng(zlib.crc32((name + case).encode()))
    s1, s2 = make_case(ds, case, rng)
    check(ds, s1, s2)


@pytest.mark.parametrize("case", ["lengths", "n_after_misses"])
def test_rolled_kmers_single_end(case):
    ds = util.dataset("synth_small")
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    s1, _ = make_case(ds, case, rng)
    check(ds, s1, None)
