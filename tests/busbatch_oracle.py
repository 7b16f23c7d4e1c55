"""TEST INFRASTRUCTURE: `kallisto bus --batch FILE` with a technology restated on top of oracle.bus_model (and
tests/aa_oracle.py for --aa): every line of the batch file is a sample of its own (read numbers and the fragment-length
quota restart), lines with the same id share a batch number (batch_id_mapping, src/ProcessReads.h:211-224), and with
--batch-barcodes (src/ProcessReads.cpp:1583-1627):
  * without a barcode read the barcode is the batch number as 16 letters;
  * with a barcode read of blen <= 32 letters it is binaryToString(batch, 32 - blen) + binaryToString(stringToBinary(bc,
    blen), blen): 32 letters, an N turned into G, no N flag in the barcode half of the flags nor in the UMI half where
    it repeats the barcode's.
That rule is applied by handing bus_model the rewritten barcode as one whole-read piece of an extra file; a read set
whose barcode pieces do not fit gets an empty one there, so it is skipped as before.  Without --batch-barcodes the
records are those of a single-sample run, and a technology without a barcode read gets 16 x 'A'.
The files a run writes follow src/main.cpp:2405-2454 and the header src/ProcessReads.h:240-253.  Imported by tests only."""
import os

import numpy as np

from oracle import oracle as O
from tests import aa_oracle as A

# technology -> (bc pieces, umi pieces (None: no UMI), seq, seq2, default strand, tag); umi[0] advanced past the tag
TECH = {
    "10XV3": ([(0, 0, 16)], [(0, 16, 28)], (1, 0), None, 1, None),
    "10XV2": ([(0, 0, 16)], [(0, 16, 26)], (1, 0), None, 1, None),
    "SMARTSEQ3": ([(0, 0, 0), (1, 0, 0)], [(2, 11, 19)], (2, 22), (3, 0), 1, b"ATTGCGCAATG"),
    "-1,-1,-1:0,16,28:1,0,0": ([], [(0, 16, 28)], (1, 0), None, 0, None),
    "0,0,16,1,0,16:0,16,28:1,0,0": ([(0, 0, 16), (1, 0, 16)], [(0, 16, 28)], (1, 0), None, 0, None),
}


def binary_to_string(x, n):
    """binaryToString (src/BUSData.cpp:38-51)"""
    return bytes(b"ACGT"[(x >> (2 * (n - 1 - i))) & 3] for i in range(n))


def read_batch_file(path):
    """-> [(id, [file, ...])] of the lines that are not empty or comments (src/main.cpp:1240-1270)"""
    out = []
    with open(path) as f:
        for line in f:
            w = line.split()
            if w and not w[0].startswith("#"):
                out.append((w[0], w[1:]))
    return out


def batch_numbers(ids):
    m = {}
    return [m.setdefault(i, len(m)) for i in ids]


def prefixed(bc_string, batch):
    """The 32-letter barcode of --batch-barcodes for a barcode of at most 32 letters."""
    blen = len(bc_string)
    assert 0 < blen <= 32
    v, _ = O.string_to_binary(bc_string)
    return binary_to_string(batch, 32 - blen) + binary_to_string(v, blen)


def batch_model(index, lines, tech, strand="default", num=False, batch_barcodes=False, aa=False, paired_flag=False):
    """lines: [(id, [list of sequences per file of the technology])], one per batch-file line.
    -> dict(records, ecs, flens, header, cells, sample_barcodes, index_saved, n_processed, [clashes])"""
    bc, umi, seq, seq2, dstrand, tag = TECH[tech]
    strand = dstrand if strand == "default" else strand
    nf = len(lines[0][1])
    files = [[] for _ in range(nf)]
    samples = []
    for _, fl in lines:
        lo = len(files[0])
        for f in range(nf):
            files[f].extend(fl[f])
        samples.append((lo, len(files[0])))
    nums = batch_numbers([i for i, _ in lines])
    sample_barcodes = nums if batch_barcodes else [0] * len(lines)      # used without a barcode read only
    if batch_barcodes and bc:
        extra = []
        for si, (lo, hi) in enumerate(samples):
            for i in range(lo, hi):
                parts = []
                for f, a, b in bc:
                    l = len(files[f][i])
                    ln = (l - a) if b == 0 else (b - a)
                    parts.append(None if (l < a + ln or ln <= 0) else files[f][i][a:a + ln])
                if any(p is None for p in parts):
                    extra.append(b"")
                    continue
                s = b"".join(parts)
                if len(s) > 32:
                    raise ValueError("read set %d: a barcode of %d letters cannot take the batch number" % (i, len(s)))
                extra.append(prefixed(s, nums[si]))
        files = files + [extra]
        bc = [(nf, 0, 0)]
    if aa:
        m = A.aa_bus_model(index, files, bc, umi, seq, strand=strand, num=num, samples=samples,
                           sample_barcodes=sample_barcodes)
    else:
        m = O.bus_model(index, files, bc, umi, seq, seq2, strand=strand, num=num, samples=samples, tag=tag,
                        sample_barcodes=sample_barcodes)
    bclen = sum(b - a for _, a, b in TECH[tech][0]) if all(b != 0 for _, _, b in TECH[tech][0]) else 0
    umilen = 0 if umi is None or any(b == 0 for _, _, b in umi) else sum(b - a for _, a, b in umi)
    m["header"] = (16 if (batch_barcodes and not TECH[tech][0]) else bclen, umilen)
    m["cells"] = [i for i, _ in lines]
    m["sample_barcodes"] = [binary_to_string(v, 16).decode() for v in nums] if batch_barcodes else None
    m["index_saved"] = bool(paired_flag or seq2 is not None or umi is None)
    if not paired_flag:
        m["flens"] = None
    return m


def read_lines(batch_path, tech):
    """The sequences of a batch file's lines, read from the files it names (relative to the batch file)."""
    d = os.path.dirname(batch_path)
    return [(i, [O.read_fastq(os.path.join(d, f)) for f in fl]) for i, fl in read_batch_file(batch_path)]


def n_unique(records, ecs):
    return int(sum(1 for e in records["ec"] if len(ecs[int(e)]) == 1))


def sorted_records(r):
    return np.sort(r, order=["barcode", "umi", "ec", "flags", "count"])
