"""TEST INFRASTRUCTURE: `kallisto bus --aa` restated on the CPU (src/ProcessReads.cpp:1629-1736) on top of the oracle's
single-end pseudoalignment (oracle/kb_oracle.cpp through oracle/oracle.py):

  1. every read set's sequence s (from the technology's start to the end of the read) gives six frames: frame j reads
     from (j < 3 ? s : revcomp(s)) + j % 3 and has l_j = len(s) - j % 3 letters; it is translated into comma-free code
     (nn_to_cfc, src/KmerIndex.cpp:19-85,118-138) and, as the device does, padded with l_j mod 3 letters N up to l_j;
  2. the 6n frames are pseudoaligned as unstranded single-end reads;
  3. intersectKmersCFC (src/MinCollector.cpp:44-119): the smallest non-empty frame set wins, the lowest frame on a tie;
     a clash for every later frame whose set is as small as the smallest set before it;
  4. with a strand mode, doStrandSpecificity with v = frame 0's hits (src/ProcessReads.cpp:45-110,1728-1735): the set is
     cut down to the members of the EC of frame 0's first mapping k-mer whose sense agrees with the strand.  That k-mer
     is the first window of frame 0, in scan order, that is in the index; the filter set is what the oracle's stranded
     single-end run gives for that window alone (its one hit is its own first hit, and its set is the block's EC).
Imported by tests only."""
import numpy as np

from oracle import oracle as O

# comma-free code of every codon, codon = b0 * 16 + b1 * 4 + b2 with A 0, C 1, G 2, T 3 (cfc_map; NNN for stops)
CFC = ("CGCCGACGCCGACTTCTTCTTCTTTGTCTATGTCTAATAATAATCATAAGGAGTAGGAGTCTCCTCCTCCTCTGTTGTTGTTGTACAACAACAACACGGCGTCGGCG"
       "TAGAAGAAGAAGATGGTGGTGGTGGATTATTATTATTNNNAGCNNNAGCCTACTACTACTANNNTGATGCTGAACAACCACAACC").encode()
_B = {ord("A"): 0, ord("C"): 1, ord("G"): 2, ord("T"): 3}
_RC = {ord("A"): b"T", ord("C"): b"G", ord("G"): b"C", ord("T"): b"A",
       ord("a"): b"T", ord("c"): b"G", ord("g"): b"C", ord("t"): b"A"}


def revcomp(s):
    """src/common.cpp:36-53: A/C/G/T in either case complemented to upper case, any other letter N."""
    return b"".join(_RC.get(c, b"N") for c in reversed(s))


def nn_to_cfc(s):
    out = []
    for i in range(0, len(s) - 2, 3):
        t = s[i:i + 3].upper()
        if all(c in _B for c in t):
            x = _B[t[0]] * 16 + _B[t[1]] * 4 + _B[t[2]]
            out.append(CFC[3 * x:3 * x + 3])
        else:
            out.append(b"NNN")
    return b"".join(out)


def frames(s):
    """The six padded cfc frames of a sequence."""
    rc = revcomp(s)
    out = []
    for j in range(6):
        src = (s if j < 3 else rc)[j % 3:]
        c = nn_to_cfc(src)
        out.append(c + b"N" * (len(src) - len(c)))
    return out


def aa_sets(index, seqs, strand=0):
    """seqs: the sequence of every read set (b"" for a skipped one).  -> (per set: tuple of targets or None, clashes)"""
    n = len(seqs)
    fr = [f for s in seqs for f in frames(s)]
    run = O.OracleRun(index, False, 0, collect_fld=False)
    b, o = O.to_batch(fr)
    ids = run.pseudoalign(b, o)
    eo, et, _ = run.ec_table()
    sets = [tuple(int(x) for x in et[int(eo[e]):int(eo[e + 1])]) for e in range(len(eo) - 1)]
    out, clashes, need_filter = [None] * n, 0, []
    for i in range(n):
        best = None
        for j in range(6):
            e = int(ids[6 * i + j])
            if e < 0:
                continue
            u = sets[e]
            if best is None or len(u) < len(best):
                best = u
            elif len(u) == len(best):
                clashes += 1
        out[i] = best
        if best is not None and strand != 0:
            need_filter.append(i)
    if need_filter:
        k = index.k
        # every window of frame 0 holding only A/C/G/T, as a read of its own
        wins, owner = [], []
        for i in need_filter:
            f0 = fr[6 * i]
            for p in range(len(f0) - k + 1):
                w = f0[p:p + k]
                if all(c in _B for c in w):
                    wins.append(w)
                    owner.append(i)
        if wins:
            b, o = O.to_batch(wins)
            hit = O.OracleRun(index, False, 0, collect_fld=False).pseudoalign(b, o)
            srun = O.OracleRun(index, False, strand, collect_fld=False)
            fid = srun.pseudoalign(b, o)
            so, st, _ = srun.ec_table()
            ssets = [set(int(x) for x in st[int(so[e]):int(so[e + 1])]) for e in range(len(so) - 1)]
            first = {}
            for w, i in enumerate(owner):
                if i not in first and hit[w] >= 0:
                    first[i] = w
            for i, w in first.items():
                keep = ssets[fid[w]] if fid[w] >= 0 else set()
                r = tuple(t for t in out[i] if t in keep)
                out[i] = r if r else None
    return out, clashes


def aa_bus_model(index, files, bc, umi, seq, strand=0, num=False, samples=None, sample_barcodes=None):
    """Records, EC sets and clashes of `kallisto bus --aa -t 1`.  Arguments as oracle.bus_model's (one sequence read, no
    tag sequence): files: one list of sequences per file; bc / umi: lists of (file, start, stop), bc == [] = no barcode
    read, umi None = no UMI; seq: (file, start); samples: (first, end) ranges that are samples of their own."""
    n = len(files[0])
    by_sample = samples is not None
    samples = samples or [(0, n)]
    rec_bc, rec_umi, rec_fl, skip = [0] * n, [0] * n, [0] * n, [False] * n

    def piece(i, f, a, b):
        l = len(files[f][i])
        ln = (l - a) if b == 0 else (b - a)
        if l < a + ln or ln <= 0:
            return None
        return files[f][i][a:a + ln]

    for si, (lo, hi) in enumerate(samples):
        for i in range(lo, hi):
            if umi is None:
                uval, uflag = 0xFFFFFFFFFFFFFFFF, None
            else:
                parts = [piece(i, *u) for u in umi]
                if any(p is None for p in parts):
                    skip[i] = True
                    continue
                uval, uflag = O.string_to_binary(b"".join(parts))
            if bc:
                parts = [piece(i, *x) for x in bc]
                if any(p is None for p in parts):
                    skip[i] = True
                    continue
                bval, bflag = O.string_to_binary(b"".join(parts))
            else:
                bval, bflag = ((sample_barcodes[si] if sample_barcodes else si) if by_sample else 0), 0
            if uflag is None:
                uflag = bflag
            rec_bc[i], rec_umi[i] = bval, uval
            rec_fl[i] = (i - lo) if num else (bflag | (uflag << 8))
    seqs = [b"" if skip[i] else files[seq[0]][i][seq[1]:] for i in range(n)]
    sets, clashes = aa_sets(index, seqs, strand)
    ids, ecs = {}, []
    for s in sets:
        if s is not None and s not in ids:
            ids[s] = len(ecs)
            ecs.append(s)
    keep = [i for i in range(n) if sets[i] is not None]
    dt = np.dtype([("barcode", "<u8"), ("umi", "<u8"), ("ec", "<i4"), ("count", "<u4"), ("flags", "<u4"), ("pad", "<u4")])
    rec = np.zeros(len(keep), dt)
    for j, i in enumerate(keep):
        rec[j] = (rec_bc[i], rec_umi[i], ids[sets[i]], 1, rec_fl[i] & 0xFFFFFFFF, 0)
    return dict(records=rec, ecs=ecs, sets=sets, clashes=clashes, n_processed=n)
