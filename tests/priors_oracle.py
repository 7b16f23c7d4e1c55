"""The reference's EM started from given abundances (EMAlgorithm::set_priors + EMAlgorithm::run, src/EMAlgorithm.h:83-221),
restated with numpy in the reference's own order of operations, and the --priors file arithmetic
(EMAlgorithm::read_priors, :52-81).  oracle.em is the same EM from the uniform start; em() here equals it bit for bit when
it is given alpha0 = 1 / T (tests/test_oracle_priors.py checks that), so the two share one model.

Every per-EC denominator and per-target numerator is a sequential sum in the reference's order: np.bincount adds its
weights one after the other in input order, so feeding it the entries in EC order reproduces the reference's loops."""
import numpy as np

ALPHA_LIMIT, ALPHA_CHANGE_LIMIT, ALPHA_CHANGE = 1e-7, 1e-2, 1e-2
TOLERANCE = np.finfo(np.float64).smallest_subnormal


def em(off, tids, counts, eff, n_targets, alpha0=None, counts_w=None, n_iter=10000, min_rounds=50):
    """-> (est_counts, rounds) of the EM over the EC table (off, tids, counts) started from alpha0 (None: 1 / T)."""
    T = int(n_targets)
    off = np.asarray(off, np.int64)
    tids = np.asarray(tids, np.int64)
    counts = np.asarray(counts, np.uint32)
    cw = counts if counts_w is None else np.asarray(counts_w, np.uint32)
    eff = np.asarray(eff, np.float64)
    n_ec = len(counts)
    lens = np.diff(off)
    ec_of = np.repeat(np.arange(n_ec), lens)
    single = lens == 1
    s_t = tids[off[:-1][single]]
    s_c = counts[single].astype(np.float64)
    # entries of the multi-target ECs with a non-zero count, in EC order (the others are skipped, :125-129)
    keep = (~single[ec_of]) & (counts[ec_of] != 0)
    m_t = tids[keep]
    m_e = ec_of[keep]
    ecs, m_loc = np.unique(m_e, return_inverse=True)
    m_w = cw[m_e].astype(np.float64) / eff[m_t]
    m_c = counts[ecs].astype(np.float64)
    idx = np.concatenate([s_t, m_t])
    alpha = np.full(T, 1.0 / T) if alpha0 is None else np.array(alpha0, np.float64, copy=True)
    final = False
    i = 0
    with np.errstate(divide="ignore", invalid="ignore"):
        while i < n_iter:
            a = alpha[m_t]
            denom = np.bincount(m_loc, weights=a * m_w, minlength=len(ecs))
            ok = ~(denom < TOLERANCE)
            norm = np.where(ok, m_c / denom, 0.0)
            contrib = np.where(ok[m_loc], (m_w * a) * norm[m_loc], 0.0)
            nxt = np.bincount(idx, weights=np.concatenate([s_c, contrib]), minlength=T)
            chcount = np.count_nonzero((nxt > ALPHA_CHANGE_LIMIT) & ((np.abs(nxt - alpha) / nxt) > ALPHA_CHANGE))
            alpha = nxt
            stop = chcount == 0 and i > min_rounds
            if final:
                break
            if stop:
                final = True
                alpha[alpha < ALPHA_LIMIT / 10.0] = 0.0
            i += 1
    return alpha, i


def read_priors_text(text):
    """EMAlgorithm::read_priors on the text of a file whose every line std::stod accepts -> float64 array."""
    lines = text.split("\n")
    if lines[-1] == "":
        lines.pop()                 # std::getline: a final newline ends the last line, it does not start another
    vals = [stod(l) for l in lines]
    v = np.array(vals, np.float64)
    s = 0.0
    for x in vals:                  # in file order
        s += x
    if s >= 1.0 + 1e-3:
        s += len(vals)
        v = (v + 1.0) / s
    return v


_strtod = None


def stod(line):
    """std::stod: strtod over the whole line (leading blanks skipped, the rest ignored, hex floats accepted); ValueError
    where std::stod throws (no number, or out of range)."""
    global _strtod
    import ctypes
    if _strtod is None:
        _strtod = ctypes.CDLL(None, use_errno=True).strtod
        _strtod.restype = ctypes.c_double
        _strtod.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]
    buf = ctypes.create_string_buffer(line.encode())
    end = ctypes.c_void_p()
    ctypes.set_errno(0)
    x = _strtod(ctypes.addressof(buf), ctypes.byref(end))
    if end.value == ctypes.addressof(buf) or ctypes.get_errno() != 0:
        raise ValueError("std::stod rejects %r" % line)
    return x
