"""Test tools for the pair HMM: ctypes over tests/sim/pairhmm_oracle.cpp (the literal restatement of the reference's
PairHMM::prob_related) and tests/sim/b2a_sim_pairhmm.cpp (the kernels' lane logic on the host), both built on first
use without FP contraction, and the input matrix the host and the GPU suites share."""
import ctypes as C
import math
import os

import numpy as np

import distance_util as du

SIM_DIR = du.SIM_DIR
ORC_SRC = os.path.join(SIM_DIR, "pairhmm_oracle.cpp")
ORC_SO = os.path.join(SIM_DIR, "libpairhmmoracle.so")
SIM_SRC = os.path.join(SIM_DIR, "b2a_sim_pairhmm.cpp")
SIM_SO = os.path.join(SIM_DIR, "libb2asimpairhmm.so")
SIM_DEPS = [SIM_SRC, os.path.join(SIM_DIR, "b2a_sim.cpp")] + [
    os.path.join(du.ROOT, "rust_bio_b200", "csrc", f) for f in ("b2a_pairhmm.cuh", "b2a_common.cuh")]
FLAGS = ["-ffp-contract=off"]
NONE = 0xFFFFFFFFFFFFFFFF  # max_edit_dist None
PT_DONE, PT_C1, PT_C2, PT_C4, PT_C5, PT_C8, PT_STRIP = range(7)  # b2a_pairhmm.cuh
TIER_C = {PT_C1: 1, PT_C2: 2, PT_C4: 4, PT_C5: 5, PT_C8: 8, PT_STRIP: 8}
LN_ZERO = float("-inf")

# Single base insertion, deletion and substitution rates of Illumina R1 (the reference's tests and bench:
# pairhmm.rs:291-293, benches/pairhmm.rs:17-19)
PROB_ILLUMINA_INS = 2.8e-6
PROB_ILLUMINA_DEL = 5.1e-6
PROB_ILLUMINA_SUBST = 0.0021
ILLUMINA_GAP = (math.log(PROB_ILLUMINA_INS), math.log(PROB_ILLUMINA_DEL), LN_ZERO, LN_ZERO)
ILLUMINA_EMIT = [[math.log(1.0 - PROB_ILLUMINA_SUBST)], [math.log(PROB_ILLUMINA_SUBST / 3.0)],
                 [math.log(1.0 - PROB_ILLUMINA_SUBST)], [math.log(1.0 - PROB_ILLUMINA_SUBST)]]

_orc = _sim = None


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def oracle():
    global _orc
    if _orc is None:
        L = C.CDLL(du._build(ORC_SO, [ORC_SRC], ORC_SRC, FLAGS + ["-pthread"]))
        for f in ("orc_fastexp",):
            getattr(L, f).restype = C.c_double
            getattr(L, f).argtypes = [C.c_double]
        L.orc_ln_add_exp.restype = C.c_double
        L.orc_ln_add_exp.argtypes = [C.c_double, C.c_double]
        L.orc_ln_sum_exp.restype = C.c_double
        L.orc_ln_sum_exp.argtypes = [C.c_void_p, C.c_uint64]
        L.orc_ln_one_minus_exp.restype = C.c_int
        L.orc_ln_one_minus_exp.argtypes = [C.c_double, C.POINTER(C.c_double)]
        L.orc_ln_sum3_exp_approx.restype = C.c_double
        L.orc_ln_sum3_exp_approx.argtypes = [C.c_double, C.c_double, C.c_double]
        L.orc_pairhmm_batch.restype = C.c_int
        L.orc_pairhmm_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_uint32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_uint64, C.c_int, C.c_void_p]
        _orc = L
    return _orc


def sim():
    global _sim
    if _sim is None:
        L = C.CDLL(du._build(SIM_SO, SIM_DEPS, SIM_SRC, FLAGS))
        L.sim_pairhmm.restype = C.c_int
        L.sim_pairhmm.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int,
                                  C.c_void_p, C.c_void_p]
        _sim = L
    return _sim


def ln_sum_exp(vals):
    v = np.asarray(vals, dtype=np.float64)
    return oracle().orc_ln_sum_exp(_ptr(v) if len(v) else None, len(v))


def ln_one_minus_exp(p):
    out = C.c_double(0.0)
    if oracle().orc_ln_one_minus_exp(p, C.byref(out)):
        raise AssertionError("assertion failed: p <= 0.0")
    return out.value


def emit_table(emit):
    """[match, mismatch, x, y] lists of one value per class -> the ABI's [4 * n_classes] float64 table"""
    t = np.asarray(emit, dtype=np.float64)
    assert t.ndim == 2 and t.shape[0] == 4
    return np.ascontiguousarray(t.reshape(-1)), t.shape[1]


def pack(pairs, classes=None):
    """(blob, cls or None, x_off, x_len, y_off, y_len): sequences back to back, pairs with equal x sharing one copy;
    classes: per pair (x_classes, y_classes) byte strings, or None"""
    parts, cparts, xo, yo, pos, seen = [], [], [], [], 0, {}
    for p, (x, y) in enumerate(pairs):
        x, y = bytes(x), bytes(y)
        cx, cy = (bytes(classes[p][0]), bytes(classes[p][1])) if classes is not None else (bytes(len(x)), bytes(len(y)))
        if (x, cx) not in seen:
            seen[(x, cx)] = pos
            parts.append(x)
            cparts.append(cx)
            pos += len(x)
        xo.append(seen[(x, cx)])
        yo.append(pos)
        parts.append(y)
        cparts.append(cy)
        pos += len(y)
    blob = np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8).copy()
    cls = np.frombuffer(b"".join(cparts) + b"\0", dtype=np.uint8).copy() if classes is not None else None
    return (blob, cls, np.array(xo, dtype=np.uint64), np.array([len(x) for x, _ in pairs], dtype=np.uint32),
            np.array(yo, dtype=np.uint64), np.array([len(y) for _, y in pairs], dtype=np.uint32))


def _call(fn, gap, mode, max_edit_dist, emit, packed, extra):
    blob, cls, xo, xl, yo, yl = packed
    n = len(xl)
    g = np.asarray(gap, dtype=np.float64)
    tab, ncls = emit_table(emit)
    out = np.zeros(max(1, n), dtype=np.float64)
    fs, fe = (1, 1) if mode == "semiglobal" else (0, 0) if mode == "global" else mode
    return fn(g, fs, fe, max_edit_dist, tab, ncls, blob, cls, xo, xl, yo, yl, n, out, *extra), out[:n]


def orc_batch(gap, mode, max_edit_dist, emit, packed, threads=1):
    """the oracle's prob_related per pair (NaN: the reference's assert); mode "global", "semiglobal" or (free_start,
    free_end); max_edit_dist None or an int.  Raises AssertionError where PairHMM::new asserts."""
    def fn(g, fs, fe, med, tab, ncls, blob, cls, xo, xl, yo, yl, n, out):
        return oracle().orc_pairhmm_batch(_ptr(g), fs, fe, 0 if med is None else 1, 0 if med is None else med,
                                          _ptr(tab), ncls, _ptr(blob), _ptr(cls), _ptr(xo), _ptr(xl), _ptr(yo),
                                          _ptr(yl), n, threads, _ptr(out))
    rc, out = _call(fn, gap, mode, max_edit_dist, emit, packed, ())
    if rc:
        raise AssertionError("assertion failed: p <= 0.0")
    return out


def sim_batch(gap, mode, max_edit_dist, emit, packed, force_tier=-1):
    """the kernels' lane logic on the host -> (results, tiers)"""
    n = len(packed[3])
    tiers = np.zeros(max(1, n), dtype=np.int32)

    def fn(g, fs, fe, med, tab, ncls, blob, cls, xo, xl, yo, yl, n, out, ft):
        return sim().sim_pairhmm(_ptr(g), fs, fe, NONE if med is None else min(int(med), NONE), _ptr(tab), ncls,
                                 _ptr(blob), _ptr(cls), _ptr(xo), _ptr(xl), _ptr(yo), _ptr(yl), n, ft, _ptr(out),
                                 _ptr(tiers))
    rc, out = _call(fn, gap, mode, max_edit_dist, emit, packed, (force_tier,))
    assert rc == 0, rc
    return out, [int(t) for t in tiers[:n]]


def bits(a):
    return np.asarray(a, dtype=np.float64).view(np.uint64)


def within(got, want, rel=1e-9):
    """the GPU tolerance rule: -inf exactly where the oracle gives -inf, NaN where it gives NaN, else |got - want| <=
    rel * max(1, |want|); -> indices outside it"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    bad = []
    for i, (g, w) in enumerate(zip(got, want)):
        if math.isnan(w) or math.isnan(g):
            ok = math.isnan(w) and math.isnan(g)
        elif math.isinf(w) or math.isinf(g):
            ok = g == w
        else:
            ok = abs(g - w) <= rel * max(1.0, abs(w))
        if not ok:
            bad.append(i)
    return bad


# the parameter sets of the matrix: (name, gap, emit)
def quality_emit(n_classes=42):
    """Phred-quality emission classes: class q has substitution probability 10^(-q/10) (q >= 2)"""
    em, mm, ex, ey = [], [], [], []
    for q in range(n_classes):
        e = 10 ** (-max(q, 2) / 10.0)
        em.append(math.log(1 - e))
        mm.append(math.log(e / 3))
        ex.append(math.log(1 - e))
        ey.append(math.log(1 - e))
    return [em, mm, ex, ey]


GAP_EXT = (math.log(1e-3), math.log(2e-3), math.log(0.1), math.log(0.2))
PARAMS = [("illumina", ILLUMINA_GAP, ILLUMINA_EMIT), ("extend", GAP_EXT, ILLUMINA_EMIT)]
MAX_EDIT = (None, 0, 2, 4, 10 ** 6)
Y_LENGTHS = (0, 1, 31, 32, 33, 63, 65, 127, 129, 159, 161, 255, 257, 600)
X_LENGTHS = (0, 1, 2, 300)


def matrix_pairs(seed=1, y_lengths=Y_LENGTHS, x_lengths=X_LENGTHS):
    """len_y at every tier and strip edge against len_x in {0, 1, 2, 300}: for each, y cut from x and mutated (similar)
    and an unrelated y; and a window shared by several reads"""
    rng = np.random.default_rng(seed)
    pairs = []
    for m in x_lengths:
        for n in y_lengths:
            x = du.rand_seq(rng, m)
            st = int(rng.integers(0, max(1, m - n) + 1))
            core = du.mutate(rng, x[st:st + n], 0.05, b"ACGT")
            y = (core + du.rand_seq(rng, max(0, n - len(core))))[:n]
            pairs.append((x, y))
            pairs.append((x, du.rand_seq(rng, n)))
    win = du.rand_seq(rng, 200)
    for _ in range(4):
        st = int(rng.integers(0, 50))
        pairs.append((win, du.mutate(rng, win[st:st + 150], 0.03, b"ACGT")))
    return pairs


def random_classes(rng, pairs, n_classes):
    return [(bytes(rng.integers(0, n_classes, len(x)).astype(np.uint8)),
             bytes(rng.integers(0, n_classes, len(y)).astype(np.uint8))) for x, y in pairs]
