"""Test tools for the Myers pattern matching: ctypes over tests/sim/myers_oracle.cpp (the semi-global definition,
with the edit-distance definitions it includes) and tests/sim/b2a_sim_myers.cpp (the kernels' lane logic on the
host), both built on first use, and the input matrix the host and the GPU suites share."""
import ctypes as C
import os

import numpy as np

import distance_util as du

SIM_DIR = du.SIM_DIR
ORC_SRC = os.path.join(SIM_DIR, "myers_oracle.cpp")
ORC_SO = os.path.join(SIM_DIR, "libmyersoracle.so")
SIM_SRC = os.path.join(SIM_DIR, "b2a_sim_myers.cpp")
SIM_SO = os.path.join(SIM_DIR, "libb2asimmyers.so")
SIM_DEPS = du.SIM_DEPS + [SIM_SRC, os.path.join(du.ROOT, "rust_bio_b200", "csrc", "b2a_myers.cuh")]
NONE = du.NONE
MT_DONE, MT_REGS1, MT_WARP = 0, 1, 5  # b2a_myers.cuh
PATTERN_LENGTHS = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049, 4097)
IUPAC = {b"M": b"AC", b"R": b"AG", b"W": b"AT", b"S": b"CG", b"Y": b"CT", b"K": b"GT", b"V": b"ACGMRS",
         b"H": b"ACTMWY", b"D": b"AGTRWK", b"B": b"CGTSYK", b"N": b"ACGTMRWSYKVHDB"}  # builder.rs:18-30

_orc = _sim = None


def myers_tier(m: int, n: int) -> int:
    """the tier b2a_myers.cuh's myers_tier picks for a pair"""
    if m == 0 or n == 0:
        return MT_DONE
    w = (m + 63) // 64
    return MT_REGS1 + w - 1 if w <= 4 else MT_WARP


def tables(ambig=None, wildcards=None):
    """b2a_myers_match's bit tables (numpy, or None) from {pattern byte: text bytes} and wildcard text bytes"""
    amb = None
    if ambig:
        amb = np.zeros((256, 32), dtype=np.uint8)
        for p, eqs in ambig.items():
            for t in bytes(eqs):
                amb[int(p), t >> 3] |= np.uint8(1 << (t & 7))
    wild = None
    if wildcards:
        wild = np.zeros(32, dtype=np.uint8)
        for t in wildcards:
            wild[int(t) >> 3] |= np.uint8(1 << (int(t) & 7))
    return amb, wild


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def oracle():
    global _orc
    if _orc is None:
        L = C.CDLL(du._build(ORC_SO, [ORC_SRC, du.ORC_SRC], ORC_SRC, []))
        L.orc_myers_row.restype = None
        L.orc_myers_row.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                    C.c_void_p]
        L.orc_levenshtein.restype = C.c_uint32
        L.orc_levenshtein.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32]
        _orc = L
    return _orc


def orc_row(x: bytes, y: bytes, ambig=None, wildcards=None):
    """[D[m][j] for j = 1..n]"""
    amb, wild = tables(ambig, wildcards)
    row = np.zeros(max(1, len(y)), dtype=np.uint32)
    oracle().orc_myers_row(x, len(x), y, len(y), _ptr(amb), _ptr(wild), _ptr(row))
    return [int(v) for v in row[:len(y)]]


def orc_search(x: bytes, y: bytes, k=None, ambig=None, wildcards=None):
    """(best_end, best_dist, hits): the first end of the least D[m][j] (None, None for an empty text) and, with k,
    every (end, dist) with dist <= k in ascending end order"""
    row = orc_row(x, y, ambig, wildcards)
    if not row:
        return None, None, [] if k is not None else None
    best = min(row)
    hits = [(j, d) for j, d in enumerate(row) if d <= k] if k is not None else None
    return row.index(best), best, hits


def orc_levenshtein(x: bytes, y: bytes) -> int:
    return int(oracle().orc_levenshtein(x, len(x), y, len(y)))


def sim():
    global _sim
    if _sim is None:
        _sim = C.CDLL(du._build(SIM_SO, SIM_DEPS, SIM_SRC, []))
    return _sim


def sim_myers(pairs, k=None, ambig=None, wildcards=None, force_warp=False):
    """the lane code's two passes on the host -> per pair (best_end, best_dist, hits or None), and the tiers"""
    blob, xo, xl, yo, yl = pack_shared(pairs)
    n = len(pairs)
    amb, wild = tables(ambig, wildcards)
    be, bd, cnt = (np.zeros(max(1, n), dtype=np.uint32) for _ in range(3))
    tiers = np.zeros(max(1, n), dtype=np.int32)
    kk = NONE if k is None else min(int(k), NONE)
    args = [_ptr(blob), C.c_uint64(blob.nbytes), _ptr(xo), _ptr(xl), _ptr(yo), _ptr(yl), C.c_uint64(n), _ptr(amb),
            _ptr(wild), C.c_uint32(kk), C.c_int(1 if force_warp else 0), _ptr(be), _ptr(bd), _ptr(cnt), _ptr(tiers)]
    assert sim().sim_myers(*args, None, None, None) == 0
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(cnt[:n], dtype=np.uint64)
    total = int(off[-1])
    he, hd = np.zeros(max(1, total), dtype=np.uint32), np.zeros(max(1, total), dtype=np.uint32)
    assert sim().sim_myers(*args, _ptr(off), _ptr(he), _ptr(hd)) == 0
    out = []
    for p in range(n):
        e, d = int(be[p]), int(bd[p])
        hits = None
        if k is not None:
            lo, hi = int(off[p]), int(off[p + 1])
            hits = list(zip(he[lo:hi].tolist(), hd[lo:hi].tolist()))
        out.append((None if e == NONE else e, None if d == NONE else d, hits))
    return out, [int(t) for t in tiers[:n]]


def pack_shared(pairs):
    """(blob, x_off, x_len, y_off, y_len) with the sequences back to back at every alignment, and every pair whose
    pattern equals an earlier pair's pointing at that pattern's one copy"""
    parts, xo, yo, pos, seen = [], [], [], 0, {}
    for x, y in pairs:
        x = bytes(x)
        if x not in seen:
            seen[x] = pos
            parts.append(x)
            pos += len(x)
        xo.append(seen[x])
        yo.append(pos)
        parts.append(bytes(y))
        pos += len(y)
    blob = np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8).copy()
    return (blob, np.array(xo, dtype=np.uint64), np.array([len(x) for x, _ in pairs], dtype=np.uint32),
            np.array(yo, dtype=np.uint64), np.array([len(y) for _, y in pairs], dtype=np.uint32))


def plant(rng, x: bytes, n: int, rate: float, alphabet: bytes = b"ACGT") -> bytes:
    """a random text of about n bytes holding a mutated copy of x at a random place"""
    core = du.mutate(rng, x, rate, alphabet)
    left = int(rng.integers(0, max(1, n - len(core)) + 1))
    return du.rand_seq(rng, left, alphabet) + core + du.rand_seq(rng, max(0, n - len(core) - left), alphabet)


def matrix_pairs(seed=1, lengths=PATTERN_LENGTHS):
    """Pattern lengths at word, register-tier and strip edges, each in a text holding a mutated copy, in an unrelated
    text, and in a text shorter than the pattern; empty texts; all 256 byte values; one pattern shared by several
    texts."""
    rng = np.random.default_rng(seed)
    pairs = [(b"A", b""), (b"ACGT" * 20, b""), (b"ACGT", b"A"), (b"CATGC", b"ATG")]
    for P in lengths:
        x = du.rand_seq(rng, P)
        pairs.append((x, plant(rng, x, P + int(rng.integers(5, 200)), 0.08)))
        pairs.append((x, du.rand_seq(rng, int(rng.integers(1, P + 40)))))
        pairs.append((x, du.mutate(rng, x[:max(1, P // 2)], 0.1, b"ACGT")))
    allb = bytes(range(256))
    pairs.append((allb, allb[::-1] + allb))
    pairs.append((bytes(rng.permutation(256).astype(np.uint8))[:100], allb * 2))
    shared = du.rand_seq(rng, 33)
    for _ in range(4):
        pairs.append((shared, plant(rng, shared, 150, 0.1)))
    return pairs
