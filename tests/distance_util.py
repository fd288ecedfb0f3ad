"""Test tools for the edit distances: ctypes over tests/sim/distance_oracle.cpp (the definitions, O(mn)) and
tests/sim/b2a_sim_distance.cpp (the kernels' lane logic on the host), both built on first use, and the input matrix
the host and the GPU suites share."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SIM_DIR = os.path.join(HERE, "sim")
ORC_SRC = os.path.join(SIM_DIR, "distance_oracle.cpp")
ORC_SO = os.path.join(SIM_DIR, "libdistoracle.so")
SIM_SRC = os.path.join(SIM_DIR, "b2a_sim_distance.cpp")
SIM_SO = os.path.join(SIM_DIR, "libb2asimdist.so")
SIM_DEPS = [SIM_SRC, os.path.join(SIM_DIR, "b2a_sim.cpp")] + [
    os.path.join(ROOT, "rust_bio_b200", "csrc", f)
    for f in ("b2a_distance.cuh", "b2a_coop.cuh", "b2a_common.cuh", "b2a_fill.cuh", "b2a_walk.cuh", "b2a_plan.h")]
NONE = 0xFFFFFFFF
DT_DONE, DT_REGS1, DT_BAND4, DT_BAND8, DT_WARP = 0, 1, 5, 6, 7  # b2a_distance.cuh


def dist_tier(m: int, n: int, k=None) -> int:
    """the tier b2a_distance.cuh's dist_tier picks for a pair (k None: unbounded)"""
    P, N = min(m, n), max(m, n)
    kk = N if k is None else min(k, N)
    if N - P > kk or P == 0:
        return DT_DONE
    words = (P + 63) // 64
    if words <= 4:
        return DT_REGS1 + words - 1
    if k is not None and 2 * kk // 64 + 2 <= 4:
        return DT_BAND4
    if k is not None and 2 * kk // 64 + 2 <= 8:
        return DT_BAND8
    return DT_WARP


def _build(so, deps, src, extra):
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                               *extra, "-o", so, src])
    return so


_orc = _sim = None


def oracle():
    global _orc
    if _orc is None:
        L = C.CDLL(_build(ORC_SO, [ORC_SRC], ORC_SRC, []))
        L.orc_levenshtein.restype = C.c_uint32
        L.orc_levenshtein.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32]
        L.orc_bounded_levenshtein.restype = C.c_uint32
        L.orc_bounded_levenshtein.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32]
        L.orc_hamming.restype = C.c_int64
        L.orc_hamming.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32]
        _orc = L
    return _orc


def orc_levenshtein(x: bytes, y: bytes) -> int:
    return int(oracle().orc_levenshtein(x, len(x), y, len(y)))


def orc_bounded(x: bytes, y: bytes, k: int):
    """simd::bounded_levenshtein's rule on the oracle's distance: the distance, or None"""
    v = int(oracle().orc_bounded_levenshtein(x, len(x), y, len(y), k))
    return None if v == NONE else v


def orc_hamming(x: bytes, y: bytes):
    v = int(oracle().orc_hamming(x, len(x), y, len(y)))
    return None if v < 0 else v


def sim():
    global _sim
    if _sim is None:
        _sim = C.CDLL(_build(SIM_SO, SIM_DEPS, SIM_SRC, []))
    return _sim


def pack_unaligned(pairs):
    """(blob, x_off, x_len, y_off, y_len) with the sequences back to back: offsets at every alignment, for the
    kernels' wide loads"""
    parts, xo, yo, pos = [], [], [], 0
    for x, y in pairs:
        xo.append(pos)
        pos += len(x)
        yo.append(pos)
        pos += len(y)
        parts += [bytes(x), bytes(y)]
    blob = np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8).copy()
    return (blob, np.array(xo, dtype=np.uint64), np.array([len(x) for x, _ in pairs], dtype=np.uint32),
            np.array(yo, dtype=np.uint64), np.array([len(y) for _, y in pairs], dtype=np.uint32))



def sim_levenshtein(pairs, k=None, force_tier=-1):
    """-> (distances as ints / None for a bounded miss, tiers)"""
    blob, xo, xl, yo, yl = pack_unaligned(pairs)
    n = len(pairs)
    out = np.zeros(max(1, n), dtype=np.uint32)
    tiers = np.zeros(max(1, n), dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = sim().sim_levenshtein(p(blob), C.c_uint64(blob.nbytes), p(xo), p(xl), p(yo), p(yl), C.c_uint64(n),
                               C.c_uint32(NONE if k is None else k), C.c_int(force_tier), p(out), p(tiers))
    assert rc == 0
    return [None if v == NONE and k is not None else int(v) for v in out[:n]], [int(t) for t in tiers[:n]]


def sim_hamming(pairs):
    blob, xo, xl, yo, yl = pack_unaligned(pairs)
    n = len(pairs)
    out = np.zeros(max(1, n), dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = sim().sim_hamming(p(blob), C.c_uint64(blob.nbytes), p(xo), p(xl), p(yo), p(yl), C.c_uint64(n), p(out))
    assert rc == 0
    return [None if v == NONE else int(v) for v in out[:n]]


def mutate(rng, s: bytes, rate: float, alphabet: bytes) -> bytes:
    """substitutions, insertions and deletions at about `rate` per base"""
    out = bytearray()
    for c in s:
        r = rng.random()
        if r < rate / 3:
            out.append(alphabet[rng.integers(0, len(alphabet))])
        elif r < 2 * rate / 3:
            out.append(c)
            out.append(alphabet[rng.integers(0, len(alphabet))])
        elif r < rate:
            continue
        else:
            out.append(c)
    return bytes(out)


def rand_seq(rng, n: int, alphabet: bytes = b"ACGT") -> bytes:
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return bytes(a[rng.integers(0, len(a), n)])


def edge_pairs(seed=1, lengths=(0, 1, 31, 32, 33, 63, 64, 65, 150, 192, 193, 255, 256, 257)):
    """Pattern lengths at word edges (64-bit words) and at the 4-word edge of the register tier, each against a
    related text (mutated copy) and an unrelated one; empty sides; all 256 byte values."""
    rng = np.random.default_rng(seed)
    pairs = [(b"", b""), (b"", b"ACGT"), (b"ACGT", b""), (b"ACCGTGGAT", b"AAAAACCGTTGAT"), (b"AAA", b"TTTT")]
    for P in lengths:
        x = rand_seq(rng, P)
        pairs.append((x, mutate(rng, x, 0.1, b"ACGT") + rand_seq(rng, int(rng.integers(0, 5)))))
        pairs.append((rand_seq(rng, int(P + rng.integers(0, 40))), x))
    allb = bytes(range(256))
    pairs.append((allb, allb[::-1]))
    pairs.append((bytes(rng.permutation(256).astype(np.uint8)), allb + allb[:40]))
    return pairs


def strip_pairs(seed=2):
    """Patterns at the edges of the warp tier's 2048-row strips (32 words of 64 rows)"""
    rng = np.random.default_rng(seed)
    pairs = []
    for P in (2047, 2048, 2049, 300, 4097):
        x = rand_seq(rng, P)
        pairs.append((x, mutate(rng, x, 0.05, b"ACGT")))
    pairs.append((rand_seq(rng, 2049), rand_seq(rng, 2100)))
    pairs.append((rand_seq(rng, 260), rand_seq(rng, 270)))  # unrelated: a distance near the length
    return pairs
