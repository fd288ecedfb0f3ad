"""Long pairs: the warp-per-pair fill reads y from the staged-sequence arena instead of a whole-y shared-memory copy,
and the plan sizes the traceback of a warp-per-pair block by its real pairs and cuts blocks to fit the budget.

On the host (tests/sim/b2a_sim_long.cpp): the 32x8 and 32x16 strip-pipelined fill against the oracle, full and
score-only, with every y load checked against the pair's own words and the arena around each pair's y poisoned; the
plan for G = 32 (per-pair traceback, block cuts, waves) and for G < 32 (unchanged, by digest); the rows-arena
index.  On the GPU: pairs past the old on-chip staging limit, long x long pairs, the traceback budget's block cuts and
waves, the over-budget refusal, and a 14-million-row x."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import threading

import numpy as np
import pytest

import sim_util
from parity_util import MODES, assert_same, oracle_batch
from rust_bio_b200 import synth

MIN = -858993459
F_TR, F_TC, F_CX, F_LUT, F_PK, F_RELU, F_PR, F_BND8, F_NOTB, F_YSTREAM = 1, 2, 4, 8, 16, 32, 128, 256, 512, 1024
CLIPS = {"custom": (-3, -7, 0, -9), "global": (MIN,) * 4, "semiglobal": (MIN,) * 4, "local": (MIN,) * 4}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plan_digests.json")

SIML_SRC = os.path.join(sim_util.HERE, "sim", "b2a_sim_long.cpp")
SIML_SO = os.path.join(sim_util.HERE, "sim", "libb2asim_long.so")
_siml = None


def siml_lib():
    """tests/sim/b2a_sim_long.cpp, built on first use"""
    global _siml
    if _siml is None:
        deps = [SIML_SRC, os.path.join(sim_util.HERE, "sim", "b2a_sim.cpp")] + sim_util.DEPS
        if not os.path.exists(SIML_SO) or any(os.path.getmtime(d) > os.path.getmtime(SIML_SO) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                                   "-o", SIML_SO, SIML_SRC])
        _siml = C.CDLL(SIML_SO)
        _siml.siml_align.restype = C.c_int
        _siml.siml_fill_flags.restype = C.c_int
        _siml.siml_plan_bytes.restype = C.c_uint64
        _siml.siml_rows_index.restype = C.c_uint64
    return _siml


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------ plan helpers

def plan_of(xl, yl, G, R, budget, flags=0):
    """-> (blocks: array [nb, 8] of first, npairs, maxm, maxn, nstrips, K, tb_off, strip_task_base;
           waves: array [nw, 3] of block_lo, block_hi, tb_bytes; total_tb; max_tb)"""
    xl = np.ascontiguousarray(xl, np.uint32)
    yl = np.ascontiguousarray(yl, np.uint32)
    n = len(xl)
    cap = n + 1
    blocks = np.zeros((cap, 8), np.uint64)
    waves = np.zeros((cap, 3), np.uint64)
    sc = np.zeros(4, np.uint64)
    siml_lib().siml_plan(_p(xl), _p(yl), C.c_uint64(n), int(G), int(R), C.c_uint64(budget), int(flags), _p(blocks),
                         C.c_uint64(cap), _p(waves), C.c_uint64(cap), _p(sc))
    return blocks[:int(sc[0])], waves[:int(sc[1])], int(sc[2]), int(sc[3])


def plan_digest(xl, yl, G, R, budget, flags=0):
    """SHA-256 of every field of the plan (siml_plan_bytes)"""
    xl = np.ascontiguousarray(xl, np.uint32)
    yl = np.ascontiguousarray(yl, np.uint32)
    L = siml_lib()
    nbytes = L.siml_plan_bytes(_p(xl), _p(yl), C.c_uint64(len(xl)), int(G), int(R), C.c_uint64(budget), int(flags),
                               None, C.c_uint64(0))
    buf = np.zeros(int(nbytes), np.uint8)
    L.siml_plan_bytes(_p(xl), _p(yl), C.c_uint64(len(xl)), int(G), int(R), C.c_uint64(budget), int(flags), _p(buf),
                      C.c_uint64(nbytes))
    return hashlib.sha256(buf.tobytes()).hexdigest()


def _lcg_lengths(seed, n, lo, hi):
    """deterministic lengths in [lo, hi] that do not depend on numpy's generators"""
    out, v = [], seed * 2654435761 % (1 << 32)
    for _ in range(n):
        v = (v * 1103515245 + 12345) % (1 << 31)
        out.append(lo + v % (hi - lo + 1))
    return np.array(out, np.uint32)


def plan_cases():
    """Batches of the shapes with fewer than 32 lanes per pair: uniform and ragged, reads and long pairs, lengths
    0-2, generous and tight budgets (several waves), full and score-only flags."""
    cases = []
    inputs = {
        "reads150": (np.full(1000, 150, np.uint32), np.full(1000, 150, np.uint32)),
        "ragged": (_lcg_lengths(1, 777, 0, 300), _lcg_lengths(2, 777, 0, 250)),
        "tiny": (_lcg_lengths(3, 70, 0, 2), _lcg_lengths(4, 70, 0, 2)),
        "long": (_lcg_lengths(5, 100, 1000, 5000), _lcg_lengths(6, 100, 1000, 5000)),
        "c5like": (np.full(200, 10000, np.uint32), np.full(200, 10000, np.uint32)),
    }
    for name, (xl, yl) in inputs.items():
        for G, R in ((1, 16), (1, 8), (2, 16), (4, 16), (8, 16), (8, 20), (8, 8)):
            for budget in ((1 << 62), 1 << 22):
                for flags in (0, F_BND8, F_NOTB):
                    cases.append((f"{name}-{G}x{R}-{budget}-{flags}", xl, yl, G, R, budget, flags))
    return cases


# ------------------------------------------------------------------------------------------------ host: plan

def test_plans_below_32_lanes_unchanged():
    """Plans with fewer than 32 lanes per pair are what they were before the warp-per-pair block cut, field by field."""
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = plan_cases()
    assert len(want) == len(cases)
    for name, xl, yl, G, R, budget, flags in cases:
        assert plan_digest(xl, yl, G, R, budget, flags) == want[name], name


def _task_tb(m, n, G, R):
    """traceback bytes of one warp-task over every strip (b2a_plan.h)"""
    nstrips = (m - 1 + G * R - 1) // (G * R) if m >= 2 else 0
    K = (n + G - 1 + 7) // 8 if n else 0
    return nstrips * K * ((R + 3) // 4) * 512


def _assert_cover(blocks, n):
    """first / npairs cover the sorted pairs 0..n-1 exactly once, in order"""
    nxt = 0
    for b in blocks:
        assert int(b[0]) == nxt and 1 <= int(b[1]) <= 32
        nxt += int(b[1])
    assert nxt == n


@pytest.mark.parametrize("R", [8, 16])
def test_plan_warp_per_pair_traceback_per_pair(R):
    """G = 32: a block's traceback is its real pairs' (blocks of 32 and a last one of 8 pairs, not 32 pairs' worth)."""
    for xl, yl in ((np.full(40, 3000, np.uint32), np.full(40, 2000, np.uint32)),
                   (_lcg_lengths(7, 71, 0, 3000), _lcg_lengths(8, 71, 0, 5000))):
        blocks, waves, total, _ = plan_of(xl, yl, 32, R, 1 << 62)
        _assert_cover(blocks, len(xl))
        assert [int(b[1]) for b in blocks] == [32] * (len(xl) // 32) + ([len(xl) % 32] if len(xl) % 32 else [])
        want = sum(int(b[1]) * _task_tb(int(b[2]), int(b[3]), 32, R) for b in blocks)
        assert total == want
        if len(set(xl.tolist())) == 1:  # uniform: the sum over the pairs themselves
            assert total == sum(_task_tb(int(m), int(n), 32, R) for m, n in zip(xl, yl))
        assert len(waves) == 1
        # the strip tasks of a block are its pairs' (pair, strip) tasks
        for b in blocks:
            nb = int(b[1]) * int(b[4])
            assert int(b[7]) + nb <= sum(int(c[1]) * int(c[4]) for c in blocks)
        # score-only: no traceback, blocks of 32 as before
        sblocks, _, stotal, _ = plan_of(xl, yl, 32, R, 1 << 62, F_NOTB)
        assert stotal == 0 and [int(b[1]) for b in sblocks] == [int(b[1]) for b in blocks]


@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_plan_warp_per_pair_blocks_cut_to_the_budget(k):
    """A budget that fits k long pairs' traceback: blocks of at most k pairs, each wave within the budget and closed
    between pairs; first / npairs cover every sorted pair once."""
    n = 40
    xl = np.full(n, 30000, np.uint32)
    yl = np.full(n, 40000, np.uint32)
    one = _task_tb(30000, 40000, 32, 16)
    budget = k * one + one // 2
    blocks, waves, total, max_tb = plan_of(xl, yl, 32, 16, budget)
    _assert_cover(blocks, n)
    assert all(int(b[1]) <= k for b in blocks) and int(blocks[0][1]) == k
    assert len(waves) == len(blocks) and len(waves) > 1  # k pairs' worth per wave: one block each
    assert max_tb <= budget and total == n * one
    lo = 0
    for w in waves:
        assert int(w[0]) == lo and int(w[2]) <= budget
        lo = int(w[1])
    assert lo == len(blocks)
    # ragged lengths: a block's traceback (its pairs times the block maxima) stays within the budget
    xl = _lcg_lengths(9, 60, 1000, 30000)
    yl = _lcg_lengths(10, 60, 1000, 40000)
    blocks, waves, _, max_tb = plan_of(xl, yl, 32, 8, budget)
    _assert_cover(blocks, 60)
    for b in blocks:
        assert int(b[1]) == 1 or int(b[1]) * _task_tb(int(b[2]), int(b[3]), 32, 8) <= budget
    assert max_tb <= budget


def test_plan_over_budget_single_pair():
    """A pair whose traceback alone is above the budget keeps a block and a wave of its own, and the plan shows it
    (max_tb > budget: the engine refuses the batch before allocating)."""
    xl = np.array([200000, 100, 100], np.uint32)
    yl = np.array([200000, 100, 100], np.uint32)
    one = _task_tb(200000, 200000, 32, 16)
    blocks, waves, _, max_tb = plan_of(xl, yl, 32, 16, one - 1)
    _assert_cover(blocks, 3)
    assert int(blocks[0][1]) == 1 and max_tb == one > one - 1
    blocks, waves, _, max_tb = plan_of(xl, yl, 32, 16, one)  # exactly fits: one wave for it, one for the rest
    assert max_tb == one and int(blocks[0][1]) == 1 and len(waves) == 2


def test_same_long_pair_twice_two_waves():
    xl = np.full(2, 200000, np.uint32)
    one = _task_tb(200000, 200000, 32, 16)
    blocks, waves, total, max_tb = plan_of(xl, xl, 32, 16, one + one // 2)
    assert [int(b[1]) for b in blocks] == [1, 1] and len(waves) == 2 and max_tb == one and total == 2 * one


def test_rows_index_is_64_bit():
    """Rows-arena offsets at m = 2^24 - 1 (the longest x the engine takes) do not wrap: the helper the fill and K2
    index with, against exact integer arithmetic."""
    L = siml_lib()
    m = (1 << 24) - 1
    for G, R in ((32, 16), (32, 8), (8, 20), (1, 16)):
        nstrips = (m - 1 + G * R - 1) // (G * R)
        rows_pad = nstrips * G * R + 2
        for arr in range(5):
            for row in (1, m - 1, rows_pad - 1):
                for pi in (0, 31):
                    want = (arr * rows_pad + row) * 32 + pi
                    assert int(L.siml_rows_index(arr, C.c_int32(rows_pad), C.c_int32(row), C.c_int32(pi))) == want
        assert (4 * rows_pad + m - 1) * 32 + 31 >= 1 << 31  # (the offsets that wrap in signed 32 bits)


# ------------------------------------------------------------------------------------------------ host: the fill

def siml_run(mode, orc_scoring, batch, R, score_only, warp_walk, poison):
    s = sim_util.SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob, x_off, x_len, y_off, y_len = [np.ascontiguousarray(a) for a in batch]
    n = len(x_len)
    cap = x_len.astype(np.uint64) + y_len.astype(np.uint64) + np.uint64(4)
    ops_off = np.concatenate([[0], np.cumsum(cap)]).astype(np.uint64)
    ops = np.zeros(int(ops_off[-1]) + 1, np.uint8)
    out = {k: np.zeros(n, np.uint32) for k in ("xstart", "xend", "ystart", "yend", "n_ops", "status")}
    out["score"] = np.zeros(n, np.int32)
    out["clip_len"] = np.zeros(4 * n, np.uint32)
    oob, loads = C.c_uint64(0), C.c_uint64(0)
    L = siml_lib()
    rc = L.siml_align(int(mode), C.byref(s), _p(blob), _p(x_off), _p(x_len), _p(y_off), _p(y_len), C.c_uint64(n),
                      int(R), int(score_only), int(warp_walk), 0x3C, int(poison), _p(out["score"]), _p(out["xstart"]),
                      _p(out["xend"]), _p(out["ystart"]), _p(out["yend"]), _p(out["n_ops"]), _p(out["clip_len"]),
                      _p(out["status"]), _p(ops), _p(ops_off), C.byref(oob), C.byref(loads))
    assert rc == 0, rc
    oplists = None
    if not score_only:
        oplists = [sim_util.decode_ops(ops[int(ops_off[i]):int(ops_off[i]) + int(out["n_ops"][i])],
                                       out["clip_len"][4 * i:4 * i + 4]) for i in range(n)]
    return out, oplists, oob.value, loads.value, L.siml_fill_flags()


# y lengths crossing word boundaries and the 31-column lane skew at both ends of a strip: short ones against x of 1-3
# strips (and m in {0, 1, 2}), long ones against x of 1-2 strips (the fill runs every pair of a block over the block's
# longest y, so the two sets are batches of their own)
NS_SHORT = [1, 2, 3, 4, 5, 31, 32, 33]
NS_LONG = [4095, 4097, 2500]


def long_batches(seed, R, alphabet):
    """-> [short-y batch, long-y batch], related and unrelated pairs"""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(alphabet, np.uint8)
    strip = 32 * R
    out = []
    for ns, ms in ((NS_SHORT, [2 * strip + 7, strip, 1, 2, strip + 1, 0, 3 * strip - 5, 40]),
                   (NS_LONG, [strip + 1, 5, strip - 1])):
        pairs = []
        for q, (n, m) in enumerate(zip(ns, ms)):
            x = alpha[rng.integers(0, len(alpha), m)]
            y = alpha[rng.integers(0, len(alpha), n)]
            if q % 2 and m > 4 and n > 4:  # a mutated copy of x inside y
                k = min(m, n)
                src = x[:k].copy()
                mut = rng.random(k) < 0.1
                src[mut] = alpha[rng.integers(0, len(alpha), int(mut.sum()))]
                off = (n - k) // 2
                y[off:off + k] = src
            pairs.append((bytes(x), bytes(y)))
        out.append(pack_pairs(pairs))
    return out


def _scoring(oracle, mode, table):
    if table is None:
        return oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    go = {"local": -10, "global": -5, "semiglobal": -11, "custom": -8}[mode]
    return oracle.make_scoring(go, -1, 0, 0, table, *CLIPS[mode])


@pytest.mark.parametrize("alphabet", ["dna", "blosum62"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("R", [8, 16])
def test_sim_streamed_y_fill_vs_oracle(oracle, R, mode, alphabet):
    """The 32xR strip-pipelined fill with y streamed from the arena, full (both walk forms) and score-only, against the
    oracle; with the arena around each pair's y poisoned the results do not change, and no y load leaves the pair's
    own words."""
    from rust_bio_b200 import scores
    table = scores.matrix_table256("blosum62") if alphabet == "blosum62" else None
    for bi, batch in enumerate(long_batches(100 + R + len(mode), R, synth.PROTEIN if table is not None else synth.DNA)):
        s, _ = _scoring(oracle, mode, table)
        ref, ref_ops = oracle_batch(oracle, mode, s, batch)
        walk = (len(mode) + R + bi) % 2  # one walk form on the plain arena, the other on the poisoned one
        got, ops, oob, loads, flags = siml_run(MODES[mode], s, batch, R, 0, walk, -1)
        assert flags & F_LUT and flags & F_YSTREAM and loads > 0 and oob == 0, (flags, loads, oob)
        assert_same(got, ops, ref, ref_ops, batch, f"{mode} 32x{R} {alphabet}")
        got2, ops2, oob, _, _ = siml_run(MODES[mode], s, batch, R, 0, 1 - walk, 0xA5)
        assert oob == 0
        assert_same(got2, ops2, ref, ref_ops, batch, f"{mode} 32x{R} {alphabet} poisoned, other walk")
        sc, _, oob, _, flags = siml_run(MODES[mode], s, batch, R, 1, walk, 0x5A)
        assert flags & F_NOTB and oob == 0
        for f in ("score", "xend", "yend"):
            assert np.array_equal(sc[f].astype(np.int64), np.asarray(ref[f]).astype(np.int64)), f
        assert not np.any(sc["status"])


# ------------------------------------------------------------------------------------------------ GPU

@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _c_scoring(go, ge, ma, mi, clips=(MIN,) * 4, table=None):
    from rust_bio_b200._lib import CScoring
    cs = CScoring(go, ge, clips[0], clips[1], clips[2], clips[3], ma, mi, 0, None, None, 0)
    keep = None
    if table is not None:
        keep = np.ascontiguousarray(table, dtype=np.int32)
        cs.table = keep.ctypes.data_as(C.c_void_p)
    return cs, keep


def _full(eng, mode, cs, batch):
    res = eng.align_batch(MODES[mode], cs, batch)
    return res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)]


def _assert_scores_equal_full(sc, got, what):
    for f in ("score", "xend", "yend"):
        assert np.array_equal(np.asarray(sc[f]).astype(np.int64), np.asarray(got[f]).astype(np.int64)), (what, f)
    assert not np.any(sc["status"]), what


def _related(rng, m, n, alphabet, rate=0.08):
    """x, and y holding a mutated copy of x's first min(m, n) symbols in the middle"""
    alpha = np.frombuffer(alphabet, np.uint8)
    x = alpha[rng.integers(0, len(alpha), m)]
    y = alpha[rng.integers(0, len(alpha), n)]
    k = min(m, n)
    src = x[:k].copy()
    mut = rng.random(k) < rate
    src[mut] = alpha[rng.integers(0, len(alpha), int(mut.sum()))]
    off = (n - k) // 2
    y[off:off + k] = src
    return bytes(x), bytes(y)


def _gpu_scoring(oracle, mode, table):
    go = -5 if table is None else {"local": -10, "global": -5, "semiglobal": -11, "custom": -8}[mode]
    ma, mi = (1, -1) if table is None else (0, 0)
    s, _ = oracle.make_scoring(go, -1, ma, mi, table, *CLIPS[mode])
    cs, keep = _c_scoring(go, -1, ma, mi, CLIPS[mode], table)
    return s, cs, keep


@pytest.mark.gpu
@pytest.mark.parametrize("alphabet", ["dna", "blosum62"])
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_past_the_old_staging_limit(eng, oracle, mode, alphabet):
    """16 pairs of 300 x 120,000 and 16 of 120,000 x 300 (y far past the ~50,000 symbols whole-y staging allowed):
    every field and the ops against the oracle, score-only against full, with the automatic shape and with 32x8 and
    32x16 forced."""
    from rust_bio_b200 import scores
    from rust_bio_b200.engine import pack_pairs
    table = scores.matrix_table256("blosum62") if alphabet == "blosum62" else None
    rng = np.random.default_rng(len(mode) * 7 + len(alphabet))
    ab = synth.PROTEIN if table is not None else synth.DNA
    pairs = [_related(rng, 300, 120000, ab) for _ in range(16)]
    pairs += [tuple(reversed(_related(rng, 300, 120000, ab))) for _ in range(16)]
    batch = pack_pairs(pairs)
    s, cs, keep = _gpu_scoring(oracle, mode, table)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
    for shape in (None, (32, 8), (32, 16)):
        if shape:
            eng.set_tuning(*shape)
        try:
            got, ops = _full(eng, mode, cs, batch)
            assert eng.stats.fill_lanes_per_pair == 32
            assert_same(got, ops, ref, ref_ops, batch, f"{mode} {alphabet} shape={shape}")
            sc = eng.align_batch_scores(MODES[mode], cs, batch)
            _assert_scores_equal_full(sc, got, f"{mode} {alphabet} shape={shape} score-only")
        finally:
            eng.set_tuning(0, 0)


def _oracle_threads(oracle, mode, s, batch, parts):
    """the oracle on `parts` slices of the batch at once, one thread each (its u16 traceback is m*n*2 bytes a pair)"""
    blob, xo, xl, yo, yl = batch
    out = [None] * len(parts)

    def work(k, idx):
        sub = (blob, xo[idx].copy(), xl[idx].copy(), yo[idx].copy(), yl[idx].copy())
        out[k] = oracle_batch(oracle, mode, s, sub, threads=1)

    th = [threading.Thread(target=work, args=(k, np.asarray(idx))) for k, idx in enumerate(parts)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["local", "global"])
def test_gpu_long_by_long(eng, oracle, mode):
    """2 pairs of 56,000 x 56,000 against the oracle (each pair's oracle on a thread of its own)."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(56 + len(mode))
    batch = pack_pairs([_related(rng, 56000, 56000, synth.DNA), _related(rng, 56000, 56000, synth.DNA, 0.2)])
    s, cs, keep = _gpu_scoring(oracle, mode, None)
    got, ops = _full(eng, mode, cs, batch)
    for k, (ref, ref_ops) in enumerate(_oracle_threads(oracle, mode, s, batch, [[0], [1]])):
        one = {f: np.asarray(v)[[k]] for f, v in got.items() if len(np.asarray(v)) == 2}
        sub = tuple(a if i == 0 else np.asarray(a)[[k]] for i, a in enumerate(batch))
        assert_same(one, [ops[k]], ref, ref_ops, sub, f"{mode} 56k pair {k}")
    _assert_scores_equal_full(eng.align_batch_scores(MODES[mode], cs, batch), got, f"{mode} 56k score-only")


@pytest.mark.gpu
def test_gpu_200k_single_pair(eng, oracle):
    """1 pair of 200,000 x 200,000 global (no oracle: its u16 traceback would be 80 GB): the path rescores to the
    score and consumes exactly m and n; score-only equals full; the same pair twice under a budget that fits one
    pair's traceback runs 2 waves and gives the same result twice."""
    from parity_util import rescore_path
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(200)
    x, y = _related(rng, 200000, 200000, synth.DNA)
    batch = pack_pairs([(x, y)])
    s, cs, keep = _gpu_scoring(oracle, "global", None)
    got, ops = _full(eng, "global", cs, batch)
    assert eng.stats.fill_lanes_per_pair == 32  # (a pair the reference panics on would fail the call)
    f = {k: int(got[k][0]) for k in ("xstart", "xend", "ystart", "yend")}
    assert (f["xstart"], f["xend"], f["ystart"], f["yend"]) == (0, 200000, 0, 200000)
    # Match / Subst / Del(3) move in x, Match / Subst / Ins(2) in y: the ops consume exactly m and n
    assert sum(1 for c, _ in ops[0] if c in (0, 1, 3)) == 200000 and sum(1 for c, _ in ops[0] if c in (0, 1, 2)) == 200000
    assert rescore_path(x, y, ops[0], f, "global", -5, -1, lambda a, b: 1 if a == b else -1, (MIN,) * 4) == \
        int(got["score"][0])
    tb_one = int(eng.stats.traceback_bytes)
    _assert_scores_equal_full(eng.align_batch_scores(MODES["global"], cs, batch), got, "200k score-only")
    twice = pack_pairs([(x, y), (x, y)])
    eng.set_traceback_budget(tb_one + tb_one // 2)
    try:
        got2, ops2 = _full(eng, "global", cs, twice)
        assert eng.stats.waves == 2
    finally:
        eng.set_traceback_budget(0)
    for k in range(2):
        for fld in ("score", "xstart", "xend", "ystart", "yend"):
            assert int(got2[fld][k]) == int(got[fld][0]), (k, fld)
        assert ops2[k] == ops[0]


@pytest.mark.gpu
def test_gpu_budget_cuts_blocks_and_waves(eng, oracle):
    """40 pairs of 30,000 x 40,000 under a budget of about 8 pairs' traceback: more than one wave (blocks of fewer
    than 32 pairs), results identical to the default budget, and 2 pairs against the oracle."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(3040)
    batch = pack_pairs([_related(rng, 30000, 40000, synth.DNA, 0.05 + 0.01 * (q % 5)) for q in range(40)])
    s, cs, keep = _gpu_scoring(oracle, "semiglobal", None)
    base, base_ops = _full(eng, "semiglobal", cs, batch)
    one = int(eng.stats.traceback_bytes) // 40
    eng.set_traceback_budget(8 * one + one // 2)
    try:
        got, ops = _full(eng, "semiglobal", cs, batch)
        assert eng.stats.waves == 5, eng.stats.waves  # blocks of 8 pairs, a wave each
    finally:
        eng.set_traceback_budget(0)
    for fld in base:
        assert np.array_equal(np.asarray(got[fld]), np.asarray(base[fld])), fld
    assert ops == base_ops
    idx = [3, 38]
    sub = tuple(a if i == 0 else np.asarray(a)[idx] for i, a in enumerate(batch))
    ref, ref_ops = oracle_batch(oracle, "semiglobal", s, sub, threads=2)
    assert_same({f: np.asarray(v)[idx] for f, v in got.items() if len(np.asarray(v)) == 40}, [ops[i] for i in idx],
                ref, ref_ops, sub, "oracle sample")


@pytest.mark.gpu
def test_gpu_over_budget_pair_is_refused(eng, oracle):
    """A pair whose traceback is above set_traceback_budget: B2A_E_UNSUPPORTED naming the bytes, the budget and the
    score-only form, before anything runs; the same batch succeeds score-only."""
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(5)
    batch = pack_pairs([_related(rng, 20000, 20000, synth.DNA), _related(rng, 300, 400, synth.DNA)])
    s, cs, keep = _gpu_scoring(oracle, "local", None)
    full, _ = _full(eng, "local", cs, batch)
    eng.set_traceback_budget(50 << 20)
    try:
        with pytest.raises(B2AError, match=r"UNSUPPORTED.*needs \d+ bytes.*budget of 52428800 bytes.*score-only"):
            eng.align_batch(MODES["local"], cs, batch)
        sc = eng.align_batch_scores(MODES["local"], cs, batch)
    finally:
        eng.set_traceback_budget(0)
    _assert_scores_equal_full(sc, full, "score-only under the budget")


@pytest.mark.gpu
def test_gpu_rows_arena_past_32_bit_offsets(eng, oracle):
    """1 pair of 14,000,000 x 64 local (rows-arena offsets past 2^31), full and score-only, against the oracle."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(14)
    y, x = _related(rng, 64, 14000000, synth.DNA, 0.05)
    batch = pack_pairs([(x, y)])
    s, cs, keep = _gpu_scoring(oracle, "local", None)
    ref, ref_ops = oracle_batch(oracle, "local", s, batch, threads=1)
    got, ops = _full(eng, "local", cs, batch)
    assert eng.stats.fill_lanes_per_pair == 32
    assert_same(got, ops, ref, ref_ops, batch, "14M x 64 local")
    _assert_scores_equal_full(eng.align_batch_scores(MODES["local"], cs, batch), got, "14M x 64 score-only")
