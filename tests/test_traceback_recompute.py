"""Recomputed traceback: a warp-per-pair pair whose traceback is above the traceback budget is aligned, with
b2a_engine_set_traceback_recompute(e, 1), by one score-only fill that checkpoints the strip boundary at the end of every
window of W = floor(budget / strip bytes) strips, and a refill of each window the walk enters (DESIGN.md §2).

On the host: the window arithmetic (W, the window count, the checkpoint bytes, the refusal below one strip) against the
plan of tests/sim/b2a_sim_long.cpp; and tests/sim/b2a_sim_recompute.cpp, the kernels' source compiled for the host,
running the whole recompute path (pass 1 with checkpoints, K2's finish, the windowed walk and the refills) on 32x8 and
32x16 with windows of 1, 2 and 3 strips against the oracle and the sim's full path, every mode, DNA and BLOSUM62, random
custom clips, windows the walk skips, and the rows arena, row-m cells and boundary row compared byte for byte around
every refill.  On the GPU: every mode at 20,000 x 20,000 DNA and local / global at 12,000 x 12,000
BLOSUM62 against the oracle under budgets of 3 to 8 windows; 100,000 x 100,000 under two window splits against each
other and the default budget; a mixed batch; the staged and compact forms; windows the walk never enters; the refusal
below one strip; and one 330,000 x 330,000 pair above the default budget."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import sim_util
from parity_util import MODES, assert_same, oracle_batch
from rust_bio_b200 import synth
from test_long_pairs import _gpu_scoring, _oracle_threads, _related, _scoring, plan_of, siml_run

MIN = -858993459


# ------------------------------------------------------------------------------------------------ window arithmetic

def shape_r(m):
    """R of the warp-per-pair shape the engine picks for a pair with m rows (b2a_engine.cu choose_shape)"""
    rows = max(m - 1, 1)
    pad16, pad8 = (rows + 511) // 512 * 512, (rows + 255) // 256 * 256
    return 16 if pad16 * 100 <= pad8 * 112 else 8


def strip_bytes(n, R):
    """traceback bytes of one strip of a warp-per-pair pair: K * TBW * 512, K = ceil((n + 31) / 8)"""
    return (n + 32 - 1 + 7) // 8 * ((R + 3) // 4) * 512


def windows_of(m, n, budget):
    """-> (W, windows, checkpoint bytes) of a recomputed pair, or None when the budget is below one strip"""
    R = shape_r(m)
    nstrips = (m - 1 + 32 * R - 1) // (32 * R)
    sb = strip_bytes(n, R)
    if budget < sb:
        return None
    W = min(budget // sb, nstrips)
    nw = (nstrips + W - 1) // W
    return W, nw, (nw - 1) * (n + 1) * 16


@pytest.mark.parametrize("m,n", [(20000, 20000), (12000, 12000), (100000, 100000), (330000, 330000), (5000, 70000)])
def test_window_arithmetic_matches_the_plan(m, n):
    """The strip bytes are what the plan gives a one-pair block per strip, and a budget of W strips (plus a little)
    gives W-strip windows that cover every strip once."""
    R = shape_r(m)
    blocks, waves, total_tb, max_tb = plan_of([m], [n], 32, R, 1 << 62)
    nstrips, K = int(blocks[0][4]), int(blocks[0][5])
    sb = strip_bytes(n, R)
    assert K * ((R + 3) // 4) * 512 == sb
    assert max_tb == nstrips * sb
    for W in (1, 2, 3, max(1, nstrips // 4), nstrips - 1):
        got = windows_of(m, n, W * sb + sb // 2)
        assert got is not None and got[0] == W
        nw = got[1]
        assert (nw - 1) * W < nstrips <= nw * W
        assert got[2] == (nw - 1) * (n + 1) * 16
    assert windows_of(m, n, sb - 1) is None
    assert windows_of(m, n, sb)[0] == 1


# ------------------------------------------------------------------------------------------------ host simulation

SIMR_SRC = os.path.join(sim_util.HERE, "sim", "b2a_sim_recompute.cpp")
SIMR_SO = os.path.join(sim_util.HERE, "sim", "libb2asim_recompute.so")
_simr = None


def simr_lib():
    """tests/sim/b2a_sim_recompute.cpp, built on first use"""
    global _simr
    if _simr is None:
        deps = [SIMR_SRC] + [os.path.join(sim_util.HERE, "sim", f) for f in ("b2a_sim_long.cpp", "b2a_sim.cpp")]
        deps += sim_util.DEPS
        if not os.path.exists(SIMR_SO) or any(os.path.getmtime(d) > os.path.getmtime(SIMR_SO) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                                   "-o", SIMR_SO, SIMR_SRC])
        _simr = C.CDLL(SIMR_SO)
        _simr.simr_align.restype = C.c_int
    return _simr


def simr_run(mode, orc_scoring, x, y, R, win):
    """-> (fields of the one pair, its ops, windows, windows refilled, bytes a refill changed)"""
    s = sim_util.SimScoring.from_buffer_copy(bytes(orc_scoring))
    xa, ya = np.frombuffer(x, np.uint8).copy(), np.frombuffer(y, np.uint8).copy()
    out = {k: np.zeros(1, np.uint32) for k in ("xstart", "xend", "ystart", "yend", "n_ops", "status")}
    out["score"] = np.zeros(1, np.int32)
    out["clip_len"] = np.zeros(4, np.uint32)
    ops = np.zeros(len(x) + len(y) + 8, np.uint8)
    counts = np.zeros(4, np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = simr_lib().simr_align(int(mode), C.byref(s), p(xa), len(x), p(ya), len(y), int(R), int(win), p(out["score"]),
                               p(out["xstart"]), p(out["xend"]), p(out["ystart"]), p(out["yend"]), p(out["n_ops"]),
                               p(out["clip_len"]), p(out["status"]), p(ops), p(counts))
    assert rc == 0, rc
    oplist = sim_util.decode_ops(ops[:int(out["n_ops"][0])], out["clip_len"])
    return out, [oplist], int(counts[0]), int(counts[1]), int(counts[2])


def _check_pair(oracle, mode, s, x, y, R, wins, what):
    """the recompute sim under each W against the oracle and the sim's full path; no refill changes the rows arena,
    the row-m cells or the boundary row"""
    from rust_bio_b200.engine import pack_pairs
    batch = pack_pairs([(x, y)])
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=1)
    full, full_ops, _, _, _ = siml_run(MODES[mode], s, batch, R, 0, 1, -1)
    assert_same(full, full_ops, ref, ref_ops, batch, f"{what} full sim")
    res = []
    for W in wins:
        got, ops, nw, filled, clobbered = simr_run(MODES[mode], s, x, y, R, W)
        assert clobbered == 0, (what, W, clobbered)
        assert 1 <= filled <= nw or (filled == 0 and nw >= 1), (what, W, nw, filled)
        assert_same(got, ops, ref, ref_ops, batch, f"{what} W={W}")
        for f in ("score", "xstart", "xend", "ystart", "yend", "n_ops"):
            assert int(got[f][0]) == int(full[f][0]), (what, W, f)
        assert np.array_equal(got["clip_len"], full["clip_len"][:4]) and ops[0] == full_ops[0], (what, W)
        res.append((nw, filled))
    return res


def _sim_pairs(rng, R, alphabet):
    """x of 3, 5 and 7 strips (full and partial last strips), y lengths crossing 32-bit words; related pairs"""
    alpha = np.frombuffer(alphabet, np.uint8)
    GR = 32 * R
    out = []
    for m, n in ((3 * GR - 3, 97), (4 * GR + 2, 130), (7 * GR - 40, 61)):
        x = alpha[rng.integers(0, len(alpha), m)]
        y = alpha[rng.integers(0, len(alpha), n)]
        off = int(rng.integers(0, m - n))
        src = x[off:off + n].copy()
        mut = rng.random(n) < 0.15
        src[mut] = alpha[rng.integers(0, len(alpha), int(mut.sum()))]
        y[:] = src
        out.append((bytes(x), bytes(y)))
    return out


@pytest.mark.parametrize("alphabet", ["dna", "blosum62"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("R", [8, 16])
def test_sim_recompute_vs_oracle(oracle, R, mode, alphabet):
    """32xR, x of 3 to 7 strips, windows of 1, 2 and 3 strips: every field and the ops against the oracle and the
    sim's full path; the refills leave the rows arena, the row-m cells and the boundary row byte-identical."""
    from rust_bio_b200 import scores
    table = scores.matrix_table256("blosum62") if alphabet == "blosum62" else None
    rng = np.random.default_rng(300 + R + len(mode) + len(alphabet))
    s, _ = _scoring(oracle, mode, table)
    for k, (x, y) in enumerate(_sim_pairs(rng, R, synth.PROTEIN if table is not None else synth.DNA)):
        _check_pair(oracle, mode, s, x, y, R, (1, 2, 3), f"{mode} 32x{R} {alphabet} pair {k}")


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("R", [8, 16])
def test_sim_recompute_random_custom_clips(oracle, R, seed):
    """custom mode with random clip penalties (some dead), windows of 1, 2 and 3 strips, against the oracle"""
    rng = np.random.default_rng(400 + 10 * seed + R)
    for k, (x, y) in enumerate(_sim_pairs(rng, R, synth.DNA)):
        clips = [MIN if rng.random() < 0.25 else -int(rng.integers(0, 25)) for _ in range(4)]
        s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *clips)
        _check_pair(oracle, "custom", s, x, y, R, (1, 2, 3), f"custom {clips} 32x{R} seed {seed} pair {k}")


@pytest.mark.parametrize("R", [8, 16])
def test_sim_recompute_skipped_windows(oracle, R):
    """Windows the walk never enters are not refilled: a local hit in the bottom window refills exactly that one
    window; a custom x-suffix clip from row m up past several windows refills only the windows of the aligned part."""
    GR = 32 * R
    rng = np.random.default_rng(500 + R)
    alpha = np.frombuffer(synth.DNA, np.uint8)
    m = 6 * GR - 3  # 6 strips
    x = alpha[rng.integers(0, 4, m)]
    y = alpha[rng.integers(0, 4, 150)]
    y[20:120] = x[m - 140:m - 40]  # the hit: inside the last strip
    s, _ = _scoring(oracle, "local", None)
    (nw, filled), = _check_pair(oracle, "local", s, bytes(x), bytes(y), R, (1,), f"local bottom hit 32x{R}")
    assert nw == 6 and filled == 1, (nw, filled)
    # x's first strip matches y; the rest of x is random and clipped off by a cheap x-suffix clip
    y2 = x[:GR - 50].copy()
    s2, _ = oracle.make_scoring(-5, -1, 2, -3, None, MIN, -2, MIN, MIN)
    (nw, filled), = _check_pair(oracle, "custom", s2, bytes(x), bytes(y2), R, (1,), f"custom x-suffix jump 32x{R}")
    assert nw == 6 and filled == 1, (nw, filled)


# ------------------------------------------------------------------------------------------------ GPU

@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _run(eng, mode, cs, batch, budget=0, recompute=False):
    """-> (fields, ops, last_recompute) of b2a_align_batch under `budget` (0: the default)"""
    eng.set_traceback_budget(budget)
    eng.set_traceback_recompute(recompute)
    try:
        res = eng.align_batch(MODES[mode], cs, batch)
        rc = eng.last_recompute()
    finally:
        eng.set_traceback_budget(0)
        eng.set_traceback_recompute(False)
    d = res.as_dict()
    d["clip_len"] = res.clip_len.copy()
    return d, [res.ops_of(i) for i in range(res.n_pairs)], rc


def _assert_equal(a, a_ops, b, b_ops, what):
    for f in ("score", "xstart", "xend", "ystart", "yend"):
        assert np.array_equal(np.asarray(a[f]).astype(np.int64), np.asarray(b[f]).astype(np.int64)), (what, f)
    n = len(np.asarray(a["score"]))
    assert np.array_equal(a["clip_len"][:4 * n], b["clip_len"][:4 * n]), (what, "clip_len")
    assert a_ops == b_ops, (what, "ops")


def _budget(m, n, W):
    sb = strip_bytes(n, shape_r(m))
    return W * sb + sb // 3


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_recompute_vs_oracle_dna(eng, oracle, mode):
    """20,000 x 20,000 DNA (40 strips) under budgets of 13 and 7 strips: 4 and 6 windows; against the oracle and the
    default-budget path."""
    rng = np.random.default_rng(20 + len(mode))
    from rust_bio_b200.engine import pack_pairs
    batch = pack_pairs([_related(rng, 20000, 20000, synth.DNA, 0.1)])
    s, cs, keep = _gpu_scoring(oracle, mode, None)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=1)
    base, base_ops, rc0 = _run(eng, mode, cs, batch)
    assert rc0 == {"pairs": 0, "windows": 0, "windows_filled": 0}
    assert_same(base, base_ops, ref, ref_ops, batch, f"{mode} default budget")
    for W in (13, 7):
        got, ops, rc = _run(eng, mode, cs, batch, _budget(20000, 20000, W), True)
        assert rc["pairs"] == 1 and rc["windows"] == windows_of(20000, 20000, _budget(20000, 20000, W))[1], rc
        assert 1 <= rc["windows_filled"] <= rc["windows"]
        assert_same(got, ops, ref, ref_ops, batch, f"{mode} W={W}")
        _assert_equal(got, ops, base, base_ops, f"{mode} W={W} against the default budget")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["local", "global"])
def test_gpu_recompute_vs_oracle_blosum62(eng, oracle, mode):
    """12,000 x 12,000 BLOSUM62 (24 strips of 32x16) under budgets of 3 and 8 windows, against the oracle."""
    from rust_bio_b200 import scores
    from rust_bio_b200.engine import pack_pairs
    table = scores.matrix_table256("blosum62")
    rng = np.random.default_rng(12 + len(mode))
    batch = pack_pairs([_related(rng, 12000, 12000, synth.PROTEIN, 0.15)])
    s, cs, keep = _gpu_scoring(oracle, mode, table)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=1)
    nstrips = (12000 - 1 + 511) // 512
    for nw in (3, 8):
        W = (nstrips + nw - 1) // nw
        got, ops, rc = _run(eng, mode, cs, batch, _budget(12000, 12000, W), True)
        assert rc["pairs"] == 1 and rc["windows"] == (nstrips + W - 1) // W, rc
        assert_same(got, ops, ref, ref_ops, batch, f"{mode} blosum62 {nw} windows")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["global", "local"])
def test_gpu_recompute_100k(eng, oracle, mode):
    """100,000 x 100,000 under two budgets with different window splits (about 4 and 16 windows): both equal the
    default-budget path, field for field and op for op."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(100 + len(mode))
    batch = pack_pairs([_related(rng, 100000, 100000, synth.DNA, 0.1)])
    s, cs, keep = _gpu_scoring(oracle, mode, None)
    base, base_ops, _ = _run(eng, mode, cs, batch)
    nstrips = (100000 - 1 + 511) // 512
    for nw in (4, 16):
        W = (nstrips + nw - 1) // nw
        got, ops, rc = _run(eng, mode, cs, batch, _budget(100000, 100000, W), True)
        assert rc["pairs"] == 1 and rc["windows"] == (nstrips + W - 1) // W, rc
        _assert_equal(got, ops, base, base_ops, f"{mode} 100k, {rc}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_recompute_32x8_small_windows(eng, oracle, mode):
    """1,200 x 40,000 (the 32x8 shape, 5 strips) under budgets of 1, 2 and 3 strips, and one pair of each under a
    budget of 1 strip in one batch: against the oracle and the default budget."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(8 + len(mode))
    m, n = 1200, 40000
    assert shape_r(m) == 8
    pairs = [_related(rng, m, n, synth.DNA, 0.1), _related(rng, m, n - 13, synth.DNA, 0.2)]
    batch = pack_pairs(pairs)
    s, cs, keep = _gpu_scoring(oracle, mode, None)
    refs = _oracle_threads(oracle, mode, s, batch, [[0], [1]])
    base, base_ops, _ = _run(eng, mode, cs, batch)
    assert eng.stats.fill_rows_per_lane == 8
    for W in (1, 2, 3):
        got, ops, rc = _run(eng, mode, cs, batch, _budget(m, n, W), True)
        assert eng.stats.fill_rows_per_lane == 8
        assert rc["pairs"] == 2 and rc["windows"] == 2 * ((5 + W - 1) // W), rc
        _assert_equal(got, ops, base, base_ops, f"{mode} 32x8 W={W}")
        for k, (ref, ref_ops) in enumerate(refs):
            one = {f: np.asarray(v)[[k]] for f, v in got.items() if f != "clip_len"}
            sub = tuple(a if i == 0 else np.asarray(a)[[k]] for i, a in enumerate(batch))
            assert_same(one, [ops[k]], ref, ref_ops, sub, f"{mode} 32x8 W={W} pair {k}")


@pytest.mark.gpu
def test_gpu_recompute_skips_windows_the_walk_never_enters(eng, oracle):
    """A local pair whose only hit lies in the last rows: the walk ends inside the bottom window, so fewer windows are
    refilled than there are; the result equals the default budget's."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(7)
    alpha = np.frombuffer(synth.DNA, np.uint8)
    m, n = 20000, 3000
    x = alpha[rng.integers(0, 4, m)]
    y = alpha[rng.integers(0, 4, n)]
    y[1000:1400] = x[m - 500:m - 100]  # the hit: 400 rows near the bottom
    batch = pack_pairs([(bytes(x), bytes(y))])
    s, cs, keep = _gpu_scoring(oracle, "local", None)
    base, base_ops, _ = _run(eng, "local", cs, batch)
    got, ops, rc = _run(eng, "local", cs, batch, _budget(m, n, 4), True)
    assert rc["pairs"] == 1 and rc["windows"] == 10 and rc["windows_filled"] == 1, rc  # rows 19,500-19,900: window 9
    _assert_equal(got, ops, base, base_ops, "local hit in the bottom window")


@pytest.mark.gpu
def test_gpu_recompute_mixed_batch(eng, oracle):
    """One over-budget pair and 64 short reads in one batch: the default budget's results for every pair."""
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(65)
    pairs = [_related(rng, 20000, 20000, synth.DNA, 0.1)] + [_related(rng, 150, 150 + (q % 7), synth.DNA, 0.1)
                                                             for q in range(64)]
    batch = pack_pairs(pairs)
    s, cs, keep = _gpu_scoring(oracle, "semiglobal", None)
    base, base_ops, _ = _run(eng, "semiglobal", cs, batch)
    got, ops, rc = _run(eng, "semiglobal", cs, batch, _budget(20000, 20000, 9), True)
    assert rc["pairs"] == 1 and rc["windows"] == 5, rc
    _assert_equal(got, ops, base, base_ops, "mixed batch")


@pytest.mark.gpu
def test_gpu_recompute_staged_and_compact_forms(eng, oracle):
    """stage / run / fetch, and compact_fixed + gathered_fetch, on a batch with a recomputed pair: both equal the
    one-shot call."""
    import torch
    from rust_bio_b200.engine import Results, pack_pairs
    rng = np.random.default_rng(66)
    batch = pack_pairs([_related(rng, 16000, 18000, synth.DNA, 0.1), _related(rng, 300, 280, synth.DNA, 0.1)])
    s, cs, keep = _gpu_scoring(oracle, "custom", None)
    budget = _budget(16000, 18000, 6)
    want, want_ops, rc = _run(eng, "custom", cs, batch, budget, True)
    assert rc["pairs"] == 1
    eng.set_traceback_budget(budget)
    eng.set_traceback_recompute(True)
    try:
        eng.stage(MODES["custom"], cs, batch)
        eng.run()
        staged = Results(2, 1 << 20)
        eng.fetch(staged)
        d = staged.as_dict()
        d["clip_len"] = staged.clip_len.copy()
        _assert_equal(d, [staged.ops_of(i) for i in range(2)], want, want_ops, "stage / run / fetch")
        eng.stage(MODES["custom"], cs, batch)
        eng.run()
        seg = 1 << 20
        buf = torch.zeros(seg, dtype=torch.uint8, device="cuda")
        eng.compact_fixed(buf.data_ptr(), seg)
        torch.cuda.synchronize()
        got = Results(2, 1 << 20)
        n_got, _ = eng.gathered_fetch(buf.data_ptr(), seg, 1, got)
        assert n_got == 2
        d = got.as_dict()
        d["clip_len"] = got.clip_len.copy()
        _assert_equal(d, [got.ops_of(i) for i in range(2)], want, want_ops, "compact_fixed + gathered_fetch")
    finally:
        eng.set_traceback_budget(0)
        eng.set_traceback_recompute(False)


@pytest.mark.gpu
def test_gpu_recompute_refuses_below_one_strip(eng, oracle):
    """A budget below one strip's traceback of the pair is still B2A_E_UNSUPPORTED, with its own message."""
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(1)
    batch = pack_pairs([_related(rng, 20000, 20000, synth.DNA)])
    s, cs, keep = _gpu_scoring(oracle, "global", None)
    sb = strip_bytes(20000, shape_r(20000))
    with pytest.raises(B2AError, match=r"UNSUPPORTED.*one strip of this pair's traceback needs %d bytes" % sb):
        _run(eng, "global", cs, batch, sb - 1, True)


@pytest.mark.gpu
def test_gpu_recompute_above_the_default_budget(eng, oracle):
    """1 pair of 330,000 x 330,000 global, about 54 GB of traceback, above the default budget: with the knob on it is
    aligned; start and end are the corners, the ops consume exactly m and n, the path rescores to the score, and score,
    xend and yend equal the score-only call."""
    from parity_util import rescore_path
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(330)
    N = 330000
    x, y = _related(rng, N, N, synth.DNA, 0.1)
    batch = pack_pairs([(x, y)])
    s, cs, keep = _gpu_scoring(oracle, "global", None)
    got, ops, rc = _run(eng, "global", cs, batch, 0, True)
    assert rc["pairs"] == 1 and rc["windows"] >= 2, rc
    f = {k: int(got[k][0]) for k in ("xstart", "xend", "ystart", "yend")}
    assert (f["xstart"], f["xend"], f["ystart"], f["yend"]) == (0, N, 0, N)
    assert sum(1 for c, _ in ops[0] if c in (0, 1, 3)) == N and sum(1 for c, _ in ops[0] if c in (0, 1, 2)) == N
    assert rescore_path(x, y, ops[0], f, "global", -5, -1, lambda a, b: 1 if a == b else -1, (MIN,) * 4) == \
        int(got["score"][0])
    sc = eng.align_batch_scores(MODES["global"], cs, batch)
    for k in ("score", "xend", "yend"):
        assert int(sc[k][0]) == int(got[k][0]), k
