"""Tabulated scoring (a MatchFunc given as a 256 x 256 table) on every kernel path.

Every site that scores a cell reads the table as [x symbol][y symbol]: the host LUT build, K0's code map, the
shared-memory LUT of each fill shape, row m in K2 and in the fused finish, the banded column loops and strip fill, and
the BitEnc unpack (where the table is indexed by rank).  BLOSUM62 and MatchParams are symmetric, so a transposed lookup
scores the same there.  The tables here are not: they are asymmetric, hold a zero row, a negative match and a mismatch
above a match, and every entry of a byte outside the alphabet is huge, so that a transposed, shifted or out-of-alphabet
lookup changes the result or trips the range guard.  Every result is compared with the oracle, field by field and op
for op."""
import ctypes as C

import numpy as np
import pytest

import sim_util
from parity_util import MODES, assert_same, oracle_batch

MIN = -858993459
SHAPES = [(1, 16), (1, 8), (4, 16), (8, 16), (8, 20), (32, 8), (32, 16)]  # test_gpu_parity.SHAPES
OUTSIDE = 1 << 29  # every table entry of a byte outside the alphabet: above the 2^27 range guard
# symbols either side of the sign bit of a byte; 0 and 255 are covered by test_gpu_edge_bytes_as_symbols
ALPHA = bytes([0x41, 0x43, 0x47, 0x54, 0x7E, 0x7F, 0x80, 0xC1, 0xFE])
GO, GE = -5, -1
# every mode, and custom with live clips, dead x clips and dead y clips
CASES = [("local", (MIN,) * 4), ("global", (MIN,) * 4), ("semiglobal", (MIN,) * 4),
         ("custom", (-3, -4, -2, -5)), ("custom", (MIN, MIN, -1, 0)), ("custom", (0, -2, MIN, MIN))]
CASE_IDS = ["local", "global", "semiglobal", "custom_live", "custom_dead_x", "custom_dead_y"]
F_LUT, F_PACKTRK, F_PACKREL = 8, 16, 128  # b2a_common.cuh


# ---------------------------------------------------------------------------------------------------------------
# tables and batches

def asym_table(seed, alphabet):
    """256 x 256 int32 table over `alphabet` (at least 4 symbols): random asymmetric entries, a mismatch (a0 -> a1)
    scoring above every match while its transpose is a heavy penalty, a zero row (x symbol a[k/2]), a negative match
    (a[k-1]), and OUTSIDE on every entry that involves a byte outside the alphabet."""
    rng = np.random.default_rng(seed)
    idx = np.frombuffer(bytes(alphabet), dtype=np.uint8)
    k = len(idx)
    sub = rng.integers(-7, 4, (k, k))
    np.fill_diagonal(sub, rng.integers(2, 7, k))
    sub[0, 1], sub[1, 0] = 9, -8
    sub[k - 1, k - 1] = -3
    sub[k // 2, :] = 0
    t = np.full((256, 256), OUTSIDE, dtype=np.int32)
    t[np.ix_(idx, idx)] = sub
    assert not np.array_equal(sub, sub.T)
    assert sub[0, 1] > np.diag(sub).min() and np.diag(sub).min() < 0 and not np.any(sub[k // 2])
    return t


def flat_table(alphabet, v=2):
    """every entry over the alphabet equal (every cell of the matrix a tie), OUTSIDE elsewhere"""
    idx = np.frombuffer(bytes(alphabet), dtype=np.uint8)
    t = np.full((256, 256), OUTSIDE, dtype=np.int32)
    t[np.ix_(idx, idx)] = v
    return t


def mutate(rng, s, alpha, sub=0.1, indel=0.04):
    """s with substitutions, deletions and insertions (each insertion a random symbol before the source symbol)"""
    s = np.asarray(s, dtype=np.uint8)
    n = len(s)
    r = rng.random(n)
    s = np.where(rng.random(n) < sub, alpha[rng.integers(0, len(alpha), n)], s)
    extra = alpha[rng.integers(0, len(alpha), n)]
    keep = np.stack([(r >= indel / 2) & (r < indel), r >= indel / 2], axis=1).reshape(-1)
    return np.stack([extra, s], axis=1).reshape(-1)[keep]


def related_pairs(seed, n_pairs, max_len, alphabet):
    """every (m, n) with m, n in 0..2, then pairs of ragged lengths up to max_len: y a mutated copy of x, some with
    random flanks on y (or x), a few unrelated"""
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(bytes(alphabet), dtype=np.uint8)
    rnd = lambda n: alpha[rng.integers(0, len(alpha), n)]
    pairs = [(bytes(rnd(m)), bytes(rnd(n))) for m in range(3) for n in range(3)]
    for q in range(n_pairs):
        m = int(rng.integers(3, max_len + 1))
        x = rnd(m)
        if q % 7 == 6:
            y = rnd(int(rng.integers(1, max_len + 1)))
        else:
            y = mutate(rng, x, alpha)
            if q % 3 == 1:
                y = np.concatenate([rnd(int(rng.integers(0, 30))), y, rnd(int(rng.integers(0, 30)))])
            y = y[:max_len]
        if q % 5 == 4:
            x, y = y, x
        pairs.append((bytes(x), bytes(y)))
    return pairs


def pack(pairs, pad=None):
    """pack_pairs; with `pad` the bytes between sequences are set to that symbol, so that a batch whose alphabet the
    engine finds itself (the padding counts as present, b2a_scoring.alphabet) has no byte outside the table's
    alphabet"""
    from rust_bio_b200.engine import pack_pairs
    batch = pack_pairs(pairs)
    if pad is not None:
        blob, xo, xl, yo, yl = batch
        inside = np.zeros(len(blob), dtype=bool)
        for off, ln in ((xo, xl), (yo, yl)):
            for o, l in zip(off, ln):
                inside[int(o):int(o) + int(l)] = True
        blob[~inside] = pad
    return batch


def present_bytes(batch):
    blob, xo, xl, yo, yl = batch
    return np.unique(np.concatenate([blob[int(o):int(o) + int(l)] for off, ln in ((xo, xl), (yo, yl))
                                     for o, l in zip(off, ln)] + [np.zeros(0, np.uint8)]))


def select(batch, idx):
    return (batch[0],) + tuple(np.ascontiguousarray(a[idx]) for a in batch[1:])


def c_scoring(clips, table=None, alphabet=None, go=GO, ge=GE, ma=0, mi=0, has_ms=0):
    from rust_bio_b200._lib import CScoring
    cs = CScoring(go, ge, clips[0], clips[1], clips[2], clips[3], ma, mi, has_ms, None, None, 0)
    keep = []
    if table is not None:
        t = np.ascontiguousarray(table, dtype=np.int32).reshape(-1)
        keep.append(t)
        cs.table = t.ctypes.data_as(C.c_void_p)
    if alphabet is not None:
        a = np.frombuffer(bytes(alphabet), dtype=np.uint8).copy()
        keep.append(a)
        cs.alphabet = a.ctypes.data_as(C.c_void_p)
        cs.alphabet_len = len(a)
    return cs, keep


def oracle_ref(oracle, mode, clips, table, batch, go=GO, ge=GE, ma=0, mi=0):
    s, keep = oracle.make_scoring(go, ge, ma, mi, table, *clips)
    return oracle_batch(oracle, mode, s, batch, threads=8)


def banded_ref(oracle, mode, clips, table, k, w, batch, has_ms, go=GO, ge=GE, ma=2, mi=-3):
    s, keep = oracle.make_scoring(go, ge, ma, mi, table, *clips, has_match_scores=has_ms)
    ref, rops, roff, _, cells = oracle.banded_align_batch(mode, s, k, w, *batch, threads=8)
    assert not np.any(ref["n_ops"] == 0xFFFFFFFF), "a pair the reference panics on"
    ops = [[(int(v) & 7, int(v) >> 3) for v in rops[int(roff[p]):int(roff[p]) + int(ref["n_ops"][p])]]
           for p in range(len(ref))]
    return ref, ops, cells


def full(eng, mode, cs, batch):
    res = eng.align_batch(MODES[mode], cs, batch)
    return res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)]


def banded_full(eng, mode, cs, k, w, batch):
    res = eng.align_batch_banded(MODES[mode], cs, k, w, batch)
    return res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)]


def eight_lane_shape(batch):
    """(G, R) the engine picks for a batch of fewer than 49,152 pairs with m <= 161 (b2a_engine.cu choose_shape): 8
    lanes, 128- or 160-row strips, whichever pads m less"""
    rows = max(int(batch[2].max()) - 1, 1)
    assert int(batch[2].max()) <= 161 and len(batch[2]) < 49152
    return 8, (20 if -(-rows // 160) * 160 < -(-rows // 128) * 128 else 16)


def assert_scores(sc, ref, what):
    """a score-only result against the oracle (or a full result): score, xend, yend; no pair flagged"""
    n = len(ref["score"])
    for f in ("score", "xend", "yend"):
        assert np.array_equal(np.asarray(sc[f])[:n].astype(np.int64), np.asarray(ref[f]).astype(np.int64)), (what, f)
    assert not np.any(sc["status"]), what


def flags_of(mode, clips, table, alphabet, batch):
    """the fill flags the engine derives for this batch (b2a_engine.cu stage_front -> scoring_flags)"""
    from test_score_range import flags_of as score_range_flags, score_bound
    maxm, maxn = int(batch[2].max()), int(batch[4].max())
    return score_range_flags(mode, clips, score_bound(GO, GE, 0, 0, table, alphabet, maxm, maxn), maxm, maxn,
                             alpha=len(alphabet))


# ---------------------------------------------------------------------------------------------------------------
# the helpers themselves

def test_asym_table_properties():
    t = asym_table(1, ALPHA)
    idx = np.frombuffer(ALPHA, dtype=np.uint8)
    sub = t[np.ix_(idx, idx)].astype(np.int64)
    assert np.count_nonzero(sub != sub.T) >= len(idx)
    assert (t != OUTSIDE).sum() == len(idx) ** 2
    batch = pack(related_pairs(2, 20, 40, ALPHA), pad=ALPHA[0])
    assert set(np.unique(batch[0]).tolist()) <= set(ALPHA)
    assert np.array_equal(present_bytes(batch), np.unique(batch[0]))


# ---------------------------------------------------------------------------------------------------------------
# host simulation: the kernels' per-lane logic compiled for the CPU (tests/sim)

SIM_SHAPES = [(1, 16, 0), (1, 16, 1), (8, 8, 0), (8, 20, 1), (4, 16, 0), (32, 8, 0), (132, 8, 1)]


@pytest.mark.parametrize("G,R,walk", SIM_SHAPES, ids=[f"{g}x{r}_walk{w}" for g, r, w in SIM_SHAPES])
def test_sim_asymmetric_table_every_mode(oracle, G, R, walk):
    """G = 1 runs the fused finish, 132 x 8 the strip-pipelined warp-per-pair fill; walk 1 the warp walk"""
    table = asym_table(10 + G + R, ALPHA)
    batch = pack(related_pairs(G + R + walk, 30, 70, ALPHA), pad=ALPHA[0])
    for mode, clips in CASES:
        s, keep = oracle.make_scoring(GO, GE, 0, 0, table, *clips)
        ref, ref_ops = oracle_batch(oracle, mode, s, batch)
        got, ops = sim_util.align_batch(MODES[mode], s, *batch, R=R, G=G, warp_walk=walk)
        assert_same(got, ops, ref, ref_ops, batch, f"sim {G}x{R} walk={walk} {mode} {clips}")


def _window_pairs(seed, n_pairs, xlen, ylen, alphabet, sub=0.06, indel=0.02):
    """x: a mutated window of y (lengths ragged around xlen / ylen)"""
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(bytes(alphabet), dtype=np.uint8)
    pairs = []
    for _ in range(n_pairs):
        n = int(rng.integers(ylen // 2, ylen + 1))
        y = alpha[rng.integers(0, len(alpha), n)]
        m = int(rng.integers(xlen // 2, xlen + 1))
        st = int(rng.integers(0, max(1, n - m)))
        pairs.append((bytes(mutate(rng, y[st:st + m], alpha, sub, indel)), bytes(y)))
    return pairs


BANDED_CASES = CASES[:5]


@pytest.mark.parametrize("has_ms", [0, 1])
def test_sim_banded_asymmetric_table(oracle, has_ms):
    """K4 + K3 of b2a_banded.cuh on the host (column loops), the W = 32 warp form and warp-tasks of the strip fill"""
    table = asym_table(20 + has_ms, ALPHA)
    pairs = _window_pairs(30 + has_ms, 16, 80, 200, ALPHA)
    batch = pack(pairs)
    k, w = 6, 7
    alpha = np.frombuffer(ALPHA, dtype=np.uint8).copy()
    strip_ran = 0
    for mode, clips in BANDED_CASES:
        s, keep = oracle.make_scoring(GO, GE, 2, -3, table, *clips, has_match_scores=has_ms)
        s.alphabet, s.alphabet_len = alpha.ctypes.data_as(C.c_void_p), len(alpha)  # (pack_pairs pads with 0)
        ref, ref_ops, cells = banded_ref(oracle, mode, clips, table, k, w, batch, has_ms)
        got, ops, _ = sim_util.banded_batch(MODES[mode], s, k, w, *batch)
        assert not np.any(got["status"])
        assert int(got["num_cells"].sum()) == cells
        assert_same(got, ops, ref, ref_ops, batch, f"sim banded {mode} {clips} has_ms={has_ms}")
        for p in range(0, len(pairs), 4):
            one = sim_util.banded_warp32_one(MODES[mode], s, k, w, *pairs[p])
            assert one is not None
            assert one[0] == {f: int(ref[f][p]) for f in one[0]} and one[1] == ref_ops[p], (mode, clips, p)
        for lo in range(0, len(pairs), 4):
            for q, r in enumerate(sim_util.banded_strip_task(MODES[mode], s, k, w, pairs[lo:lo + 4])):
                if r is None:
                    continue
                strip_ran += 1
                p = lo + q
                assert r[0] == {f: int(ref[f][p]) for f in r[0]} and r[1] == ref_ops[p], (mode, clips, p, "strip")
    assert strip_ran >= len(pairs)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the full aligner

@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def main_case(oracle):
    """300 related ragged pairs (m <= 150: the automatic shape has 8 lanes per pair), padded with an alphabet symbol,
    the asymmetric table and the oracle's answer for every CASES entry"""
    table = asym_table(7, ALPHA)
    batch = pack(related_pairs(7, 300, 150, ALPHA), pad=ALPHA[0])
    refs = {(mode, clips): oracle_ref(oracle, mode, clips, table, batch) for mode, clips in CASES}
    return table, batch, refs


@pytest.mark.gpu
@pytest.mark.parametrize("G,R", [(0, 0)] + SHAPES, ids=["auto"] + [f"{g}x{r}" for g, r in SHAPES])
def test_gpu_every_shape_mode_and_walk(eng, main_case, G, R):
    table, batch, refs = main_case
    shape = (G, R) if G else eight_lane_shape(batch)
    try:
        eng.set_tuning(G, R)
        for walk in (1, 2):
            eng.set_walk(walk)
            for mode, clips in CASES:
                cs, keep = c_scoring(clips, table, ALPHA)
                got, ops = full(eng, mode, cs, batch)
                assert (eng.stats.fill_lanes_per_pair, eng.stats.fill_rows_per_lane) == shape
                assert_same(got, ops, *refs[(mode, clips)], batch, f"{G}x{R} walk={walk} {mode} {clips}")
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,clips", CASES, ids=CASE_IDS)
def test_gpu_caller_and_discovered_alphabet(eng, oracle, main_case, mode, clips):
    """alphabet=NULL: the engine finds the alphabet in the batch (padding included) and gives the same results as with
    the caller's alphabet; last_alphabet() reports the alphabet each form used"""
    table, batch, refs = main_case
    cs, keep = c_scoring(clips, table, ALPHA)
    cs_found, keep_found = c_scoring(clips, table, None)
    got, ops = full(eng, mode, cs, batch)
    assert eng.last_alphabet().tolist() == sorted(ALPHA)
    assert_same(got, ops, *refs[(mode, clips)], batch, f"caller alphabet {mode} {clips}")
    got2, ops2 = full(eng, mode, cs_found, batch)
    assert eng.last_alphabet().tolist() == present_bytes(batch).tolist() == sorted(ALPHA)
    assert_same(got2, ops2, *refs[(mode, clips)], batch, f"discovered alphabet {mode} {clips}")
    # two symbols fewer in the batch: the discovered alphabet is smaller than the caller's, so every symbol after the
    # first one removed has another code in the two forms
    gone = [ALPHA[3], ALPHA[6]]
    b2 = (np.where(np.isin(batch[0], gone), ALPHA[1], batch[0]).astype(np.uint8),) + batch[1:]
    ref, ref_ops = oracle_ref(oracle, mode, clips, table, b2)
    got3, ops3 = full(eng, mode, cs_found, b2)
    assert eng.last_alphabet().tolist() == present_bytes(b2).tolist() == sorted(set(ALPHA) - set(gone))
    assert_same(got3, ops3, ref, ref_ops, b2, f"discovered smaller alphabet {mode} {clips}")
    got4, ops4 = full(eng, mode, cs, b2)
    assert eng.last_alphabet().tolist() == sorted(ALPHA)
    assert_same(got4, ops4, ref, ref_ops, b2, f"caller alphabet, symbols absent {mode} {clips}")


@pytest.mark.gpu
@pytest.mark.parametrize("G,R", [(0, 0), (1, 16), (8, 20), (32, 8)], ids=["auto", "1x16", "8x20", "32x8"])
def test_gpu_degenerate_table_every_cell_a_tie(eng, oracle, G, R):
    """all entries equal: every choice is a tie, so only the tie-breaking order decides the path"""
    table = flat_table(ALPHA, 2)
    batch = pack(related_pairs(8, 120, 90, ALPHA), pad=ALPHA[0])
    try:
        eng.set_tuning(G, R)
        for walk in (1, 2):
            eng.set_walk(walk)
            for mode, clips in CASES:
                ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch, go=-3, ge=-1)
                cs, keep = c_scoring(clips, table, None, go=-3, ge=-1)
                got, ops = full(eng, mode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"flat table {G}x{R} walk={walk} {mode} {clips}")
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("G,R", [(0, 0), (1, 16), (8, 16), (8, 20), (32, 8), (32, 16)],
                         ids=["auto", "1x16", "8x16", "8x20", "32x8", "32x16"])
def test_gpu_score_only_equals_full_and_oracle(eng, main_case, G, R):
    table, batch, refs = main_case
    shape = (G, R) if G else eight_lane_shape(batch)
    try:
        eng.set_tuning(G, R)
        for mode, clips in CASES:
            cs, keep = c_scoring(clips, table, ALPHA)
            sc = eng.align_batch_scores(MODES[mode], cs, batch)
            assert (eng.stats.fill_lanes_per_pair, eng.stats.fill_rows_per_lane) == shape
            got, ops = full(eng, mode, cs, batch)
            assert_scores(sc, got, f"score-only vs full {G}x{R} {mode} {clips}")
            assert_scores(sc, refs[(mode, clips)][0], f"score-only vs oracle {G}x{R} {mode} {clips}")
    finally:
        eng.set_tuning(0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,clips", [CASES[0], CASES[1], CASES[3]], ids=["local", "global", "custom_live"])
def test_gpu_streamed_y(eng, oracle, mode, clips):
    """y of 60,000 symbols (past what whole-y staging holds: the warp-per-pair fill streams y, F_YSTREAM), with 32 x 16
    forced and the automatic shape; full and score-only"""
    rng = np.random.default_rng(60 + len(mode))
    alpha = np.frombuffer(ALPHA, dtype=np.uint8)
    pairs = []
    for _ in range(4):
        x = alpha[rng.integers(0, len(alpha), 300)]
        y = alpha[rng.integers(0, len(alpha), 60000)]
        off = int(rng.integers(0, 60000 - 400))
        src = mutate(rng, x, alpha)
        y[off:off + len(src)] = src
        pairs.append((bytes(x), bytes(y)))
    table = asym_table(61, ALPHA)
    batch = pack(pairs)
    ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch)
    cs, keep = c_scoring(clips, table, ALPHA)
    try:
        for shape in ((32, 16), (0, 0)):
            eng.set_tuning(*shape)
            got, ops = full(eng, mode, cs, batch)
            assert eng.stats.fill_lanes_per_pair == 32
            assert_same(got, ops, ref, ref_ops, batch, f"streamed y {mode} {shape}")
            assert_scores(eng.align_batch_scores(MODES[mode], cs, batch), ref, f"streamed y score-only {mode} {shape}")
    finally:
        eng.set_tuning(0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,clips", [CASES[0], CASES[2], CASES[3]], ids=["local", "semiglobal", "custom_live"])
def test_gpu_long_pairs_relative_trackers(eng, oracle, mode, clips):
    """m, n above 4,095 with a LUT: the relative packed trackers (F_PACKREL | F_LUT)"""
    rng = np.random.default_rng(4500 + len(mode))
    alpha = np.frombuffer(ALPHA, dtype=np.uint8)
    pairs = []
    for m in (4200, 4700):
        x = alpha[rng.integers(0, len(alpha), m)]
        pairs.append((bytes(x), bytes(mutate(rng, x, alpha, 0.12, 0.04)[:4400])))
    pairs.append((pairs[0][1][::-1], pairs[0][0]))
    table = asym_table(45, ALPHA)
    batch = pack(pairs)
    assert int(batch[2].min()) > 4095 and int(batch[4].min()) > 4095
    flags = flags_of(mode, clips, table, ALPHA, batch)
    assert flags & F_PACKREL and not flags & F_PACKTRK, flags
    ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch)
    cs, keep = c_scoring(clips, table, ALPHA)
    got, ops = full(eng, mode, cs, batch)
    assert eng.stats.fill_lanes_per_pair == 32
    assert_same(got, ops, ref, ref_ops, batch, f"long pairs {mode}")
    assert_scores(eng.align_batch_scores(MODES[mode], cs, batch), ref, f"long pairs score-only {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode,clips", [CASES[0], CASES[1], CASES[3]], ids=["local", "global", "custom_live"])
def test_gpu_recomputed_traceback(eng, oracle, mode, clips):
    """one 6,000 x 6,000 pair above a traceback budget of 4 strips, refilled in 3 windows"""
    from test_traceback_recompute import strip_bytes, windows_of
    rng = np.random.default_rng(6000 + len(mode))
    alpha = np.frombuffer(ALPHA, dtype=np.uint8)
    x = alpha[rng.integers(0, len(alpha), 6000)]
    y = mutate(rng, x, alpha, 0.1, 0.03)
    y = np.concatenate([y, alpha[rng.integers(0, len(alpha), 6000)]])[:6000]
    batch = pack([(bytes(x), bytes(y))])
    table = asym_table(6, ALPHA)
    ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch)
    cs, keep = c_scoring(clips, table, ALPHA)
    sb = strip_bytes(6000, 16)
    budget = 4 * sb + sb // 3
    W, nw, _ = windows_of(6000, 6000, budget)
    assert (W, nw) == (4, 3)
    eng.set_traceback_budget(budget)
    eng.set_traceback_recompute(True)
    try:
        got, ops = full(eng, mode, cs, batch)
        rc = eng.last_recompute()
    finally:
        eng.set_traceback_budget(0)
        eng.set_traceback_recompute(False)
    assert eng.stats.fill_lanes_per_pair == 32
    assert rc["pairs"] == 1 and rc["windows"] == nw and 1 <= rc["windows_filled"] <= nw, rc
    assert_same(got, ops, ref, ref_ops, batch, f"recomputed traceback {mode}")


def _pipeline_batch(seed, n, alphabet):
    """n short ragged pairs without padding; y begins with a mutated copy of x"""
    from rust_bio_b200 import synth
    rng = np.random.default_rng(seed)
    blob, xo, xl, yo, yl = synth.ragged_pairs(seed, n, 36, 44, alphabet=alphabet, min_len=1)
    k = np.minimum(xl, yl).astype(np.int64)
    rep = np.repeat(np.arange(n), k)
    within = np.arange(int(k.sum())) - np.repeat(np.cumsum(k) - k, k)
    keep = rng.random(len(within)) >= 0.15
    blob[yo[rep][keep].astype(np.int64) + within[keep]] = blob[xo[rep][keep].astype(np.int64) + within[keep]]
    return blob, xo, xl, yo, yl


@pytest.mark.gpu
def test_gpu_chunk_pipeline(eng, oracle):
    """280,000 pairs go through the chunk pipeline: equal to the one-shot batch (set_pipeline(0)) field for field and
    op for op, and to the oracle on a sample"""
    n = 280_000
    alpha = ALPHA[:-1]
    batch = _pipeline_batch(91, n, alpha)
    table = asym_table(91, alpha)
    mode, clips = CASES[3]
    cs, keep = c_scoring(clips, table, alpha)
    eng.set_pipeline(0)
    try:
        a = eng.align_batch(MODES[mode], cs, batch)
    finally:
        eng.set_pipeline(5)
    b = eng.align_batch(MODES[mode], cs, batch)
    for k in ("score", "xstart", "xend", "ystart", "yend", "ops_off", "clip_len"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    tot = int(a.ops_off[-1])
    assert np.array_equal(a.ops[:tot], b.ops[:tot])
    idx = np.concatenate([np.arange(300), np.random.default_rng(1).integers(0, n, 500), np.arange(n - 300, n)])
    sub = select(batch, idx)
    ref, ref_ops = oracle_ref(oracle, mode, clips, table, sub)
    assert_same({k: v[idx] for k, v in b.as_dict().items()}, [b.ops_of(int(p)) for p in idx], ref, ref_ops, sub,
                "pipelined sample")


@pytest.mark.gpu
def test_gpu_chunk_pipeline_symbol_first_in_a_late_chunk(eng, oracle):
    """a symbol that first appears in the last chunk: outside the caller's alphabet the batch is refused
    (B2A_E_INVALID); without a caller alphabet the pipeline's reuse of chunk 0's alphabet fails for that chunk and the
    batch is redone in one shot, with the right results"""
    from rust_bio_b200._lib import B2AError
    n = 270_000
    alpha = ALPHA[:-1]
    batch = list(_pipeline_batch(92, n, alpha))
    blob = batch[0].copy()
    last = n - 7
    blob[int(batch[1][last]) + int(batch[2][last]) // 2] = ALPHA[-1]
    batch[0] = blob
    batch = tuple(batch)
    table = asym_table(92, ALPHA)
    mode, clips = CASES[0]
    cs, keep = c_scoring(clips, table, alpha)
    with pytest.raises(B2AError, match="alphabet") as err:
        eng.align_batch(MODES[mode], cs, batch)
    assert err.value.code == -1  # B2A_E_INVALID
    cs2, keep2 = c_scoring(clips, table, None)
    b = eng.align_batch(MODES[mode], cs2, batch)
    idx = np.concatenate([np.arange(200), np.arange(n - 200, n)])
    sub = select(batch, idx)
    ref, ref_ops = oracle_ref(oracle, mode, clips, table, sub)
    assert_same({k: v[idx] for k, v in b.as_dict().items()}, [b.ops_of(int(p)) for p in idx], ref, ref_ops, sub,
                "late symbol, discovered alphabet")


# ---------------------------------------------------------------------------------------------------------------
# GPU: BitEnc input, the table indexed by rank

@pytest.mark.gpu
@pytest.mark.parametrize("width,ranks", [(2, 4), (3, 6), (5, 23)])
def test_gpu_bitenc_packed_input_with_a_table_by_rank(eng, oracle, width, ranks):
    """b2a_align_batch_packed and b2a_align_batch_banded_packed with table[a * 256 + b] over ranks: against the oracle
    on the rank sequences and against the byte path on the same ranks.  Width 2 leaves the alphabet to the engine
    (every rank the width holds); the others pass the ranks present, since the width holds ranks the table does not"""
    from rust_bio_b200.data_structures import BitEnc
    from rust_bio_b200.engine import Engine
    rank_alpha = bytes(range(ranks))
    table = asym_table(width, rank_alpha)
    alphabet = None if ranks == 1 << width else rank_alpha
    pairs = related_pairs(width, 200, 120, rank_alpha)
    batch = pack(pairs, pad=0)
    packed = Engine.pack_bitenc_pairs([(BitEnc.from_values(width, np.frombuffer(x, np.uint8)),
                                        BitEnc.from_values(width, np.frombuffer(y, np.uint8))) for x, y in pairs])
    assert packed[5] == width
    for mode, clips in CASES:
        cs, keep = c_scoring(clips, table, alphabet)
        ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch)
        res = eng.align_batch_packed(MODES[mode], cs, packed)
        assert_same(res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)], ref, ref_ops, batch,
                    f"packed w={width} {mode} {clips}")
        got, ops = full(eng, mode, cs, batch)
        assert_same(got, ops, ref, ref_ops, batch, f"byte path on the ranks w={width} {mode} {clips}")
    wpairs = _window_pairs(50 + width, 60, 100, 260, rank_alpha)
    wbatch = pack(wpairs, pad=0)
    wpacked = Engine.pack_bitenc_pairs([(BitEnc.from_values(width, np.frombuffer(x, np.uint8)),
                                         BitEnc.from_values(width, np.frombuffer(y, np.uint8))) for x, y in wpairs])
    for mode, clips in BANDED_CASES[:4]:
        ref, ref_ops, cells = banded_ref(oracle, mode, clips, table, 6, 8, wbatch, 1)
        cs, keep = c_scoring(clips, table, alphabet, ma=2, mi=-3, has_ms=1)
        res = eng.align_batch_packed(MODES[mode], cs, wpacked, banded=(6, 8))
        assert_same(res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)], ref, ref_ops, wbatch,
                    f"banded packed w={width} {mode} {clips}")


# ---------------------------------------------------------------------------------------------------------------
# GPU: the banded aligner

BANDED_ENVS = {"strip": {}, "column_loops": {"B2A_BANDED_STRIP": "0"}, "literal": {"B2A_BANDED_LITERAL": "1"}}


@pytest.fixture(scope="module")
def banded_engines():
    """one engine per banded fill path (the knobs are read when an engine is created)"""
    import os
    from rust_bio_b200.engine import Engine
    engines = {}
    for name, env in BANDED_ENVS.items():
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            engines[name] = Engine(0)
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    yield engines
    for e in engines.values():
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("has_ms", [0, 1])
@pytest.mark.parametrize("mode,clips", BANDED_CASES, ids=CASE_IDS[:5])
def test_gpu_banded_every_path(banded_engines, oracle, mode, clips, has_ms):
    """mutated windows with the asymmetric table through the strip fill, the column loops (B2A_BANDED_STRIP=0), the
    literal column loop (B2A_BANDED_LITERAL=1) and banded score-only; with has_match_scores 0 the band is built from
    the default match score"""
    table = asym_table(70 + has_ms, ALPHA)
    batch = pack(_window_pairs(71 + has_ms + len(mode), 200, 300, 900, ALPHA))
    k, w = 6, 8
    ref, ref_ops, cells = banded_ref(oracle, mode, clips, table, k, w, batch, has_ms)
    cs, keep = c_scoring(clips, table, ALPHA, ma=2, mi=-3, has_ms=has_ms)
    results = {}
    for name, e in banded_engines.items():
        got, ops = banded_full(e, mode, cs, k, w, batch)
        assert int(e.stats.cells) == cells, name
        assert_same(got, ops, ref, ref_ops, batch, f"banded {name} {mode} {clips} has_ms={has_ms}")
        results[name] = e.banded_strip_pairs()
        assert_scores(e.align_batch_banded_scores(MODES[mode], cs, k, w, batch), ref,
                      f"banded score-only {name} {mode} {clips} has_ms={has_ms}")
    assert results["column_loops"] == 0
    if mode != "custom":
        assert results["strip"] * 2 >= len(batch[2]), results


# ---------------------------------------------------------------------------------------------------------------
# GPU: alphabet edges

def _spread_alphabet(k):
    """k byte values spread over 1..255, both ends included (0 excluded: pack_pairs pads with it)"""
    return bytes(sorted(set(np.linspace(1, 255, k).round().astype(int).tolist())))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [64, 65])
def test_gpu_matchparams_at_64_and_65_symbols(eng, oracle, k):
    """MatchParams over 64 distinct bytes run from the LUT, over 65 from compare / select in the kernel, where K0 stages
    the bytes unmapped: byte 0xFF is then a symbol, not the code of a byte outside the alphabet"""
    from rust_bio_b200 import synth
    alpha = _spread_alphabet(k)
    assert len(alpha) == k and alpha[-1] == 0xFF
    batch = synth.ragged_pairs(64 + k, 300, 120, 140, alphabet=alpha, min_len=0)
    assert len(present_bytes(batch)) == k
    try:
        for G, R in [(0, 0), (1, 16), (8, 16), (32, 8)]:
            eng.set_tuning(G, R)
            for mode, clips in CASES:
                ref, ref_ops = oracle_ref(oracle, mode, clips, None, batch, ma=3, mi=-2)
                cs, keep = c_scoring(clips, ma=3, mi=-2)
                got, ops = full(eng, mode, cs, batch)
                assert eng.last_alphabet().tolist() == list(alpha)
                assert_same(got, ops, ref, ref_ops, batch, f"{k} symbols {G}x{R} {mode} {clips}")
    finally:
        eng.set_tuning(0, 0)


@pytest.mark.gpu
def test_gpu_table_at_128_and_129_symbols(eng, oracle):
    """a table over exactly 128 symbols is accepted (a 128 x 128 LUT beside the staged sequences on 8 x 20 and 1 x 16),
    over 129 refused"""
    from rust_bio_b200._lib import B2AError
    alpha = _spread_alphabet(128)
    assert len(alpha) == 128
    table = asym_table(128, alpha)
    batch = pack(related_pairs(128, 200, 60, alpha))
    try:
        for G, R in [(0, 0), (8, 20), (1, 16), (32, 8)]:
            eng.set_tuning(G, R)
            shape = (G, R) if G else eight_lane_shape(batch)
            for mode, clips in CASES:
                ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch)
                cs, keep = c_scoring(clips, table, alpha)
                got, ops = full(eng, mode, cs, batch)
                assert (eng.stats.fill_lanes_per_pair, eng.stats.fill_rows_per_lane) == shape
                assert_same(got, ops, ref, ref_ops, batch, f"128 symbols {G}x{R} {mode} {clips}")
    finally:
        eng.set_tuning(0, 0)
    wide = alpha + b"\x00"
    cs, keep = c_scoring(CASES[0][1], asym_table(129, wide), wide)
    with pytest.raises(B2AError, match="128 distinct") as err:
        eng.align_batch(MODES["local"], cs, batch)
    assert err.value.code == -7  # B2A_E_UNSUPPORTED
    # the same count found in the batch (alphabet=NULL): 128 symbols and the padding byte 0
    cs, keep = c_scoring(CASES[0][1], asym_table(129, wide), None)
    with pytest.raises(B2AError, match="128 distinct"):
        eng.align_batch(MODES["local"], cs, batch)


EDGE = bytes([0, 1, 126, 127, 128, 129, 254, 255])


@pytest.mark.gpu
@pytest.mark.parametrize("scoring", ["table", "matchparams"])
def test_gpu_edge_bytes_as_symbols(eng, oracle, scoring):
    """bytes 0, 127, 128 and 255 as real sequence symbols (the signedness of the code-map load, and 0xFF as the code
    of a byte outside the alphabet), full and banded"""
    table = asym_table(255, EDGE) if scoring == "table" else None
    alphabet = EDGE if scoring == "table" else None
    ma, mi = (0, 0) if scoring == "table" else (3, -2)
    batch = pack(related_pairs(255, 200, 120, EDGE))
    try:
        for G, R in [(0, 0), (1, 16), (8, 16), (32, 8)]:
            eng.set_tuning(G, R)
            for mode, clips in CASES:
                ref, ref_ops = oracle_ref(oracle, mode, clips, table, batch, ma=ma, mi=mi)
                cs, keep = c_scoring(clips, table, alphabet, ma=ma, mi=mi)
                got, ops = full(eng, mode, cs, batch)
                assert eng.last_alphabet().tolist() == list(EDGE)
                assert_same(got, ops, ref, ref_ops, batch, f"edge bytes {scoring} {G}x{R} {mode} {clips}")
    finally:
        eng.set_tuning(0, 0)
    wbatch = pack(_window_pairs(256, 120, 300, 900, EDGE))
    for mode, clips in BANDED_CASES[:3]:
        ref, ref_ops, cells = banded_ref(oracle, mode, clips, table, 6, 8, wbatch, 1, ma=2, mi=-3)
        cs, keep = c_scoring(clips, table, alphabet, ma=2, mi=-3, has_ms=1)
        got, ops = banded_full(eng, mode, cs, 6, 8, wbatch)
        assert eng.banded_strip_pairs() * 2 >= 120
        assert_same(got, ops, ref, ref_ops, wbatch, f"edge bytes banded {scoring} {mode}")


@pytest.mark.gpu
def test_gpu_banded_strip_byte_outside_the_callers_alphabet(eng, oracle):
    """a sequence byte outside the caller's alphabet on the banded strip path is B2A_E_INVALID, not a score"""
    from rust_bio_b200._lib import B2AError
    table = asym_table(3, ALPHA)
    pairs = _window_pairs(3, 40, 300, 900, ALPHA)
    cs, keep = c_scoring(CASES[2][1], table, ALPHA, ma=2, mi=-3, has_ms=1)
    batch = pack(pairs)
    banded_full(eng, "semiglobal", cs, 6, 8, batch)
    assert eng.banded_strip_pairs() * 2 >= len(pairs)
    x, y = pairs[5]
    pairs[5] = (x[:40] + b"Z" + x[41:], y)
    with pytest.raises(B2AError, match="alphabet") as err:
        banded_full(eng, "semiglobal", cs, 6, 8, pack(pairs))
    assert err.value.code == -1  # B2A_E_INVALID
