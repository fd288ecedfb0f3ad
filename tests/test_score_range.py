"""The aligner at the edges of its score range and of its packed-index limits.

The engine picks its kernel form from numeric thresholds on score_bound = (maxm + maxn + 2) * unit - gap_open, where
unit = max(|score|, -gap_open, -gap_extend) over the batch's alphabet (b2a_engine.cu stage_front):
  * F_PACKTRK (keys 4096 * S + (4095 - index)): score_bound < 2^17 and maxm, maxn <= 4095;
  * F_PACKREL (the same keys over chunk- / strip-relative indices): score_bound < 2^18;
  * explicit (value, index) trackers above that;
  * the banded strip-wavefront fill: score_bound < 2^26, with live trackers only below 2^17 (banded_strip_gate);
  * the range guard: score_bound <= 2^27, |LUT entry| <= 2^27, live clips >= -2^27.
Every group below builds its scoring from a target bound, asserts which form the batch ran on each side of the edge,
and compares every Alignment field and the ops with the oracle; paths are re-scored independently of it.  Scores are
pushed to the edge, not only the bound: local mode on related pairs (S up to about half the bound) and global /
suffix-clip custom modes on pairs over disjoint alphabets, long against short, where S comes close to -bound."""
import ctypes as C

import numpy as np
import pytest

import sim_util
from parity_util import MODES, assert_same, oracle_batch, rescore_path

MIN = -858993459
DEAD_CLIP = -429496729  # MIN_SCORE / 2 rounded toward zero (b2a_common.cuh): clips at or below it are dead
F_TR, F_TC, F_PK, F_PR = 1, 2, 16, 128  # b2a_common.cuh: F_TRACK_ROWS, F_TRACK_COLS, F_PACKTRK, F_PACKREL
LOCAL, GLOBAL, SEMI = (0, 0, 0, 0), (MIN,) * 4, (MIN, MIN, 0, 0)
SHAPES = [(1, 16), (1, 8), (4, 16), (8, 16), (8, 20), (32, 8), (32, 16)]  # test_gpu_parity.SHAPES


def score_bound(go, ge, match, mismatch, table, alphabet, maxm, maxn):
    """stage_front's bound: (maxm + maxn + 2) * max(|scores|, -go, -ge) - go, the scores taken over the alphabet's
    table entries for a tabulated MatchFunc (alphabet: the bytes present in the batch, or the caller's)."""
    if table is not None:
        idx = np.frombuffer(bytes(alphabet), dtype=np.uint8)
        t = np.asarray(table, dtype=np.int64).reshape(256, 256)
        unit = int(np.abs(t[np.ix_(idx, idx)]).max())
    else:
        unit = max(abs(match), abs(mismatch))
    unit = max(unit, -go, -ge)
    return (maxm + maxn + 2) * unit - go


def unit_go(target, L, above=False):
    """(unit, gap_open) with -gap_open <= unit (so that unit stays the largest magnitude) and the bound
    L * unit - gap_open as close to target as it gets: at most target, or with `above` at least target; exactly target
    whenever target >= L * (L + 1).  gap_open stays within L of -unit: with gap_extend = -unit, every gap symbol then
    costs about a unit (a cheap gap_open would let the recurrence re-open every symbol)."""
    u = -(-target // (L + 1))
    rem = target - L * u
    if 0 <= rem <= u:
        return u, -rem
    if above:
        u = -(-target // (L + 1))
        return u, -max(0, target - L * u)
    return target // (L + 1), -(target // (L + 1))


def effective_clips(mode, clips):
    return {"global": GLOBAL, "semiglobal": SEMI, "local": LOCAL}.get(mode, clips)


def flags_of(mode, clips, bound, maxm, maxn, alpha=4):
    return int(sim_util.lib().sim_scoring_flags(*[C.c_int32(c) for c in effective_clips(mode, clips)], C.c_int32(alpha),
                                                C.c_int64(bound), C.c_uint32(maxm), C.c_uint32(maxn)))


def strip_gate(mode, clips, bound, maxm):
    L = sim_util.lib()
    return L.sim_banded_strip_gate(*[C.c_int32(c) for c in effective_clips(mode, clips)], C.c_int64(bound),
                                   C.c_uint32(maxm)) == 1


def tracker_form(flags):
    if flags & F_PK:
        return "packed"
    if flags & F_PR:
        return "relative"
    return "explicit" if flags & (F_TR | F_TC) else "none"


# ---------------------------------------------------------------------------------------------------------------
# batches

DNA = np.frombuffer(b"ACGT", dtype=np.uint8)


def _mutate(rng, s, rate=0.08, alphabet=DNA):
    s = s.copy()
    mut = rng.random(len(s)) < rate
    s[mut] = alphabet[rng.integers(0, len(alphabet), int(mut.sum()))]
    return s


def make_pair(rng, m, n, kind, alphabet=DNA):
    """related: y starts with a mutated copy of x; tail: the shorter sequence is a mutated copy of the longer one's
    last symbols, the last eight kept exact (the best local alignment ends at the largest index); disjoint: x over the
    alphabet's first half, y over its second half (every cell a mismatch or a gap)."""
    if kind == "disjoint":
        h = len(alphabet) // 2
        return (bytes(alphabet[:h][rng.integers(0, h, m)]), bytes(alphabet[h:][rng.integers(0, len(alphabet) - h, n)]))
    x = alphabet[rng.integers(0, len(alphabet), m)]
    y = alphabet[rng.integers(0, len(alphabet), n)]
    k = min(m, n)
    if kind == "related":
        y[:k] = _mutate(rng, x[:k], alphabet=alphabet)
    elif kind == "tail":
        t = min(8, k)
        if m >= n:
            y = _mutate(rng, x[m - n:], 0.04, alphabet)
            y[n - t:] = x[m - t:]
        else:
            x = _mutate(rng, y[n - m:], 0.04, alphabet)
            x[m - t:] = y[n - t:]
    return bytes(x), bytes(y)


def pack(pairs):
    from rust_bio_b200.engine import pack_pairs
    return pack_pairs(pairs)


def short_batch(seed, kind):
    """40-60 long pairs, maxm = maxn = 60 (L = 122): uniform 60 x 60 (masked last strips for R = 16 / 8 x 8's 64 rows)
    or ragged; related, identical and disjoint pairs mixed, plus a long-against-short pair each way."""
    rng = np.random.default_rng(seed)
    pairs = []
    for q in range(40):
        m, n = (60, 60) if kind == "uniform" else (int(rng.integers(40, 61)), int(rng.integers(40, 61)))
        pairs.append(make_pair(rng, m, n, ("related", "tail", "disjoint")[q % 3]))
    if kind == "ragged":
        pairs += [make_pair(rng, 60, 60, "related"), make_pair(rng, 60, 3, "disjoint"), make_pair(rng, 2, 60, "disjoint")]
    return pack(pairs)


def pairs_of(batch):
    blob, xo, xl, yo, yl = batch
    return [(bytes(blob[int(xo[p]):int(xo[p]) + int(xl[p])]), bytes(blob[int(yo[p]):int(yo[p]) + int(yl[p])]))
            for p in range(len(xl))]


def check_rescore(batch, got, ops, mode, go, ge, score_fn, clips):
    """rescore_path on every pair; with gap_extend < gap_open not on paths that start with a gap: the first row and
    column charge go + (k - 1) ge for k leading gap symbols, where re-opening (rescore_path's model) would be cheaper"""
    eff = effective_clips(mode, clips)
    for p, (x, y) in enumerate(pairs_of(batch)):
        if ge < go and [c for c, _ in ops[p] if c < 4][:1] in ([2], [3]):
            continue
        f = {k: got[k][p] for k in ("xstart", "xend", "ystart", "yend")}
        assert rescore_path(x, y, ops[p], f, mode, go, ge, score_fn, eff) == int(got["score"][p]), (mode, p)


def _unit_fn(ma, mi):
    return lambda a, b: ma if a == b else mi


def _table_fn(table):
    flat = np.asarray(table).reshape(-1)
    return lambda a, b: int(flat[a * 256 + b])


def sim_run(mode, s, batch, G, R, warp_walk):
    return sim_util.align_batch(MODES[mode], s, *batch, R=R, G=G, warp_walk=warp_walk)


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers

def c_scoring(go, ge, ma, mi, clips=GLOBAL, table=None, alphabet=None, has_ms=0):
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


def gpu_run(eng, mode, cs, batch):
    res = eng.align_batch(MODES[mode], cs, batch)
    return res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)]


@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


# ---------------------------------------------------------------------------------------------------------------
# helpers themselves

def test_score_bound_and_unit_go():
    assert score_bound(-5, -1, 1, -1, None, None, 150, 150) == 302 * 5 + 5  # C1: the gap open is the unit
    for target, L in [((1 << 17) - 1, 122), (1 << 17, 122), ((1 << 27), 1022), ((1 << 18) - 1, 20483), (1 << 17, 802)]:
        for above in (False, True):
            u, go = unit_go(target, L, above)
            b = score_bound(go, -u, u, -u, None, None, L - 2, 0)
            assert -go <= u and (b >= target if above else b <= target) and abs(b - target) < 2 * L
            assert b == target or target < L * (L + 1)
    table = np.zeros((256, 256), dtype=np.int64)
    table[ord("A"), ord("C")] = -70
    table[ord("Z"), ord("Z")] = 2 ** 31 - 1  # not in the alphabet: ignored
    assert score_bound(-3, -1, 0, 0, table, b"AC", 10, 10) == 22 * 70 + 3


# ---------------------------------------------------------------------------------------------------------------
# a. packed keys over absolute indices (F_PACKTRK) at 2^17 - 1, relative keys at 2^17 and at 2^18 - 1 (S up to about
# 2^17, keys 4096 * S + index near +-2^30)

A_SIDES = {"packed": (1 << 17) - 1, "relative": 1 << 17, "relative_2^18-1": (1 << 18) - 1}
A_MODES = {"local": LOCAL, "semiglobal": SEMI, "custom_suffix": (MIN, "xs", 0, "ys"), "custom_prefix": ("xp", MIN, "yp", "ys")}


def _a_scoring(mode, side):
    u, go = unit_go(A_SIDES[side], 122)
    clips = A_MODES[mode]
    clips = tuple({"xs": -3 * u, "ys": -2 * u, "xp": -u, "yp": -5 * u}.get(c, c) for c in clips)
    omode = "custom" if mode.startswith("custom") else mode
    return omode, clips, go, -u, u, -u


@pytest.mark.parametrize("G,R", [(1, 16), (8, 8), (32, 8), (132, 8)], ids=["1x16", "8x8", "32x8", "strip_pipelined_32x8"])
@pytest.mark.parametrize("mode", list(A_MODES))
@pytest.mark.parametrize("side", list(A_SIDES))
def test_sim_packed_keys_at_2_17(oracle, side, mode, G, R):
    omode, clips, go, ge, ma, mi = _a_scoring(mode, side)
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
    assert score_bound(go, ge, ma, mi, None, None, 60, 60) == A_SIDES[side]
    assert tracker_form(flags_of(omode, clips, A_SIDES[side], 60, 60)) == side.split("_")[0]
    for kind in ("uniform", "ragged"):
        batch = short_batch(11 + len(mode), kind)
        ref, ref_ops = oracle_batch(oracle, omode, s, batch)
        assert int(np.abs(ref["score"]).max()) > A_SIDES[side] // 3  # the scores reach the edge, not only the bound
        walk = 1 if kind == "ragged" else 0  # the one-lane walk on one batch, the warp walk on the other
        got, ops = sim_run(omode, s, batch, G, R, walk)
        assert_same(got, ops, ref, ref_ops, batch, f"{side} {mode} {kind} G={G} R={R} walk={walk}")
        check_rescore(batch, got, ops, omode, go, ge, _unit_fn(ma, mi), clips)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(A_MODES))
@pytest.mark.parametrize("side", list(A_SIDES))
def test_gpu_packed_keys_at_2_17(eng, oracle, side, mode):
    omode, clips, go, ge, ma, mi = _a_scoring(mode, side)
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
    cs, keep = c_scoring(go, ge, ma, mi, clips)
    assert tracker_form(flags_of(omode, clips, A_SIDES[side], 60, 60)) == side.split("_")[0]
    try:
        for kind in ("uniform", "ragged"):
            batch = short_batch(11 + len(mode), kind)
            ref, ref_ops = oracle_batch(oracle, omode, s, batch)
            assert int(np.abs(ref["score"]).max()) > A_SIDES[side] // 3
            for G, R in SHAPES:
                eng.set_tuning(G, R)
                for walk in (1, 2):
                    eng.set_walk(walk)
                    got, ops = gpu_run(eng, omode, cs, batch)
                    assert eng.stats.fill_lanes_per_pair == G
                    assert_same(got, ops, ref, ref_ops, batch, f"GPU {side} {mode} {kind} G={G} R={R} walk={walk}")
            check_rescore(batch, got, ops, omode, go, ge, _unit_fn(ma, mi), clips)
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)


# ---------------------------------------------------------------------------------------------------------------
# b. the index limit 4,095 of the packed keys

def _limit_batch(m, n, seed):
    """m x n: a tail copy (the best alignment ends at the long sequence's last index) and a disjoint pair"""
    rng = np.random.default_rng(seed)
    return pack([make_pair(rng, m, n, "tail"), make_pair(rng, m, n, "disjoint"), make_pair(rng, m, n - 1, "tail")])


B_MODES = {"local": LOCAL, "semiglobal": SEMI, "custom": (MIN, -40, 0, -25)}


def _b_scoring(L):
    u, go = unit_go((1 << 17) - 1, L)
    return go, -u, u, -u


@pytest.mark.parametrize("lim,G,R", [(4095, 1, 16), (4095, 132, 8), (4096, 1, 16)],
                         ids=["4095-1x16", "4095-strip_pipelined_32x8", "4096-1x16"])
@pytest.mark.parametrize("mode", list(B_MODES))
def test_sim_index_limit_4095(oracle, lim, mode, G, R):
    """4095 x 32 puts the limit index into the column tracker, 32 x 4095 into the row tracker (j = n = 4095 is packed
    as 0); one more and the batch runs the relative keys.  Each direction is a batch of its own, so that x and y are
    held to the limit separately."""
    clips = B_MODES[mode]
    for m, n in ((lim, 32), (32, lim)):
        go, ge, ma, mi = _b_scoring(m + n + 2)
        bound = score_bound(go, ge, ma, mi, None, None, m, n)
        assert (1 << 17) - 2 * (m + n + 3) < bound < 1 << 17
        assert tracker_form(flags_of(mode, clips, bound, m, n)) == ("packed" if lim == 4095 else "relative")
        s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
        batch = _limit_batch(m, n, 5)
        ref, ref_ops = oracle_batch(oracle, mode, s, batch)
        if mode == "local":  # the tail copy's best alignment ends at (m, n): index lim goes into the key
            assert (int(ref["xend"][0]), int(ref["yend"][0])) == (m, n)
        got, ops = sim_run(mode, s, batch, G, R, 1 if G == 132 else 0)
        assert_same(got, ops, ref, ref_ops, batch, f"{m} x {n} {mode} G={G} R={R}")
        check_rescore(batch, got, ops, mode, go, ge, _unit_fn(ma, mi), clips)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(B_MODES))
@pytest.mark.parametrize("lim", [4095, 4096])
def test_gpu_index_limit_4095(eng, oracle, lim, mode):
    """lim x lim, lim x 300 and 300 x lim on the automatic shape, 8x16 and 32x8, both walks"""
    clips = B_MODES[mode]
    go, ge, ma, mi = _b_scoring(2 * lim + 2)
    bound = score_bound(go, ge, ma, mi, None, None, lim, lim)
    assert (1 << 17) - 2 * (2 * lim + 3) < bound < 1 << 17
    assert tracker_form(flags_of(mode, clips, bound, lim, lim)) == ("packed" if lim == 4095 else "relative")
    rng = np.random.default_rng(lim)
    batch = pack([make_pair(rng, lim, lim, "related"), make_pair(rng, lim, 300, "tail"), make_pair(rng, 300, lim, "tail"),
                  make_pair(rng, lim, 300, "disjoint"), make_pair(rng, 300, lim, "disjoint")])
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
    if mode == "local":  # the tail copies' best alignments end at index lim
        assert [(int(ref["xend"][p]), int(ref["yend"][p])) for p in (1, 2)] == [(lim, 300), (300, lim)]
    cs, keep = c_scoring(go, ge, ma, mi, clips)
    try:
        for G, R in [(0, 0), (8, 16), (32, 8)]:
            eng.set_tuning(G, R)
            for walk in (1, 2):
                eng.set_walk(walk)
                got, ops = gpu_run(eng, mode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"GPU {lim} {mode} G={G} R={R} walk={walk}")
        check_rescore(batch, got, ops, mode, go, ge, _unit_fn(ma, mi), clips)
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)


# ---------------------------------------------------------------------------------------------------------------
# c. relative keys (F_PACKREL) around the 4,096-step chunk edges, bound just under 2^18 (GPU: the host harness
# covers 32-column chunks)

# custom_ys_only: both prefix clips dead, so S(m, j) on the disjoint 300 x 12288 pair runs to about -12288 units
# (more than half the bound) in the row whose keys the tracker compares
C_MODES = {"semiglobal": SEMI, "custom_ys": (MIN, MIN, -30, -20), "custom_ys_only": (MIN, MIN, MIN, -20), "local": LOCAL,
           "custom_xs": (MIN, -20, 0, MIN)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(C_MODES))
def test_gpu_relative_keys_at_chunk_edges(eng, oracle, mode):
    """300-long reads ending at the chunk edges, a disjoint 300 x 12288 pair, and related 8193 x 12288 / 8193 x 8193
    pairs whose scores reach about a third of the bound"""
    rng = np.random.default_rng(len(mode))
    pairs = []
    # n at the chunk edges, and shifted by the wavefront skew G - 1 of the 32-lane shapes (the ones that stage y this long)
    for n in (8191, 8192, 8193, 12288, 8192 - 31, 8192 - 30, 12288 - 31):
        e = 8192 if n >= 8192 else n
        y = DNA[rng.integers(0, 4, n)]
        pairs.append((bytes(_mutate(rng, y[e - 300:e], 0.04)), bytes(y)))  # the read ends at the chunk edge
        pairs.append(make_pair(rng, 300, n, "tail"))
    pairs += [make_pair(rng, 300, 12288, "disjoint"), make_pair(rng, 4097, 300, "tail"), make_pair(rng, 8193, 300, "tail"),
              make_pair(rng, 8193, 290, "disjoint"), make_pair(rng, 8193, 12288, "related"),
              make_pair(rng, 8193, 8193, "related")]  # (y dead-ended in custom_xs: the whole of y aligns)
    batch = pack(pairs)
    clips = C_MODES[mode]
    omode = "custom" if mode.startswith("custom") else mode
    L = 8193 + 12288 + 2
    u, go = unit_go((1 << 18) - 1, L)
    ge, ma, mi = -u, u, -u
    bound = score_bound(go, ge, ma, mi, None, None, 8193, 12288)
    assert (1 << 18) - 2 * L < bound < 1 << 18
    assert tracker_form(flags_of(omode, clips, bound, 8193, 12288)) == "relative"
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
    ref, ref_ops = oracle_batch(oracle, omode, s, batch, threads=8)
    assert int(np.abs(ref["score"]).max()) > bound // 4  # the scores reach the edge, not only the bound
    cs, keep = c_scoring(go, ge, ma, mi, clips)
    try:
        for G, R in [(0, 0), (32, 8), (32, 16)]:  # (the 12,288-long y is too long for the smaller shapes' staging)
            eng.set_tuning(G, R)
            for walk in (1, 2):
                eng.set_walk(walk)
                got, ops = gpu_run(eng, omode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"GPU relative keys {mode} G={G} R={R} walk={walk}")
        check_rescore(batch, got, ops, omode, go, ge, _unit_fn(ma, mi), clips)
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)


# ---------------------------------------------------------------------------------------------------------------
# d. explicit (value, index) trackers, reached by the score range alone

D_BOUNDS = {"2^18": 1 << 18, "under_2^27": (1 << 27) - 1000}
D_MODES = {"local": LOCAL, "semiglobal": SEMI, "custom": (-2, -3, -1, -1)}  # custom: the clips in units


def _reads_batch(seed):
    """150-long reads (related / disjoint), and 10 x 150 / 150 x 10 disjoint pairs whose S runs to about -bound"""
    rng = np.random.default_rng(seed)
    pairs = [make_pair(rng, 150, 150, ("related", "tail", "disjoint")[q % 3]) for q in range(36)]
    pairs += [make_pair(rng, 150, 2, "disjoint"), make_pair(rng, 2, 150, "disjoint"), make_pair(rng, 150, 0, "related")]
    return pack(pairs)


def _d_scoring(bound, mode, maxm, maxn):
    """-> (clips, go, ge, match, mismatch): at least 2^18, or at most 2^27 - 1000"""
    u, go = unit_go(D_BOUNDS[bound], maxm + maxn + 2, above=bound == "2^18")
    clips = tuple(c * u for c in D_MODES[mode]) if mode == "custom" else D_MODES[mode]
    return clips, go, -u, u, -u


@pytest.mark.parametrize("G,R", [(1, 16), (8, 20), (132, 8)], ids=["1x16", "8x20", "strip_pipelined_32x8"])
@pytest.mark.parametrize("mode", list(D_MODES))
@pytest.mark.parametrize("bound", list(D_BOUNDS))
def test_sim_explicit_trackers_by_score_range(oracle, bound, mode, G, R):
    omode = mode
    clips, go, ge, ma, mi = _d_scoring(bound, mode, 150, 150)
    b = score_bound(go, ge, ma, mi, None, None, 150, 150)
    assert b == D_BOUNDS[bound]
    assert tracker_form(flags_of(omode, clips, b, 150, 150)) == "explicit"
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
    batch = _reads_batch(3)
    ref, ref_ops = oracle_batch(oracle, omode, s, batch)
    got, ops = sim_run(omode, s, batch, G, R, 1 if G != 1 else 0)
    assert_same(got, ops, ref, ref_ops, batch, f"{bound} {mode} G={G} R={R}")
    check_rescore(batch, got, ops, omode, go, ge, _unit_fn(ma, mi), clips)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(D_MODES))
@pytest.mark.parametrize("bound", list(D_BOUNDS))
def test_gpu_explicit_trackers_by_score_range(eng, oracle, bound, mode):
    omode = mode
    rng = np.random.default_rng(17)
    long_batch = pack([make_pair(rng, 4200, 4200, "related"), make_pair(rng, 4200, 4150, "tail"),
                       make_pair(rng, 40, 4200, "disjoint"), make_pair(rng, 4200, 30, "disjoint")])
    for batch, (maxm, maxn), shapes in [(_reads_batch(3), (150, 150), [(0, 0), (1, 16), (8, 20), (32, 8)]),
                                        (long_batch, (4200, 4200), [(0, 0), (8, 16), (32, 8)])]:
        cl, go, ge, ma, mi = _d_scoring(bound, mode, maxm, maxn)
        b = score_bound(go, ge, ma, mi, None, None, maxm, maxn)
        assert abs(b - D_BOUNDS[bound]) < 2 * (maxm + maxn + 3) and (b >= 1 << 18) and b <= (1 << 27)
        assert tracker_form(flags_of(omode, cl, b, maxm, maxn)) == "explicit"
        s, _ = oracle.make_scoring(go, ge, ma, mi, None, *cl)
        ref, ref_ops = oracle_batch(oracle, omode, s, batch, threads=8)
        cs, keep = c_scoring(go, ge, ma, mi, cl)
        try:
            for G, R in shapes:
                eng.set_tuning(G, R)
                for walk in (1, 2):
                    eng.set_walk(walk)
                    got, ops = gpu_run(eng, omode, cs, batch)
                    assert_same(got, ops, ref, ref_ops, batch, f"GPU {bound} {mode} {maxm} G={G} R={R} walk={walk}")
        finally:
            eng.set_walk(0)
            eng.set_tuning(0, 0)
        check_rescore(batch, got, ops, omode, go, ge, _unit_fn(ma, mi), cl)


# ---------------------------------------------------------------------------------------------------------------
# e. the range guard: accepted just inside it (bit-exact), refused just outside it;  g. gap models and an asymmetric
# table at those magnitudes

def _asym_table(rng, alphabet, u):
    """an asymmetric table over `alphabet` with entries in [-u, u] (the diagonal at +u), and INT32_MAX / MIN outside"""
    t = np.full((256, 256), 2 ** 31 - 1, dtype=np.int64)
    t[::2, :] = -2 ** 31
    idx = np.frombuffer(alphabet, dtype=np.uint8)
    sub = rng.integers(-u, u + 1, (len(idx), len(idx)))
    np.fill_diagonal(sub, u)
    t[np.ix_(idx, idx)] = sub
    # byte 0 pads the blob between sequences (pack_pairs); without a caller alphabet the engine finds the alphabet in
    # one flat pass over the whole blob, padding included (b2a_scoring.alphabet, b200align.h), so its entries stay small
    # here and test_sim_banded_padding_counts_without_a_caller_alphabet checks the rule
    t[0, :] = t[:, 0] = 0
    assert not np.array_equal(sub, sub.T)
    return t.astype(np.int32)


AA = b"ACDEFGHIKLMNPQRSTVWYBZX*abcdefghijklmnopqrstuvwxyz0123456789"[:40]


def _e_case(case):
    """-> (mode, clips, go, ge, ma, mi, table, batch) with score_bound at (or just under) 2^27"""
    rng = np.random.default_rng(E_CASES.index(case))
    if case in ("global_x_short", "custom_y_short"):  # S(m, n) runs to within a few percent of -bound
        long_x = case == "custom_y_short"
        pairs = []
        for q in range(24):
            a, b = int(rng.integers(1, 13)), int(rng.integers(250, 301))
            m, n = (b, a) if long_x else (a, b)
            pairs.append(make_pair(rng, m, n, ("disjoint", "disjoint", "related")[q % 3]))
        pairs.append(make_pair(rng, *((300, 12) if long_x else (12, 300)), "disjoint"))
        u, go = unit_go(1 << 27, 314)
        if long_x:
            return "custom", (MIN, -u * 200, MIN, -u * 5), go, -u, u, -u, None, pack(pairs)
        return "global", GLOBAL, go, -u, u, -u, None, pack(pairs)
    if case == "asym_table":
        pairs = [make_pair(rng, 150, 150, k, np.frombuffer(AA, dtype=np.uint8)) for k in ("related", "tail", "disjoint") * 6]
        pairs += [make_pair(rng, 150, 4, "disjoint", np.frombuffer(AA, dtype=np.uint8))]
        batch = pack(pairs)
        u, go = unit_go(1 << 27, 302)
        table = _asym_table(rng, AA, u)
        return "local", LOCAL, go, -u // 3, 0, 0, table, batch
    batch = _reads_batch(9)
    u, go = unit_go(1 << 27, 302)
    if case == "exact_2^27_global":
        return "global", GLOBAL, go, -u, u, -u, None, batch
    if case == "exact_2^27_custom":
        return "custom", (MIN, -u * 7, -(1 << 27), -u * 3), go, -u, u, -u, None, batch
    if case == "clip_minus_2^27":
        return "custom", (-(1 << 27), -(1 << 27), -(1 << 27), -(1 << 27)), go, -u, u, -u, None, batch
    # gap models at a bound just under 2^27 (unit set by the mismatch / the larger gap penalty)
    u = ((1 << 27) - 1) // 303
    if case == "ge_below_go":   # extending costs more than opening
        return "semiglobal", SEMI, -u // 4, -u, u, -u, None, batch
    if case == "go_zero":
        return "local", LOCAL, 0, -u // 2, u, -u, None, batch
    if case == "go_eq_ge":
        return "global", GLOBAL, -u, -u, u // 2, -u, None, batch
    raise ValueError(case)


E_CASES = ["exact_2^27_global", "exact_2^27_custom", "clip_minus_2^27", "global_x_short", "custom_y_short", "ge_below_go",
           "go_zero", "go_eq_ge", "asym_table"]


def _e_bound(go, ge, ma, mi, table, batch):
    blob, xo, xl, yo, yl = batch
    present = np.unique(np.concatenate([blob[int(xo[p]):int(xo[p]) + int(xl[p])] for p in range(len(xl))] +
                                       [blob[int(yo[p]):int(yo[p]) + int(yl[p])] for p in range(len(xl))]))
    return score_bound(go, ge, ma, mi, table, present.tobytes(), int(xl.max()), int(yl.max()))


@pytest.mark.parametrize("G,R", [(1, 16), (32, 8)])
@pytest.mark.parametrize("case", E_CASES)
def test_sim_range_guard_accepted_is_exact(oracle, case, G, R):
    mode, clips, go, ge, ma, mi, table, batch = _e_case(case)
    b = _e_bound(go, ge, ma, mi, table, batch)
    assert (1 << 27) * 0.99 < b <= 1 << 27 and (b == 1 << 27 or case.startswith("g"))
    assert tracker_form(flags_of(mode, clips, b, int(batch[2].max()), int(batch[4].max()))) in ("explicit", "none")
    s, keep = oracle.make_scoring(go, ge, ma, mi, table, *clips)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch)
    assert int(np.abs(ref["score"]).max()) > (1 << 27) // (4 if table is not None else 3)
    if case.endswith("short"):  # real 4 * S below -2^28
        assert int(ref["score"].min()) < -(1 << 26)
    for walk in (0, 1):
        got, ops = sim_run(mode, s, batch, G, R, walk)
        assert_same(got, ops, ref, ref_ops, batch, f"{case} G={G} R={R} walk={walk}")
    check_rescore(batch, got, ops, mode, go, ge, _table_fn(table) if table is not None else _unit_fn(ma, mi), clips)


def _dead_clip_batch(seed):
    rng = np.random.default_rng(seed)
    pairs = [make_pair(rng, m, n, "related") for m in range(5) for n in range(5)]
    pairs += [make_pair(rng, int(rng.integers(0, 70)), int(rng.integers(0, 70)), ("related", "disjoint")[q % 2])
              for q in range(40)]
    return pack(pairs)


DEAD_VALUES = [DEAD_CLIP, DEAD_CLIP - 1, MIN + 1, MIN, -(1 << 27), 0, -3]  # (DEAD_CLIP + 1 is live and refused)


@pytest.mark.parametrize("G,R,walk", [(1, 16, 0), (8, 8, 1), (132, 8, 1)])
def test_sim_dead_clip_boundary(oracle, G, R, walk):
    """clips at DEAD_CLIP, just below / above it, MIN_SCORE + 1, MIN_SCORE and -2^27, mixed at random: live but never
    winning penalties behave as the reference's."""
    rng = np.random.default_rng(G + R)
    batch = _dead_clip_batch(G)
    for trial in range(6):
        clips = tuple(int(rng.choice(DEAD_VALUES)) for _ in range(4))
        s, _ = oracle.make_scoring(-5, -2, 3, -4, None, *clips)
        ref, ref_ops = oracle_batch(oracle, "custom", s, batch)
        got, ops = sim_run("custom", s, batch, G, R, walk)
        assert_same(got, ops, ref, ref_ops, batch, f"dead clips {clips} G={G} R={R}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", E_CASES)
def test_gpu_range_guard_accepted_is_exact(eng, oracle, case):
    mode, clips, go, ge, ma, mi, table, batch = _e_case(case)
    s, keep = oracle.make_scoring(go, ge, ma, mi, table, *clips)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
    cs, keep2 = c_scoring(go, ge, ma, mi, clips, table)
    try:
        for G, R in [(0, 0), (1, 16), (8, 20), (32, 8)]:
            eng.set_tuning(G, R)
            for walk in (1, 2):
                eng.set_walk(walk)
                got, ops = gpu_run(eng, mode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"GPU {case} G={G} R={R} walk={walk}")
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)
    check_rescore(batch, got, ops, mode, go, ge, _table_fn(table) if table is not None else _unit_fn(ma, mi), clips)
    if table is not None:  # the entries outside the batch's alphabet change nothing, found or given by the caller
        clean = np.where(np.isin(np.arange(256), np.frombuffer(AA, dtype=np.uint8)), 1, 0)
        clean = (np.asarray(table, dtype=np.int64) * np.outer(clean, clean)).astype(np.int32)
        for alpha in (None, AA):
            cs2, keep3 = c_scoring(go, ge, ma, mi, clips, clean if alpha is None else table, alpha)
            got2, ops2 = gpu_run(eng, mode, cs2, batch)
            assert_same(got2, ops2, ref, ref_ops, batch, f"GPU {case} alphabet={alpha}")


@pytest.mark.gpu
def test_gpu_dead_clip_boundary(eng, oracle):
    rng = np.random.default_rng(71)
    batch = _dead_clip_batch(4)
    for trial in range(10):
        clips = tuple(int(rng.choice(DEAD_VALUES)) for _ in range(4))
        s, _ = oracle.make_scoring(-5, -2, 3, -4, None, *clips)
        ref, ref_ops = oracle_batch(oracle, "custom", s, batch)
        cs, keep = c_scoring(-5, -2, 3, -4, clips)
        got, ops = gpu_run(eng, "custom", cs, batch)
        assert_same(got, ops, ref, ref_ops, batch, f"GPU dead clips {clips}")


REFUSED = {
    "bound_2^27+1": "i32-safe range",
    "table_entry_2^27+1": "substitution score magnitude above 2\\^27",
    "clip_minus_2^27-1": "clip penalty between -2\\^27",
    "clip_below_MIN_SCORE": "clip penalty below MIN_SCORE",
}


@pytest.mark.gpu
@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("case", list(REFUSED))
def test_gpu_range_guard_refuses(eng, case, banded):
    from rust_bio_b200._lib import B2AError
    rng = np.random.default_rng(1)
    batch = pack([make_pair(rng, 150, 150, "related") for _ in range(4)])
    u, go = unit_go(1 << 27, 302)
    table = None
    clips = GLOBAL
    if case == "bound_2^27+1":
        go -= 1
        assert score_bound(go, -u, u, -u, None, None, 150, 150) == (1 << 27) + 1
    elif case == "table_entry_2^27+1":
        u, go = 1000, -5
        table = np.full((256, 256), -3, dtype=np.int32)
        table[ord("G"), ord("T")] = (1 << 27) + 1  # G and T both occur
    elif case == "clip_minus_2^27-1":
        u, go = 1000, -5
        clips = (MIN, -(1 << 27) - 1, MIN, MIN)
    else:
        u, go = 1000, -5
        clips = (MIN - 1, MIN, MIN, MIN)
    cs, keep = c_scoring(go, -u, u, -u, clips, table)
    with pytest.raises(B2AError, match="B2A_E_RANGE: .*" + REFUSED[case]):
        if banded:
            eng.align_batch_banded(MODES["custom"], cs, 8, 8, batch)
        else:
            eng.align_batch(MODES["custom"], cs, batch)
    # and one step back inside the guard runs
    if case == "bound_2^27+1":
        go += 1
    elif case == "table_entry_2^27+1":  # on a 1 x 1 pair (L = 4) an entry of 2^25 makes the bound 2^27 exactly
        table[ord("G"), ord("T")] = 1 << 25
        go = 0
        batch = pack([(b"G", b"T")])
    elif case == "clip_minus_2^27-1":
        clips = (MIN, -(1 << 27), MIN, MIN)
    else:
        clips = (MIN, MIN, MIN, MIN)
    cs, keep = c_scoring(go, -u, u, -u, clips, table)
    if banded:
        eng.align_batch_banded(MODES["custom"], cs, 8, 8, batch)
    else:
        eng.align_batch(MODES["custom"], cs, batch)


# ---------------------------------------------------------------------------------------------------------------
# f. the banded strip gate (b2a_plan.h banded_strip_gate)

def _window_pairs(seed, n_pairs, xlen, ylen, sub=0.05):
    """reads that are mutated windows of longer sequences (the banded aligner's use)"""
    rng = np.random.default_rng(seed)
    pairs = []
    for _ in range(n_pairs):
        xl = int(rng.integers(xlen // 2, xlen + 1)) if n_pairs > 1 else xlen
        yl = int(rng.integers(max(xl + 50, ylen // 2), ylen + 1)) if n_pairs > 1 else ylen
        y = DNA[rng.integers(0, 4, yl)]
        st = int(rng.integers(0, yl - xl + 1)) if yl > xl else 0
        x = _mutate(rng, y[st:st + xl], sub)
        pairs.append((bytes(x), bytes(y)))
    return pairs


# (mode, clips, bound inside the gate, bound outside it)
F_CASES = {
    "local": ("local", LOCAL, (1 << 17) - 1, 1 << 17),
    "custom_yp_ys": ("custom", (MIN, MIN, "c", "c"), (1 << 17) - 1, 1 << 17),
    "custom_yp_xs": ("custom", (MIN, "c", 0, MIN), (1 << 17) - 1, 1 << 17),
    "semiglobal": ("semiglobal", SEMI, (1 << 17) - 1, 1 << 17),  # the y clips of the preset are live: row trackers
    "global": ("global", GLOBAL, (1 << 26) - 1, 1 << 26),  # no trackers: the strip fill's own range
    "custom_xp": ("custom", ("c", MIN, MIN, MIN), (1 << 26) - 1, 1 << 26),
}


def _f_scoring(case, target, maxm, maxn):
    """at most the inside bound, at least the outside one"""
    omode, clips, _, outside = F_CASES[case]
    u, go = unit_go(target, maxm + maxn + 2, above=target == outside)
    clips = tuple(-2 * u if c == "c" else c for c in clips)
    return omode, clips, go, -max(1, u // 3), u, -u


def _band_ref(oracle, omode, s, k, w, pairs):
    return [oracle.banded_align(omode, s, k, w, x, y) for x, y in pairs]


@pytest.mark.parametrize("has_ms", [1, 0], ids=["sdpkpp_bands", "lcskpp_bands"])
@pytest.mark.parametrize("case", list(F_CASES))
def test_sim_banded_strip_gate(oracle, case, has_ms):
    pairs = _window_pairs(31 + len(case), 4, 200, 600)
    maxm, maxn = max(len(x) for x, _ in pairs), max(len(y) for _, y in pairs)
    k, w = 6, 8
    for side, target in (("inside", F_CASES[case][2]), ("outside", F_CASES[case][3])):
        omode, clips, go, ge, ma, mi = _f_scoring(case, target, maxm, maxn)
        b = score_bound(go, ge, ma, mi, None, None, maxm, maxn)
        assert abs(b - target) < 2 * (maxm + maxn + 3), (b, target)
        assert strip_gate(omode, clips, b, maxm) == (side == "inside"), (case, side, b)
        s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips, has_match_scores=has_ms)
        got = sim_util.banded_strip_task(MODES[omode], s, k, w, pairs)
        if side == "outside":
            assert all(g is None for g in got), case
            continue
        assert sum(g is not None for g in got) >= (1 if case == "custom_xp" else 2), case
        for (x, y), g, (ref, ref_ops) in zip(pairs, got, _band_ref(oracle, omode, s, k, w, pairs)):
            if g is not None:
                assert g[0] == {f: ref[f] for f in g[0]} and g[1] == ref_ops, (case, len(x), len(y))
        # the column loops (K4 + K3 on the host) agree on both sides
        res = sim_util.banded_batch(MODES[omode], s, k, w, *pack(pairs))
        for p, (ref, ref_ops) in enumerate(_band_ref(oracle, omode, s, k, w, pairs)):
            assert int(res[0]["score"][p]) == ref["score"] and res[1][p] == ref_ops, (case, p)


def test_sim_banded_strip_gate_edges():
    """the gate's own edges, with the mode presets applied"""
    for mode, clips in [("local", LOCAL), ("custom", (MIN, MIN, 0, -3)), ("custom", (MIN, -3, 0, MIN))]:
        assert strip_gate(mode, clips, (1 << 17) - 1, 4095) and not strip_gate(mode, clips, 1 << 17, 4095)
    assert strip_gate("custom", (MIN, -3, 0, MIN), 1000, 4095) and not strip_gate("custom", (MIN, -3, 0, MIN), 1000, 4096)
    assert strip_gate("custom", (MIN, MIN, 0, -3), 1000, 4096)  # no column tracker: x may be longer
    assert not strip_gate("custom", (MIN, MIN, MIN, -3), 1000, 100)  # live tracker, y prefix dead: S not always real
    assert strip_gate("semiglobal", None, (1 << 17) - 1, 10000) and not strip_gate("semiglobal", None, 1 << 17, 10000)
    for mode, clips in [("global", None), ("custom", (-3, MIN, MIN, MIN))]:
        assert strip_gate(mode, clips, (1 << 26) - 1, 10000) and not strip_gate(mode, clips, 1 << 26, 10000)
    assert strip_gate("custom", (DEAD_CLIP, DEAD_CLIP, DEAD_CLIP, DEAD_CLIP), (1 << 26) - 1, 10)  # DEAD_CLIP is dead
    assert not strip_gate("custom", (MIN, DEAD_CLIP + 1, 0, MIN), 1000, 10000)


def _padding_table():
    """+2 / -3 over ACGT, and 5,000 in the row and column of byte 0 (pack_pairs' padding between sequences)"""
    t = np.zeros((256, 256), dtype=np.int32)
    idx = np.frombuffer(b"ACGT", dtype=np.uint8)
    t[np.ix_(idx, idx)] = -3
    t[idx, idx] = 2
    t[0, :] = t[:, 0] = 5000
    return t


def test_sim_banded_padding_counts_without_a_caller_alphabet(oracle):
    """Without a caller alphabet the alphabet is every byte value of the blob, the padding between sequences included
    (b2a_scoring.alphabet in b200align.h): byte 0's entries then set score_bound (about 800 x 5,000 here, over the
    gate's 2^17), and the local batch stays with the column loops.  With the alphabet "ACGT" the bound is about 4,000
    and the strip fill takes the pairs, with the oracle's results."""
    pairs = _window_pairs(5, 4, 200, 600)
    assert 0 in np.frombuffer(pack(pairs)[0], dtype=np.uint8)
    t = _padding_table()
    s, keep = oracle.make_scoring(-5, -1, 0, 0, t)
    assert all(g is None for g in sim_util.banded_strip_task(MODES["local"], s, 6, 8, pairs))
    alpha = np.frombuffer(b"ACGT", dtype=np.uint8).copy()
    s.alphabet, s.alphabet_len = alpha.ctypes.data_as(C.c_void_p), len(alpha)
    got = sim_util.banded_strip_task(MODES["local"], s, 6, 8, pairs)
    assert sum(g is not None for g in got) >= 2
    for (x, y), g in zip(pairs, got):
        if g is not None:
            ref, ref_ops = oracle.banded_align("local", s, 6, 8, x, y)
            assert g[0] == {f: ref[f] for f in g[0]} and g[1] == ref_ops


@pytest.mark.gpu
def test_gpu_padding_counts_without_a_caller_alphabet(eng, oracle):
    """The same rule at the range guard: an entry above 2^27 in byte 0's row refuses the batch unless the caller
    gives the alphabet; given, the results are the oracle's."""
    from rust_bio_b200._lib import B2AError
    pairs = _window_pairs(6, 40, 150, 400)
    batch = pack(pairs)
    t = _padding_table()
    t[0, :] = t[:, 0] = (1 << 27) + 1
    cs, keep = c_scoring(-5, -1, 0, 0, LOCAL, t)
    with pytest.raises(B2AError, match="B2A_E_RANGE: substitution score magnitude above 2\\^27"):
        gpu_run(eng, "local", cs, batch)
    cs, keep = c_scoring(-5, -1, 0, 0, LOCAL, t, b"ACGT")
    s, keep2 = oracle.make_scoring(-5, -1, 0, 0, t)
    ref, ref_ops = oracle_batch(oracle, "local", s, batch)
    got, ops = gpu_run(eng, "local", cs, batch)
    assert_same(got, ops, ref, ref_ops, batch, "caller alphabet over a padded blob")


def test_sim_banded_x_limit_4095_with_x_suffix_clip(oracle):
    """x = 4095 (strip path) against 4096 (column loops) with a live x-suffix clip and a live y prefix clip"""
    for lim in (4095, 4096):
        pairs = _window_pairs(lim, 1, lim, 4400, 0.03)
        L = lim + 4400 + 2
        u, go = unit_go((1 << 17) - 1, L)
        clips = (MIN, -2 * u, 0, MIN)
        b = score_bound(go, -u, u, -u, None, None, lim, 4400)
        assert strip_gate("custom", clips, b, lim) == (lim == 4095)
        s, _ = oracle.make_scoring(go, -u, u, -u, None, *clips, has_match_scores=1)
        g = sim_util.banded_strip_task(MODES["custom"], s, 12, 10, pairs)[0]
        if lim == 4096:
            assert g is None
            continue
        ref, ref_ops = oracle.banded_align("custom", s, 12, 10, *pairs[0])
        assert g is not None and g[0] == {f: ref[f] for f in g[0]} and g[1] == ref_ops


@pytest.mark.gpu
@pytest.mark.parametrize("has_ms", [1, 0], ids=["sdpkpp_bands", "lcskpp_bands"])
@pytest.mark.parametrize("case", list(F_CASES) + ["x_limit", "under_2^27"])
def test_gpu_banded_strip_gate(oracle, case, has_ms, monkeypatch):
    """banded_strip_pairs() shows which path ran; results equal the oracle, the column loops (B2A_BANDED_STRIP=0) and,
    for dead trackers, the literal K3 loop (B2A_BANDED_LITERAL=1)"""
    from rust_bio_b200.engine import Engine
    engines = {"strip": Engine(0)}
    monkeypatch.setenv("B2A_BANDED_STRIP", "0")
    engines["loops"] = Engine(0)
    monkeypatch.delenv("B2A_BANDED_STRIP")
    monkeypatch.setenv("B2A_BANDED_LITERAL", "1")
    engines["literal"] = Engine(0)
    monkeypatch.delenv("B2A_BANDED_LITERAL")
    k, w = 6, 8
    try:
        if case == "x_limit":
            sides = []
            for lim in (4095, 4096):
                pairs = _window_pairs(lim, 1, lim, 4400, 0.03) * 3
                u, go = unit_go((1 << 17) - 1, lim + 4400 + 2)
                sides.append(("inside" if lim == 4095 else "outside", pairs, ("custom", (MIN, -2 * u, 0, MIN), go, -u, u, -u)))
        elif case == "under_2^27":  # the K3 column loops, whose arithmetic is in the plain domain
            pairs = _window_pairs(77, 60, 300, 900)
            maxm, maxn = max(len(x) for x, _ in pairs), max(len(y) for _, y in pairs)
            u, go = unit_go((1 << 27) - 1, maxm + maxn + 2)
            sides = [("outside", pairs, ("semiglobal", SEMI, go, -u, u, -u)), ("outside", pairs, ("local", LOCAL, go, -u, u, -u)),
                     ("outside", pairs, ("custom", (-u, -3 * u, 0, -2 * u), go, -u, u, -u))]
        else:
            pairs = _window_pairs(131 + len(case), 80, 300, 900)
            maxm, maxn = max(len(x) for x, _ in pairs), max(len(y) for _, y in pairs)
            sides = [(side, pairs, _f_scoring(case, F_CASES[case][2 if side == "inside" else 3], maxm, maxn))
                     for side in ("inside", "outside")]
        for side, pairs, (omode, clips, go, ge, ma, mi) in sides:
            batch = pack(pairs)
            maxm, maxn = int(batch[2].max()), int(batch[4].max())
            b = score_bound(go, ge, ma, mi, None, None, maxm, maxn)
            assert strip_gate(omode, clips, b, maxm) == (side == "inside"), (case, side, b)
            s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips, has_match_scores=has_ms)
            cs, keep = c_scoring(go, ge, ma, mi, clips, has_ms=has_ms)
            ref, rops, roff, _, ref_cells = oracle.banded_align_batch(omode, s, k, w, *batch, threads=8)
            out = {}
            for name, e in engines.items():
                out[name] = e.align_batch_banded(MODES[omode], cs, k, w, batch)
                taken = e.banded_strip_pairs()
                if name != "strip" or side == "outside":
                    assert taken == 0, (case, side, name)
                else:  # (x-prefix-only pairs whose final score is not real are handed back to the column loops)
                    assert taken * (10 if case == "custom_xp" else 2) >= len(pairs), (case, taken)
                assert int(e.stats.cells) == ref_cells
            for name, a in out.items():
                for f in ("score", "xstart", "xend", "ystart", "yend"):
                    assert np.array_equal(getattr(a, f).astype(np.int64), ref[f].astype(np.int64)), (case, side, name, f)
                for p in range(len(pairs)):
                    want = [(int(v) & 7, int(v) >> 3) for v in rops[int(roff[p]):int(roff[p]) + int(ref["n_ops"][p])]]
                    assert a.ops_of(p) == want, (case, side, name, p)
    finally:
        for e in engines.values():
            e.close()
