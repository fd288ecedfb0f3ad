"""Score-only batches (b2a_batch_stage_scores / b2a_align_batch_scores): Alignment.score, xend and yend without the
traceback.  On the host (tests/sim/b2a_sim_scores.cpp: the F_NOTB fill and the score-only K2 against the oracle, with
no traceback arena and with a poisoned one that must stay untouched; the score-only plan) and on the GPU (against the
full path for every mode, fill shape and walk form; long sequences; a C2-sized batch; waves; the error paths)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import sim_util
from parity_util import MODES, oracle_batch
from rust_bio_b200 import synth

MIN = -858993459
F_TR, F_TC, F_CX, F_LUT, F_PK, F_RELU, F_PR, F_BND8, F_NOTB = 1, 2, 4, 8, 16, 32, 128, 256, 512
FIELDS = ("score", "xend", "yend")
CLIPS = {"custom": (-3, -7, 0, -9), "global": (MIN,) * 4, "semiglobal": (MIN,) * 4, "local": (MIN,) * 4}

SIMS_SRC = os.path.join(sim_util.HERE, "sim", "b2a_sim_scores.cpp")
SIMS_SO = os.path.join(sim_util.HERE, "sim", "libb2asim_scores.so")
_sims = None


def _sims_lib():
    """tests/sim/b2a_sim_scores.cpp, built on first use"""
    global _sims
    if _sims is None:
        deps = [SIMS_SRC] + sim_util.DEPS
        if not os.path.exists(SIMS_SO) or any(os.path.getmtime(d) > os.path.getmtime(SIMS_SO) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                                   "-o", SIMS_SO, SIMS_SRC])
        _sims = C.CDLL(SIMS_SO)
        for fn in (_sims.sims_align_scores, _sims.sims_fill_flags, _sims.sims_plan_waves):
            fn.restype = C.c_int
    return _sims


def _sims_run(mode, orc_scoring, batch, G, R, warp_walk, poison):
    s = sim_util.SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob, x_off, x_len, y_off, y_len = [np.ascontiguousarray(a) for a in batch]
    n = len(x_len)
    out = {"score": np.zeros(n, np.int32), "xend": np.zeros(n, np.uint32), "yend": np.zeros(n, np.uint32),
           "status": np.zeros(n, np.uint32)}
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    L = _sims_lib()
    rc = L.sims_align_scores(int(mode), C.byref(s), p(blob), p(x_off), p(x_len), p(y_off), p(y_len), C.c_uint64(n),
                             int(G), int(R), int(warp_walk), 0x3C, int(poison), p(out["score"]), p(out["xend"]),
                             p(out["yend"]), p(out["status"]))
    assert rc != -3, "the score-only fill or walk wrote into the traceback arena"
    assert rc == 0, rc
    return out, L.sims_fill_flags()


def sim_scores(mode, orc_scoring, batch, G, R, warp_walk):
    """The score-only fill + K2 on the host with tb = nullptr, then again with a poisoned traceback arena (of the full
    path's size), which must come back byte for byte unchanged and give the same results."""
    a, flags = _sims_run(mode, orc_scoring, batch, G, R, warp_walk, -1)
    b, _ = _sims_run(mode, orc_scoring, batch, G, R, warp_walk, 0xA5)
    for k in a:
        assert np.array_equal(a[k], b[k]), ("result depends on the traceback arena", k)
    assert flags & F_NOTB, flags
    return a, flags


def assert_scores_match_oracle(got, ref, batch, what):
    """every pair whose oracle call returns: score, xend, yend equal, status 0"""
    ok = ref["n_ops"] != 0xFFFFFFFF
    for f in FIELDS:
        bad = np.nonzero(ok & (np.asarray(got[f]).astype(np.int64) != ref[f].astype(np.int64)))[0]
        if len(bad):
            p = int(bad[0])
            raise AssertionError(f"{what}: {f} differs for {len(bad)} pairs; first pair {p} (m={batch[2][p]}, "
                                 f"n={batch[4][p]}): got {got[f][p]} ref {ref[f][p]}")
    assert not np.any(got["status"][ok]), what


def edge_batch(seed, n, max_m, max_n, alphabet=synth.DNA):
    """ragged lengths in [0, max], with every combination of m, n in {0, 1, 2} present"""
    rng = np.random.default_rng(seed)
    xl = rng.integers(0, max_m + 1, n).astype(np.uint32)
    yl = rng.integers(0, max_n + 1, n).astype(np.uint32)
    small = [(a, b) for a in range(3) for b in range(3)] + [(a, max_n) for a in range(3)] + [(max_m, b) for b in range(3)]
    for k, (a, b) in enumerate(small):
        xl[k * 3 % n], yl[k * 3 % n] = a, b
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    lens = np.stack([xl, yl], axis=1).reshape(-1).astype(np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    blob = alpha[rng.integers(0, len(alpha), int(lens.sum()) + 1)]
    for p in range(n):  # related pairs, so that local / clipped alignments end inside the matrix
        xo, yo, k = int(offs[2 * p]), int(offs[2 * p + 1]), int(min(xl[p], yl[p]))
        if k > 4 and p % 2:
            src = blob[xo:xo + k].copy()
            mut = rng.random(k) < 0.15
            src[mut] = alpha[rng.integers(0, len(alpha), int(mut.sum()))]
            blob[yo:yo + k] = src
    return blob, offs[0::2].copy(), xl, offs[1::2].copy(), yl


# (Gsel, R, warp_walk): Gsel 132 = 32x8 with strip-pipelined (pair, strip) tasks
SIM_SHAPES = [(1, 16, 0), (1, 16, 1), (8, 20, 0), (8, 20, 1), (132, 8, 0), (132, 8, 1)]
SIM_IDS = ["1x16-lane", "1x16-warp", "8x20-lane", "8x20-warp", "32x8piped-lane", "32x8piped-warp"]


# ------------------------------------------------------------------------------------------------ host (not-gpu)

@pytest.mark.parametrize("G,R,warp_walk", SIM_SHAPES, ids=SIM_IDS)
@pytest.mark.parametrize("mode", list(MODES))
def test_sim_scores_vs_oracle(oracle, mode, G, R, warp_walk):
    """Ragged batches with m, n in {0, 1, 2} among them; the piped shape gets pairs of 1-3 strips of 256 rows."""
    batch = edge_batch(31 + G + R, 24, 600, 300) if G == 132 else edge_batch(7 + G + R, 80, 70, 60)
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    ref, _ = oracle_batch(oracle, mode, s, batch)
    got, flags = sim_scores(MODES[mode], s, batch, G, R, warp_walk)
    if mode != "global":
        assert flags & (F_PK | F_PR), flags
    assert_scores_match_oracle(got, ref, batch, f"{mode} G={G} R={R} warp_walk={warp_walk}")


def test_sim_scores_take_the_8_byte_record(oracle):
    """C2-like scoring: the score-only fill runs with F_BND8 as the full one does (stage_front's choice)."""
    batch = edge_batch(3, 64, 100, 100)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, _ = oracle_batch(oracle, "local", s, batch)
    got, flags = sim_scores(MODES["local"], s, batch, 1, 16, 0)
    assert flags & F_BND8 and flags & F_PK, flags
    assert_scores_match_oracle(got, ref, batch, "local bnd8")


@pytest.mark.parametrize("seed", range(6))
def test_sim_scores_random_custom_clips(oracle, seed):
    """Arbitrary live / dead mixes of the four clip penalties (the suffix clips decide xend / yend)."""
    rng = np.random.default_rng(700 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    go, ge = int(rng.choice([0, -1, -2, -5])), int(rng.choice([0, -1, -2]))
    ma, mi = int(rng.choice([1, 2, 4])), int(rng.choice([-1, -3, 0]))
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, pick(), pick(), pick(), pick())
    batch = edge_batch(seed, 64, 50, 45, alphabet=b"AC" if seed % 2 else b"ACGT")
    ref, _ = oracle_batch(oracle, "custom", s, batch)
    G, R, ww = SIM_SHAPES[seed % 4]
    got, _ = sim_scores(MODES["custom"], s, batch, G, R, ww)
    assert_scores_match_oracle(got, ref, batch, f"custom seed={seed} G={G} warp_walk={ww}")


@pytest.mark.parametrize("G,R,warp_walk", [(1, 16, 0), (8, 20, 1)], ids=["1x16-lane", "8x20-warp"])
def test_sim_scores_blosum62(oracle, G, R, warp_walk):
    """A tabulated MatchFunc through the LUT (protein, BLOSUM62)."""
    from rust_bio_b200 import scores
    table = scores.matrix_table256("blosum62")
    batch = edge_batch(11, 64, 60, 60, alphabet=synth.PROTEIN)
    for mode, go in (("local", -10), ("global", -5), ("semiglobal", -11), ("custom", -8)):
        s, keep = oracle.make_scoring(go, -1, 0, 0, table, *CLIPS[mode])
        ref, _ = oracle_batch(oracle, mode, s, batch)
        got, flags = sim_scores(MODES[mode], s, batch, G, R, warp_walk)
        assert flags & F_LUT, flags
        assert_scores_match_oracle(got, ref, batch, f"blosum62 {mode}")


def test_sim_score_only_plan():
    """The score-only plan stores no traceback, and a batch that needs >= 10 waves of traceback on the full path's
    budget (C5's shape: 10,000 pairs of 10k x 10k against 48 GB, 60 % of a free H100) fits in one."""
    L = _sims_lib()
    n = 10000
    xl = np.full(n, 10000, np.uint32)
    yl = np.full(n, 10000, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    tb = C.c_uint64(0)
    budget = C.c_uint64(48 * 10 ** 9)
    flags = F_TR | F_TC | F_CX | F_LUT | F_RELU | F_PR
    full = L.sims_plan_waves(p(xl), p(yl), C.c_uint64(n), 32, 16, budget, flags, C.byref(tb))
    assert full >= 10 and tb.value > 10 * budget.value, (full, tb.value)
    so = L.sims_plan_waves(p(xl), p(yl), C.c_uint64(n), 32, 16, budget, flags | F_NOTB, C.byref(tb))
    assert so == 1 and tb.value == 0, (so, tb.value)
    # a budget below the batch's other scratch still cuts score-only waves (and C2's shape)
    xl2 = np.full(100000, 150, np.uint32)
    so2 = L.sims_plan_waves(p(xl2), p(xl2), C.c_uint64(100000), 1, 16, C.c_uint64(64 << 20),
                            F_TR | F_TC | F_CX | F_LUT | F_RELU | F_PK | F_BND8 | F_NOTB, C.byref(tb))
    assert so2 > 1 and tb.value == 0


# ------------------------------------------------------------------------------------------------ GPU

def _cs(mode, go=-5, ge=-1, ma=2, mi=-3, table=None, alphabet=None):
    from rust_bio_b200._lib import CScoring
    c = CLIPS[mode]
    cs = CScoring(go, ge, c[0], c[1], c[2], c[3], ma, mi, 1 if table is None else 0, None, None, 0)
    if table is not None:
        cs.table = table.ctypes.data_as(C.c_void_p)
        cs.alphabet = alphabet.ctypes.data_as(C.c_void_p)
        cs.alphabet_len = len(alphabet)
    return cs


def _full(eng, mode, cs, batch):
    from rust_bio_b200.engine import Results
    res = eng.align_batch(MODES[mode], cs, batch, results=Results(len(batch[2]), eng.default_ops_capacity(batch),
                                                                  pair_status=True))
    out = {f: getattr(res, f)[:res.n_pairs].copy() for f in FIELDS}
    out["status"] = res.status[:res.n_pairs].copy()
    return out


def assert_same_as_full(got, full, what):
    """score, xend, yend and status of every pair equal the full path's (pairs the full path reports as panicking:
    see test_gpu_scores_panicking_pairs)"""
    ok = full["status"] == 0
    for f in FIELDS:
        bad = np.nonzero(ok & (got[f].astype(np.int64) != full[f].astype(np.int64)))[0]
        assert not len(bad), f"{what}: {f} differs for {len(bad)} pairs; first {int(bad[0])}: " \
                             f"{got[f][bad[0]]} vs {full[f][bad[0]]}"
    assert np.array_equal(got["status"][ok], full["status"][ok]), what
    check_panicking(got, full, what)


def check_panicking(got, full, what):
    """The documented behaviour on pairs the full path reports as panicking: a panic met on row m / column n is
    B2A_PAIR_PANIC here too (score MIN_SCORE); one only the interior walk meets cannot be seen, so the pair reports a
    score.  A pair the full path finishes never panics here."""
    for p in np.nonzero(full["status"] != 0)[0]:
        s = int(got["status"][p])
        print(f"{what}: pair {p}: full path status {int(full['status'][p])}, score-only status {s}, "
              f"score {int(got['score'][p])}")
        assert s in (0, 1)
        if s:
            assert int(got["score"][p]) == MIN and int(got["xend"][p]) == 0 and int(got["yend"][p]) == 0
    assert not np.any(got["status"][full["status"] == 0])


GPU_SHAPES = [(1, 16), (8, 16), (8, 20), (32, 8), (32, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("walk", [1, 2], ids=["lane_walk", "warp_walk"])
@pytest.mark.parametrize("G,R", GPU_SHAPES, ids=[f"{g}x{r}" for g, r in GPU_SHAPES])
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_scores_vs_full(oracle, mode, G, R, walk):
    from rust_bio_b200.engine import Engine
    batch = edge_batch(100 + G + R, 600, 300, 260)
    cs = _cs(mode)
    eng = Engine(0)
    try:
        eng.set_tuning(G, R)
        eng.set_walk(walk)
        full = _full(eng, mode, cs, batch)
        got = eng.align_batch_scores(MODES[mode], cs, batch)
        assert (eng.stats.fill_lanes_per_pair, eng.stats.fill_rows_per_lane) == (G, R)
        assert eng.stats.traceback_bytes == 0
    finally:
        eng.close()
    assert_same_as_full(got, full, f"{mode} {G}x{R} walk={walk}")
    # an oracle sample
    k = 96
    sample = tuple(a[:k].copy() if i else a for i, a in enumerate(batch))
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    ref, _ = oracle_batch(oracle, mode, s, sample)
    assert_scores_match_oracle({f: got[f][:k] for f in got}, ref, sample, f"oracle sample {mode} {G}x{R}")


@pytest.mark.gpu
@pytest.mark.parametrize("walk", [1, 2], ids=["lane_walk", "warp_walk"])
@pytest.mark.parametrize("G,R", GPU_SHAPES, ids=[f"{g}x{r}" for g, r in GPU_SHAPES])
def test_gpu_scores_c1(G, R, walk):
    """C1: 1,000 pairs of 150 x 150, local, MatchParams(1, -1), gap -5 / -1."""
    from rust_bio_b200.engine import Engine
    batch = synth.uniform_pairs(synth.BASES["C1"], 0, 1000, 150, 150)
    cs = _cs("local", -5, -1, 1, -1)
    eng = Engine(0)
    try:
        eng.set_tuning(G, R)
        eng.set_walk(walk)
        full = _full(eng, "local", cs, batch)
        got = eng.align_batch_scores(MODES["local"], cs, batch)
    finally:
        eng.close()
    assert_same_as_full(got, full, f"C1 {G}x{R} walk={walk}")


@pytest.mark.gpu
@pytest.mark.parametrize("no_packrel", [0, 1], ids=["relative_keys", "explicit_trackers"])
@pytest.mark.parametrize("mode", ["local", "custom", "semiglobal"])
def test_gpu_scores_long_4200(monkeypatch, mode, no_packrel):
    """4,200-long pairs: the long-sequence trackers (F_PACKREL), and with B2A_NO_PACKREL=1 the explicit ones."""
    from rust_bio_b200.engine import Engine
    monkeypatch.setenv("B2A_NO_PACKREL", str(no_packrel))
    batch = synth.mutated_window_pairs(synth.BASES["C4"], 0, 12, 4200, 4800)
    cs = _cs(mode)
    eng = Engine(0)
    try:
        full = _full(eng, mode, cs, batch)
        got = eng.align_batch_scores(MODES[mode], cs, batch)
    finally:
        eng.close()
    assert_same_as_full(got, full, f"4200 {mode} no_packrel={no_packrel}")


@pytest.mark.gpu
def test_gpu_scores_10k_blosum62():
    """8 pairs of 10k x 10k protein, BLOSUM62, local (C5's shape)."""
    from rust_bio_b200 import scores
    from rust_bio_b200.engine import Engine
    table = np.ascontiguousarray(scores.matrix_table256("blosum62"), dtype=np.int32)
    alphabet = np.frombuffer(bytes(range(65, 91)) + b"*", dtype=np.uint8).copy()
    batch = synth.uniform_pairs(synth.BASES["C5"], 0, 8, 10000, 10000, alphabet=synth.PROTEIN)
    cs = _cs("local", -11, -1, 0, 0, table, alphabet)
    eng = Engine(0)
    try:
        full = _full(eng, "local", cs, batch)
        got = eng.align_batch_scores(MODES["local"], cs, batch)
        assert eng.stats.traceback_bytes == 0
    finally:
        eng.close()
    assert_same_as_full(got, full, "10k blosum62 local")


@pytest.mark.gpu
def test_gpu_scores_c2_1m():
    """C2: 1,000,000 pairs of 150 x 150 local; the full call runs its chunk pipeline, the score-only call one shot."""
    from rust_bio_b200.engine import Engine
    batch = synth.uniform_pairs(synth.BASES["C2"], 0, 1_000_000, 150, 150)
    cs = _cs("local", -5, -1, 1, -1)
    eng = Engine(0)
    try:
        full = _full(eng, "local", cs, batch)
        got = eng.align_batch_scores(MODES["local"], cs, batch)
        assert eng.stats.traceback_bytes == 0
        assert eng.stats.waves == 1
    finally:
        eng.close()
    assert_same_as_full(got, full, "C2 1M")
    assert not np.any(full["status"])


@pytest.mark.gpu
def test_gpu_scores_wave_budget():
    """A traceback budget that cuts the full path into many waves: the score-only batch runs in one, same results."""
    from rust_bio_b200.engine import Engine
    batch = synth.uniform_pairs(synth.BASES["C3"], 0, 1000, 1000, 1000)
    cs = _cs("global", -5, -1, 1, -1)
    eng = Engine(0)
    try:
        eng.set_traceback_budget(48 << 20)
        full = _full(eng, "global", cs, batch)
        full_waves = eng.stats.waves
        got = eng.align_batch_scores(MODES["global"], cs, batch)
        assert eng.stats.waves == 1, eng.stats.waves
    finally:
        eng.close()
    assert full_waves >= 5, full_waves
    assert_same_as_full(got, full, "wave budget")


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [0, 1], ids=["tail_split", "small_batch_overlap"])
def test_gpu_scores_small_batch_paths(monkeypatch, overlap):
    """The launch structures of small batches (tail-aware split by default, sub-range overlap with B2A_OVERLAP=1):
    10k uniform local and 5,000 ragged custom."""
    from rust_bio_b200.engine import Engine
    monkeypatch.setenv("B2A_OVERLAP", str(overlap))
    eng = Engine(0)
    try:
        for mode, batch, cs in (("local", synth.uniform_pairs(synth.BASES["C2"], 0, 10000, 150, 150), _cs("local", -5, -1, 1, -1)),
                                ("custom", edge_batch(5, 5000, 200, 180), _cs("custom"))):
            full = _full(eng, mode, cs, batch)
            got = eng.align_batch_scores(MODES[mode], cs, batch)
            assert_same_as_full(got, full, f"small batch {mode} overlap={overlap}")
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_scores_error_paths():
    from rust_bio_b200._lib import B2AError, CStats
    from rust_bio_b200.engine import Engine, Results, ScoreResults
    batch = edge_batch(9, 200, 120, 100)
    cs = _cs("custom")
    eng = Engine(0)
    L, h = eng._L, eng._h
    try:
        first = _full(eng, "custom", cs, batch)
        # a forced shape without a score-only fill
        eng.set_tuning(1, 8)
        with pytest.raises(B2AError) as ei:
            eng.align_batch_scores(MODES["custom"], cs, batch)
        assert ei.value.code == -7 and "score-only" in str(ei.value)
        eng.set_tuning(0, 0)
        eng.stage_scores(MODES["custom"], cs, batch)
        eng.run()
        # fetch with any of the full path's outputs
        res = Results(len(batch[2]), eng.default_ops_capacity(batch), pair_status=True)
        assert L.b2a_batch_fetch(h, C.byref(res.c), C.byref(CStats())) == -1
        for f in ("xstart", "ystart", "ops", "ops_off", "clip_len"):  # one of them set at a time
            sr = ScoreResults(len(batch[2]))
            setattr(sr.c, f, res.c.score)
            assert L.b2a_batch_fetch(h, C.byref(sr.c), None) == -1, f
        # records, compact segments, gathered fetch
        buf, stride, nrec = C.c_void_p(), C.c_uint32(), C.c_uint64()
        assert L.b2a_batch_records(h, C.byref(buf), C.byref(stride), C.byref(nrec)) == -6
        assert L.b2a_batch_records_into(h, C.c_void_p(1), C.c_uint64(1 << 30), C.byref(stride)) == -6
        nb = C.c_uint64()
        assert L.b2a_batch_compact_bytes(h, C.byref(nb)) == -6
        assert L.b2a_batch_compact_into(h, C.c_void_p(1), C.c_uint64(1 << 30)) == -6
        assert L.b2a_batch_compact_fixed(h, C.c_void_p(1), C.c_uint64(1 << 30)) == -6
        assert L.b2a_gathered_fetch(h, C.c_void_p(1), C.c_uint64(1 << 20), 1, C.byref(res.c), C.byref(nrec),
                                    C.byref(nrec)) == -6
        got = eng.fetch_scores()
        assert_same_as_full(got, first, "staged score-only")
        # full -> score-only -> full on one engine gives the first result again
        again = _full(eng, "custom", cs, batch)
        for f in first:
            assert np.array_equal(first[f], again[f]), f
        assert eng.stats.traceback_bytes > 0
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_gpu_scores_panicking_pairs(seed):
    """Random custom clips and gap costs (the setting where the reference's walk can panic): every pair the full path
    finishes agrees; pairs it reports as panicking are printed and follow the documented behaviour."""
    from rust_bio_b200.engine import Engine
    from rust_bio_b200._lib import CScoring
    rng = np.random.default_rng(900 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    cs = CScoring(int(rng.choice([0, -1, -2, -5])), int(rng.choice([0, -1, -2])), pick(), pick(), pick(), pick(),
                  int(rng.choice([1, 2, 4])), int(rng.choice([-1, -3, 0])), 1, None, None, 0)
    batch = edge_batch(seed, 2000, 90, 80, alphabet=b"AC" if seed % 2 else b"ACGT")
    eng = Engine(0)
    try:
        full = _full(eng, "custom", cs, batch)
        got = eng.align_batch_scores(MODES["custom"], cs, batch)
    finally:
        eng.close()
    print(f"seed {seed}: {int(np.count_nonzero(full['status']))} pairs the full path reports as panicking")
    assert_same_as_full(got, full, f"random clips seed={seed}")
