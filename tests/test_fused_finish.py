"""The thread-per-pair fill that finishes each pair's matrix itself (F_FINISH, b2a_fill.cuh): row m, the literal cells
of column n and both last-column fix-ups run in K1, and K2 loads each pair's EndState instead of running its own finish.
On the host (tests/sim/b2a_sim_finish.cpp: the fused fill + K2 against the oracle and against the same fill without
F_FINISH plus K2's finish, field for field and op for op) and on the GPU (the 1x16 path against the same batch forced
to 8x16, which keeps K2's finish, and against the oracle on a sample)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import sim_util
from parity_util import MODES, assert_same, oracle_batch
from rust_bio_b200 import synth
from test_score_only import edge_batch

MIN = -858993459
F_PK, F_LUT, F_PR, F_BND8, F_NOTB, F_FINISH = 16, 8, 128, 256, 512, 2048
CLIPS = {"custom": (-3, -7, 0, -9), "global": (MIN,) * 4, "semiglobal": (MIN,) * 4, "local": (MIN,) * 4}
OUT = ("score", "xstart", "xend", "ystart", "yend", "n_ops", "status", "clip_len")

SIMF_SRC = os.path.join(sim_util.HERE, "sim", "b2a_sim_finish.cpp")
SIMF_SO = os.path.join(sim_util.HERE, "sim", "libb2asim_finish.so")
_simf = None


def _lib():
    """tests/sim/b2a_sim_finish.cpp, built on first use"""
    global _simf
    if _simf is None:
        deps = [SIMF_SRC] + sim_util.DEPS
        if not os.path.exists(SIMF_SO) or any(os.path.getmtime(d) > os.path.getmtime(SIMF_SO) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                                   "-o", SIMF_SO, SIMF_SRC])
        _simf = C.CDLL(SIMF_SO)
        for fn in (_simf.simf_align_batch, _simf.simf_fill_flags):
            fn.restype = C.c_int
    return _simf


def _run(mode, orc_scoring, batch, R, bits, garbage):
    s = sim_util.SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob, x_off, x_len, y_off, y_len = batch
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    x_off = np.ascontiguousarray(x_off, dtype=np.uint64)
    y_off = np.ascontiguousarray(y_off, dtype=np.uint64)
    x_len = np.ascontiguousarray(x_len, dtype=np.uint32)
    y_len = np.ascontiguousarray(y_len, dtype=np.uint32)
    n = len(x_len)
    cap = x_len.astype(np.uint64) + y_len.astype(np.uint64) + np.uint64(4)
    ops_off = np.concatenate([[0], np.cumsum(cap)]).astype(np.uint64)
    ops = np.zeros(int(ops_off[-1]), dtype=np.uint8)
    out = {k: np.zeros(n, dtype=np.uint32) for k in ("xstart", "xend", "ystart", "yend", "n_ops", "status")}
    out["score"] = np.zeros(n, dtype=np.int32)
    out["clip_len"] = np.zeros(4 * n, dtype=np.uint32)
    untouched = C.c_int32(0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    L = _lib()
    rc = L.simf_align_batch(int(mode), C.byref(s), p(blob), p(x_off), p(x_len), p(y_off), p(y_len), C.c_uint64(n),
                            int(R), int(bits), int(garbage), p(out["score"]), p(out["xstart"]), p(out["xend"]),
                            p(out["ystart"]), p(out["yend"]), p(out["n_ops"]), p(out["clip_len"]), p(out["status"]),
                            p(ops), p(ops_off), C.byref(untouched))
    assert rc == 0, rc
    lists = [sim_util.decode_ops(ops[int(ops_off[i]):int(ops_off[i]) + int(out["n_ops"][i])],
                                 out["clip_len"][4 * i:4 * i + 4]) for i in range(n)]
    return out, lists, L.simf_fill_flags(), untouched.value


def fused_and_unfused(mode, orc_scoring, batch, R=16, bits=0):
    """The fused fill + K2 (its rows arena poisoned: S, I and Sn of every finished pair must come back untouched) and
    the same fill without F_FINISH + K2's finish (other scratch garbage); every output must agree.  -> fused result"""
    a, a_ops, a_flags, untouched = _run(mode, orc_scoring, batch, R, bits | 128, 0x5A)
    b, b_ops, b_flags, _ = _run(mode, orc_scoring, batch, R, bits | 64, 0x00)
    assert a_flags & F_FINISH and not b_flags & F_FINISH, (a_flags, b_flags)
    assert a_flags == b_flags | F_FINISH
    assert untouched == 1, "the fused fill or K2 wrote S, I or Sn of a finished pair into the rows arena"
    for k in OUT:
        if bits & 32 and k not in ("score", "xend", "yend", "status"):
            continue
        bad = np.nonzero(a[k] != b[k])[0]
        assert not len(bad), f"{k} differs from K2's finish at {len(bad)} entries; first {int(bad[0])}"
    if not bits & 32:
        assert a_ops == b_ops
    return a, a_ops, a_flags


def assert_scores(got, ref, what):
    for f in ("score", "xend", "yend"):
        assert np.array_equal(got[f].astype(np.int64), ref[f].astype(np.int64)), (what, f)


# ------------------------------------------------------------------------------------------------ host (not-gpu)

@pytest.mark.parametrize("walk", [0, 8], ids=["lane_walk", "warp_walk"])
@pytest.mark.parametrize("R", [16, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_sim_fused_vs_oracle(oracle, mode, R, walk):
    """Ragged blocks (row m-1 in different strips, m and n in {0, 1, 2} among them, a partial last block)."""
    batch = edge_batch(7 + R, 80, 70, 60)
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    ref, ref_ops = oracle_batch(oracle, mode, s, batch)
    got, ops, flags = fused_and_unfused(MODES[mode], s, batch, R, walk)
    if mode != "global":
        assert flags & F_PK and flags & F_BND8, flags
    assert_same(got, ops, ref, ref_ops, batch, f"{mode} R={R} walk={walk}")


@pytest.mark.parametrize("bits", [2, 4], ids=["explicit_trackers", "matchparams"])
@pytest.mark.parametrize("mode", ["custom", "local", "global"])
def test_sim_fused_tracker_and_score_forms(oracle, mode, bits):
    """The explicit (value, row) trackers with the 16-byte record, and the compare path without the LUT."""
    batch = edge_batch(40 + bits, 70, 50, 50)
    s, _ = oracle.make_scoring(-4, -2, 3, -2, None, *CLIPS[mode])
    ref, ref_ops = oracle_batch(oracle, mode, s, batch)
    got, ops, flags = fused_and_unfused(MODES[mode], s, batch, 16, bits)
    if bits == 2:
        assert not flags & (F_PK | F_BND8), flags
    else:
        assert not flags & F_LUT, flags
    assert_same(got, ops, ref, ref_ops, batch, f"{mode} bits={bits}")


@pytest.mark.parametrize("seed", range(8))
def test_sim_fused_random_custom_clips(oracle, seed):
    """Arbitrary live / dead mixes of the four clips, live suffix clips among them; two-letter alphabets make ties."""
    rng = np.random.default_rng(1700 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    go, ge = int(rng.choice([0, -1, -2, -5])), int(rng.choice([0, -1, -2]))
    ma, mi = int(rng.choice([1, 2, 4])), int(rng.choice([-1, -3, 0]))
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, pick(), pick(), pick(), pick())
    batch = edge_batch(seed, 96, 50, 45, alphabet=b"AC" if seed % 2 else b"ACGT")
    got, ops, _ = fused_and_unfused(MODES["custom"], s, batch, 16 if seed % 4 < 2 else 8, 8 if seed % 3 == 0 else 0)
    ref, ref_ops = oracle_batch(oracle, "custom", s, batch)
    ok = got["status"] == 0  # pairs on which the reference's walk panics are reported, not aligned
    for f in ("score", "xstart", "xend", "ystart", "yend"):
        assert np.array_equal(got[f][ok].astype(np.int64), ref[f][ok].astype(np.int64)), (seed, f)
    assert all(ops[p] == ref_ops[p] for p in np.nonzero(ok)[0])


def test_sim_fused_blosum62(oracle):
    """A tabulated MatchFunc through the LUT (protein, BLOSUM62)."""
    from rust_bio_b200 import scores
    table = scores.matrix_table256("blosum62")
    batch = edge_batch(11, 64, 60, 60, alphabet=synth.PROTEIN)
    for mode, go in (("local", -10), ("global", -5), ("semiglobal", -11), ("custom", -8)):
        s, keep = oracle.make_scoring(go, -1, 0, 0, table, *CLIPS[mode])
        ref, ref_ops = oracle_batch(oracle, mode, s, batch)
        got, ops, flags = fused_and_unfused(MODES[mode], s, batch, 16, 0)
        assert flags & F_LUT, flags
        assert_same(got, ops, ref, ref_ops, batch, f"blosum62 {mode}")


@pytest.mark.parametrize("mode", list(MODES))
def test_sim_fused_score_only(oracle, mode):
    """The F_NOTB twin: the score-only fill finishes the pairs too, the score-only K2 loads their EndState."""
    batch = edge_batch(23, 80, 70, 60)
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    ref, _ = oracle_batch(oracle, mode, s, batch)
    for walk in (0, 8):
        got, _, flags = fused_and_unfused(MODES[mode], s, batch, 16, 32 | walk)
        assert flags & F_NOTB, flags
        assert_scores(got, ref, f"{mode} walk={walk}")


M_SIDES = [0, 1, 2, 3, 16, 17, 18, 33, 150]
N_SIDES = [0, 1, 2, 150]


def _pairs_batch(pairs, seed):
    rng = np.random.default_rng(seed)
    blob, xo, xl, yo, yl, pos = [], [], [], [], [], 0
    for m, n in pairs:
        x = rng.integers(0, 4, m)
        y = x[:n].copy() if n <= m else np.concatenate([x, rng.integers(0, 4, n - m)])
        y = np.where(rng.random(n) < 0.2, rng.integers(0, 4, n), y)
        for arr, o, ln in ((x, xo, xl), (y, yo, yl)):
            o.append(pos)
            ln.append(len(arr))
            blob.append(np.frombuffer(b"ACGT", np.uint8)[arr.astype(np.int64)])
            pos += len(arr)
    return (np.concatenate(blob + [np.zeros(1, np.uint8)]), np.array(xo, np.uint64), np.array(xl, np.uint32),
            np.array(yo, np.uint64), np.array(yl, np.uint32))


@pytest.mark.parametrize("R", [16, 8])
@pytest.mark.parametrize("mode", ["local", "custom"])
def test_sim_fused_shapes(oracle, mode, R):
    """Every m in {0, 1, 2, 3, 16, 17, 18, 33, 150} against every n in {0, 1, 2, 150}: as one ragged batch (row m-1
    in every strip position, full final strips among them: m-1 = 16 and 32 with R = 16 and 8), and as uniform blocks
    of each shape."""
    pairs = [(m, n) for m in M_SIDES for n in N_SIDES]
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    ragged = _pairs_batch(pairs, 5)
    ref, ref_ops = oracle_batch(oracle, mode, s, ragged)
    got, ops, _ = fused_and_unfused(MODES[mode], s, ragged, R)
    assert_same(got, ops, ref, ref_ops, ragged, f"ragged {mode} R={R}")
    for m, n in pairs:
        uni = _pairs_batch([(m, n)] * 33, 100 + m + n)  # a full block and a partial last one
        ref, ref_ops = oracle_batch(oracle, mode, s, uni)
        got, ops, _ = fused_and_unfused(MODES[mode], s, uni, R)
        assert_same(got, ops, ref, ref_ops, uni, f"uniform {m}x{n} {mode} R={R}")


@pytest.mark.parametrize("m,n", [(4095, 2), (2, 4095), (4095, 150), (150, 4095)])
def test_sim_fused_longest_packed(oracle, m, n):
    """The packed trackers' longest sides (4,095 rows / columns) with short and medium partners."""
    batch = _pairs_batch([(m, n), (m - 1, n), (17, 3)], 9)
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS["local"])
    ref, ref_ops = oracle_batch(oracle, "local", s, batch)
    got, ops, flags = fused_and_unfused(MODES["local"], s, batch, 16)
    assert flags & F_PK, flags
    assert_same(got, ops, ref, ref_ops, batch, f"{m}x{n}")


# ------------------------------------------------------------------------------------------------ GPU

def _cs(mode, go=-5, ge=-1, ma=2, mi=-3, clips=None):
    from rust_bio_b200._lib import CScoring
    c = clips or CLIPS[mode]
    return CScoring(go, ge, c[0], c[1], c[2], c[3], ma, mi, 1, None, None, 0)


def _gpu_full(eng, mode, cs, batch):
    from rust_bio_b200.engine import Results
    res = eng.align_batch(MODES[mode], cs, batch, results=Results(len(batch[2]), eng.default_ops_capacity(batch),
                                                                  pair_status=True))
    out = {f: getattr(res, f)[:res.n_pairs].copy() for f in ("score", "xstart", "xend", "ystart", "yend", "status")}
    out["ops"] = [res.ops_of(p) if out["status"][p] == 0 else None for p in range(res.n_pairs)]
    return out, (eng.stats.fill_lanes_per_pair, eng.stats.fill_rows_per_lane)


def _assert_gpu_same(a, b, what):
    for f in ("score", "xstart", "xend", "ystart", "yend", "status"):
        bad = np.nonzero(a[f] != b[f])[0]
        assert not len(bad), f"{what}: {f} differs at {len(bad)} pairs; first {int(bad[0])}"
    assert a["ops"] == b["ops"], what


def _fused_vs_8x16(mode, cs, batch, walk=0, budget=0):
    """The batch on the 1x16 fill (F_FINISH) and forced to 8x16 (K2's finish): the same answer, ops included"""
    from rust_bio_b200.engine import Engine
    eng = Engine(0)
    try:
        eng.set_walk(walk)
        if budget:
            eng.set_traceback_budget(budget)
        eng.set_tuning(1, 16)
        a, shape_a = _gpu_full(eng, mode, cs, batch)
        if budget:
            assert eng.stats.waves >= 2, eng.stats.waves
        eng.set_tuning(8, 16)
        b, shape_b = _gpu_full(eng, mode, cs, batch)
    finally:
        eng.close()
    assert shape_a == (1, 16) and shape_b == (8, 16)
    _assert_gpu_same(a, b, f"{mode} walk={walk}")
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("walk", [1, 2], ids=["lane_walk", "warp_walk"])
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_fused_vs_k2_finish(oracle, mode, walk):
    batch = edge_batch(300 + walk, 3000, 160, 150)
    got = _fused_vs_8x16(mode, _cs(mode), batch, walk)
    k = 128
    sample = tuple(a[:k].copy() if i else a for i, a in enumerate(batch))
    s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *CLIPS[mode])
    ref, ref_ops = oracle_batch(oracle, mode, s, sample)
    assert_same({f: got[f][:k] for f in ("score", "xstart", "xend", "ystart", "yend", "status")}, got["ops"][:k],
                ref, ref_ops, sample, f"oracle sample {mode} walk={walk}")


@pytest.mark.gpu
def test_gpu_fused_waves():
    """Several traceback waves under a small budget: each wave's finish region starts at its own first block."""
    batch = edge_batch(77, 20000, 150, 150)
    _fused_vs_8x16("local", _cs("local"), batch, 0, budget=64 << 20)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_fused_score_only(mode):
    from rust_bio_b200.engine import Engine
    batch = edge_batch(500, 4000, 150, 150)
    eng = Engine(0)
    try:
        eng.set_tuning(1, 16)
        a = eng.align_batch_scores(MODES[mode], _cs(mode), batch)
        eng.set_tuning(8, 16)
        b = eng.align_batch_scores(MODES[mode], _cs(mode), batch)
    finally:
        eng.close()
    for f in ("score", "xend", "yend", "status"):
        assert np.array_equal(a[f], b[f]), (mode, f)


@pytest.mark.gpu
def test_gpu_fused_chunked_batch():
    """b2a_align_batch's chunk pipeline at 262,144 pairs of 150 x 150 (the C2 shape): the 1x16 fill of every chunk."""
    from rust_bio_b200.engine import Engine
    batch = synth.uniform_pairs(synth.BASES["C1"], 3, 262144, 150, 150)
    cs = _cs("local", -5, -1, 1, -1)
    eng = Engine(0)
    try:
        a, shape = _gpu_full(eng, "local", cs, batch)
        eng.set_tuning(8, 16)
        b, _ = _gpu_full(eng, "local", cs, batch)
    finally:
        eng.close()
    assert shape == (1, 16)
    _assert_gpu_same(a, b, "chunked C2 shape")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_gpu_fused_random_clips(seed):
    """Random custom clips: every pair, the panicking ones included, as K2's finish reports it."""
    rng = np.random.default_rng(2900 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    clips = (pick(), pick(), pick(), pick())
    cs = _cs("custom", int(rng.choice([0, -1, -2, -5])), int(rng.choice([0, -1, -2])), int(rng.choice([1, 2, 4])),
             int(rng.choice([-1, -3, 0])), clips)
    batch = edge_batch(seed, 4000, 90, 80, alphabet=b"AC" if seed % 2 else b"ACGT")
    got = _fused_vs_8x16("custom", cs, batch)
    print(f"seed {seed}: {int(np.count_nonzero(got['status']))} panicking pairs")
