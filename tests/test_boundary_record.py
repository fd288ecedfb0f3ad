"""The 8-byte strip boundary record (F_BND8, b2a_common.cuh): when the engine picks it (boundary8_ok in b2a_plan.h),
and that the fill + walk give the oracle's answer with it and just beyond its 16-bit bound, where the 16-byte record
is kept: on the host (tests/sim/b2a_sim_bnd8.cpp) and on the GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import sim_util
from parity_util import MODES, assert_same, oracle_batch

MIN = -858993459
F_TR, F_TC, F_CX, F_LUT, F_PK, F_RELU, F_PR, F_BND8 = 1, 2, 4, 8, 16, 32, 128, 256
LOCAL, GLOBAL, SEMI = (0, 0, 0, 0), (MIN,) * 4, (MIN, MIN, 0, 0)
CUSTOM = (MIN, -7, MIN, -9)  # suffix clips only: S runs as negative as in global mode, the record's halves go negative

# Batches whose maxm + maxn is 202, so score_bound = (202 + 2) * unit - gap_open with unit = 40 (mismatch -40) is
# 8191 = the largest bound the record takes (4 * 8191 + 3 < 2^15) with gap_open -31, and 8192 with gap_open -32.
SIDES = {"inside": -31, "outside": -32}
MATCH, MISMATCH, GAP_EXTEND = 25, -40, -3


SIM8_SRC = os.path.join(sim_util.HERE, "sim", "b2a_sim_bnd8.cpp")
SIM8_SO = os.path.join(sim_util.HERE, "sim", "libb2asim_bnd8.so")
_sim8 = None


def _flags_lib():
    """tests/sim/b2a_sim_bnd8.cpp: the host harness with the engine's record choice (built on first use)."""
    global _sim8
    if _sim8 is None:
        deps = [SIM8_SRC] + sim_util.DEPS
        if not os.path.exists(SIM8_SO) or any(os.path.getmtime(d) > os.path.getmtime(SIM8_SO) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                                   "-o", SIM8_SO, SIM8_SRC])
        _sim8 = C.CDLL(SIM8_SO)
        for fn in (_sim8.sim_scoring_flags, _sim8.sim8_boundary8_ok, _sim8.sim8_fill_flags, _sim8.sim8_align_batch):
            fn.restype = C.c_int
    return _sim8


def _sim8_run(mode, orc_scoring, batch, G, R, warp_walk, garbage):
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
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    L = _flags_lib()
    rc = L.sim8_align_batch(int(mode), C.byref(s), p(blob), p(x_off), p(x_len), p(y_off), p(y_len), C.c_uint64(n),
                            int(G), int(R), int(warp_walk), int(garbage), p(out["score"]), p(out["xstart"]),
                            p(out["xend"]), p(out["ystart"]), p(out["yend"]), p(out["n_ops"]), p(out["clip_len"]),
                            p(out["status"]), p(ops), p(ops_off))
    assert rc == 0, rc
    oplists = [sim_util.decode_ops(ops[int(ops_off[i]):int(ops_off[i]) + int(out["n_ops"][i])],
                                   out["clip_len"][4 * i:4 * i + 4]) for i in range(n)]
    return out, oplists, L.sim8_fill_flags()


def sim8_align_batch(mode, orc_scoring, batch, G, R, warp_walk=0):
    """-> (fields, ops, fill flags); run on two scratch fills that must give the same result"""
    a = _sim8_run(mode, orc_scoring, batch, G, R, warp_walk, 0x00)
    b = _sim8_run(mode, orc_scoring, batch, G, R, warp_walk, 0x7F)
    for k in a[0]:
        assert np.array_equal(a[0][k], b[0][k]), ("scratch-dependent result", k)
    assert a[1] == b[1] and a[2] == b[2], "scratch-dependent ops"
    return a


def test_boundary8_selection():
    """C2 (150 x 150 DNA local, score_bound 1500) takes the 8-byte record; one past the 16-bit bound, the long-sequence
    packed form (F_PACKREL), the explicit (value, index) trackers and global mode (no trackers) keep 16 bytes."""
    L = _flags_lib()
    f = lambda clips, alpha, bound, m, n: L.sim_scoring_flags(*[C.c_int32(c) for c in clips], C.c_int32(alpha),
                                                           C.c_int64(bound), C.c_uint32(m), C.c_uint32(n))
    ok = lambda flags, bound: L.sim8_boundary8_ok(C.c_int(flags), C.c_int64(bound)) == 1
    c2 = f(LOCAL, 4, 1500, 150, 150)
    assert c2 & F_PK and ok(c2, 1500)
    assert ok(f(LOCAL, 4, 8191, 150, 150), 8191) and not ok(f(LOCAL, 4, 8192, 150, 150), 8192)
    assert ok(f(SEMI, 4, 1500, 150, 150), 1500)  # row trackers only: still the packed form
    assert ok(f(CUSTOM, 4, 1500, 150, 150), 1500)
    assert not ok(f(LOCAL, 25, 220032, 10000, 10000), 220032)  # C5: F_PACKREL
    assert not ok(F_TR | F_TC | F_CX | F_LUT | F_RELU | F_PR, 1500)  # F_PACKREL even with small scores
    assert not ok(f(LOCAL, 25, 1 << 19, 10000, 10000), 1 << 19)  # explicit pairs
    assert not ok(F_TR | F_TC | F_CX | F_LUT | F_RELU, 1500)  # explicit pairs (packing disabled)
    assert not ok(f(GLOBAL, 4, 1500, 150, 150), 1500)  # C3-like: global, no trackers


def _batch(kind, seed):
    """uniform: 101 x 101 (100 interior rows: masked last strip for R = 16 and for 8 x 20's 160-row strip);
    ragged: lengths in [1, 101] with one 101 x 101 pair, so every block's shape differs"""
    rng = np.random.default_rng(seed)
    n = 96
    if kind == "uniform":
        xl = np.full(n, 101, dtype=np.uint32)
        yl = np.full(n, 101, dtype=np.uint32)
    else:
        xl = rng.integers(1, 102, n).astype(np.uint32)
        yl = rng.integers(1, 102, n).astype(np.uint32)
        xl[5], yl[5] = 101, 101
    alpha = np.frombuffer(b"ACGT", dtype=np.uint8)
    lens = np.stack([xl, yl], axis=1).reshape(-1).astype(np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    blob = alpha[rng.integers(0, 4, int(lens.sum()) + 1)]
    # related pairs (y a mutated copy of x where it fits) so that the alignments are long and the scores large
    for p in range(n):
        xo, yo, k = int(offs[2 * p]), int(offs[2 * p + 1]), int(min(xl[p], yl[p]))
        src = blob[xo:xo + k].copy()
        mut = rng.random(k) < 0.1
        src[mut] = alpha[rng.integers(0, 4, int(mut.sum()))]
        blob[yo:yo + k] = src
    return blob, offs[0::2].copy(), xl, offs[1::2].copy(), yl


def _mode_clips(mode):
    return {"local": LOCAL, "semiglobal": SEMI, "custom": CUSTOM}[mode]


@pytest.mark.parametrize("side", list(SIDES))
@pytest.mark.parametrize("mode", ["local", "custom", "semiglobal"])
@pytest.mark.parametrize("kind", ["uniform", "ragged"])
@pytest.mark.parametrize("G,R,warp_walk", [(1, 16, 0), (8, 20, 1)], ids=["1x16", "8x20_warp_walk"])
def test_sim_boundary_record_vs_oracle(oracle, side, mode, kind, G, R, warp_walk):
    """fill_lane + the walk on the host with the 8-byte record (inside) and the 16-byte one (outside); both K2 forms."""
    go = SIDES[side]
    batch = _batch(kind, 7 + G + R)
    s, _ = oracle.make_scoring(go, GAP_EXTEND, MATCH, MISMATCH, None, *_mode_clips(mode))
    ref, ref_ops = oracle_batch(oracle, mode, s, batch)
    got, ops, flags = sim8_align_batch(MODES[mode], s, batch, G, R, warp_walk)
    assert flags & F_PK, flags
    assert bool(flags & F_BND8) == (side == "inside"), flags
    assert_same(got, ops, ref, ref_ops, batch, f"{mode} {kind} G={G} R={R} {side}")


@pytest.mark.parametrize("mismatch,bnd8", [(-1, True), (-20, False)], ids=["inside", "outside"])
@pytest.mark.parametrize("mode", ["local", "custom"])
def test_sim_boundary_record_strip_pipelined(oracle, mode, mismatch, bnd8):
    """The warp-per-pair shape with strip-pipelined tasks (G = 132 in the harness): [pair][column] records handed from
    strip to strip through progress words while both strips run, over 1-3 strips of 256 rows.  score_bound is
    (maxm + maxn + 2) * 5 + 5 <= 4,515 with mismatch -1 (8-byte record) and above 8,191 with mismatch -20 (16 bytes)."""
    from rust_bio_b200 import synth
    clips = [MIN, -4, 0, -6] if mode == "custom" else [MIN] * 4
    s, _ = oracle.make_scoring(-5, -1, 1, mismatch, None, *clips)
    for batch in (synth.ragged_pairs(503, 9, 700, 200), synth.uniform_pairs(5, 0, 3, 600, 300)):
        ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=4)
        got, ops, flags = sim8_align_batch(MODES[mode], s, batch, 132, 8)
        assert bool(flags & F_BND8) == bnd8
        assert_same(got, ops, ref, ref_ops, batch, f"strip-pipelined 32x8 {mode} bnd8={bnd8}")


@pytest.mark.gpu
@pytest.mark.parametrize("side", list(SIDES))
@pytest.mark.parametrize("mode", ["local", "custom", "semiglobal"])
@pytest.mark.parametrize("kind", ["uniform", "ragged"])
@pytest.mark.parametrize("G,R", [(1, 16), (8, 20)])
def test_gpu_boundary_record_vs_oracle(oracle, side, mode, kind, G, R):
    """The same batches on the device for the shapes 1x16 (C2's) and 8x20: every Alignment field and the ops."""
    from rust_bio_b200._lib import CScoring
    from rust_bio_b200.engine import Engine
    go = SIDES[side]
    clips = _mode_clips(mode)
    batch = _batch(kind, 7 + G + R)
    s, _ = oracle.make_scoring(go, GAP_EXTEND, MATCH, MISMATCH, None, *clips)
    name = mode
    ref, ref_ops = oracle_batch(oracle, name, s, batch)
    cs = CScoring(go, GAP_EXTEND, clips[0], clips[1], clips[2], clips[3], MATCH, MISMATCH, 1, None, None, 0)
    eng = Engine(0)
    try:
        eng.set_tuning(G, R)
        res = eng.align_batch(MODES[name], cs, batch)
        assert (eng.stats.fill_lanes_per_pair, eng.stats.fill_rows_per_lane) == (G, R)
        got = res.as_dict()  # (a pair the reference would panic on fails the whole batch)
        ops = [res.ops_of(i) for i in range(res.n_pairs)]
    finally:
        eng.close()
    assert_same(got, ops, ref, ref_ops, batch, f"GPU {mode} {kind} G={G} R={R} {side}")


@pytest.mark.gpu
@pytest.mark.parametrize("mismatch", [-1, -20], ids=["inside", "outside"])
@pytest.mark.parametrize("mode", ["local", "custom"])
def test_gpu_boundary_record_strip_pipelined(oracle, mode, mismatch):
    """The strip-pipelined warp-per-pair fill (32x8, 1-3 strips per pair) on the device, both record sizes."""
    from rust_bio_b200 import synth
    from rust_bio_b200._lib import CScoring
    from rust_bio_b200.engine import Engine
    clips = [MIN, -4, 0, -6] if mode == "custom" else [MIN] * 4
    s, _ = oracle.make_scoring(-5, -1, 1, mismatch, None, *clips)
    cs = CScoring(-5, -1, clips[0], clips[1], clips[2], clips[3], 1, mismatch, 1, None, None, 0)
    eng = Engine(0)
    try:
        eng.set_tuning(32, 8)
        for batch in (synth.ragged_pairs(503, 9, 700, 200), synth.uniform_pairs(5, 0, 3, 600, 300)):
            ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=4)
            res = eng.align_batch(MODES[mode], cs, batch)
            assert eng.stats.fill_lanes_per_pair == 32
            ops = [res.ops_of(i) for i in range(res.n_pairs)]
            assert_same(res.as_dict(), ops, ref, ref_ops, batch, f"GPU strip-pipelined 32x8 {mode} mismatch {mismatch}")
    finally:
        eng.close()
