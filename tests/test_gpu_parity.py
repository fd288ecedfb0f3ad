"""GPU parity: the CUDA path (through the C ABI) against the oracle and the reference's golden vectors.
Bit-exact on every Alignment field and on the operation vectors."""
import numpy as np
import pytest

from golden_util import load_cases, parse_ops, scoring_fields
from parity_util import MODES, assert_same, oracle_batch, rescore_path

pytestmark = pytest.mark.gpu
MIN = -858993459
CASES = load_cases()
SHAPES = [(1, 16), (1, 8), (4, 16), (8, 16), (8, 20), (32, 8), (32, 16)]


@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _mirror_scoring(sc):
    from rust_bio_b200 import scores
    from rust_bio_b200.pairwise import MatchParams, Scoring
    f = scoring_fields(sc)
    if f["matrix"]:
        fn = getattr(scores, f["matrix"])
        s = Scoring.new(f["gap_open"], f["gap_extend"], fn)
    elif f["from_scores"]:
        s = Scoring.from_scores(f["gap_open"], f["gap_extend"], f["match"], f["mismatch"])
    else:
        ma, mi = f["match"], f["mismatch"]
        s = Scoring.new(f["gap_open"], f["gap_extend"], lambda a, b: ma if a == b else mi)
    s.xclip_prefix, s.xclip_suffix = f["xclip_prefix"], f["xclip_suffix"]
    s.yclip_prefix, s.yclip_suffix = f["yclip_prefix"], f["yclip_suffix"]
    return s


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_reference_known_answers_through_the_mirror(eng, case):
    """Reads like the reference's tests (mod.rs:1203-1769): Aligner::with_scoring(..).<mode>(x, y)."""
    from rust_bio_b200.pairwise import Aligner
    aligner = Aligner.with_scoring(_mirror_scoring(case["scoring"]), engine=eng)
    method = {"custom": aligner.custom, "global": aligner.global_, "semiglobal": aligner.semiglobal,
              "local": aligner.local}[case["mode"]]
    alignment = method(case["x"].encode(), case["y"].encode())
    exp = case["expect"]
    for k in ("score", "xstart", "xend", "ystart", "yend"):
        if k in exp:
            assert getattr(alignment, k) == exp[k], (case["name"], k, alignment)
    if "ops" in exp:
        assert [(o.code, o.len) for o in alignment.operations] == parse_ops(exp["ops"])
    assert alignment.xlen == len(case["x"]) and alignment.ylen == len(case["y"])


def _c_scoring(go, ge, ma, mi, clips=(MIN, MIN, MIN, MIN), table=None, alphabet=None):
    import ctypes as C
    from rust_bio_b200._lib import CScoring
    cs = CScoring(go, ge, clips[0], clips[1], clips[2], clips[3], ma, mi, 0, None, None, 0)
    keep = []
    if table is not None:
        t = np.ascontiguousarray(table, dtype=np.int32)
        keep.append(t)
        cs.table = t.ctypes.data_as(C.c_void_p)
        if alphabet is not None:
            a = np.frombuffer(alphabet, dtype=np.uint8).copy()
            keep.append(a)
            cs.alphabet = a.ctypes.data_as(C.c_void_p)
            cs.alphabet_len = len(a)
    return cs, keep


def _engine_result(eng, mode, cs, batch):
    res = eng.align_batch(MODES[mode], cs, batch)
    got = res.as_dict()
    ops = [res.ops_of(i) for i in range(res.n_pairs)]
    return got, ops


@pytest.mark.parametrize("G,R", SHAPES)
def test_c1_1k_pairs_150x150_local_every_field(eng, oracle, G, R):
    """BASELINE config 1: 1k pairs of 150x150 random DNA, local affine (1,-1,-5,-1), all fill shapes."""
    from rust_bio_b200 import synth
    batch = synth.uniform_pairs(synth.BASES["C1"], 0, 1000, 150, 150)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "local", s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    eng.set_tuning(G, R)
    try:
        got, ops = _engine_result(eng, "local", cs, batch)
    finally:
        eng.set_tuning(0, 0)
    assert eng.stats.fill_lanes_per_pair == G and eng.stats.fill_rows_per_lane == R
    assert_same(got, ops, ref, ref_ops, batch, f"C1 local G={G} R={R}")


@pytest.mark.parametrize("G,R", SHAPES)
@pytest.mark.parametrize("mode", ["local", "global", "semiglobal"])
def test_ragged_presets(eng, oracle, mode, G, R):
    from rust_bio_b200 import synth
    batch = synth.ragged_pairs(40 + G, 500, 200, 260)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    eng.set_tuning(G, R)
    try:
        got, ops = _engine_result(eng, mode, cs, batch)
    finally:
        eng.set_tuning(0, 0)
    assert_same(got, ops, ref, ref_ops, batch, f"ragged {mode} G={G} R={R}")


@pytest.mark.parametrize("G,R", [(1, 16), (8, 16), (32, 8)])
def test_tiny_and_empty_shapes(eng, oracle, G, R):
    xs, ys = [], []
    for m in range(0, 5):
        for n in range(0, 5):
            for rep in range(3):
                xs.append(m)
                ys.append(n)
    rng = np.random.default_rng(5)
    total = sum(xs) + sum(ys)
    blob = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 2, size=total + 1)]
    lens = np.array([v for pair in zip(xs, ys) for v in pair], dtype=np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    batch = (blob, offs[0::2].copy(), np.array(xs, dtype=np.uint32), offs[1::2].copy(),
             np.array(ys, dtype=np.uint32))
    eng.set_tuning(G, R)
    try:
        for mode in ("custom", "local", "global", "semiglobal"):
            for clips in [(MIN, MIN, MIN, MIN), (0, 0, 0, 0), (-1, 0, MIN, -2), (0, MIN, MIN, 0)]:
                s, _ = oracle.make_scoring(-2, -1, 2, -1, None, *clips)
                ref, ref_ops = oracle_batch(oracle, mode, s, batch)
                cs, keep = _c_scoring(-2, -1, 2, -1, clips)
                got, ops = _engine_result(eng, mode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"tiny {mode} {clips} G={G}")
    finally:
        eng.set_tuning(0, 0)


@pytest.mark.parametrize("seed", range(8))
def test_random_custom_clip_penalties(eng, oracle, seed):
    from rust_bio_b200 import synth
    rng = np.random.default_rng(100 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    go, ge = int(rng.choice([0, -1, -2, -5, -6])), int(rng.choice([0, -1, -1, -2]))
    ma, mi = int(rng.choice([1, 2, 4])), int(rng.choice([-1, -3, -7, 0]))
    clips = (pick(), pick(), pick(), pick())
    s, _ = oracle.make_scoring(go, ge, ma, mi, None, *clips)
    batch = synth.ragged_pairs(seed, 300, 90, 110, alphabet=b"AC" if seed % 2 else b"ACGT")
    ref, ref_ops = oracle_batch(oracle, "custom", s, batch, threads=8)
    cs, keep = _c_scoring(go, ge, ma, mi, clips)
    for G, R in [(1, 16), (8, 16), (32, 8)]:
        eng.set_tuning(G, R)
        try:
            got, ops = _engine_result(eng, "custom", cs, batch)
        finally:
            eng.set_tuning(0, 0)
        assert_same(got, ops, ref, ref_ops, batch, f"custom seed={seed} clips={clips} G={G}")


@pytest.mark.parametrize("G,R", [(1, 16), (8, 16), (32, 8)])
def test_blosum62_protein_lut_path(eng, oracle, G, R):
    from rust_bio_b200 import scores, synth
    table = scores.matrix_table256("blosum62")
    alpha = bytes(range(65, 91)) + b"*"
    batch = synth.ragged_pairs(3, 300, 180, 170, alphabet=synth.PROTEIN, min_len=1)
    eng.set_tuning(G, R)
    try:
        for mode, go in (("local", -10), ("global", -5), ("semiglobal", -11)):
            s, keep1 = oracle.make_scoring(go, -1, 0, 0, table)
            ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
            cs, keep2 = _c_scoring(go, -1, 0, 0, table=table, alphabet=alpha)
            got, ops = _engine_result(eng, mode, cs, batch)
            assert_same(got, ops, ref, ref_ops, batch, f"blosum62 {mode} G={G}")
    finally:
        eng.set_tuning(0, 0)


def test_c3_shape_global_1000x1000_sample(eng, oracle):
    """BASELINE config 3 shape (global 1000x1000), a 96-pair sample, warp-per-pair and 8-lane shapes."""
    from rust_bio_b200 import synth
    batch = synth.uniform_pairs(synth.BASES["C3"], 0, 96, 1000, 1000)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "global", s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    for G, R in [(32, 8), (32, 16), (8, 16), (4, 16)]:
        eng.set_tuning(G, R)
        try:
            got, ops = _engine_result(eng, "global", cs, batch)
        finally:
            eng.set_tuning(0, 0)
        assert_same(got, ops, ref, ref_ops, batch, f"C3 global G={G}")
    # thread-per-pair staging of 32 x (1000+1000) bytes per warp does not fit on chip: refused, not wrong
    from rust_bio_b200._lib import B2AError
    eng.set_tuning(1, 16)
    try:
        with pytest.raises(B2AError, match="UNSUPPORTED"):
            eng.align_batch(MODES["global"], cs, batch)
    finally:
        eng.set_tuning(0, 0)
    got, ops = _engine_result(eng, "global", cs, batch)  # automatic shape
    assert_same(got, ops, ref, ref_ops, batch, "C3 global auto shape")


def test_waves_give_identical_results(eng, oracle):
    """A traceback budget that forces several waves must not change any result."""
    from rust_bio_b200 import synth
    batch = synth.uniform_pairs(synth.BASES["C1"] + 77, 0, 2000, 150, 150)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    got1, ops1 = _engine_result(eng, "local", cs, batch)
    assert eng.stats.waves == 1
    eng.set_traceback_budget(3 << 20)
    try:
        got2, ops2 = _engine_result(eng, "local", cs, batch)
        assert eng.stats.waves > 1
    finally:
        eng.set_traceback_budget(0)
    for k in got1:
        assert np.array_equal(got1[k], got2[k])
    assert ops1 == ops2


def test_pipelined_batch_equals_single_shot(eng, oracle):
    """b2a_align_batch pipelines >= 262,144 pairs in chunks over two internal engines: same results,
    ops placed contiguously in caller order (ragged lengths, so chunks have different plans)."""
    from rust_bio_b200 import synth
    n = 300_000
    batch = synth.ragged_pairs(77, n, 36, 44, min_len=1)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    eng.set_pipeline(0)
    try:
        a = eng.align_batch(MODES["semiglobal"], cs, batch)
    finally:
        eng.set_pipeline(5)
    b = eng.align_batch(MODES["semiglobal"], cs, batch)
    for k in ("score", "xstart", "xend", "ystart", "yend", "ops_off"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    tot = int(a.ops_off[-1])
    assert np.array_equal(a.ops[:tot], b.ops[:tot])
    idx = np.random.default_rng(0).integers(0, n, 500)
    sub = (batch[0], batch[1][idx], batch[2][idx], batch[3][idx], batch[4][idx])
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "semiglobal", s, sub, threads=8)
    got = {k: v[idx] for k, v in b.as_dict().items()}
    assert_same(got, [b.ops_of(int(p)) for p in idx], ref, ref_ops, sub, "pipelined sample")


def test_pipeline_alphabet_reuse_falls_back_when_a_later_chunk_has_new_symbols(eng, oracle):
    """The pipeline reuses chunk 0's discovered alphabet; a symbol that first appears in a later chunk must
    not change results (the batch is redone in one shot)."""
    from rust_bio_b200 import synth
    n = 280_000
    batch = list(synth.ragged_pairs(78, n, 20, 24, alphabet=b"ACG", min_len=1))
    blob = batch[0].copy()
    last = n - 5
    blob[int(batch[1][last])] = ord("T")          # a 'T' only in the last chunk
    batch[0] = blob
    batch = tuple(batch)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    b = eng.align_batch(MODES["local"], cs, batch)
    idx = np.concatenate([np.arange(200), np.arange(n - 200, n)])
    sub = (batch[0], batch[1][idx], batch[2][idx], batch[3][idx], batch[4][idx])
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "local", s, sub, threads=8)
    got = {k: v[idx] for k, v in b.as_dict().items()}
    assert_same(got, [b.ops_of(int(p)) for p in idx], ref, ref_ops, sub, "alphabet fallback")


def test_full_size_c2_properties(eng, oracle):
    """BASELINE config 2 at full size (1M pairs): size-independent properties + sampled oracle parity.
    - every returned path re-scores to the returned score (4.0 gap model, mod.rs:9-15);
    - coordinates are consistent with the ops; scores are >= 0 (local);
    - the first 2,000 and 2,000 random pairs are bit-exact against the oracle."""
    from rust_bio_b200 import synth
    n = 1_000_000
    batch = synth.uniform_pairs(synth.BASES["C2"], 0, n, 150, 150)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    res = eng.align_batch(MODES["local"], cs, batch)
    blob, xo, xl, yo, yl = batch
    assert int(res.score.min()) >= 0
    ops_off = res.ops_off.astype(np.int64)
    codes = res.ops[:ops_off[-1]]
    assert codes.max() <= 3  # clips are filtered in local mode (mod.rs:1006)
    # vectorised consistency: #ops consuming x == xend-xstart, consuming y == yend-ystart
    cons_x = np.add.reduceat(np.concatenate([(codes != 2).astype(np.int64), [0]]), np.minimum(ops_off[:-1], len(codes)))
    cons_y = np.add.reduceat(np.concatenate([(codes != 3).astype(np.int64), [0]]), np.minimum(ops_off[:-1], len(codes)))
    nops = np.diff(ops_off)
    cons_x = np.where(nops > 0, cons_x, 0)
    cons_y = np.where(nops > 0, cons_y, 0)
    assert np.array_equal(cons_x, res.xend.astype(np.int64) - res.xstart)
    assert np.array_equal(cons_y, res.yend.astype(np.int64) - res.ystart)
    rng = np.random.default_rng(1)
    idx = np.unique(np.concatenate([np.arange(2000), rng.integers(0, n, size=2000)]))
    # re-score sampled paths
    for p in idx[::8]:
        i, j = int(res.xstart[p]), int(res.ystart[p])
        x = blob[int(xo[p]):int(xo[p]) + 150]
        y = blob[int(yo[p]):int(yo[p]) + 150]
        score, last = 0, None
        for c, _ in res.ops_of(int(p)):
            if c in (0, 1):
                assert (x[i] == y[j]) == (c == 0)
                score += 1 if c == 0 else -1
                i += 1
                j += 1
            elif c == 2:
                score += -1 if last == 2 else -5
                j += 1
            else:
                score += -1 if last == 3 else -5
                i += 1
            last = c
        assert (i, j) == (int(res.xend[p]), int(res.yend[p]))
        assert score == int(res.score[p])
    sub = (blob, xo[idx], xl[idx], yo[idx], yl[idx])
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "local", s, sub, threads=8)
    got = {k: v[idx] for k, v in res.as_dict().items()}
    assert_same(got, [res.ops_of(int(p)) for p in idx], ref, ref_ops, sub, "C2 sample")


def test_result_wire_formats_equal_fetch(eng, oracle):
    """The two all-gather wire formats (fixed-stride records, compact segment) decode to what fetch returns."""
    import torch
    from rust_bio_b200 import dist as bdist, synth
    from rust_bio_b200.engine import Results
    batch = synth.ragged_pairs(77, 300, 5, 90)
    n = len(batch[2])
    cs, keep = _c_scoring(-5, -1, 1, -1)
    for mode in ("local", "global"):
        eng.stage(MODES[mode], cs, batch)
        eng.run()
        want = Results(n, 64 * 1024)
        eng.fetch(want)
        total = int(want.ops_off[n])
        # compact segment, through both decoders
        nb = eng.compact_bytes()
        assert nb == 64 + 40 * n + total
        seg = torch.zeros(nb + 100, dtype=torch.uint8, device="cuda")
        eng.compact_into(seg.data_ptr(), seg.numel())
        torch.cuda.synchronize()
        host = seg.cpu().numpy()
        got = eng.decode_compact(host, host.size, 1, n, 64 * 1024)
        for k in ("score", "xstart", "xend", "ystart", "yend", "clip_len"):
            assert np.array_equal(getattr(got, k), getattr(want, k)), (mode, k)
        assert np.array_equal(got.ops_off[:n + 1], want.ops_off[:n + 1])
        assert np.array_equal(got.ops[:total], want.ops[:total])
        fields, ops_lists = bdist.decode_compact(host, host.size, 1)
        assert np.array_equal(fields["score"], want.score)
        assert ops_lists == [want.ops_of(p) for p in range(n)]
        # fixed-stride records
        stride = eng.record_stride(int(batch[2].max()), int(batch[4].max()))
        rec = torch.zeros(n * stride, dtype=torch.uint8, device="cuda")
        assert eng.records_into(rec.data_ptr(), rec.numel()) == stride
        torch.cuda.synchronize()
        f2, o2 = bdist.decode_records(rec.cpu().numpy(), stride, n)
        assert np.array_equal(f2["score"], want.score) and o2 == ops_lists


def test_error_paths(eng):
    """Bad parameters are refused like the reference's assert!s; out-of-alphabet bytes are an error."""
    from rust_bio_b200 import scores, synth
    from rust_bio_b200._lib import B2AError
    batch = synth.uniform_pairs(1, 0, 4, 20, 20)
    cs, _ = _c_scoring(1, -1, 1, -1)
    with pytest.raises(B2AError, match="gap_open can't be positive"):
        eng.align_batch(MODES["local"], cs, batch)
    cs, _ = _c_scoring(-1, -1, 1, -1, clips=(1, 0, 0, 0))
    with pytest.raises(B2AError, match="x prefix"):
        eng.align_batch(MODES["custom"], cs, batch)
    table = scores.matrix_table256("blosum62")
    bad = (np.full(64, ord("a"), dtype=np.uint8), batch[1][:1] * 0, batch[2][:1], batch[1][:1] * 0 + 32, batch[4][:1])
    cs, keep = _c_scoring(-5, -1, 0, 0, table=table, alphabet=bytes(range(65, 91)) + b"*")
    with pytest.raises(B2AError, match="alphabet"):
        eng.align_batch(MODES["local"], cs, bad)
    cs, _ = _c_scoring(-5, -1, 1 << 20, -1)
    with pytest.raises(B2AError, match="RANGE"):
        eng.align_batch(MODES["local"], cs, synth.uniform_pairs(1, 0, 4, 2000, 2000))


# --------------------------------------------------------------------------------------------------------
# Kernel variants and sizes checked against the oracle on hardware

def _blosum62():
    from rust_bio_b200 import scores
    return scores.matrix_table256("blosum62"), bytes(range(65, 91)) + b"*"


def test_c5_shape_8_pairs_10k_x_10k_blosum62_local(eng, oracle):
    """BASELINE config 5 (SURVEY 8d: 8 pairs): 10,000 x 10,000 protein, BLOSUM62, gap_open -10, gap_extend -1,
    local (the reference's own BLOSUM62-local example, mod.rs:41-54, 1323-1337).  m, n > 4095, so K1 runs its
    explicit (value, index) trackers (no F_PACKTRK) and K2's decode_boundary its unpacked branch."""
    from rust_bio_b200 import synth
    table, alpha = _blosum62()
    batch = synth.uniform_pairs(synth.BASES["C5"], 0, 8, 10000, 10000, alphabet=synth.PROTEIN)
    s, keep1 = oracle.make_scoring(-10, -1, 0, 0, table)
    ref, ref_ops = oracle_batch(oracle, "local", s, batch, threads=8)
    cs, keep2 = _c_scoring(-10, -1, 0, 0, table=table, alphabet=alpha)
    got, ops = _engine_result(eng, "local", cs, batch)  # the shape choose_shape() picks for C5
    assert eng.stats.fill_lanes_per_pair == 32
    assert_same(got, ops, ref, ref_ops, batch, "C5 local blosum62 auto shape")
    blob, xo, xl, yo, yl = batch
    flat = np.asarray(table).reshape(-1)
    for p in range(8):  # and independent of the oracle: the path re-scores to the score
        x = bytes(blob[int(xo[p]):int(xo[p]) + 10000])
        y = bytes(blob[int(yo[p]):int(yo[p]) + 10000])
        f = {k: got[k][p] for k in ("xstart", "xend", "ystart", "yend")}
        assert rescore_path(x, y, ops[p], f, "local", -10, -1, lambda a, b: int(flat[a * 256 + b])) == int(got["score"][p])


@pytest.mark.parametrize("G,R", [(8, 16), (8, 20), (32, 16), (32, 8)])
@pytest.mark.parametrize("lut", [True, False], ids=["lut", "matchparams_wide_alphabet"])
@pytest.mark.parametrize("trackers", ["relative_keys", "explicit_pairs"])
def test_unpacked_tracker_variants_4200(oracle, G, R, lut, trackers, monkeypatch):
    """m, n > 4095 in every mode: the fill_kernel<G,R,FLAGS> instantiations without F_PACKTRK -- with the packed keys
    over chunk- / strip-relative indices (F_PACKREL, what long sequences run: 0, TRACK_ROWS, ALL, ALL|RELU, each with
    and without F_LUT) and with explicit (value, index) trackers (B2A_NO_PACKREL=1: what scores above 2^18 would run).
    A 200-symbol alphabet keeps MatchParams on its compare/select path (no LUT above 64 symbols)."""
    from rust_bio_b200.engine import Engine
    if trackers == "explicit_pairs":
        monkeypatch.setenv("B2A_NO_PACKREL", "1")
    eng = Engine(0)
    from rust_bio_b200 import synth
    alphabet = b"ACGT" if lut else bytes(range(33, 233))
    rng = np.random.default_rng(G * 100 + R + (1 if lut else 0))
    pairs = []
    for m, n in [(4200, 4200), (4100, 4301), (4333, 4097), (4099, 5000)]:
        a = np.frombuffer(alphabet, dtype=np.uint8)
        x = a[rng.integers(0, len(a), m)]
        y = a[rng.integers(0, len(a), n)]
        if not lut:  # plant matches so that the 100-symbol case is not all mismatches
            k = min(m, n) - 50
            y = y.copy()
            y[20:20 + k:3] = x[30:30 + k:3]
        pairs.append((bytes(x), bytes(y)))
    from rust_bio_b200.engine import pack_pairs
    batch = pack_pairs(pairs)
    cases = [("global", (MIN,) * 4), ("semiglobal", (MIN,) * 4), ("local", (MIN,) * 4),
             ("custom", (-3, -4, -2, -5)), ("custom", (MIN, 0, MIN, -1)), ("custom", (0, MIN, 0, MIN))]
    eng.set_tuning(G, R)
    try:
        for mode, clips in cases:
            s, _ = oracle.make_scoring(-5, -1, 2, -1, None, *clips)
            ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=4)
            cs, keep = _c_scoring(-5, -1, 2, -1, clips)
            got, ops = _engine_result(eng, mode, cs, batch)
            assert eng.stats.fill_lanes_per_pair == G
            assert_same(got, ops, ref, ref_ops, batch, f"4200 {mode} {clips} G={G} R={R} lut={lut} {trackers}")
    finally:
        eng.close()


@pytest.mark.parametrize("mode", ["global", "semiglobal", "local", "custom"])
def test_paths_rescore_to_their_score_every_mode(eng, mode):
    """The fuzz target's property (fuzz/fuzz_targets/banded_aligner.rs:10-56), independent of the oracle, on
    every pair of a batch, for every mode incl. custom clips: the returned path re-scores to the returned score."""
    from rust_bio_b200 import synth
    rng = np.random.default_rng(23)
    for trial in range(4):
        go, ge = int(rng.choice([0, -1, -2, -5, -6])), int(rng.choice([0, -1, -1, -2]))
        ge = max(ge, go)  # the affine model the property is stated for: opening costs at least as much as extending
        ma, mi = int(rng.choice([1, 2, 4])), int(rng.choice([-1, -3, -7]))
        clips = (MIN, MIN, MIN, MIN)
        if mode == "custom":
            clips = tuple(int(rng.choice([MIN, 0, -1, -3, -7, -20])) for _ in range(4))
        batch = synth.ragged_pairs(300 + trial, 2000, 150, 180, alphabet=b"AC" if trial % 2 else b"ACGT")
        cs, keep = _c_scoring(go, ge, ma, mi, clips)
        got, ops = _engine_result(eng, mode, cs, batch)
        blob, xo, xl, yo, yl = batch
        eff = {"global": (MIN,) * 4, "semiglobal": (MIN, MIN, 0, 0), "local": (0, 0, 0, 0)}.get(mode, clips)
        for p in range(len(xl)):
            x = bytes(blob[int(xo[p]):int(xo[p]) + int(xl[p])])
            y = bytes(blob[int(yo[p]):int(yo[p]) + int(yl[p])])
            f = {k: got[k][p] for k in ("xstart", "xend", "ystart", "yend")}
            sc = rescore_path(x, y, ops[p], f, mode, go, ge, lambda a, b: ma if a == b else mi, eff)
            assert sc == int(got["score"][p]), (mode, trial, p, clips)


def test_c3_full_shape_1000_pairs_global_with_rescoring(eng, oracle):
    """BASELINE config 3 parity sample (SURVEY 8d: 1,000 pairs of 1000x1000 global) on the automatic shape."""
    from rust_bio_b200 import synth
    batch = synth.uniform_pairs(synth.BASES["C3"], 0, 1000, 1000, 1000)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "global", s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    got, ops = _engine_result(eng, "global", cs, batch)
    assert_same(got, ops, ref, ref_ops, batch, "C3 1000 pairs")
    blob, xo, xl, yo, yl = batch
    for p in range(0, 1000, 10):
        x = bytes(blob[int(xo[p]):int(xo[p]) + 1000])
        y = bytes(blob[int(yo[p]):int(yo[p]) + 1000])
        f = {k: got[k][p] for k in ("xstart", "xend", "ystart", "yend")}
        assert rescore_path(x, y, ops[p], f, "global", -5, -1, lambda a, b: 1 if a == b else -1) == int(got["score"][p])


def test_long_reference_falls_back_to_warp_per_pair_staging(eng, oracle):
    """A read against a 15 kb reference (semiglobal): the 8-lanes-per-pair shape would stage 4 x 4 x (m + n)
    bytes per CTA (> 200 KB); the engine falls back to the warp-per-pair shape instead of refusing (ADVICE r1)."""
    from rust_bio_b200 import synth
    batch = synth.uniform_pairs(77, 0, 64, 100, 15000)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "semiglobal", s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    got, ops = _engine_result(eng, "semiglobal", cs, batch)
    assert eng.stats.fill_lanes_per_pair == 32
    assert_same(got, ops, ref, ref_ops, batch, "100 x 15000 semiglobal")
    from rust_bio_b200._lib import B2AError
    eng.set_tuning(8, 16)  # a forced shape is not replaced
    try:
        with pytest.raises(B2AError, match="UNSUPPORTED"):
            eng.align_batch(MODES["semiglobal"], cs, batch)
    finally:
        eng.set_tuning(0, 0)


def test_fixed_capacity_segments_and_gathered_fetch(eng, oracle):
    """b2a_batch_compact_fixed + b2a_gathered_fetch (the N > 1 reassembly without a size agreement): segments of a
    caller-fixed capacity, 'gathered' here by placing two batches' segments side by side, decode on the host to
    exactly what fetch returns; a capacity below the ops bytes is reported, not silently cut."""
    import torch
    from rust_bio_b200 import synth
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import Results
    cs, keep = _c_scoring(-5, -1, 1, -1)
    batches = [synth.ragged_pairs(5, 700, 60, 90), synth.ragged_pairs(6, 300, 120, 40)]
    seg = 1 << 20
    allbuf = torch.zeros(2 * seg, dtype=torch.uint8, device="cuda")
    wants = []
    for g, batch in enumerate(batches):
        n = len(batch[2])
        eng.stage(MODES["global"], cs, batch)
        eng.run()
        eng.compact_fixed(allbuf.data_ptr() + g * seg, seg)
        want = Results(n, 1 << 20)
        eng.fetch(want)
        wants.append(want)
    torch.cuda.synchronize()
    got = Results(1000, 2 << 20)
    n_got, moved = eng.gathered_fetch(allbuf.data_ptr(), seg, 2, got)
    assert n_got == 1000 and moved > 0
    base, obase = 0, 0
    for want in wants:
        n = want.n_pairs
        for k in ("score", "xstart", "xend", "ystart", "yend"):
            assert np.array_equal(getattr(got, k)[base:base + n], getattr(want, k)[:n]), k
        assert np.array_equal(got.clip_len[4 * base:4 * (base + n)], want.clip_len[:4 * n])
        tot = int(want.ops_off[n])
        assert np.array_equal(got.ops_off[base:base + n + 1].astype(np.int64) - obase, want.ops_off[:n + 1].astype(np.int64))
        assert np.array_equal(got.ops[obase:obase + tot], want.ops[:tot])
        base += n
        obase += tot
    # too small a capacity: the header says so and the fetch refuses the segment
    small = 64 + 40 * 300 + 100
    eng.compact_fixed(allbuf.data_ptr(), small)
    torch.cuda.synchronize()
    with pytest.raises(B2AError, match="CAPACITY"):
        eng.gathered_fetch(allbuf.data_ptr(), small, 1, Results(300, 1 << 20))
    with pytest.raises(B2AError, match="CAPACITY"):
        eng.compact_fixed(allbuf.data_ptr(), 64)


@pytest.mark.parametrize("walk", [1, 2], ids=["lane_per_pair", "warp_per_pair"])
def test_both_walk_kernels_every_mode(eng, oracle, walk):
    """K2 as one lane per pair and as one warp per pair (prefix-maximum passes + prefetched walk) give the
    reference's results in every mode, on ragged batches, custom clips, every fill shape family."""
    from rust_bio_b200 import synth
    eng.set_walk(walk)
    try:
        for (G, R) in [(0, 0), (1, 16), (8, 20), (8, 16), (32, 8)]:
            eng.set_tuning(G, R)
            for mode, clips in [("local", (MIN,) * 4), ("global", (MIN,) * 4), ("semiglobal", (MIN,) * 4),
                                ("custom", (-3, -4, -2, -5)), ("custom", (MIN, 0, MIN, -1)), ("custom", (0, MIN, 0, 0))]:
                batch = synth.ragged_pairs(60 + G, 400, 200, 230)
                s, _ = oracle.make_scoring(-5, -1, 2, -3, None, *clips)
                ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
                cs, keep = _c_scoring(-5, -1, 2, -3, clips)
                got, ops = _engine_result(eng, mode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"walk={walk} {mode} {clips} G={G} R={R}")
        eng.set_tuning(0, 0)
        # tiny and empty shapes
        xs, ys = [], []
        for m in range(0, 5):
            for n in range(0, 5):
                xs.append(m)
                ys.append(n)
        rng = np.random.default_rng(5)
        blob = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 2, size=sum(xs) + sum(ys) + 1)]
        lens = np.array([v for pair in zip(xs, ys) for v in pair], dtype=np.uint64)
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        batch = (blob, offs[0::2].copy(), np.array(xs, dtype=np.uint32), offs[1::2].copy(), np.array(ys, dtype=np.uint32))
        for mode in ("custom", "local", "global", "semiglobal"):
            for clips in [(MIN, MIN, MIN, MIN), (0, 0, 0, 0), (-1, 0, MIN, -2)]:
                s, _ = oracle.make_scoring(-2, -1, 2, -1, None, *clips)
                ref, ref_ops = oracle_batch(oracle, mode, s, batch)
                cs, keep = _c_scoring(-2, -1, 2, -1, clips)
                got, ops = _engine_result(eng, mode, cs, batch)
                assert_same(got, ops, ref, ref_ops, batch, f"walk={walk} tiny {mode} {clips}")
        # C1, C3 sample, blosum
        batch = synth.uniform_pairs(synth.BASES["C1"], 0, 1000, 150, 150)
        s, _ = oracle.make_scoring(-5, -1, 1, -1)
        ref, ref_ops = oracle_batch(oracle, "local", s, batch, threads=8)
        cs, keep = _c_scoring(-5, -1, 1, -1)
        got, ops = _engine_result(eng, "local", cs, batch)
        assert_same(got, ops, ref, ref_ops, batch, f"walk={walk} C1")
        batch = synth.uniform_pairs(synth.BASES["C3"], 0, 64, 1000, 1000)
        ref, ref_ops = oracle_batch(oracle, "global", s, batch, threads=8)
        got, ops = _engine_result(eng, "global", cs, batch)
        assert_same(got, ops, ref, ref_ops, batch, f"walk={walk} C3 sample")
        table, alpha = _blosum62()
        batch = synth.ragged_pairs(3, 200, 180, 170, alphabet=synth.PROTEIN, min_len=1)
        s, keep1 = oracle.make_scoring(-10, -1, 0, 0, table)
        ref, ref_ops = oracle_batch(oracle, "local", s, batch, threads=8)
        cs, keep2 = _c_scoring(-10, -1, 0, 0, table=table, alphabet=alpha)
        got, ops = _engine_result(eng, "local", cs, batch)
        assert_same(got, ops, ref, ref_ops, batch, f"walk={walk} blosum62 local")
    finally:
        eng.set_walk(0)
        eng.set_tuning(0, 0)


@pytest.mark.parametrize("mode,clips", [("local", (MIN,) * 4), ("global", (MIN,) * 4), ("custom", (-3, 0, -2, -5))])
def test_small_batch_overlap_of_fills_and_walks(oracle, mode, clips, monkeypatch):
    """2,048 .. 16,384 pairs: the wave is cut into four sub-ranges whose fills alternate between two streams and
    whose warp-per-pair walks run on a high-priority stream (b2a_batch_run): same results as the oracle, run
    three times in a row on the same staged batch (stale scratch must not leak)."""
    from rust_bio_b200 import synth
    from rust_bio_b200.engine import Engine, Results
    monkeypatch.setenv("B2A_OVERLAP", "1")  # read at engine creation (off by default: no gain measured)
    eng = Engine(0)
    batch = synth.ragged_pairs(4242, 6000, 150, 170, min_len=100)
    s, _ = oracle.make_scoring(-5, -1, 1, -1, None, *clips)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1, clips)
    eng.stage(MODES[mode], cs, batch)
    for rep in range(3):
        eng.run()
        res = Results(6000, int(eng.default_ops_capacity(batch)))
        eng.fetch(res)
        assert_same(res.as_dict(), [res.ops_of(i) for i in range(6000)], ref, ref_ops, batch, f"overlap {mode} rep {rep}")
    assert eng.stats.kernel_launches >= 9  # K0 + 4 fills + 4 walks (+ compaction): the overlapped form ran
    eng.close()


@pytest.mark.parametrize("cta_warps", [4, 16])
@pytest.mark.parametrize("kind", ["uniform_10k_local", "ragged_5000_custom"])
def test_tail_split_of_the_small_batch_fill(oracle, kind, cta_warps, monkeypatch):
    """Small batches whose equal tasks leave a thin last round on the persistent fill (10k reads on 8x20: two
    rounds of 1,184 tasks + 132): the whole rounds and the remainder are filled back to back and the warp-per-pair
    walk of the first part runs beside the fill of the second (b2a_batch_run).  Every pair against the oracle,
    three runs on the same staged batch; and K2's CTA size (pairs of a block that share L1 sectors)."""
    from rust_bio_b200 import synth
    from rust_bio_b200.engine import Engine, Results
    monkeypatch.setenv("B2A_TAIL_SPLIT", "1")
    monkeypatch.setenv("B2A_WALK_CTA_WARPS", str(cta_warps))
    eng = Engine(0)
    if kind == "uniform_10k_local":
        n, mode, clips = 10000, "local", (MIN,) * 4
        batch = synth.uniform_pairs(synth.BASES["C2"], 0, n, 150, 150)
    else:
        n, mode, clips = 5000, "custom", (-3, 0, -2, -5)  # 1,250 tasks on 1,184 resident warps
        batch = synth.ragged_pairs(777, n, 150, 170, min_len=120)
    s, _ = oracle.make_scoring(-5, -1, 1, -1, None, *clips)
    ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
    cs, keep = _c_scoring(-5, -1, 1, -1, clips)
    eng.stage(MODES[mode], cs, batch)
    for rep in range(3):
        eng.run()
        res = Results(n, int(eng.default_ops_capacity(batch)))
        eng.fetch(res)
        assert_same(res.as_dict(), [res.ops_of(i) for i in range(n)], ref, ref_ops, batch, f"tail split {kind} rep {rep}")
    assert eng.stats.kernel_launches >= 5  # K0 + 2 fills + 2 walks (+ compaction): the split form ran
    eng.close()


def _bitenc_batch(seed, n_pairs, max_m, max_n, alphabet, min_len=0):
    """ragged batch + the same sequences as BitEnc storages of RankTransform ranks"""
    from rust_bio_b200 import synth
    from rust_bio_b200.alphabets import Alphabet, RankTransform
    batch = synth.ragged_pairs(seed, n_pairs, max_m, max_n, alphabet=alphabet, min_len=min_len)
    rt = RankTransform.new(Alphabet.new(alphabet))
    blob, xo, xl, yo, yl = batch
    ranks_blob = rt.transform(bytes(blob))
    return batch, (ranks_blob, xo, xl, yo, yl), rt


@pytest.mark.parametrize("alphabet", [b"ACGT", b"ACGTN"], ids=["width2", "width3"])
def test_bitenc_packed_input_every_mode(eng, oracle, alphabet):
    """SURVEY 8f rank 2: BitEnc storage (bitenc.rs:50-56) of RankTransform ranks (alphabets/mod.rs:220-283) as
    the batch input, through b2a_align_batch_packed: same alignments as the oracle on the rank sequences (MatchParams
    scores by equality, so ranks and symbols score alike) and as the byte path on the original symbols."""
    from rust_bio_b200.data_structures import BitEnc
    from rust_bio_b200.engine import Engine
    batch, rank_batch, rt = _bitenc_batch(17, 700, 140, 170, alphabet)
    width = max(1, rt.get_width())
    blob, xo, xl, yo, yl = rank_batch
    pairs = [(BitEnc.from_values(width, blob[int(xo[p]):int(xo[p]) + int(xl[p])]),
              BitEnc.from_values(width, blob[int(yo[p]):int(yo[p]) + int(yl[p])])) for p in range(len(xl))]
    packed = Engine.pack_bitenc_pairs(pairs)
    assert packed[0].nbytes * (3 if width == 2 else 2) < int(xl.sum() + yl.sum()) * 1 + 4096
    cs, keep = _c_scoring(-5, -1, 2, -3)
    s, _ = oracle.make_scoring(-5, -1, 2, -3)
    for mode in ("local", "global", "semiglobal"):
        ref, ref_ops = oracle_batch(oracle, mode, s, rank_batch, threads=8)
        res = eng.align_batch_packed(MODES[mode], cs, packed)
        assert_same(res.as_dict(), [res.ops_of(i) for i in range(res.n_pairs)], ref, ref_ops, rank_batch, f"bitenc {mode}")
        got2, ops2 = _engine_result(eng, mode, cs, batch)  # the byte path on the original symbols
        assert np.array_equal(got2["score"], res.score) and ops2 == [res.ops_of(i) for i in range(res.n_pairs)]
    # the mirror: Aligner.batch_bitenc
    from rust_bio_b200.pairwise import Aligner, MatchParams, Scoring
    al = Aligner.with_scoring(Scoring.new(-5, -1, MatchParams.new(2, -3)), engine=eng)
    alns = al.batch_bitenc(MODES["local"], pairs[:50])
    ref, ref_ops = oracle_batch(oracle, "local", s, tuple(a[:50] if i else a for i, a in enumerate(rank_batch)), threads=4)
    assert [a.score for a in alns] == [int(v) for v in ref["score"][:50]]
    assert [[(o.code, o.len) for o in a.operations] for a in alns] == ref_ops[:50]


def test_bitenc_packed_input_through_the_chunk_pipeline_and_banded(eng, oracle):
    """>= 262,144 pairs of packed input go through the chunked H2D / kernel / D2H pipeline (block-indexed slices);
    the banded aligner takes the same packed input."""
    from rust_bio_b200.data_structures import BitEnc
    from rust_bio_b200.engine import Engine
    n = 270_000
    batch, rank_batch, rt = _bitenc_batch(23, n, 30, 36, b"ACGT", min_len=1)
    blob, xo, xl, yo, yl = rank_batch
    # vectorised packing: every sequence starts a new block (16 symbols per block at width 2)
    xb = np.zeros(n, dtype=np.uint64)
    yb = np.zeros(n, dtype=np.uint64)
    nblk = lambda l: (l.astype(np.uint64) + np.uint64(15)) // np.uint64(16)
    sizes = np.stack([nblk(xl), nblk(yl)], axis=1).reshape(-1)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    xb[:], yb[:] = offs[0:-1:2], offs[1::2]
    blocks = np.zeros(int(offs[-1]) + 4, dtype=np.uint32)
    for arr_off, arr_len, arr_blk in ((xo, xl, xb), (yo, yl, yb)):
        for k in range(36):
            sel = arr_len > k
            v = blob[(arr_off[sel] + np.uint64(k)).astype(np.int64)].astype(np.uint32)
            np.bitwise_or.at(blocks, (arr_blk[sel] + np.uint64(k // 16)).astype(np.int64), v << np.uint32(2 * (k % 16)))
    packed = (blocks, xb, xl, yb, yl, 2)
    assert BitEnc.from_values(2, blob[int(xo[5]):int(xo[5]) + int(xl[5])]).storage.tolist() == \
        blocks[int(xb[5]):int(xb[5]) + int(nblk(xl[5:6])[0])].tolist()
    cs, keep = _c_scoring(-5, -1, 1, -1)
    res = eng.align_batch_packed(MODES["semiglobal"], cs, packed)
    got2 = eng.align_batch(MODES["semiglobal"], cs, batch)
    for k in ("score", "xstart", "xend", "ystart", "yend", "ops_off"):
        assert np.array_equal(getattr(res, k), getattr(got2, k)), k
    tot = int(res.ops_off[-1])
    assert np.array_equal(res.ops[:tot], got2.ops[:tot])
    idx = np.random.default_rng(0).integers(0, n, 400)
    sub = (blob, xo[idx], xl[idx], yo[idx], yl[idx])
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    ref, ref_ops = oracle_batch(oracle, "semiglobal", s, sub, threads=8)
    assert_same({k: v[idx] for k, v in res.as_dict().items()}, [res.ops_of(int(p)) for p in idx], ref, ref_ops, sub, "packed pipeline")
    # banded, packed
    from test_sim_banded import _mutated_window_batch
    from rust_bio_b200.alphabets import Alphabet, RankTransform
    bb = _mutated_window_batch(5, 200, 120, 500)
    rt = RankTransform.new(Alphabet.new(b"ACGT"))
    rb = (rt._table[np.asarray(bb[0])],) + tuple(bb[1:])  # (the blob's padding bytes are not symbols: no transform())
    pairs = [(BitEnc.from_values(2, rb[0][int(rb[1][p]):int(rb[1][p]) + int(rb[2][p])]),
              BitEnc.from_values(2, rb[0][int(rb[3][p]):int(rb[3][p]) + int(rb[4][p])])) for p in range(200)]
    from rust_bio_b200._lib import CScoring
    csb = CScoring(-5, -1, MIN, MIN, MIN, MIN, 1, -1, 1, None, None, 0)
    resb = eng.align_batch_packed(MODES["semiglobal"], csb, Engine.pack_bitenc_pairs(pairs), banded=(12, 8))
    so, _ = oracle.make_scoring(-5, -1, 1, -1, has_match_scores=1)
    refb, rops, roff, _, _ = oracle.banded_align_batch("semiglobal", so, 12, 8, *rb, threads=8)
    assert np.array_equal(resb.score.astype(np.int64), refb["score"].astype(np.int64))
    for p in range(200):
        want = [(int(v) & 7, int(v) >> 3) for v in rops[int(roff[p]):int(roff[p]) + int(refb["n_ops"][p])]]
        assert resb.ops_of(p) == want, p


def test_scattered_blob_layout_through_the_chunk_pipeline(eng, oracle):
    """A caller blob laid out as all x, then all y: each chunk of the pipeline gathers its own sequences into a
    compact blob instead of uploading (almost) the whole span once per chunk (ADVICE r1); results equal those of
    the interleaved layout."""
    from rust_bio_b200 import synth
    n = 270_000
    a = synth.ragged_pairs(501, n, 24, 30, min_len=1)
    blob, xo, xl, yo, yl = a
    # rebuild as [all x][gap][all y]
    xs = np.concatenate([[0], np.cumsum(xl.astype(np.uint64))]).astype(np.uint64)
    ys = np.concatenate([[0], np.cumsum(yl.astype(np.uint64))]).astype(np.uint64)
    gap = 3_000_000
    nb = np.zeros(int(xs[-1]) + gap + int(ys[-1]) + 16, dtype=np.uint8)
    # vectorised copy of every sequence: positions = offset + running index
    def place(dst_off, src_off, lens, base):
        total = int(lens.astype(np.uint64).sum())
        rep = np.repeat(np.arange(len(lens)), lens.astype(np.int64))
        within = np.arange(total) - np.repeat((np.cumsum(lens.astype(np.int64)) - lens.astype(np.int64)), lens.astype(np.int64))
        nb[base + dst_off[rep].astype(np.int64) + within] = blob[src_off[rep].astype(np.int64) + within]
    place(xs[:-1], xo, xl, 0)
    place(ys[:-1], yo, yl, int(xs[-1]) + gap)
    b = (nb, xs[:-1].copy(), xl, ys[:-1] + np.uint64(int(xs[-1]) + gap), yl)
    cs, keep = _c_scoring(-5, -1, 1, -1)
    r1 = eng.align_batch(MODES["local"], cs, a)
    r2 = eng.align_batch(MODES["local"], cs, b)
    assert int(eng.stats.h2d_bytes) < 3 * (int(xl.sum()) + int(yl.sum()) + 40 * n)  # not one blob upload per chunk
    for k in ("score", "xstart", "xend", "ystart", "yend", "ops_off"):
        assert np.array_equal(getattr(r1, k), getattr(r2, k)), k
    tot = int(r1.ops_off[-1])
    assert np.array_equal(r1.ops[:tot], r2.ops[:tot])


def test_tabulated_matchfunc_over_100_symbols(eng, oracle):
    """A closure MatchFunc (mod.rs:221-228) over a 100-symbol alphabet: tabulated into a 100 x 100 LUT in shared
    memory (round 1 refused tables over 64 symbols); beyond 128 distinct symbols the table is still refused."""
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import pack_pairs
    rng = np.random.default_rng(12)
    alphabet = np.arange(33, 133, dtype=np.uint8)
    fn = lambda a, b: (5 if a == b else (1 if (a ^ b) < 4 else -((a * 7 + b * 3) % 5)))
    table = np.zeros((256, 256), dtype=np.int32)
    for a in alphabet:
        for b in alphabet:
            table[a, b] = fn(int(a), int(b))
    pairs = []
    for _ in range(60):
        m, n = int(rng.integers(1, 180)), int(rng.integers(1, 200))
        x = alphabet[rng.integers(0, 100, m)]
        y = alphabet[rng.integers(0, 100, n)].copy()
        k = min(m, n) // 2
        y[:k] = x[:k]
        pairs.append((bytes(x), bytes(y)))
    batch = pack_pairs(pairs)
    for mode, go in (("local", -6), ("global", -4), ("semiglobal", -5)):
        s, keep1 = oracle.make_scoring(go, -1, 0, 0, table)
        ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=4)
        cs, keep2 = _c_scoring(go, -1, 0, 0, table=table, alphabet=bytes(alphabet))
        got, ops = _engine_result(eng, mode, cs, batch)
        assert_same(got, ops, ref, ref_ops, batch, f"100-symbol table {mode}")
    wide = bytes(range(20, 220))
    cs, keep = _c_scoring(-5, -1, 0, 0, table=table, alphabet=wide)
    with pytest.raises(B2AError, match="128 distinct"):
        eng.align_batch(MODES["local"], cs, batch)
