"""bio::stats::pairhmm::PairHMM::prob_related on the H100 (b2a_pairhmm_batch and its multi-GPU form) against the oracle
(tests/sim/pairhmm_oracle.cpp) under the tolerance rule: -inf exactly where the oracle gives -inf, else |gpu - oracle|
<= 1e-9 * max(1, |oracle|).  The device log1p against glibc's is the only expected difference.  Covers the host
suite's matrix with every tier reached, 100k read-window pairs with quality classes, 10k x 10k pairs, the golden
vectors through the mirror, NaN statuses, repeatability and two engines on one card against one."""
import json
import os

import numpy as np
import pytest

import distance_util as du
import pairhmm_util as pu

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pairhmm_vectors.json")))
MODES = {"global": (False, False), "semiglobal": (True, True), (1, 0): (True, False), (0, 1): (False, True)}


@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _threads():
    from oracle import oracle as orc
    return orc.hardware_threads()


def _gpu(eng, packed, gap, mode, med, emit, pair_status=True):
    blob, cls, xo, xl, yo, yl = packed
    fs, fe = MODES[mode]
    return eng.pairhmm_batch((blob, xo, xl, yo, yl), gap, emit, fs, fe, med, cls, pair_status=pair_status)


def _compare(eng, pairs, gap, mode, med, emit, classes=None):
    pk = pu.pack(pairs, classes)
    got, st = _gpu(eng, pk, gap, mode, med, emit)
    want = pu.orc_batch(gap, mode, med, emit, pk, threads=_threads())
    bad = pu.within(got, want)
    assert not bad, (mode, med, [(int(pk[3][i]), int(pk[5][i]), got[i], want[i]) for i in bad[:5]])
    assert np.array_equal(st != 0, np.isnan(want))
    tiers = [0] * 7
    for x, y in pairs:
        tiers[_tier(len(x), len(y))] += 1
    assert eng.pairhmm_tier_pairs() == tiers  # every pair ran the tier its len_y picks
    return got, want


def _tier(m, n):
    if m == 0 or n == 0:
        return pu.PT_DONE
    for t, hi in ((pu.PT_C1, 32), (pu.PT_C2, 64), (pu.PT_C4, 128), (pu.PT_C5, 160), (pu.PT_C8, 256)):
        if n <= hi:
            return t
    return pu.PT_STRIP


def test_matrix(eng):
    pairs = pu.matrix_pairs(seed=1)
    seen = set()
    for name, gap, emit in pu.PARAMS:
        for mode in MODES:
            for med in pu.MAX_EDIT:
                _compare(eng, pairs, gap, mode, med, emit)
                seen |= {i for i, c in enumerate(eng.pairhmm_tier_pairs()) if c}
    assert seen == set(range(7))


def test_matrix_classes(eng):
    rng = np.random.default_rng(5)
    pairs = pu.matrix_pairs(seed=2)
    cls = pu.random_classes(rng, pairs, 42)
    for mode in ("global", "semiglobal"):
        for med in pu.MAX_EDIT:
            _compare(eng, pairs, pu.GAP_EXT, mode, med, pu.quality_emit(42), cls)


def _reads_in_windows(rng, n_reads, read_len, win_len, n_windows, rate=0.02):
    wins = [du.rand_seq(rng, win_len) for _ in range(n_windows)]
    pairs = []
    for r in range(n_reads):
        w = wins[r % n_windows]
        st = int(rng.integers(0, win_len - read_len + 1))
        y = du.mutate(rng, w[st:st + read_len], rate, b"ACGT")
        pairs.append((w, y if r % 10 else du.rand_seq(rng, read_len)))  # every tenth read unrelated
    return pairs


def test_100k_reads_with_quality_classes(eng):
    rng = np.random.default_rng(17)
    pairs = _reads_in_windows(rng, 100_000, 150, 200, 2000)
    cls = pu.random_classes(rng, pairs, 42)
    _compare(eng, pairs, pu.GAP_EXT, "semiglobal", 4, pu.quality_emit(42), cls)


def test_10k_by_10k(eng):
    rng = np.random.default_rng(23)
    pairs = []
    for i in range(8):
        x = du.rand_seq(rng, 10_000)
        pairs.append((x, du.mutate(rng, x, 0.01 if i % 2 else 0.2, b"ACGT")[:10_000]))
    _compare(eng, pairs, pu.ILLUMINA_GAP, "global", None, pu.ILLUMINA_EMIT)
    _compare(eng, pairs[:4], pu.GAP_EXT, "semiglobal", 20, pu.ILLUMINA_EMIT)


@pytest.mark.parametrize("case", GOLDEN["prob_related"], ids=lambda c: c["name"])
def test_golden_through_mirror(eng, case):
    from rust_bio_b200.stats import pairhmm as ph
    hmm = ph.PairHMM.new(ph.GapParams(*[float(v) for v in case["gap"]]), engine=eng)
    mode = ph.SEMIGLOBAL if case["mode"] == "semiglobal" else ph.GLOBAL
    em = ph.ClassEmission(case["x"].encode(), case["y"].encode(), case["emit"])
    p = hmm.prob_related(em, mode, case["max_edit_dist"])
    pk = pu.pack([(case["x"].encode(), case["y"].encode())])
    want = pu.orc_batch([float(v) for v in case["gap"]], case["mode"], case["max_edit_dist"], case["emit"], pk)
    assert not pu.within([p], want)
    for chk in case["checks"]:
        if chk["kind"] == "eq":
            assert p == float(chk["value"])
        elif chk["kind"] == "le":
            assert p <= chk["value"]
        elif chk["kind"] == "relative_eq":
            assert abs(p - chk["value"]) <= chk["epsilon"]
        elif chk["kind"] == "relative_eq_unbanded":
            assert abs(p - hmm.prob_related(em, mode, None)) <= chk["epsilon"]


def test_nan_class_entry_statuses(eng):
    """A NaN class entry is B2A_PAIR_PANIC for exactly the pairs whose result it makes NaN; without a status array the
    call fails with B2A_E_INVALID naming the first.  The NaN class sits on y's last column: its fm is NaN on every row,
    and a NaN in the first or maximum slot of a sum stays NaN.  (Elsewhere a NaN can be absorbed: fastexp(NaN) is 0,
    so a NaN beside a finite maximum drops out of a sum, in the reference too.)"""
    from rust_bio_b200._lib import B2AError
    rng = np.random.default_rng(31)
    pairs = _reads_in_windows(rng, 400, 60, 100, 8)
    cls = [(bytes(len(x)), bytes(len(y))) for x, y in pairs]
    uses = sorted(int(i) for i in rng.choice(len(pairs), 25, replace=False))
    for i in uses:
        c = bytearray(cls[i][1])
        c[-1] = 3
        cls[i] = (cls[i][0], bytes(c))
    emit = pu.quality_emit(4)
    emit[0][3] = emit[1][3] = float("nan")
    pk = pu.pack(pairs, cls)
    for mode in ("semiglobal", "global"):
        got, st = _gpu(eng, pk, pu.GAP_EXT, mode, None, emit)
        want = pu.orc_batch(pu.GAP_EXT, mode, None, emit, pk)
        panics = [int(i) for i in np.nonzero(st)[0]]
        assert panics == uses == [int(i) for i in np.nonzero(np.isnan(want))[0]]
        assert np.all(np.isnan(got[uses])) and not pu.within(got, want)
        with pytest.raises(B2AError) as ei:
            _gpu(eng, pk, pu.GAP_EXT, mode, None, emit, pair_status=False)
        assert ei.value.code == -1 and f"pair {uses[0]}:" in str(ei.value)


def test_input_errors(eng):
    from rust_bio_b200._lib import B2AError
    pk = pu.pack([(b"ACGT", b"ACG")], [(b"\0\0\0\0", b"\0\5\0")])
    with pytest.raises(B2AError) as ei:
        _gpu(eng, pk, pu.GAP_EXT, "global", None, pu.quality_emit(4))
    assert ei.value.code == -1 and "class byte 5" in str(ei.value)
    pk = pu.pack([(b"ACGT", b"ACG")])
    for gap in ((0.1, -1.0, -np.inf, -np.inf), (-1.0, -1.0, 0.5, -np.inf), (-1.0, -1.0, -np.inf, float("nan"))):
        with pytest.raises(B2AError) as ei:
            _gpu(eng, pk, gap, "global", None, pu.ILLUMINA_EMIT)
        assert ei.value.code == -1 and "p <= 0.0" in str(ei.value)


def test_repeatable(eng):
    rng = np.random.default_rng(41)
    pairs = _reads_in_windows(rng, 3000, 150, 400, 30) + pu.matrix_pairs(seed=6)
    cls = pu.random_classes(rng, pairs, 42)
    pk = pu.pack(pairs, cls)
    a, _ = _gpu(eng, pk, pu.GAP_EXT, "semiglobal", 4, pu.quality_emit(42))
    b, _ = _gpu(eng, pk, pu.GAP_EXT, "semiglobal", 4, pu.quality_emit(42))
    assert np.array_equal(pu.bits(a), pu.bits(b))


def test_multi_engine_two_on_one_card(eng):
    from rust_bio_b200.engine import MultiEngine
    from rust_bio_b200._lib import B2AError
    rng = np.random.default_rng(43)
    pairs = _reads_in_windows(rng, 5001, 150, 200, 40) + pu.matrix_pairs(seed=7)
    cls = [(cx.replace(b"\7", b"\10"), cy.replace(b"\7", b"\10")) for cx, cy in pu.random_classes(rng, pairs, 42)]
    half = len(pairs) // 2
    nan_pairs = [half + 17, half + 300, len(pairs) - 40]  # class 7 (NaN below) on y's last column, second share only
    for p in nan_pairs:
        cls[p] = (cls[p][0], cls[p][1][:-1] + b"\7")
    pk = pu.pack(pairs, cls)
    emit = pu.quality_emit(42)
    me = MultiEngine([0, 0])
    try:
        for mode, med in (("semiglobal", None), ("semiglobal", 2), ("global", None)):
            a, sa = _gpu(eng, pk, pu.GAP_EXT, mode, med, emit)
            b, sb = _gpu(me, pk, pu.GAP_EXT, mode, med, emit)
            assert np.array_equal(pu.bits(a), pu.bits(b)) and np.array_equal(sa, sb)
        emit[0][7] = emit[1][7] = float("nan")  # a panic in the second share is named by its index in the whole batch
        a, sa = _gpu(eng, pk, pu.GAP_EXT, "semiglobal", None, emit)
        b, sb = _gpu(me, pk, pu.GAP_EXT, "semiglobal", None, emit)
        assert [int(i) for i in np.nonzero(sa)[0]] == nan_pairs and np.array_equal(sa, sb)
        assert np.array_equal(pu.bits(a), pu.bits(b))
        with pytest.raises(B2AError) as ei:
            _gpu(me, pk, pu.GAP_EXT, "semiglobal", None, emit, pair_status=False)
        assert f"pair {nan_pairs[0]}:" in str(ei.value)
    finally:
        me.close()
