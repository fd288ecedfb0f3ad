"""bio::alignment::distance on the H100 (b2a_levenshtein_batch, b2a_hamming_batch and their multi-GPU forms) against
the oracle (tests/sim/distance_oracle.cpp): the host suite's input matrix with every tier reached, a 100k-pair batch
against the aligner under unit costs, long protein pairs, bounded long similar pairs, Hamming statuses, and two
engines on one card against one."""
import numpy as np
import pytest

import distance_util as du
from distance_util import NONE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _lev(eng, pairs, k=None):
    d = eng.levenshtein_batch(du.pack_unaligned(pairs), k)
    want = [0] * 8
    for x, y in pairs:
        want[du.dist_tier(len(x), len(y), k)] += 1
    assert eng.distance_tier_pairs() == want, k  # every pair ran the tier its lengths and bound pick
    return [None if (k is not None and v == NONE) else int(v) for v in d]


def test_matrix_every_tier(eng):
    rng = np.random.default_rng(5)
    pairs = du.edge_pairs() + du.strip_pairs()
    for P in (300, 700, 1500):
        x = du.rand_seq(rng, P)
        pairs.append((x, du.mutate(rng, x, 0.02, b"ACGT")))
    want = [du.orc_levenshtein(x, y) for x, y in pairs]
    assert _lev(eng, pairs) == want
    assert eng.stats.cells == sum(len(x) * len(y) for x, y in pairs)
    tiers = eng.distance_tier_pairs()
    assert all(tiers[t] for t in (1, 2, 3, 4, 7))  # the register tier's four word counts and the warp tier
    assert eng.stats.kernel_launches == 1 + 5  # the rewrite into codes, one launch per tier
    seen = set()
    # the bounds around each distance: every pair of one batch per bound, so the band tiers, the warp tier's early
    # exit and |m - n| > k all run
    for delta in (-1, 0, 1):
        ks = [max(w + delta, 0) for w in want]
        for kk in sorted(set(ks)):
            sel = [i for i, v in enumerate(ks) if v == kk]
            got = _lev(eng, [pairs[i] for i in sel], kk)
            assert got == [du.orc_bounded(*pairs[i], kk) for i in sel], kk
            seen |= {t for t, c in enumerate(eng.distance_tier_pairs()) if c}
    assert _lev(eng, pairs, 0) == [du.orc_bounded(x, y, 0) for x, y in pairs]
    assert _lev(eng, pairs, 20) == [du.orc_bounded(x, y, 20) for x, y in pairs]
    assert _lev(eng, pairs, 150) == [du.orc_bounded(x, y, 150) for x, y in pairs]
    seen |= {t for t, c in enumerate(eng.distance_tier_pairs()) if c}
    assert {0, 5, 6, 7} <= seen  # host-answered, both bands, and the warp tier under a bound


def test_100k_reads_equal_the_aligner(eng):
    from rust_bio_b200 import synth
    from rust_bio_b200._lib import MIN_SCORE, MODE_GLOBAL, CScoring
    batch = synth.uniform_pairs(synth.BASES["C2"], 0, 100_000, 150, 150)
    unit = CScoring(-1, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 0, -1, 1, None, None, 0)
    d = eng.levenshtein_batch(batch)
    s = eng.align_batch_scores(MODE_GLOBAL, unit, batch)
    assert np.array_equal(d.astype(np.int64), -s["score"].astype(np.int64))


def test_long_protein_pairs(eng):
    rng = np.random.default_rng(9)
    prot = b"ACDEFGHIKLMNPQRSTVWY"
    x = du.rand_seq(rng, 10000, prot)
    pairs = [(x, du.mutate(rng, x, 0.3, prot)), (du.rand_seq(rng, 10000, prot), du.rand_seq(rng, 10000, prot))]
    assert _lev(eng, pairs) == [du.orc_levenshtein(a, b) for a, b in pairs]


def test_bounded_long_similar_pairs(eng):
    rng = np.random.default_rng(10)
    pairs = []
    for L in (5000, 8000, 12000):
        x = du.rand_seq(rng, L)
        pairs.append((x, du.mutate(rng, x, 0.01, b"ACGT")))
    ds = [du.orc_levenshtein(x, y) for x, y in pairs]
    for k in (10, 60, 100, 200, 400):
        assert _lev(eng, pairs, k) == [d if d <= k else None for d in ds], k


def test_hamming_statuses(eng):
    rng = np.random.default_rng(12)
    pairs = [(b"GTCTGCATGCG", b"TTTAGCTAGCG"), (b"GACTATATCGA", b"TTTAGCTC"), (b"", b"")]
    for L in (1, 3, 4, 5, 129, 1000, 100000):
        x = du.rand_seq(rng, L)
        pairs.append((x, du.mutate(rng, x, 0.0, b"ACGT")))
        pairs.append((x, bytes(rng.integers(0, 256, L).astype(np.uint8))))
    batch = du.pack_unaligned(pairs)
    d, st = eng.hamming_batch(batch)
    want = [du.orc_hamming(x, y) for x, y in pairs]
    assert [None if s else int(v) for v, s in zip(d, st)] == want
    assert [int(s) for s in st] == [0 if w is not None else 1 for w in want]
    from rust_bio_b200._lib import B2AError
    with pytest.raises(B2AError, match=r"pair 1: hamming distance cannot be calculated for texts of different length \(11!=8\)"):
        eng.hamming_batch(batch, pair_status=False)
    ok = [p for p, w in zip(pairs, want) if w is not None]
    assert [int(v) for v in eng.hamming_batch(du.pack_unaligned(ok), pair_status=False)] == [w for w in want if w is not None]


def test_python_mirror(eng):
    from rust_bio_b200 import distance
    assert distance.levenshtein(b"ACCGTGGAT", b"AAAAACCGTTGAT", engine=eng) == 5
    assert distance.simd.levenshtein(b"TTTT", b"AAA", engine=eng) == 4
    assert distance.simd.bounded_levenshtein(b"ACCGTGGAT", b"AAAAACCGTTGAT", 5, engine=eng) == 5
    assert distance.simd.bounded_levenshtein(b"ACCGTGGAT", b"AAAAACCGTTGAT", 4, engine=eng) is None
    assert distance.simd.bounded_levenshtein(b"AAA", b"TTTT", 0xFFFFFFFF, engine=eng) == 4
    assert distance.hamming(b"GTCTGCATGCG", b"TTTAGCTAGCG", engine=eng) == 5
    assert distance.hamming_batch([(b"AC", b"AG"), (b"A", b"AC")], on_panic="none", engine=eng) == [1, None]


def test_multi_engine_equals_one(eng):
    from rust_bio_b200.engine import MultiEngine
    rng = np.random.default_rng(13)
    pairs = du.edge_pairs() + du.strip_pairs()
    for _ in range(200):
        x = du.rand_seq(rng, int(rng.integers(0, 400)))
        pairs.append((x, du.mutate(rng, x, 0.05, b"ACGT")))
    batch = du.pack_unaligned(pairs)
    m = MultiEngine([0, 0])
    try:
        for k in (None, 5, 40):
            assert np.array_equal(m.levenshtein_batch(batch, k), eng.levenshtein_batch(batch, k)), k
        hp = [(x, y[:len(x)] if len(y) >= len(x) else y) for x, y in pairs]
        hb = du.pack_unaligned(hp)
        d1, s1 = m.hamming_batch(hb)
        d0, s0 = eng.hamming_batch(hb)
        assert np.array_equal(d1, d0) and np.array_equal(s1, s0)
        from rust_bio_b200._lib import B2AError
        with pytest.raises(B2AError, match=r"pair %d: hamming distance" % int(np.flatnonzero(s0)[0])):
            m.hamming_batch(hb, pair_status=False)
        # the only unequal pair is the last, in the second device's share: the error names the caller's index
        ok = [p for p, st in zip(hp, s0) if st == 0] + [(b"ACGT", b"AC")]
        with pytest.raises(B2AError, match=r"pair %d: hamming distance" % (len(ok) - 1)):
            m.hamming_batch(du.pack_unaligned(ok), pair_status=False)
    finally:
        m.close()
