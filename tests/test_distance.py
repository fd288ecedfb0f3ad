"""bio::alignment::distance without a GPU: the reference's known answers (tests/golden/distance_vectors.json) against
the oracle (tests/sim/distance_oracle.cpp, the definitions) and the Python mirror's panics; the oracle tied to the
pinned pairwise oracle; and the kernels' lane logic (tests/sim/b2a_sim_distance.cpp: every tier, the warp tier on 32
emulated lanes) against the oracle."""
import json
import os

import numpy as np
import pytest

import distance_util as du
from distance_util import DT_BAND4, DT_BAND8, DT_WARP, NONE

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "distance_vectors.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_oracle_matches_reference_answers(golden):
    for v in golden["levenshtein"]:
        assert du.orc_levenshtein(v["x"].encode(), v["y"].encode()) == v["d"]
    for v in golden["bounded_levenshtein"]:
        assert du.orc_bounded(v["x"].encode(), v["y"].encode(), v["k"]) == v["d"]
    for v in golden["hamming"]:
        assert du.orc_hamming(v["x"].encode(), v["y"].encode()) == v["d"]
    for v in golden["hamming_panics"]:
        assert du.orc_hamming(v["x"].encode(), v["y"].encode()) is None


def test_mirror_raises_reference_messages(golden):
    from rust_bio_b200 import distance
    for v in golden["hamming_panics"]:
        fn = distance.simd.hamming if v["simd"] else distance.hamming
        with pytest.raises(AssertionError) as ei:
            fn(v["x"].encode(), v["y"].encode())
        assert str(ei.value) == v["message"]
    with pytest.raises(AssertionError, match=r"^hamming distance cannot be calculated for texts of different length \(1!=2\)$"):
        distance.hamming_batch([(b"A", b"A"), (b"A", b"AC")])
    with pytest.raises(OverflowError):
        distance.bounded_levenshtein_batch([(b"A", b"C")], 1 << 32)


def test_oracle_is_global_alignment_under_unit_costs():
    """levenshtein(x, y) == -(global score) under gap_open = -1, gap_extend = -1, match 0, mismatch -1: a gap of length
    L costs gap_open + (L - 1) gap_extend = -L (pairwise/mod.rs:9-15)"""
    from oracle import oracle as orc
    s, _ = orc.make_scoring(-1, -1, 0, -1)
    rng = np.random.default_rng(11)
    for i in range(300):
        alpha = b"ACGT" if i % 3 else b"ACDEFGHIKLMNPQRSTVWY"
        x = du.rand_seq(rng, int(rng.integers(0, 60)), alpha)
        y = du.mutate(rng, x, 0.2, alpha) if i % 2 else du.rand_seq(rng, int(rng.integers(0, 60)), alpha)
        d, _ = orc.align("global", s, x, y)
        assert du.orc_levenshtein(x, y) == -d["score"], (x, y)


def _check_levenshtein(pairs, force_tier=-1):
    got, tiers = du.sim_levenshtein(pairs, None, force_tier)
    for (x, y), g in zip(pairs, got):
        assert g == du.orc_levenshtein(x, y), (len(x), len(y))
    return tiers


def test_sim_levenshtein_every_tier():
    pairs = du.edge_pairs()
    tiers = _check_levenshtein(pairs)
    assert {1, 2, 3, 4, DT_WARP} <= set(tiers)  # the register tier's 1..4 words, the warp tier beyond 256 rows
    _check_levenshtein(pairs, force_tier=DT_WARP)  # the warp tier on short patterns too: one strip, idle lanes


def test_sim_levenshtein_strip_edges():
    pairs = du.strip_pairs()
    assert set(_check_levenshtein(pairs)) == {DT_WARP}


def _bounds(d):
    return sorted({0, max(d - 1, 0), d, d + 1, NONE})


def test_tier_rule_mirror():
    """tests' copy of dist_tier (used to check the engine's per-tier counts on the GPU) against the kernels' own"""
    pairs = du.edge_pairs() + du.strip_pairs()
    rng = np.random.default_rng(4)
    for P in (300, 700, 1500):
        x = du.rand_seq(rng, P)
        pairs.append((x, du.mutate(rng, x, 0.02, b"ACGT")))
    for k in (None, 0, 5, 95, 96, 223, 224):
        _, tiers = du.sim_levenshtein(pairs, k)
        assert tiers == [du.dist_tier(len(x), len(y), k) for x, y in pairs], k


def test_sim_bounded_levenshtein():
    """k in {0, d-1, d, d+1, none}, in the engine's tier and forced into each band width and the warp tier"""
    rng = np.random.default_rng(5)
    pairs = du.edge_pairs()
    for P in (300, 700, 1500):  # long patterns with few edits: the band tiers
        x = du.rand_seq(rng, P)
        pairs.append((x, du.mutate(rng, x, 0.02, b"ACGT")))
    seen = set()
    for x, y in pairs:
        d = du.orc_levenshtein(x, y)
        for k in _bounds(d):
            want = du.orc_bounded(x, y, k)
            for force in (-1, DT_BAND4, DT_BAND8, DT_WARP):
                got, tiers = du.sim_levenshtein([(x, y)], k, force)
                assert got[0] == want, (len(x), len(y), k, force, tiers)
                seen.add(tiers[0])
    assert {DT_BAND4, DT_BAND8, DT_WARP} <= seen


def test_sim_bounded_length_gap_and_early_exit():
    rng = np.random.default_rng(6)
    # |m - n| > k: None without DP
    got, tiers = du.sim_levenshtein([(b"ACGT" * 10, b"ACGT" * 12)], 7)
    assert got == [None] and tiers == [0]
    # unrelated long pairs with a small bound: the band's cutoff (every window cell above k) and the lower bound
    # D[P][j] - (n - j) > k stop early; the answer is still None
    for P in (200, 900, 2500):
        x, y = du.rand_seq(rng, P), du.rand_seq(rng, P + 3)
        for force in (-1, DT_BAND4, DT_BAND8, DT_WARP):
            got, _ = du.sim_levenshtein([(x, y)], 20, force)
            assert got == [None]
    # a pair that only goes wrong at the very end
    x = du.rand_seq(rng, 1000)
    y = x[:-30] + du.rand_seq(rng, 30)
    d = du.orc_levenshtein(x, y)
    for force in (-1, DT_BAND4, DT_BAND8, DT_WARP):
        assert du.sim_levenshtein([(x, y)], d - 1, force)[0] == [None]
        assert du.sim_levenshtein([(x, y)], d, force)[0] == [d]


def test_sim_hamming():
    rng = np.random.default_rng(7)
    pairs = [(b"GTCTGCATGCG", b"TTTAGCTAGCG"), (b"", b""), (b"GACTATATCGA", b"TTTAGCTC")]
    for L in (1, 3, 4, 5, 127, 128, 129, 1000):
        x = du.rand_seq(rng, L)
        pairs.append((x, du.mutate(rng, x, 0.0, b"ACGT")))
        pairs.append((x, bytes(rng.integers(0, 256, L).astype(np.uint8))))
    got = du.sim_hamming(pairs)
    assert got == [du.orc_hamming(x, y) for x, y in pairs]
