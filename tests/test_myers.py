"""bio::pattern_matching::myers without a GPU: the reference's known answers (tests/golden/myers_vectors.json) against
the semi-global oracle (tests/sim/myers_oracle.cpp), the oracle tied to the edit-distance definition by brute force,
the Python mirror's panics and empty-text values, and the kernels' lane logic (tests/sim/b2a_sim_myers.cpp: the
register tier at 1..4 words, the warp tier on 32 emulated lanes) against the oracle."""
import json
import os

import numpy as np
import pytest

import distance_util as du
import myers_util as mu
from myers_util import MT_REGS1, MT_WARP

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "myers_vectors.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def golden_match(v):
    """(ambig, wildcards) of a golden vector in myers_util's form"""
    ambig = None
    if "ambig" in v:
        ambig = {}
        for b, eqs in v["ambig"]:
            ambig[ord(b)] = ambig.get(ord(b), b"") + eqs.encode()
    return ambig, v["wildcards"].encode() if "wildcards" in v else None


def test_oracle_matches_reference_answers(golden):
    for v in golden["find_all_end"]:
        _, _, hits = mu.orc_search(v["pattern"].encode(), v["text"].encode(), v["k"])
        assert [list(h) for h in hits] == v["hits"], v["cite"]
    for v in golden["first_hits"]:
        _, _, hits = mu.orc_search(v["pattern"].encode(), v["text"].encode(), v["k"])
        assert [list(h) for h in hits[:len(v["hits"])]] == v["hits"], v["cite"]
    for v in golden["distance"]:
        ambig, wild = golden_match(v)
        end, d, _ = mu.orc_search(v["pattern"].encode(), v["text"].encode(), None, ambig, wild)
        assert d == v["d"], v["cite"]
        if "best_end" in v:
            assert end == v["best_end"], v["cite"]
    for v in golden["max_hit_dist"]:
        _, _, hits = mu.orc_search(v["pattern"].encode(), v["text"].encode(), v["k"])
        assert max(d for _, d in hits) == v["max_dist"], v["cite"]


def test_oracle_is_min_levenshtein_over_starts():
    """D[m][j] == min over s of levenshtein(pattern, text[s:j]) (Sellers' semi-global recurrence restated)"""
    rng = np.random.default_rng(12)
    for i in range(120):
        alpha = b"ACGT" if i % 2 else b"AB"
        x = du.rand_seq(rng, int(rng.integers(1, 12)), alpha)
        y = du.rand_seq(rng, int(rng.integers(0, 16)), alpha)
        row = mu.orc_row(x, y)
        for j in range(1, len(y) + 1):
            assert row[j - 1] == min(mu.orc_levenshtein(x, y[s:j]) for s in range(j + 1)), (x, y, j)


def test_mirror_panics_and_empty_texts(golden):
    from rust_bio_b200.pattern_matching.myers import Myers, MyersBuilder, long
    for v in golden["panics"]:
        pat = b"T" * v["length"]
        with pytest.raises(AssertionError) as ei:
            if v.get("long"):
                long.Myers(pat, v["bits"])
            elif v.get("builder"):
                MyersBuilder().build_64(pat)
            else:
                Myers(pat, v["bits"])
        assert str(ei.value) == v["message"], v["cite"]
    Myers(b"T" * 64), Myers(b"T" * 128, 128), long.Myers(b"T" * 5000)  # at the limits: no panic
    # empty text: the reference's initial max_dist, no hits, and find_best_end's unwrap on None
    assert Myers(b"ACGT").distance(b"") == 255
    assert Myers(b"ACGT", 128).distance(b"") == 255
    assert long.Myers(b"ACGT").distance(b"") == (1 << 64) - 1 - 64
    assert long.Myers(b"ACGT", 128).distance(b"") == (1 << 64) - 1 - 128
    assert Myers(b"ACGT").find_all_end(b"", 3) == []
    with pytest.raises(AssertionError, match="unwrap"):
        Myers(b"ACGT").find_best_end(b"")
    with pytest.raises(OverflowError):
        Myers(b"ACGT").find_all_end(b"ACGT", 256)


def _check(pairs, k=None, ambig=None, wildcards=None, force_warp=False):
    got, tiers = mu.sim_myers(pairs, k, ambig, wildcards, force_warp)
    for (x, y), g in zip(pairs, got):
        assert g == mu.orc_search(x, y, k, ambig, wildcards), (len(x), len(y), k, force_warp)
    return got, tiers


def test_sim_every_tier():
    pairs = mu.matrix_pairs()
    got, tiers = _check(pairs, k=5)
    assert {MT_REGS1, MT_REGS1 + 1, MT_REGS1 + 2, MT_REGS1 + 3, MT_WARP} <= set(tiers)
    assert tiers == [mu.myers_tier(len(x), len(y)) for x, y in pairs]
    _check(pairs, k=5, force_warp=True)  # the warp tier on short patterns too: one strip, idle lanes


def test_sim_bounds_around_each_distance():
    """k = 0, each best distance - 1, itself and + 1, and k >= P (every end listed)"""
    pairs = mu.matrix_pairs(seed=3, lengths=(1, 63, 64, 65, 128, 129, 256, 257, 2049))
    best, _ = mu.sim_myers(pairs)
    for (x, y), (_, d, _) in zip(pairs, best):
        ks = {0, len(x), len(x) + 7} | ({max(d - 1, 0), d, d + 1} if d is not None else set())
        for k in sorted(ks):
            for force in (False, True):
                got, _ = _check([(x, y)], k, force_warp=force)
                if k >= len(x):
                    assert len(got[0][2]) == len(y)


def test_sim_ambiguity_and_wildcards():
    rng = np.random.default_rng(8)
    ambig = {ord(b): eqs for b, eqs in mu.IUPAC.items()}
    ambig[ord("Z")] = b"QX"  # equivalents absent from the batch drop out
    wild = b"N*#"            # N also occurs in patterns; # is absent from the batch
    pairs = [(b"TRANCGG", b"GGATGNGCGCCATAG"), (b"TRRRCGTR", b"TGATCRTR"), (b"ZZACGT", b"ACGTACG")]
    for P in (20, 64, 65, 200, 300, 2100):
        x = bytearray(du.rand_seq(rng, P))
        for q in rng.integers(0, P, max(1, P // 10)):
            x[q] = b"RYNKMSWBDHV"[rng.integers(0, 11)]
        y = bytearray(mu.plant(rng, bytes(x), P + 50, 0.05))
        for q in rng.integers(0, len(y), max(1, len(y) // 20)):
            y[q] = b"N*R"[rng.integers(0, 3)]  # wildcards and an ambiguous symbol in the text
        pairs.append((bytes(x), bytes(y)))
    for force in (False, True):
        _check(pairs, 4, ambig, wild, force)
        _check(pairs, 4, None, wild, force)
        _check(pairs, 4, ambig, None, force)


def test_sim_all_byte_values_and_shared_patterns():
    rng = np.random.default_rng(9)
    allb = bytes(range(256))
    pat = bytes(rng.permutation(256).astype(np.uint8))[:70]
    pairs = [(pat, allb + pat + allb[::-1]), (allb, allb), (pat, pat[5:60])]
    shared = du.rand_seq(rng, 40)
    pairs += [(shared, mu.plant(rng, shared, 150, 0.1)) for _ in range(6)]
    for force in (False, True):
        _check(pairs, 3, force_warp=force)
        _check(pairs, 3, {0: b"\xff\x01"}, b"\x80", force)
