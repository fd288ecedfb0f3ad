"""bio::pattern_matching::myers on the H100 (b2a_myers_batch, b2a_myers_hits_fetch and their multi-GPU forms) against
the oracle (tests/sim/myers_oracle.cpp): the host suite's input matrix with every tier reached, ambiguity and
wildcards, bounds around each distance, 100k reads against the semi-global aligner under unit costs, a listing of
every end of 10k texts, empty-pattern statuses, the held hit list, the Python mirror on the reference's examples, and
two engines on one card against one."""
import json
import os

import numpy as np
import pytest

import distance_util as du
import myers_util as mu
from myers_util import NONE

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "myers_vectors.json")


@pytest.fixture(scope="module")
def eng():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _run(eng, pairs, k=None, ambig=None, wildcards=None):
    """-> per pair (best_end, best_dist, hits) as myers_util's oracle gives them, after checking the tier counts"""
    r = eng.myers_batch(mu.pack_shared(pairs), k, ambig=ambig, wildcards=wildcards)
    want = [0] * 6
    for x, y in pairs:
        want[mu.myers_tier(len(x), len(y))] += 1
    assert eng.myers_tier_pairs()[:6] == want  # every pair ran the tier its pattern length picks
    out = []
    for p in range(len(pairs)):
        e, d = int(r["best_end"][p]), int(r["best_dist"][p])
        hits = None
        if k is not None:
            lo, hi = int(r["hit_off"][p]), int(r["hit_off"][p + 1])
            hits = list(zip(r["hit_end"][lo:hi].tolist(), r["hit_dist"][lo:hi].tolist()))
        out.append((None if e == NONE else e, None if d == NONE else d, hits))
    return out


def _check(eng, pairs, k=None, ambig=None, wildcards=None):
    got = _run(eng, pairs, k, ambig, wildcards)
    for (x, y), g in zip(pairs, got):
        assert g == mu.orc_search(x, y, k, ambig, wildcards), (len(x), len(y), k)
    return got


def test_matrix_every_tier(eng):
    pairs = mu.matrix_pairs()
    _check(eng, pairs, 5)
    assert all(eng.myers_tier_pairs()[t] for t in range(1, 6))
    assert eng.myers_tier_pairs()[6] == sum(1 for x, y in pairs if mu.orc_search(x, y, 5)[2])  # pass 2's pairs
    _check(eng, pairs)  # no listing: best ends only


def test_bounds_around_each_distance(eng):
    pairs = mu.matrix_pairs(seed=3)
    best = _run(eng, pairs)
    ks = {0}
    for (x, _), (_, d, _) in zip(pairs, best):
        ks |= {len(x)} | ({max(d - 1, 0), d, d + 1} if d is not None else set())
    for k in sorted(ks)[:40] + [max(ks)]:
        _check(eng, pairs, k)


def test_ambiguity_and_wildcards(eng):
    rng = np.random.default_rng(8)
    ambig = {ord(b): eqs for b, eqs in mu.IUPAC.items()}
    ambig[ord("Z")] = b"QX"
    wild = b"N*#"
    pairs = [(b"TRANCGG", b"GGATGNGCGCCATAG"), (b"TRRRCGTR", b"TGATCRTR"), (b"ZZACGT", b"ACGTACG")]
    for P in (20, 64, 65, 200, 300, 2100, 4097):
        x = bytearray(du.rand_seq(rng, P))
        for q in rng.integers(0, P, max(1, P // 10)):
            x[q] = b"RYNKMSWBDHV"[rng.integers(0, 11)]
        y = bytearray(mu.plant(rng, bytes(x), P + 50, 0.05))
        for q in rng.integers(0, len(y), max(1, len(y) // 20)):
            y[q] = b"N*R"[rng.integers(0, 3)]
        pairs.append((bytes(x), bytes(y)))
    for a, w in ((ambig, wild), (None, wild), (ambig, None), ({0: b"\xff"}, b"\x80")):
        _check(eng, pairs, 4, a, w)


def test_100k_reads_equal_the_semiglobal_aligner(eng):
    """best_dist == -(semiglobal score) under gap_open = gap_extend = -1, match 0, mismatch -1"""
    from rust_bio_b200._lib import MIN_SCORE, MODE_SEMIGLOBAL, CScoring
    rng = np.random.default_rng(21)
    pairs = []
    for _ in range(100_000):
        x = du.rand_seq(rng, int(rng.integers(20, 150)))
        pairs.append((x, mu.plant(rng, x, 150, 0.1) if rng.random() < 0.5 else du.rand_seq(rng, 150)))
    batch = mu.pack_shared(pairs)
    r = eng.myers_batch(batch)
    unit = CScoring(-1, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 0, -1, 1, None, None, 0)
    s = eng.align_batch_scores(MODE_SEMIGLOBAL, unit, batch)
    assert np.array_equal(r["best_dist"].astype(np.int64), -s["score"].astype(np.int64))
    for p in rng.integers(0, len(pairs), 300):
        x, y = pairs[p]
        assert (int(r["best_end"][p]), int(r["best_dist"][p])) == mu.orc_search(x, y)[:2]


def test_every_end_listed(eng):
    """k >= P on 10k x 1,000: 10M hits; the offsets are the text lengths and a sample equals the oracle"""
    rng = np.random.default_rng(22)
    x = du.rand_seq(rng, 150)
    pairs = [(x, mu.plant(rng, x, 1000, 0.1)) for _ in range(10_000)]
    r = eng.myers_batch(mu.pack_shared(pairs), 150)
    assert int(r["hit_off"][-1]) == 10_000 * 1000
    assert np.array_equal(np.diff(r["hit_off"]), np.full(10_000, 1000, dtype=np.uint64))
    for p in rng.integers(0, len(pairs), 40):
        lo = int(r["hit_off"][p])
        row = mu.orc_row(*pairs[p])
        assert r["hit_end"][lo:lo + 1000].tolist() == list(range(1000))
        assert r["hit_dist"][lo:lo + 1000].tolist() == row


def test_empty_pattern_statuses_and_held_hits(eng):
    from rust_bio_b200._lib import B2AError
    pairs = [(b"ACGT", b"TTACGTT"), (b"", b"ACGT"), (b"ACG", b""), (b"GG", b"AGGA")]
    r = eng.myers_batch(mu.pack_shared(pairs), 1)
    assert r["status"].tolist() == [0, 1, 0, 0]
    assert r["best_dist"].tolist()[1:3] == [NONE, NONE] and r["best_end"].tolist()[1:3] == [NONE, NONE]
    assert np.diff(r["hit_off"]).tolist()[1:3] == [0, 0]
    with pytest.raises(B2AError, match=r"pair 1: Pattern is empty"):
        eng.myers_batch(mu.pack_shared(pairs), 1, pair_status=False)
    # the held hits: gone after a call without a listing, or after any other call
    eng.myers_batch(mu.pack_shared(pairs[:1]), 1)
    eng.levenshtein_batch(du.pack_unaligned(pairs[:1]))
    with pytest.raises(B2AError, match="B2A_E_STATE"):
        eng._check(eng._c_myers_fetch(None, None, None))
    eng.myers_batch(mu.pack_shared(pairs[:1]))
    with pytest.raises(B2AError, match="B2A_E_STATE"):
        eng._check(eng._c_myers_fetch(None, None, None))


def test_listing_above_the_budget_is_refused():
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    try:
        e.set_traceback_budget(8 * 999)
        pairs = [(b"ACGT", b"A" * 1000)]
        with pytest.raises(B2AError, match="B2A_E_CAPACITY.*1000 hits"):
            e.myers_batch(mu.pack_shared(pairs), 4)
        assert len(e.myers_batch(mu.pack_shared([(b"ACGT", b"A" * 999)]), 4)["hit_end"]) == 999
    finally:
        e.close()


def test_python_mirror_reference_examples(eng):
    from rust_bio_b200.pattern_matching.myers import Myers, MyersBuilder, long
    with open(GOLDEN) as f:
        golden = json.load(f)
    for v in golden["find_all_end"]:
        for m in (Myers(v["pattern"].encode(), engine=eng), long.Myers(v["pattern"].encode(), engine=eng)):
            assert [list(h) for h in m.find_all_end(v["text"].encode(), v["k"])] == v["hits"], v["cite"]
    for v in golden["first_hits"]:
        m = long.Myers(v["pattern"].encode(), engine=eng)
        assert [list(h) for h in m.find_all_end(v["text"].encode(), v["k"])][:len(v["hits"])] == v["hits"]
    for v in golden["distance"]:
        b = MyersBuilder()
        for sym, eqs in v.get("ambig", []):
            b.ambig(ord(sym), eqs.encode())
        for w in v.get("wildcards", "").encode():
            b.text_wildcard(w)
        for build in (b.build_64, b.build_128, b.build_long_64, b.build_long_128):
            m = build(v["pattern"].encode(), engine=eng)
            assert m.distance(v["text"].encode()) == v["d"], v["cite"]
            if "best_end" in v:
                assert m.find_best_end(v["text"].encode()) == (v["best_end"], v["d"])
    for v in golden["max_hit_dist"]:
        hits = Myers(v["pattern"].encode(), engine=eng).find_all_end(v["text"].encode(), v["k"])
        assert max(d for _, d in hits) == v["max_dist"]
    m = Myers(b"TCCTAGGGC", engine=eng)  # the batch forms: one pattern, many texts (and an empty one)
    texts = [b"CGGTCCTGAGGGATTAGCAC", b"", b"TCCTAGGGC"]
    assert m.find_all_end_batch(texts, 2) == [m.find_all_end(t, 2) for t in texts]
    assert m.distance_batch(texts) == [2, 255, 0]
    assert m.find_best_end_batch([texts[0], texts[2]]) == [(11, 2), (8, 0)]


def test_multi_engine_equals_one(eng):
    from rust_bio_b200.engine import MultiEngine
    from rust_bio_b200._lib import B2AError
    pairs = mu.matrix_pairs(seed=5)
    batch = mu.pack_shared(pairs)
    one = eng.myers_batch(batch, 7, wildcards=b"N")
    m = MultiEngine([0, 0])
    try:
        got = m.myers_batch(batch, 7, wildcards=b"N")
        for f in ("best_end", "best_dist", "status", "hit_off", "hit_end", "hit_dist"):
            assert np.array_equal(got[f], one[f]), f
        small = mu.pack_shared(pairs[:1])  # fewer pairs than devices: the whole batch on entry 0
        assert np.array_equal(m.myers_batch(small, 7)["hit_end"], eng.myers_batch(small, 7)["hit_end"])
        with pytest.raises(B2AError, match=r"pair 2: Pattern is empty"):
            m.myers_batch(mu.pack_shared([(b"A", b"A"), (b"A", b"C"), (b"", b"A"), (b"C", b"A")]), 1,
                          pair_status=False)
        m.levenshtein_batch(du.pack_unaligned(pairs[:4]))
        with pytest.raises(B2AError, match="B2A_E_STATE"):
            m._check(m._c_myers_fetch(None, None, None))
    finally:
        m.close()
