"""The banded and score-only aligners on several devices from one process (b2a_multi_align_batch_banded,
b2a_multi_align_batch_scores, b2a_multi_align_batch_banded_scores) and the per-pair statuses of
b2a_multi_align_batch: every result equals the single engine's on the same batch.  Device lists that repeat device 0
run everywhere (one engine and stream per entry, peer copies onto entry 0); lists of distinct devices run where that
many GPUs exist.  Also the compaction of a single engine's banded results (b2a_batch_compact_* after a banded call)."""
import ctypes as C

import numpy as np
import pytest

from parity_util import MODES
from rust_bio_b200 import synth

pytestmark = pytest.mark.gpu

MIN = -858993459
FIELDS = ("score", "xstart", "xend", "ystart", "yend")
LISTS = {"0,0": [0, 0], "0,0,0": [0, 0, 0], "gpus2": [0, 1], "gpus4": [0, 1, 2, 3]}


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.fixture(scope="module")
def single():
    from rust_bio_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module", params=list(LISTS))
def me(request):
    from rust_bio_b200.engine import MultiEngine
    ids = LISTS[request.param]
    if max(ids) >= _n_gpus():
        pytest.skip(f"needs {max(ids) + 1} GPUs")
    m = MultiEngine(ids)
    m.ids = ids  # the list this engine was made from
    assert m.n_devices == len(ids)
    yield m
    m.close()


def _cs(clips=(MIN, MIN, MIN, MIN), table=None, alpha=None, go=-5, ge=-1, match=1, mismatch=-1):
    from rust_bio_b200._lib import CScoring
    return CScoring(go, ge, *clips, match, mismatch, 1 if table is None else 0,
                    table.ctypes.data_as(C.c_void_p) if table is not None else None,
                    alpha.ctypes.data_as(C.c_void_p) if alpha is not None else None, 0 if alpha is None else len(alpha))


def _window_pair(rng, xlen, ylen, nsub=5, alphabet=b"ACGT"):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    y = bytes(a[rng.integers(0, len(a), ylen)])
    st = int(rng.integers(0, max(1, ylen - xlen)))
    x = bytearray(y[st:st + xlen])
    for q in rng.integers(0, max(1, len(x)), nsub if len(x) else 0):
        x[int(q)] = int(a[rng.integers(0, len(a))])
    return bytes(x), y


def _ragged(seed, n, xmax, ymax, alphabet=b"ACGT"):
    rng = np.random.default_rng(seed)
    return [_window_pair(rng, int(rng.integers(0, xmax)), int(rng.integers(0, ymax)), int(rng.integers(0, 8)), alphabet)
            for _ in range(n)]


def _batch_of(pairs):
    from rust_bio_b200.engine import pack_pairs
    return pack_pairs(pairs)


def _c4_with_refusals(n, n_random, seed):
    """C4's generator (500 x 10,000) with independent random 500 x 10,000 pairs (bands above MAX_CELLS) spread
    through the batch, so every share holds some"""
    c4 = synth.mutated_window_pairs(synth.BASES["C4"], seed * n, n, 500, 10000)
    rnd = synth.uniform_pairs(synth.BASES["C4"] + 7, seed, n_random, 500, 10000)
    get = lambda b, p: (bytes(b[0][int(b[1][p]):int(b[1][p]) + int(b[2][p])]),
                        bytes(b[0][int(b[3][p]):int(b[3][p]) + int(b[4][p])]))
    pairs = [get(c4, p) for p in range(n)]
    where = np.linspace(0, n, n_random, endpoint=False).astype(int)
    for q, at in enumerate(where[::-1]):
        pairs.insert(int(at), get(rnd, q))
    refused = set(int(a) + q for q, a in enumerate(sorted(where)))
    return pairs, refused


def _full(eng, mode, cs, k, w, batch, hints=None):
    from rust_bio_b200.engine import Engine, Results
    res = Results(len(batch[2]), Engine.default_ops_capacity(batch), pair_status=True)
    if hints is None:
        eng.align_batch_banded(mode, cs, k, w, batch, results=res)
    else:
        eng.align_batch_banded_hinted(mode, cs, k, w, batch, results=res, **hints)
    return res


def _assert_same(a, b, n, what):
    for f in FIELDS + (("status",) if a.status is not None and b.status is not None else ()):
        ga, gb = getattr(a, f)[:n], getattr(b, f)[:n]
        bad = np.nonzero(ga != gb)[0]
        assert not len(bad), f"{what}: {f} differs at {len(bad)} pairs, first {bad[0]}: {ga[bad[0]]} vs {gb[bad[0]]}"
    assert np.array_equal(a.ops_off[:n + 1], b.ops_off[:n + 1]), what
    tot = int(a.ops_off[n])
    assert np.array_equal(a.ops[:tot], b.ops[:tot]), what
    assert np.array_equal(a.clip_len[:4 * n], b.clip_len[:4 * n]), what


def _assert_scores_same(got, want, what, fields=("score", "xend", "yend", "status")):
    for f in fields:
        g = got[f] if isinstance(got, dict) else getattr(got, f)
        wv = want[f] if isinstance(want, dict) else getattr(want, f)
        n = min(len(g), len(wv))
        assert np.array_equal(np.asarray(g)[:n], np.asarray(wv)[:n]), (what, f)


def _oracle_sample(oracle, mode, orc_args, k, w, batch, got, n_sample, what, table=None):
    n = len(batch[2])
    idx = np.unique(np.linspace(0, n - 1, min(n, n_sample)).astype(int))
    sub = _batch_of([(bytes(batch[0][int(batch[1][p]):int(batch[1][p]) + int(batch[2][p])]),
                      bytes(batch[0][int(batch[3][p]):int(batch[3][p]) + int(batch[4][p])])) for p in idx])
    s, _keep = oracle.make_scoring(*orc_args)
    ref, rops, roff, _, _ = oracle.banded_align_batch(mode, s, k, w, *sub, threads=8)
    for i, p in enumerate(idx):
        if got.status[p]:  # a pair the reference panics on: the oracle has no result for it
            continue
        for f in FIELDS:
            assert int(getattr(got, f)[p]) == int(ref[f][i]), (what, int(p), f)
        want = [(int(v) & 7, int(v) >> 3) for v in rops[int(roff[i]):int(roff[i]) + int(ref["n_ops"][i])]]
        assert got.ops_of(int(p)) == want, (what, int(p))


@pytest.mark.parametrize("mode", list(MODES))
def test_banded_c4_all_modes_with_refusals(me, single, oracle, mode):
    """1,000 C4 pairs plus random 500 x 10,000 pairs in every share: equal to one engine on every field, the ops, the
    clips and the statuses; the random pairs are the empty MIN_SCORE alignment; an oracle sample agrees."""
    pairs, refused = _c4_with_refusals(1000, 4 * len(LISTS) + 3, MODES[mode])
    batch = _batch_of(pairs)
    cs = _cs()
    got = _full(me, MODES[mode], cs, 32, 32, batch)
    one = _full(single, MODES[mode], cs, 32, 32, batch)
    _assert_same(got, one, len(pairs), f"{mode} C4")
    assert int(me.stats.cells) == int(single.stats.cells)
    for p in refused:
        assert int(got.score[p]) == MIN and int(got.ops_off[p + 1]) == int(got.ops_off[p]), p
    assert not np.any(got.status[:len(pairs)])
    _oracle_sample(oracle, mode, (-5, -1, 1, -1, None, MIN, MIN, MIN, MIN, 1), 32, 32, batch, got, 24, f"{mode} oracle")


RAGGED = {
    "local": dict(mode="local", clips=(MIN, MIN, MIN, MIN)),
    "custom_clips": dict(mode="custom", clips=(-3, -7, 0, -9)),
    "blosum62": dict(mode="semiglobal", clips=(MIN, MIN, MIN, MIN), table=True),
}


@pytest.mark.parametrize("case", list(RAGGED))
def test_banded_ragged(me, single, oracle, case):
    """Ragged batches (empty sequences among them): local, custom with live clips, and BLOSUM62 protein."""
    from rust_bio_b200 import scores
    c = RAGGED[case]
    table = alpha = None
    if c.get("table"):
        table = np.ascontiguousarray(scores.matrix_table256("blosum62"), dtype=np.int32)
        alpha = np.frombuffer(bytes(range(65, 91)) + b"*", dtype=np.uint8).copy()
        pairs = _ragged(31, 1500, 300, 900, alphabet=synth.PROTEIN)
        cs = _cs(table=table, alpha=alpha, go=-10, match=0, mismatch=0)
        orc_args = (-10, -1, 0, 0, table)
    else:
        pairs = _ragged(30 + len(case), 2000, 300, 900)
        cs = _cs(clips=c["clips"])
        orc_args = (-5, -1, 1, -1, None, *c["clips"], 1)
    batch = _batch_of(pairs)
    mode = MODES[c["mode"]]
    got = _full(me, mode, cs, 6, 8, batch)
    one = _full(single, mode, cs, 6, 8, batch)
    _assert_same(got, one, len(pairs), case)
    assert int(me.stats.cells) == int(single.stats.cells)
    _oracle_sample(oracle, c["mode"], orc_args, 6, 8, batch, got, 40, f"{case} oracle")


def _hint_inputs(oracle, n):
    """window pairs with their 6-mer matches; some lists emptied, so shares start and end on empty lists and on long
    ones alike"""
    rng = np.random.default_rng(77)
    pairs = [_window_pair(rng, int(rng.integers(40, 120)), int(rng.integers(130, 260))) for _ in range(n)]
    matches = [oracle.find_kmer_matches(x, y, 6) for x, y in pairs]
    for p in list(range(0, n, 5)) + [n // 2 - 1, n // 2, n // 3, n - 1]:
        matches[p] = []
    return pairs, matches


def test_banded_hinted(me, single, oracle):
    """custom_with_matches, custom_with_expanded_matches (allowed mismatches; lcskpp union) and
    custom_with_match_path with ragged match counts, empty lists included: equal to one engine."""
    pairs, matches = _hint_inputs(oracle, 700)
    batch = _batch_of(pairs)
    cs = _cs(clips=(-3, MIN, 0, -4))
    for kw in (dict(), dict(allowed_mismatches=1), dict(use_lcskpp_union=True)):
        hints = dict(matches=matches, **kw)
        got = _full(me, MODES["custom"], cs, 6, 4, batch, hints)
        one = _full(single, MODES["custom"], cs, 6, 4, batch, hints)
        _assert_same(got, one, len(pairs), f"hinted {kw}")
        sc = me.align_batch_banded_scores(MODES["custom"], cs, 6, 4, batch, **hints)
        _assert_scores_same(sc, single.align_batch_banded_scores(MODES["custom"], cs, 6, 4, batch, **hints), f"scores {kw}")
    paths = [oracle.lcskpp(m, 6)[0] if m else [] for m in matches]
    sub = [m if m else [(0, 0)] for m in matches]
    paths = [p if p else [0] for p in paths]
    got = _full(me, MODES["custom"], cs, 6, 4, batch, dict(matches=sub, paths=paths))
    one = _full(single, MODES["custom"], cs, 6, 4, batch, dict(matches=sub, paths=paths))
    _assert_same(got, one, len(pairs), "match path")


def test_statuses_of_a_failing_pair_in_the_last_share(me, single, oracle):
    """A reversed (invalid) match list on a pair of the last share: with a status array only that pair is
    B2A_PAIR_INVALID_HINT and the rest equal one engine; without one the call is B2A_E_INVALID."""
    from rust_bio_b200._lib import B2AError, CPairs, CStats
    from rust_bio_b200.engine import Engine, Results
    pairs, matches = _hint_inputs(oracle, 300)
    bad = len(pairs) - 3
    while len(matches[bad]) < 2:
        bad -= 1
    matches[bad] = matches[bad][::-1]
    batch = _batch_of(pairs)
    cs = _cs(clips=(-3, MIN, 0, -4))
    got = _full(me, MODES["custom"], cs, 6, 4, batch, dict(matches=matches))
    one = _full(single, MODES["custom"], cs, 6, 4, batch, dict(matches=matches))
    assert list(np.nonzero(got.status[:len(pairs)])[0]) == [bad] and int(got.status[bad]) == 4
    _assert_same(got, one, len(pairs), "invalid hint")
    with pytest.raises(B2AError) as ei:
        me.align_batch_banded_hinted(MODES["custom"], cs, 6, 4, batch, matches)
    assert ei.value.code == -1
    # a match_off that does not ascend is refused before any device runs
    h, keep = Engine._band_hints(len(pairs), matches, None, None, False)
    keep[0][5] = keep[0][6] + 1
    cp = Engine._cpairs(batch)
    res = Results(len(pairs), Engine.default_ops_capacity(batch), pair_status=True)
    assert me._L.b2a_multi_align_batch_banded(me._h, MODES["custom"], C.byref(cs), 6, 4, C.byref(cp), C.byref(h),
                                              C.byref(res.c), C.byref(CStats())) == -1


@pytest.mark.parametrize("seed", range(2))
def test_full_aligner_statuses(me, single, seed):
    """b2a_multi_align_batch with a status array: every device fetches its own slice of it (the exchanged segments
    carry no statuses), so every entry is written -- a sentinel left anywhere fails -- and statuses and results equal
    one engine's, under random custom clips (where the reference's walk can panic).  Where a trial does hold a pair
    the full aligner reports as panicking, the call without a status array fails with one engine's code."""
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import Results
    rng = np.random.default_rng(900 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    for trial in range(4):
        cs = _cs(clips=(pick(), pick(), pick(), pick()), go=int(rng.choice([0, -1, -2, -5])), ge=int(rng.choice([0, -1, -2])),
                 match=int(rng.choice([1, 2, 4])), mismatch=int(rng.choice([-1, -3, 0])))
        batch = synth.ragged_pairs(seed * 10 + trial, 1500, 90, 80, alphabet=b"AC" if trial % 2 else b"ACGT")
        n = len(batch[2])
        mk = lambda: Results(n, single.default_ops_capacity(batch), pair_status=True)
        one = single.align_batch(MODES["custom"], cs, batch, results=mk())
        got = mk()
        got.status[:] = 0xDEADBEEF
        me.align_batch(MODES["custom"], cs, batch, results=got)
        assert not np.any(got.status[:n] == 0xDEADBEEF), f"seed {seed} trial {trial}: a status entry was not written"
        _assert_same(got, one, n, f"seed {seed} trial {trial}")
        if np.any(one.status[:n]):
            with pytest.raises(B2AError) as e1:
                single.align_batch(MODES["custom"], cs, batch)
            with pytest.raises(B2AError) as e2:
                me.align_batch(MODES["custom"], cs, batch)
            assert e1.value.code == e2.value.code and "device" in str(e2.value)


@pytest.mark.parametrize("mode", ["custom", "local", "semiglobal"])
def test_score_only(me, single, mode):
    """Full and banded score-only on several devices equal one engine's score-only calls and the full calls'
    score / xend / yend."""
    pairs = _ragged(50 + MODES[mode], 2500, 300, 700)
    batch = _batch_of(pairs)
    cs = _cs(clips=(-3, -7, 0, -9) if mode == "custom" else (MIN, MIN, MIN, MIN))
    got = me.align_batch_scores(MODES[mode], cs, batch)
    _assert_scores_same(got, single.align_batch_scores(MODES[mode], cs, batch), f"{mode} scores")
    full = single.align_batch(MODES[mode], cs, batch)
    _assert_scores_same(got, full, f"{mode} scores vs full", ("score", "xend", "yend"))
    assert int(me.stats.cells) == int(single.stats.cells)
    got = me.align_batch_banded_scores(MODES[mode], cs, 8, 10, batch)
    _assert_scores_same(got, single.align_batch_banded_scores(MODES[mode], cs, 8, 10, batch), f"{mode} banded scores")
    bfull = _full(single, MODES[mode], cs, 8, 10, batch)
    _assert_scores_same(got, bfull, f"{mode} banded scores vs full", ("score", "xend", "yend", "status"))
    assert int(me.stats.cells) == int(single.stats.cells)


def test_edges(me, single):
    """An empty batch, one pair, and fewer pairs than devices, in every form."""
    pairs = _ragged(60, 8, 120, 300)
    cs = _cs()
    for n in (0, 1, me.n_devices - 1, me.n_devices):
        batch = _batch_of(pairs[:n])
        _assert_same(_full(me, 2, cs, 6, 8, batch), _full(single, 2, cs, 6, 8, batch), n, f"banded n={n}")
        _assert_scores_same(me.align_batch_scores(2, cs, batch), single.align_batch_scores(2, cs, batch), f"scores n={n}")
        _assert_scores_same(me.align_batch_banded_scores(2, cs, 6, 8, batch),
                            single.align_batch_banded_scores(2, cs, 6, 8, batch), f"banded scores n={n}")
        _assert_same(me.align_batch(2, cs, batch), single.align_batch(2, cs, batch), n, f"full n={n}")


def test_mirrors_and_exchange_kind(me):
    """banded.Aligner and pairwise.Aligner on a MultiEngine equal the default-engine mirrors; visualize raises."""
    from rust_bio_b200 import banded, pairwise
    from rust_bio_b200.pairwise import MatchParams
    assert ("listed more than once" in me.exchange_kind) == (len(set(me.ids)) < len(me.ids)), me.exchange_kind
    pairs = _ragged(70, 300, 150, 400)
    a_me = banded.Aligner.new(-5, -1, MatchParams(1, -1), 8, 10, engine=me)
    a_one = banded.Aligner.new(-5, -1, MatchParams(1, -1), 8, 10)
    for name in ("custom", "global", "semiglobal", "local"):
        assert getattr(a_me, f"{name}_batch")(pairs, on_panic="none") == getattr(a_one, f"{name}_batch")(pairs, on_panic="none")
        assert (getattr(a_me, f"{name}_scores_batch")(pairs, on_panic="none") ==
                getattr(a_one, f"{name}_scores_batch")(pairs, on_panic="none"))
    ms = [banded.find_kmer_matches(x, y, 8) for x, y in pairs]
    assert a_me.custom_with_matches_batch(pairs, ms, on_panic="none") == a_one.custom_with_matches_batch(pairs, ms, on_panic="none")
    assert (a_me.custom_with_expanded_matches_batch(pairs, ms, 1, False, on_panic="none") ==
            a_one.custom_with_expanded_matches_batch(pairs, ms, 1, False, on_panic="none"))
    one = a_me.semiglobal(*pairs[3])
    with pytest.raises(NotImplementedError):
        a_me.visualize(one)
    p_me = pairwise.Aligner.new(-5, -1, MatchParams(1, -1), engine=me) if _takes_engine() else None
    if p_me is not None:
        p_one = pairwise.Aligner.new(-5, -1, MatchParams(1, -1))
        for name in ("global", "semiglobal", "local"):
            assert getattr(p_me, f"{name}_batch")(pairs) == getattr(p_one, f"{name}_batch")(pairs)
            assert getattr(p_me, f"{name}_scores_batch")(pairs) == getattr(p_one, f"{name}_scores_batch")(pairs)


def _takes_engine():
    import inspect
    from rust_bio_b200 import pairwise
    return "engine" in inspect.signature(pairwise.Aligner.new).parameters


def test_single_engine_compaction_after_a_banded_call(single):
    """After align_batch_banded the compact segment (bytes / into / fixed) decodes to what the call returned, through
    gathered_fetch and decode_compact; run() stays B2A_E_STATE, and so does compaction after a banded score-only call."""
    import torch
    from rust_bio_b200._lib import B2AError
    from rust_bio_b200.engine import Results
    pairs = _ragged(80, 400, 200, 500)
    batch = _batch_of(pairs)
    n = len(pairs)
    cs = _cs()
    ref = _full(single, 3, cs, 8, 10, batch)
    nb = single.compact_bytes()
    for form in ("into", "fixed"):
        buf = torch.zeros(nb + 256, dtype=torch.uint8, device="cuda:0")
        if form == "into":
            single.compact_into(buf.data_ptr(), nb + 256)
        else:
            single.compact_fixed(buf.data_ptr(), nb + 256)
        torch.cuda.synchronize()
        res = Results(n, single.default_ops_capacity(batch))
        assert single.gathered_fetch(buf.data_ptr(), nb + 256, 1, res)[0] == n
        _assert_same(res, ref, n, f"gathered {form}")
        dec = single.decode_compact(buf.cpu().numpy(), nb + 256, 1, n, single.default_ops_capacity(batch))
        for f in FIELDS:
            assert np.array_equal(getattr(dec, f)[:n], getattr(ref, f)[:n]), (form, f)
        assert [dec.ops_of(p) for p in range(n)] == [ref.ops_of(p) for p in range(n)]
    with pytest.raises(B2AError) as ei:
        single.run()
    assert ei.value.code == -6
    single.align_batch_banded_scores(3, cs, 8, 10, batch)
    with pytest.raises(B2AError) as ei:
        single.compact_bytes()
    assert ei.value.code == -6
