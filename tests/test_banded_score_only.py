"""Score-only banded batches (b2a_align_batch_banded_scores): the banded aligner's Alignment.score, xend and yend
without the interior traceback.  On the host (tests/sim/b2a_sim_banded_scores.cpp: every K3 path in score-only form
against the banded oracle, each run twice -- on slabs / strip areas of the score-only size, then on full-size ones
whose interior-cell and traceback regions are poisoned and must come back unchanged; the scratch sizes) and on the GPU
(against the full banded call on the same engine and an oracle sample: every mode and K3 path, C4, sub-waves, the
strip hand-backs, the capacity retry, hints, random clips, error paths, band ranges after the call)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import sim_util
from parity_util import MODES
from rust_bio_b200 import synth

MIN = -858993459
FIELDS = ("score", "xend", "yend")

SIMB_SRC = os.path.join(sim_util.HERE, "sim", "b2a_sim_banded_scores.cpp")
SIMB_SO = os.path.join(sim_util.HERE, "sim", "libb2asim_banded_scores.so")
_simb = None


def _simb_lib():
    """tests/sim/b2a_sim_banded_scores.cpp, built on first use"""
    global _simb
    if _simb is None:
        deps = [SIMB_SRC] + sim_util.DEPS
        if not os.path.exists(SIMB_SO) or any(os.path.getmtime(d) > os.path.getmtime(SIMB_SO) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                                   "-o", SIMB_SO, SIMB_SRC])
        _simb = C.CDLL(SIMB_SO)
        _simb.simb_warp32_one.restype = C.c_int
        _simb.simb_strip_task.restype = C.c_int
    return _simb


LOOPS = {"device": 0, "literal32": 1, "literal1": 2}
HANDED_BACK = "handed back"
# the first pair of C4's generator (DESIGN.md §4): band cells, K3 slab full / score-only, strip area full / score-only
C4_PAIR_BYTES = (64659, 267520, 138240, 82944, 13824)
C4_PAIR_SAVED, C4_PAIR_SAVED_PCT = 198400, 57


def simb_one(mode, orc_scoring, k, w, x: bytes, y: bytes, loop="device", matches=None, path=None,
             allowed_mismatches=None, use_lcskpp_union=False, cap_matches=4096):
    """One pair through K4 and the score-only K3 on the host: on a slab of the score-only size, then on a full-size one
    whose interior-cell region is poisoned (it must come back unchanged, the results must agree).
    -> ({score, xend, yend}, status, cells, fast)"""
    s = sim_util.SimScoring.from_buffer_copy(bytes(orc_scoring))
    xy = np.array([v for mt in (matches or []) for v in mt] or [0, 0], dtype=np.uint32)
    pi = np.array(path if path else [0], dtype=np.uint32)
    res = []
    for poison in (-1, 0xA5):
        score, xe, ye, st = C.c_int32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        cells, fast = C.c_uint64(0), C.c_int(0)
        rc = _simb_lib().simb_warp32_one(
            C.c_int(int(mode)), C.byref(s), C.c_uint32(k), C.c_uint32(w), x, C.c_uint32(len(x)), y, C.c_uint32(len(y)),
            C.c_int(1 if matches is not None else 0), xy.ctypes.data_as(C.c_void_p),
            C.c_uint64(len(matches) if matches is not None else 0), pi.ctypes.data_as(C.c_void_p),
            C.c_uint64(len(path) if path is not None else 0), C.c_int(1 if path is not None else 0),
            C.c_int(-1 if allowed_mismatches is None else int(allowed_mismatches)), C.c_int(1 if use_lcskpp_union else 0),
            C.c_uint32(cap_matches), C.c_int(LOOPS[loop]), C.c_int(poison), C.byref(score), C.byref(xe), C.byref(ye),
            C.byref(st), C.byref(cells), C.byref(fast))
        assert rc != -3, "the score-only K3 wrote into the interior-cell region"
        assert rc == 0, rc
        res.append(({"score": score.value, "xend": xe.value, "yend": ye.value}, st.value, cells.value, fast.value))
    assert res[0] == res[1], "the result depends on the interior-cell region"
    return res[0]


def simb_task(mode, orc_scoring, k, w, pairs, cap_matches=4096):
    """Up to four pairs through K4, one warp-task of the F_NOTB strip fill, the score-only finish pass and the walk,
    on score-only-sized arenas and then on full-size ones with poisoned interior and traceback regions.
    -> per pair {score, xend, yend}, HANDED_BACK (K4 marked it, the strip path handed it back to the column loops) or
    None (not marked)"""
    from rust_bio_b200.engine import pack_pairs
    s = sim_util.SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob, x_off, x_len, y_off, y_len = [np.ascontiguousarray(a) for a in pack_pairs(pairs)]
    n = len(pairs)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    res = []
    for poison in (-1, 0xA5):
        out = {f: np.zeros(n, np.int32 if f == "score" else np.uint32) for f in FIELDS + ("status", "path")}
        rc = _simb_lib().simb_strip_task(int(mode), C.byref(s), C.c_uint32(k), C.c_uint32(w), p(blob),
                                         C.c_uint64(len(blob)), p(x_off), p(x_len), p(y_off), p(y_len), C.c_uint32(n),
                                         C.c_uint32(cap_matches), C.c_int(poison), p(out["score"]), p(out["xend"]),
                                         p(out["yend"]), p(out["status"]), p(out["path"]))
        assert rc != -3, "the score-only strip path wrote into a poisoned region"
        assert rc == 0, rc
        res.append([{f: int(out[f][i]) for f in FIELDS} if out["path"][i] == 1 else
                    (HANDED_BACK if out["path"][i] == 2 else None) for i in range(n)])
    assert res[0] == res[1], "the result depends on a poisoned region"
    return res[0]


def _window_pair(rng, xlen, ylen, nsub=5, alphabet=b"ACGT"):
    """x = a window of y with nsub substitutions"""
    a = np.frombuffer(alphabet, dtype=np.uint8)
    y = bytes(a[rng.integers(0, len(a), ylen)])
    st = int(rng.integers(0, max(1, ylen - xlen)))
    x = bytearray(y[st:st + xlen])
    for q in rng.integers(0, max(1, len(x)), nsub if len(x) else 0):
        x[int(q)] = int(a[rng.integers(0, len(a))])
    return bytes(x), y


def _oracle(oracle, mode, s, k, w, x, y):
    """the banded oracle's {score, xend, yend}, or None where the reference panics"""
    try:
        ref, _ = oracle.banded_align(mode, s, k, w, x, y)
    except RuntimeError:
        return None
    return {f: ref[f] for f in FIELDS}


def _check_one(got, status, ref, what):
    """status 0 and the oracle's fields; where the reference panics, B2A_PAIR_PANIC with no result or (a panic only
    the interior walk meets) a reported score"""
    if ref is None:
        assert status in (0, 1), what
        if status:
            assert got == {"score": MIN, "xend": 0, "yend": 0}, what
        return False
    assert status == 0 and got == ref, (what, got, ref)
    return True


# ------------------------------------------------------------------------------------------------ host (not-gpu)

@pytest.mark.parametrize("loop", list(LOOPS))
@pytest.mark.parametrize("mode", list(MODES))
def test_sim_banded_scores_column_loops(oracle, mode, loop):
    """The register-resident loop (as the device picks it), the literal loop at W = 32 and at W = 1, against the oracle;
    random gap costs, custom clips, and lengths 0-2 among the pairs."""
    rng = np.random.default_rng({"custom": 1, "global": 2, "semiglobal": 3, "local": 4}[mode] * 10 + LOOPS[loop])
    pick = lambda: int(rng.choice([MIN, 0, 0, -2, -9]))
    n_ok = n_fast = 0
    for trial in range(18):
        go, ge = int(rng.choice([0, -1, -5])), int(rng.choice([0, -1, -2]))
        clips = (pick(), pick(), pick(), pick()) if mode == "custom" else (MIN, MIN, MIN, MIN)
        s, _ = oracle.make_scoring(go, ge, int(rng.choice([1, 2])), int(rng.choice([-1, -3])), None, *clips,
                                   has_match_scores=int(trial % 2))
        if trial < 4:  # lengths 0-2
            x, y = _window_pair(rng, trial % 3, int(rng.integers(0, 3)) if trial < 2 else 40, nsub=0)
        else:
            xl = int(rng.integers(20, 160))
            x, y = _window_pair(rng, xl, xl + int(rng.integers(30, 300)), nsub=int(rng.integers(0, 9)))
        k, w = int(rng.choice([4, 6, 9])), int(rng.choice([2, 5, 11, 45]))
        got, st, cells, fast = simb_one(MODES[mode], s, k, w, x, y, loop=loop)
        n_ok += _check_one(got, st, _oracle(oracle, mode, s, k, w, x, y), (mode, loop, trial, len(x), len(y)))
        n_fast += fast
    assert n_ok >= 12
    if loop == "device":
        assert n_fast >= 6, n_fast
    else:
        assert n_fast == 0


@pytest.mark.parametrize("seed", range(6))
def test_sim_banded_scores_random_clips(oracle, seed):
    """Arbitrary live / dead mixes of the four clip penalties and gap costs, on two- and four-letter alphabets."""
    rng = np.random.default_rng(600 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    s, _ = oracle.make_scoring(int(rng.choice([0, -1, -2, -5])), int(rng.choice([0, -1, -2])), int(rng.choice([1, 2, 4])),
                               int(rng.choice([-1, -3, 0])), None, pick(), pick(), pick(), pick())
    n_ok = 0
    for trial in range(16):
        xl = int(rng.integers(0, 90))
        x, y = _window_pair(rng, xl, xl + int(rng.integers(0, 120)), nsub=int(rng.integers(0, 6)),
                            alphabet=b"AC" if seed % 2 else b"ACGT")
        k, w = int(rng.choice([3, 5, 8])), int(rng.choice([2, 6, 20]))
        loop = list(LOOPS)[trial % 3]
        got, st, _, _ = simb_one(MODES["custom"], s, k, w, x, y, loop=loop)
        n_ok += _check_one(got, st, _oracle(oracle, "custom", s, k, w, x, y), (seed, trial, loop))
    assert n_ok >= 8


def test_sim_banded_scores_blosum62(oracle):
    """A tabulated MatchFunc through the LUT: the column loops and the strip path, local and semiglobal."""
    from rust_bio_b200 import scores
    table = scores.matrix_table256("blosum62")
    rng = np.random.default_rng(91)
    n_strip = 0
    for trial in range(4):
        s, keep = oracle.make_scoring(int(rng.choice([-10, -5])), -1, 0, 0, table)
        pairs = [_window_pair(rng, int(rng.integers(40, 250)), int(rng.integers(260, 420)), nsub=8,
                              alphabet=synth.PROTEIN) for _ in range(3)]
        for mode in ("local", "semiglobal"):
            for x, y in pairs:
                got, st, _, _ = simb_one(MODES[mode], s, 5, 7, x, y, loop=list(LOOPS)[trial % 3])
                _check_one(got, st, _oracle(oracle, mode, s, 5, 7, x, y), (trial, mode))
            for (x, y), g in zip(pairs, simb_task(MODES[mode], s, 5, 7, pairs)):
                if isinstance(g, dict):
                    n_strip += 1
                    assert g == _oracle(oracle, mode, s, 5, 7, x, y), (trial, mode)
    assert n_strip >= 8, n_strip


@pytest.mark.parametrize("mode", ["semiglobal", "local", "global", "custom_y", "custom_xsuffix", "custom_xy"])
def test_sim_banded_scores_strip_path(oracle, mode):
    """The F_NOTB strip fill, the score-only finish pass and the walk: tasks of one to four ragged pairs."""
    rng = np.random.default_rng({"semiglobal": 31, "local": 32, "global": 33, "custom_y": 34, "custom_xsuffix": 35,
                                 "custom_xy": 36}[mode])
    n_strip = n_tot = 0
    for trial in range(10):
        go, ge = int(rng.choice([0, -1, -5, -5])), int(rng.choice([0, -1, -1, -2]))
        omode, clips = (mode, (MIN,) * 4) if mode in ("semiglobal", "local", "global") else ("custom", {
            "custom_y": (MIN, MIN, int(rng.choice([0, -2, -7])), int(rng.choice([0, -1, -6]))),
            "custom_xsuffix": (int(rng.choice([MIN, 0, -3])), int(rng.choice([0, -2, -5])), int(rng.choice([0, -1])),
                               int(rng.choice([MIN, 0, -4]))),
            "custom_xy": (int(rng.choice([0, -2, -8])), MIN, int(rng.choice([0, -3])), int(rng.choice([0, -4])))}[mode])
        s, _ = oracle.make_scoring(go, ge, int(rng.choice([1, 2])), int(rng.choice([-1, -3])), None, *clips,
                                   has_match_scores=int(trial % 2))
        k, w = int(rng.choice([4, 6, 9])), int(rng.choice([2, 5, 11, 20]))
        pairs = []
        for q in range(int(rng.integers(1, 5))):
            xl = int(rng.integers(12, 420))  # one to four strips of 128 rows
            pairs.append(_window_pair(rng, xl, xl + int(rng.integers(30, 500)), nsub=int(rng.integers(0, 9))))
        for (x, y), g in zip(pairs, simb_task(MODES[omode], s, k, w, pairs)):
            n_tot += 1
            if not isinstance(g, dict):
                continue
            n_strip += 1
            assert g == _oracle(oracle, omode, s, k, w, x, y), (mode, trial, len(x), len(y), k, w)
    assert n_strip >= {"custom_y": 4, "custom_xsuffix": 2, "custom_xy": 2}.get(mode, n_tot // 3), (n_strip, n_tot)


def _handback_pairs(seed, n):
    """Odd pairs: a read inside its reference.  Even pairs: 200 against 5,000 unrelated bases -- no 32-mer matches, so
    the band is the full matrix, whose strip windows span more than the 4,095 columns the packed row-tracker key holds
    (semiglobal: the y-suffix clip is live), and the strip fill hands the pair back to the column loops."""
    rng = np.random.default_rng(seed)
    a = np.frombuffer(b"ACGT", dtype=np.uint8)
    return [_window_pair(rng, 200, 600, nsub=6) if p % 2 else
            (bytes(a[rng.integers(0, 4, 200)]), bytes(a[rng.integers(0, 4, 5000)])) for p in range(n)]


def test_sim_banded_scores_strip_handbacks(oracle):
    """The pairs of _handback_pairs on the strip path: the unrelated ones are handed back, the others give the oracle's
    result."""
    s, _ = oracle.make_scoring(-5, -1, 1, -1, has_match_scores=1)
    pairs = _handback_pairs(8, 4)
    got = simb_task(MODES["semiglobal"], s, 32, 32, pairs)
    for p, ((x, y), g) in enumerate(zip(pairs, got)):
        assert g == (_oracle(oracle, "semiglobal", s, 32, 32, x, y) if p % 2 else HANDED_BACK), (p, g)


def test_sim_banded_scores_c4_shape(oracle):
    """C4's shape (500 x 10,000, k = 32, w = 32, semiglobal): the strip path and the register-resident loop."""
    blob, xo, xl, yo, yl = synth.mutated_window_pairs(synth.BASES["C4"], 0, 4, 500, 10000)
    s, _ = oracle.make_scoring(-5, -1, 1, -1, has_match_scores=1)
    pairs = [(bytes(blob[int(xo[p]):int(xo[p]) + 500]), bytes(blob[int(yo[p]):int(yo[p]) + 10000])) for p in range(4)]
    refs = [_oracle(oracle, "semiglobal", s, 32, 32, x, y) for x, y in pairs]
    assert simb_task(MODES["semiglobal"], s, 32, 32, pairs) == refs
    for (x, y), ref in zip(pairs[:2], refs):
        got, st, _, fast = simb_one(MODES["semiglobal"], s, 32, 32, x, y)
        assert fast == 1 and st == 0 and got == ref


def test_sim_banded_scores_refused_band(oracle):
    """A band above MAX_CELLS: MIN_SCORE, 0, 0 and status 0, as the full call returns."""
    rng = np.random.default_rng(3)
    alpha = np.frombuffer(b"ACGT", dtype=np.uint8)
    x, y = bytes(alpha[rng.integers(0, 4, 500)]), bytes(alpha[rng.integers(0, 4, 10000)])
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    got, st, cells, _ = simb_one(MODES["semiglobal"], s, 32, 32, x, y)
    assert cells == 501 * 10001 and st == 0 and got == {"score": MIN, "xend": 0, "yend": 0}


def test_sim_banded_scores_caller_inputs(oracle):
    """custom_with_matches / _expanded_matches / _match_path against banded_align_hinted; reversed matches and an
    out-of-range path index are B2A_PAIR_INVALID_HINT."""
    rng = np.random.default_rng(321)
    s, _ = oracle.make_scoring(-5, -1, 1, -1, None, -3, MIN, 0, -4, has_match_scores=1)
    n_ok = 0
    for trial in range(5):
        x, y = _window_pair(rng, 90, 220)
        k, w = int(rng.choice([5, 7])), int(rng.choice([3, 6]))
        m = oracle.find_kmer_matches(x, y, k)
        variants = [dict(), dict(allowed_mismatches=1), dict(use_lcskpp_union=True)]
        if m:
            variants.append(dict(path=oracle.lcskpp(m, k)[0]))
        for kw in variants:
            want = oracle.banded_align_hinted(s, k, w, x, y, m, **kw)
            got, st, cells, _ = simb_one(0, s, k, w, x, y, loop=list(LOOPS)[trial % 3], matches=m, **kw)
            if want is None:
                assert st != 0
                continue
            assert st == 0 and cells == want[2] and got == {f: want[0][f] for f in FIELDS}, (trial, kw)
            n_ok += 1
    assert n_ok >= 12
    x, y = b"ACGTACGTTGCAACGT", b"TTACGTACGTTGCAACGTAA"
    m = oracle.find_kmer_matches(x, y, 6)
    assert simb_one(0, s, 6, 3, x, y, matches=m[::-1])[1] == 4
    assert simb_one(0, s, 6, 3, x, y, matches=m, path=[0, len(m)])[1] == 4


def test_sim_banded_scores_scratch_sizes(oracle):
    """Score-only K3 slabs and strip areas hold no interior bytes, and what a C4-shaped pair saves (DESIGN.md §4)."""
    L = _simb_lib()
    L.simb_sizes.restype = None
    out = (C.c_uint64 * 4)()

    def sizes(m, n, cells, band_cols, strip_cols):
        L.simb_sizes(C.c_uint64(m), C.c_uint64(n), C.c_uint64(cells), C.c_uint64(band_cols), C.c_uint64(strip_cols), out)
        return list(out)

    for m, n, cells in ((500, 10000, 1_100_000), (150, 600, 20_000), (3, 5, 9)):
        k3f, k3s, _, _ = sizes(m, n, cells, 0, 0)
        assert k3s == sizes(m, n, 0, 0, 0)[0]  # a slab without its `cells` region
        assert abs(k3f - k3s - 2 * cells) < 256  # (both totals are rounded up to 256 bytes)
    # the first pair of C4's generator (500 x 10,000, k = 32, w = 32, semiglobal), a strip pair: its K3 slab and strip
    # area, with band columns and strip columns counted as banded_strip_ok counts them
    blob, xo, xl, yo, yl = synth.mutated_window_pairs(synth.BASES["C4"], 0, 1, 500, 10000)
    s, _ = oracle.make_scoring(-5, -1, 1, -1, has_match_scores=1)
    x, y = bytes(blob[int(xo[0]):int(xo[0]) + 500]), bytes(blob[int(yo[0]):int(yo[0]) + 10000])
    _, _, cells, rng = sim_util.banded_warp32_one(MODES["semiglobal"], s, 32, 32, x, y, want_ranges=True)
    m, n = 500, 10000
    band = [j for j in range(1, n) if rng[j][0] < rng[j][1]]
    strip_cols = sum((min(e, m) - 2) // 128 - (max(1, st) - 1) // 128 + 1
                     for st, e in (rng[j] for j in band) if max(1, st) < min(e, m))
    k3f, k3s, ksf, kss = sizes(m, n, cells, band[-1] - band[0] + 1, strip_cols)
    assert (cells, k3f, k3s, ksf, kss) == C4_PAIR_BYTES, (cells, k3f, k3s, ksf, kss)
    saved = k3f + ksf - (k3s + kss)
    assert saved == C4_PAIR_SAVED and round(100 * saved / (k3f + ksf)) == C4_PAIR_SAVED_PCT


# ------------------------------------------------------------------------------------------------ GPU

def _cs(mode, go=-5, ge=-1, ma=1, mi=-1, clips=None, table=None, alphabet=None):
    from rust_bio_b200._lib import CScoring
    c = clips if clips is not None else ((-3, -7, 0, -9) if mode == "custom" else (MIN,) * 4)
    cs = CScoring(go, ge, c[0], c[1], c[2], c[3], ma, mi, 1, None, None, 0)
    if table is not None:
        cs.has_match_scores = 0
        cs.table = table.ctypes.data_as(C.c_void_p)
        cs.alphabet = alphabet.ctypes.data_as(C.c_void_p)
        cs.alphabet_len = len(alphabet)
    return cs


def _full(eng, mode, cs, k, w, batch, hints=None):
    from rust_bio_b200.engine import Results
    res = Results(len(batch[2]), eng.default_ops_capacity(batch), pair_status=True)
    if hints is None:
        eng.align_batch_banded(MODES[mode], cs, k, w, batch, results=res)
    else:
        eng.align_batch_banded_hinted(MODES[mode], cs, k, w, batch, results=res, **hints)
    out = {f: getattr(res, f)[:res.n_pairs].copy() for f in FIELDS}
    out["status"] = res.status[:res.n_pairs].copy()
    return out


def assert_same_as_full(got, full, what):
    """score, xend, yend and status of every pair the full call finishes; the pairs it reports as panicking are printed
    and follow the documented rule (B2A_PAIR_PANIC with no result, or a reported score)"""
    ok = full["status"] != 1
    for f in FIELDS:
        bad = np.nonzero(ok & (got[f].astype(np.int64) != full[f].astype(np.int64)))[0]
        assert not len(bad), f"{what}: {f} differs for {len(bad)} pairs; first {int(bad[0])}: " \
                             f"{got[f][bad[0]]} vs {full[f][bad[0]]}"
    assert np.array_equal(got["status"][ok], full["status"][ok]), what
    for p in np.nonzero(~ok)[0]:
        s = int(got["status"][p])
        print(f"{what}: pair {p}: full call status 1, score-only status {s}, score {int(got['score'][p])}")
        assert s in (0, 1)
        if s:
            assert int(got["score"][p]) == MIN and int(got["xend"][p]) == 0 and int(got["yend"][p]) == 0


def _oracle_sample(oracle, mode, cs_args, k, w, batch, got, count, what):
    blob, xo, xl, yo, yl = batch
    s, keep = oracle.make_scoring(*cs_args)
    for p in range(min(count, len(xl))):
        x = bytes(blob[int(xo[p]):int(xo[p]) + int(xl[p])])
        y = bytes(blob[int(yo[p]):int(yo[p]) + int(yl[p])])
        ref = _oracle(oracle, mode, s, k, w, x, y)
        if ref is not None:
            assert {f: int(got[f][p]) for f in FIELDS} == ref and got["status"][p] == 0, (what, p)


def _ragged(seed, n, xmax, ymin, ymax):
    rng = np.random.default_rng(seed)
    return [_window_pair(rng, int(rng.integers(0, xmax)), int(rng.integers(ymin, ymax)), nsub=int(rng.integers(0, 8)))
            for _ in range(n)]


ENV_PATHS = {"strip": {}, "no_strip": {"B2A_BANDED_STRIP": "0"}, "literal": {"B2A_BANDED_LITERAL": "1"}}
ORACLE_ARGS = {"custom": (-5, -1, 1, -1, None, -3, -7, 0, -9, 1), "global": (-5, -1, 1, -1, None, MIN, MIN, MIN, MIN, 1),
               "semiglobal": (-5, -1, 1, -1, None, MIN, MIN, MIN, MIN, 1),
               "local": (-5, -1, 1, -1, None, MIN, MIN, MIN, MIN, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(ENV_PATHS))
@pytest.mark.parametrize("mode", list(MODES))
def test_gpu_banded_scores_vs_full(oracle, monkeypatch, mode, path):
    from rust_bio_b200.engine import Engine, pack_pairs
    for kk, v in ENV_PATHS[path].items():
        monkeypatch.setenv(kk, v)
    pairs = _ragged(40 + MODES[mode], 1500, 400, 200, 900)
    batch = pack_pairs(pairs)
    cs = _cs(mode)
    eng = Engine(0)
    try:
        full = _full(eng, mode, cs, 8, 10, batch)
        strip_full = eng.banded_strip_pairs()
        got = eng.align_batch_banded_scores(MODES[mode], cs, 8, 10, batch)
        assert eng.banded_strip_pairs() == strip_full
    finally:
        eng.close()
    if path == "strip" and mode != "custom":
        assert strip_full > len(pairs) // 4, strip_full
    if path != "strip":
        assert strip_full == 0
    assert_same_as_full(got, full, f"{mode} {path}")
    _oracle_sample(oracle, mode, ORACLE_ARGS[mode], 8, 10, batch, got, 60, f"oracle {mode} {path}")


@pytest.mark.gpu
def test_gpu_banded_scores_c4(oracle):
    """C4's generator: 2,000 pairs against the oracle, then the full 200k-pair batch against the full call."""
    from rust_bio_b200.engine import Engine
    cs = _cs("semiglobal")
    eng = Engine(0)
    try:
        small = synth.mutated_window_pairs(synth.BASES["C4"], 0, 2000, 500, 10000)
        got = eng.align_batch_banded_scores(MODES["semiglobal"], cs, 32, 32, small)
        assert not np.any(got["status"])
        _oracle_sample(oracle, "semiglobal", ORACLE_ARGS["semiglobal"], 32, 32, small, got, 2000, "C4 2k")
        batch = synth.mutated_window_pairs(synth.BASES["C4"], 0, 200_000, 500, 10000)
        full = _full(eng, "semiglobal", cs, 32, 32, batch)
        sp = eng.banded_strip_pairs()
        got = eng.align_batch_banded_scores(MODES["semiglobal"], cs, 32, 32, batch)
        assert eng.banded_strip_pairs() == sp
    finally:
        eng.close()
    assert_same_as_full(got, full, "C4 200k")
    assert not np.any(full["status"])


@pytest.mark.gpu
def test_gpu_banded_scores_sub_waves_and_retry(monkeypatch):
    """K3 sub-waves forced by a small budget, and the K4 capacity retry (B2A_BANDED_CAP=64)."""
    from rust_bio_b200.engine import Engine
    batch = synth.mutated_window_pairs(synth.BASES["C4"], 1, 3000, 500, 3000)
    cs = _cs("local")
    eng = Engine(0)
    try:
        ref = _full(eng, "local", cs, 16, 16, batch)
        eng.set_traceback_budget(16 << 20)
        full = _full(eng, "local", cs, 16, 16, batch)
        got = eng.align_batch_banded_scores(MODES["local"], cs, 16, 16, batch)
        assert_same_as_full(got, full, "sub-waves")
        assert_same_as_full(got, ref, "sub-waves vs one wave")
        eng.set_traceback_budget(0)
        monkeypatch.setenv("B2A_BANDED_CAP", "64")
        full = _full(eng, "local", cs, 16, 16, batch)
        got = eng.align_batch_banded_scores(MODES["local"], cs, 16, 16, batch)
    finally:
        eng.close()
    assert_same_as_full(got, full, "capacity retry")
    assert_same_as_full(got, ref, "capacity retry vs default")


@pytest.mark.gpu
def test_gpu_banded_scores_strip_handbacks(oracle):
    """Strip pairs handed back to the column loops (bit 10): the pairs test_sim_banded_scores_strip_handbacks shows the
    strip path hands back, in a batch of 400, against the full call and the oracle."""
    from rust_bio_b200.engine import Engine, pack_pairs
    pairs = _handback_pairs(8, 400)
    batch = pack_pairs(pairs)
    cs = _cs("semiglobal")
    eng = Engine(0)
    try:
        full = _full(eng, "semiglobal", cs, 32, 32, batch)
        sp = eng.banded_strip_pairs()
        got = eng.align_batch_banded_scores(MODES["semiglobal"], cs, 32, 32, batch)
        assert eng.banded_strip_pairs() == sp == len(pairs)  # every pair marked, half of them handed back
    finally:
        eng.close()
    assert_same_as_full(got, full, "hand-backs")
    assert not np.any(got["status"])
    s, _ = oracle.make_scoring(*ORACLE_ARGS["semiglobal"])
    for p in range(0, 40):
        assert {f: int(got[f][p]) for f in FIELDS} == _oracle(oracle, "semiglobal", s, 32, 32, *pairs[p]), p


@pytest.mark.gpu
def test_gpu_banded_scores_hinted(oracle):
    """Caller-supplied matches (and paths, expansion, lcskpp union), with reversed matches on some pairs
    (B2A_PAIR_INVALID_HINT per pair, as the full call reports)."""
    from rust_bio_b200.engine import Engine, pack_pairs
    rng = np.random.default_rng(77)
    pairs = [_window_pair(rng, 90, 220) for _ in range(300)]
    batch = pack_pairs(pairs)
    matches = [oracle.find_kmer_matches(x, y, 6) for x, y in pairs]
    for p in range(0, len(pairs), 7):
        matches[p] = matches[p][::-1]
    cs = _cs("custom", clips=(-3, MIN, 0, -4))
    eng = Engine(0)
    try:
        for kw in (dict(), dict(allowed_mismatches=1), dict(use_lcskpp_union=True)):
            hints = dict(matches=matches, **kw)
            full = _full(eng, "custom", cs, 6, 4, batch, hints)
            got = eng.align_batch_banded_scores(MODES["custom"], cs, 6, 4, batch, **hints)
            assert np.count_nonzero(full["status"] == 4) >= len(pairs) // 10
            assert_same_as_full(got, full, f"hinted {kw}")
        ok = [p for p in range(len(pairs)) if p % 7 and matches[p]]
        paths = [oracle.lcskpp(matches[p], 6)[0] if p in ok else [0] for p in range(len(pairs))]
        sub = [matches[p] if p in ok else [(0, 0)] for p in range(len(pairs))]
        full = _full(eng, "custom", cs, 6, 4, batch, dict(matches=sub, paths=paths))
        got = eng.align_batch_banded_scores(MODES["custom"], cs, 6, 4, batch, matches=sub, paths=paths)
        assert_same_as_full(got, full, "hinted paths")
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_gpu_banded_scores_random_clips(seed):
    """Random custom clips and gap costs (where the reference's walk can panic): pairs the full call finishes agree;
    the ones it reports as panicking are printed and follow the documented rule."""
    from rust_bio_b200.engine import Engine, pack_pairs
    rng = np.random.default_rng(900 + seed)
    pick = lambda: int(rng.choice([MIN, 0, 0, -1, -3, -7, -20]))
    cs = _cs("custom", int(rng.choice([0, -1, -2, -5])), int(rng.choice([0, -1, -2])), int(rng.choice([1, 2, 4])),
             int(rng.choice([-1, -3, 0])), clips=(pick(), pick(), pick(), pick()))
    batch = pack_pairs(_ragged(seed, 2000, 120, 0, 200))
    eng = Engine(0)
    try:
        full = _full(eng, "custom", cs, 5, 6, batch)
        got = eng.align_batch_banded_scores(MODES["custom"], cs, 5, 6, batch)
    finally:
        eng.close()
    print(f"seed {seed}: {int(np.count_nonzero(full['status'] == 1))} pairs the full call reports as panicking")
    assert_same_as_full(got, full, f"random clips seed={seed}")


@pytest.mark.gpu
def test_gpu_banded_scores_error_paths_and_state():
    """Any start, ops or clip output is B2A_E_INVALID; band ranges after a score-only call equal the full call's; full,
    then score-only, then full again on one engine gives the first results."""
    from rust_bio_b200._lib import CBandHints, CStats, MODE_SEMIGLOBAL
    from rust_bio_b200.engine import Engine, Results, ScoreResults, pack_pairs
    pairs = _ragged(12, 200, 150, 200, 400)
    batch = pack_pairs(pairs)
    cs = _cs("semiglobal")
    eng = Engine(0)
    L, h = eng._L, eng._h
    try:
        res1 = Results(len(pairs), eng.default_ops_capacity(batch), pair_status=True)
        eng.align_batch_banded(MODE_SEMIGLOBAL, cs, 8, 10, batch, results=res1)
        first = {f: getattr(res1, f)[:len(pairs)].copy() for f in ("score", "xstart", "xend", "ystart", "yend", "status")}
        ops1 = [res1.ops_of(p) for p in range(len(pairs))]
        ranges_full = [eng.banded_band_ranges(p, len(pairs[p][1])).copy() for p in range(len(pairs))]
        cp = eng._cpairs(batch)
        full_res = Results(len(pairs), eng.default_ops_capacity(batch), pair_status=True)
        for f in ("xstart", "ystart", "ops", "ops_off", "clip_len"):  # one of them set at a time
            sr = ScoreResults(len(pairs))
            setattr(sr.c, f, getattr(full_res.c, f))
            assert L.b2a_align_batch_banded_scores(h, MODE_SEMIGLOBAL, C.byref(cs), 8, 10, C.byref(cp), None,
                                                   C.byref(sr.c), C.byref(CStats())) == -1, f
        bad = CBandHints(None, None, None, None, -1, 0)  # hints without match_off
        sr = ScoreResults(len(pairs))
        assert L.b2a_align_batch_banded_scores(h, MODE_SEMIGLOBAL, C.byref(cs), 8, 10, C.byref(cp), C.byref(bad),
                                               C.byref(sr.c), None) == -1
        got = eng.align_batch_banded_scores(MODE_SEMIGLOBAL, cs, 8, 10, batch)
        for p in range(len(pairs)):
            assert np.array_equal(eng.banded_band_ranges(p, len(pairs[p][1])), ranges_full[p]), p
        for f in FIELDS + ("status",):
            assert np.array_equal(got[f], first[f]), f
        res2 = Results(len(pairs), eng.default_ops_capacity(batch), pair_status=True)
        eng.align_batch_banded(MODE_SEMIGLOBAL, cs, 8, 10, batch, results=res2)
        for f in first:
            assert np.array_equal(first[f], getattr(res2, f)[:len(pairs)]), f
        assert ops1 == [res2.ops_of(p) for p in range(len(pairs))]
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_banded_aligner_scores_batch(oracle):
    """banded.Aligner.*_scores_batch: AlignmentScore per pair, equal to the *_batch form's fields."""
    from rust_bio_b200 import banded
    from rust_bio_b200.pairwise import AlignmentScore, MatchParams, Scoring
    pairs = _ragged(21, 50, 200, 150, 400)
    al = banded.Aligner.new(-5, -1, MatchParams(1, -1), 8, 10)
    for name in ("custom", "global", "semiglobal", "local"):
        full = getattr(al, f"{name}_batch")(pairs, on_panic="none")
        got = getattr(al, f"{name}_scores_batch")(pairs, on_panic="none")
        for a, g in zip(full, got):
            if a is not None:
                assert g == AlignmentScore(a.score, a.xend, a.yend), name
