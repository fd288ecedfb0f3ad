"""Pair HMM without a GPU: the oracle (a literal restatement of PairHMM::prob_related) against the reference's known
answers, the reference's quirks as explicit cases, the kernels' lane logic on the host (b2a_pairhmm.cuh on 32
emulated lanes) bit-identical to the oracle over a seeded matrix, and the mirror's input errors."""
import json
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import pairhmm_util as pu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "pairhmm_vectors.json")))
F64_EPS = 2.220446049250313e-16
MODES = ("global", "semiglobal", (1, 0), (0, 1))


def _f(v):
    return float(v)  # (the fixtures write ln_zero as "-inf")


def _relative_eq(a, b, eps):
    """approx::assert_relative_eq! with max_relative = f64::EPSILON"""
    if a == b:
        return True
    d = abs(a - b)
    return d <= eps or d <= F64_EPS * max(abs(a), abs(b))


def _run_case(c, max_edit_dist="case"):
    med = c["max_edit_dist"] if max_edit_dist == "case" else max_edit_dist
    pk = pu.pack([(c["x"].encode(), c["y"].encode())])
    gap = [_f(v) for v in c["gap"]]
    return float(pu.orc_batch(gap, c["mode"], med, c["emit"], pk)[0])


@pytest.mark.parametrize("case", GOLDEN["prob_related"], ids=lambda c: c["name"])
def test_oracle_golden_prob_related(case):
    p = _run_case(case)
    for chk in case["checks"]:
        if chk["kind"] == "eq":
            assert p == _f(chk["value"]), chk
        elif chk["kind"] == "le":
            assert p <= chk["value"], chk
        elif chk["kind"] == "relative_eq":
            assert _relative_eq(p, chk["value"], chk["epsilon"]), (p, chk)
        elif chk["kind"] == "relative_eq_unbanded":
            assert _relative_eq(p, _run_case(case, None), chk["epsilon"]), chk
        else:
            raise AssertionError(chk)


def test_oracle_golden_fastexp_and_logprob():
    o = pu.oracle()
    for v in GOLDEN["fastexp"]:
        assert _relative_eq(o.orc_fastexp(v["x"]), v["expect"], v["epsilon"]), v
    for v in GOLDEN["logprob"]:
        args = [_f(a) for a in v["args"]]
        if v["op"] == "ln_sum_exp":
            assert pu.ln_sum_exp(args) == _f(v["expect"]), v
        elif v["op"] == "ln_add_exp":
            assert o.orc_ln_add_exp(*args) == _f(v["expect"]), v
        elif v["op"] == "ln_one_minus_exp":
            assert pu.ln_one_minus_exp(args[0]) == _f(v["expect"]), v
        elif v["op"] == "ln_cumsum_exp":  # a scan of ln_add_exp from ln_zero (probs/mod.rs:298-302, 369-372)
            s = float("-inf")
            for a, want, eps in zip(args, v["expect"], v["epsilon"]):
                s = o.orc_ln_add_exp(s, a)
                assert _relative_eq(s, _f(want), eps), v
        else:
            raise AssertionError(v)
    with pytest.raises(AssertionError):
        pu.ln_one_minus_exp(1e-9)  # ln_1m_exp's assert!(p <= 0.0)


# ---- a second, Python restatement of the literal loop for tiny pairs: it ties the oracle to the reference's text once
# more and, with reset_all, shows which cases depend on the stale values of quirk 1

def _py_fastexp(v):
    if not v > -500.0:
        return 0.0
    x = 1.442695041 * v
    bits = int(x)
    x -= float(bits)
    f2 = x * 0.006935931
    xt = x + 4.831794110
    f2 += 0.019890581
    xt *= x
    f2 *= x
    f2 += 0.143440676
    f2 *= xt
    f2 += 1.0
    return math.ldexp(1.0, bits) * f2


def _py_sum_exp(ps):
    if not ps:
        return -math.inf
    imax = 0
    for i in range(1, len(ps)):
        if ps[i] > ps[imax]:
            imax = i
    pmax = ps[imax]
    if pmax == -math.inf:
        return -math.inf
    s = -0.0
    for i, p in enumerate(ps):
        if i != imax and p != -math.inf:
            s += _py_fastexp(p - pmax)
    return pmax + math.log1p(s)


def _py_add_exp(a, b):
    if b == -math.inf:
        return a
    p0, p1 = (b, a) if b > a else (a, b)
    if p0 == -math.inf:
        return -math.inf
    return p0 + math.log1p(_py_fastexp(p1 - p0))


def _py_sum3(p0, p1, p2):
    if p1 < p2:
        p1, p2 = p2, p1
    if p1 > p0:
        p1, p0 = p0, p1
    return p0 if p0 - p1 > 10.0 else _py_sum_exp([p0, p1, p2])


def _py_prob_related(x, y, gap, emit, fs, fe, med, reset_all=False):
    gx, gy, gxe, gye = gap
    one_m = lambda p: math.log1p(-_py_fastexp(p)) if p < -0.693 else math.log(-math.expm1(p))
    ng, ngx, ngy = one_m(_py_add_exp(gx, gy)), one_m(gxe), one_m(gye)
    ninf, umax = -math.inf, (1 << 64) - 1
    n = len(y)
    fm = [[ninf] * (n + 1) for _ in range(2)]
    fx = [[ninf] * (n + 1) for _ in range(2)]
    fy = [[ninf] * (n + 1) for _ in range(2)]
    md = [[umax] * (n + 1) for _ in range(2)]
    cols = []
    prev, curr = 0, 1
    fm[prev][0] = 0.0
    for i in range(len(x)):
        fm[prev][0] = _py_add_exp(fm[prev][0], 0.0 if fs else ninf)
        if fs:
            md[prev][0] = 0
        for j in range(n):
            tl, top, left = md[prev][j], md[curr][j], md[prev][j + 1]
            if med is not None and min(tl, min(top, left)) > med:
                continue
            match = x[i] == y[j]
            e = emit[0][0] if match else emit[1][0]
            pm = e + _py_sum3(ng + fm[prev][j], ngx + fx[prev][j], ngy + fy[prev][j])
            pgy = emit[2][0] + (gy + fm[prev][j + 1])
            if gye != ninf:
                pgy = _py_add_exp(pgy, gye + fx[prev][j + 1])
            pgx = emit[3][0] + (gx + fm[curr][j])
            if gxe != ninf:
                pgx = _py_add_exp(pgx, gxe + fy[curr][j])
            sat = lambda v: v if v == umax else v + 1
            fm[curr][j + 1], fx[curr][j + 1], fy[curr][j + 1] = pm, pgy, pgx
            if med is not None:
                md[curr][j + 1] = min(tl if match else sat(tl), min(sat(left), sat(top)))
        if fe:
            cols += [fm[curr][n], fx[curr][n], fy[curr][n]]
        prev, curr = curr, prev
        fm[curr] = [ninf] * (n + 1)
        if reset_all:
            fx[curr], fy[curr], md[curr] = [ninf] * (n + 1), [ninf] * (n + 1), [umax] * (n + 1)
    p = _py_sum_exp(cols) if fe else _py_sum_exp([fm[prev][n], fx[prev][n], fy[prev][n]])
    return min(p, 0.0) if not math.isnan(p) else p


# (x, y, max_edit_dist, gap): pairs whose banded result reads stale values (found by a seeded search)
STALE_CASES = [(b"TTTGT", b"TTTC", 0, pu.GAP_EXT), (b"TTTGT", b"TTTC", 0, pu.ILLUMINA_GAP),
               (b"AGCGTTTGTTA", b"AGCGTTGTCA", 2, pu.GAP_EXT), (b"ATAAACCGGGCCA", b"AAAACTGGCA", 2, pu.ILLUMINA_GAP)]


@pytest.mark.parametrize("x,y,med,gap", STALE_CASES)
def test_quirk_stale_values_under_band(x, y, med, gap):
    """Only fm is reset between rows: a skipped cell keeps fx, fy and min_edit_dist of two rows earlier, and its
    computed neighbours read them.  The oracle and the lane logic keep them; resetting them changes the result."""
    want = _py_prob_related(x, y, gap, pu.ILLUMINA_EMIT, True, True, med)
    pk = pu.pack([(x, y)])
    got = pu.orc_batch(gap, "semiglobal", med, pu.ILLUMINA_EMIT, pk)
    sim, _ = pu.sim_batch(gap, "semiglobal", med, pu.ILLUMINA_EMIT, pk)
    assert pu.bits(got)[0] == pu.bits([want])[0] == pu.bits(sim)[0]
    assert want > -np.inf
    assert _py_prob_related(x, y, gap, pu.ILLUMINA_EMIT, True, True, med, reset_all=True) != want


def test_quirk_global_banded_is_ln_zero():
    """Without a free start every min_edit_dist stays usize::MAX, so a banded global call skips every cell."""
    pairs = [(b"ACGT", b"ACGT"), (b"A", b"A"), (b"ACGTACGTAC" * 30, b"ACGTACGTAC" * 30)]
    pk = pu.pack(pairs)
    for med in (0, 4, 10 ** 6, (1 << 64) - 2):
        assert np.all(pu.orc_batch(pu.ILLUMINA_GAP, "global", med, pu.ILLUMINA_EMIT, pk) == -np.inf)
        s, _ = pu.sim_batch(pu.ILLUMINA_GAP, "global", med, pu.ILLUMINA_EMIT, pk)
        assert np.all(s == -np.inf)
    # Some(usize::MAX) skips nothing: None's result
    none = pu.orc_batch(pu.ILLUMINA_GAP, "global", None, pu.ILLUMINA_EMIT, pk)
    s, _ = pu.sim_batch(pu.ILLUMINA_GAP, "global", (1 << 64) - 1, pu.ILLUMINA_EMIT, pk)
    assert np.all(none > -np.inf) and np.array_equal(pu.bits(s), pu.bits(none))


def test_quirk_sum3_two_swaps():
    """After two swaps p0 is the maximum but p1 need not be the second: the > 10 shortcut drops a close p2."""
    o = pu.oracle()
    assert o.orc_ln_sum3_exp_approx(-20.0, -5.0, -5.5) == -5.0
    assert pu.ln_sum_exp([-5.0, -20.0, -5.5]) > -4.6
    assert o.orc_ln_sum3_exp_approx(-5.0, -20.0, -5.5) != -5.0  # p2 is swapped into p1 and counted


def test_quirk_empty_sides():
    pairs = [(b"", b""), (b"", b"ACG"), (b"ACG", b""), (b"A", b"")]
    pk = pu.pack(pairs)
    want = {"global": [0.0, -np.inf, -np.inf, -np.inf], "semiglobal": [-np.inf] * 4, (1, 0): [0.0, -np.inf, -np.inf, -np.inf],
            (0, 1): [-np.inf] * 4}
    for mode in MODES:
        for med in (None, 0):
            o = pu.orc_batch(pu.GAP_EXT, mode, med, pu.ILLUMINA_EMIT, pk)
            s, tiers = pu.sim_batch(pu.GAP_EXT, mode, med, pu.ILLUMINA_EMIT, pk)
            assert list(o) == want[mode] and np.array_equal(pu.bits(o), pu.bits(s))
            assert tiers == [pu.PT_DONE] * 4


def _matrix_check(pairs, classes=None, emit=None, params=None, modes=MODES, meds=pu.MAX_EDIT):
    pk = pu.pack(pairs, classes)
    tiers_seen = set()
    for name, gap, em in params or pu.PARAMS:
        em = emit or em
        for mode in modes:
            for med in meds:
                o = pu.orc_batch(gap, mode, med, em, pk)
                s, tiers = pu.sim_batch(gap, mode, med, em, pk)
                bad = np.nonzero(pu.bits(o) != pu.bits(s))[0]
                assert len(bad) == 0, (name, mode, med, [(len(pairs[i][0]), len(pairs[i][1]), o[i], s[i]) for i in bad[:5]])
                tiers_seen |= set(tiers)
    return tiers_seen


def test_sim_matrix_bit_identical():
    tiers = _matrix_check(pu.matrix_pairs(seed=1), modes=("global", "semiglobal"))
    assert tiers == set(range(pu.PT_STRIP + 1))  # every tier, and the host-answered pairs


def test_sim_matrix_classes_bit_identical():
    rng = np.random.default_rng(5)
    pairs = pu.matrix_pairs(seed=2, y_lengths=(1, 33, 129, 161, 257), x_lengths=(1, 2, 300))
    cls = pu.random_classes(rng, pairs, 42)
    _matrix_check(pairs, cls, pu.quality_emit(42), params=[("extend", pu.GAP_EXT, None)])


def test_sim_independent_start_end_flags():
    pairs = pu.matrix_pairs(seed=3, y_lengths=(5, 40, 300), x_lengths=(2, 60))
    _matrix_check(pairs, modes=((1, 0), (0, 1)), meds=(None, 2), params=[pu.PARAMS[1]])


def test_sim_tier_choice_does_not_change_results():
    """Every C, with strips whenever len_y is above 32 * C, gives the bits of the engine's choice."""
    rng = np.random.default_rng(9)
    pairs = pu.matrix_pairs(seed=4, y_lengths=(1, 31, 33, 70, 161, 300), x_lengths=(2, 40))
    cls = pu.random_classes(rng, pairs, 8)
    pk = pu.pack(pairs, cls)
    for mode, med in (("semiglobal", 2), ("global", None), ("semiglobal", None)):
        base, _ = pu.sim_batch(pu.GAP_EXT, mode, med, pu.quality_emit(8), pk)
        for t in (pu.PT_C1, pu.PT_C2, pu.PT_C4, pu.PT_C5, pu.PT_C8):
            got, _ = pu.sim_batch(pu.GAP_EXT, mode, med, pu.quality_emit(8), pk, force_tier=t)
            assert np.array_equal(pu.bits(got), pu.bits(base)), (mode, med, t)


def test_tier_rule():
    want = {0: 0, 1: 1, 32: 1, 33: 2, 64: 2, 65: 3, 128: 3, 129: 4, 160: 4, 161: 5, 256: 5, 257: 6, 10000: 6}
    pk = pu.pack([(b"A", b"A" * n) for n in want])
    _, tiers = pu.sim_batch(pu.ILLUMINA_GAP, "global", None, pu.ILLUMINA_EMIT, pk)
    assert tiers == list(want.values())


def test_nan_emission_is_nan_result_for_pairs_using_it():
    """A NaN class entry gives NaN (the reference's assert) exactly for the pairs that reach it."""
    em = pu.quality_emit(4)
    em[1][3] = float("nan")  # mismatch of class 3
    pairs = [(b"ACGT", b"ACGT"), (b"ACGT", b"ACGA"), (b"ACGT", b"ACGA")]
    cls = [(b"\0\0\0\0", b"\0\0\0\0"), (b"\0\0\0\0", b"\0\0\0\3"), (b"\0\0\0\0", b"\0\0\0\1")]
    pk = pu.pack(pairs, cls)
    o = pu.orc_batch(pu.GAP_EXT, "global", None, em, pk)
    s, _ = pu.sim_batch(pu.GAP_EXT, "global", None, em, pk)
    assert [math.isnan(v) for v in o] == [False, True, False]
    assert np.array_equal(pu.bits(o), pu.bits(s))


# ---- the mirror's input errors (raised before the engine is used)

def test_mirror_input_errors():
    from rust_bio_b200.stats import pairhmm as ph
    with pytest.raises(AssertionError):
        ph.PairHMM.new(ph.GapParams(0.5, -1.0, -math.inf, -math.inf))
    with pytest.raises(AssertionError):
        ph.PairHMM.new(ph.GapParams(-1.0, -1.0, 1e-3, -math.inf))
    with pytest.raises(AssertionError):
        ph.PairHMM.new(ph.GapParams(-1.0, -1.0, -math.inf, float("nan")))
    hmm = ph.PairHMM.new(ph.GapParams(*pu.ILLUMINA_GAP))
    with pytest.raises(TypeError):
        hmm.prob_related(object(), ph.GLOBAL)
    with pytest.raises(ValueError):
        ph.ClassEmission(b"AC", b"AC", [[0.0], [0.0], [0.0]])
    with pytest.raises(ValueError):
        ph.ClassEmission(b"AC", b"AC", pu.ILLUMINA_EMIT, x_classes=b"\0")
    with pytest.raises(ValueError):
        ph.ClassEmission(b"AC", b"AC", pu.ILLUMINA_EMIT, y_classes=b"\0\1")
    a = ph.ClassEmission(b"AC", b"AC", pu.ILLUMINA_EMIT)
    b = ph.ClassEmission(b"AC", b"AC", pu.quality_emit(2))
    with pytest.raises(ValueError):
        hmm.prob_related_batch([a, b], ph.GLOBAL)
    with pytest.raises(OverflowError):
        hmm.prob_related(a, ph.GLOBAL, -1)
    with pytest.raises(OverflowError):
        hmm.prob_related(a, ph.GLOBAL, 1 << 64)


# ---- the fast exp compiles without contraction (a DFMA would change its bits)

def test_fastexp_sass_has_no_dfma(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc is not installed")
    src = os.path.join(HERE, "sim", "pairhmm_fastexp_probe.cu")
    cubin = str(tmp_path / "probe.cubin")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "--expt-relaxed-constexpr", "-cubin", "-o", cubin, src])
    sass = subprocess.check_output([cuobjdump, "-sass", cubin], text=True)
    funcs = {}
    for block in sass.split("Function : ")[1:]:
        funcs[block.split()[0]] = block
    fast = [b for k, b in funcs.items() if "fastexp_probe" in k]
    ctrl = [b for k, b in funcs.items() if "contract_probe" in k]
    assert fast and ctrl
    assert "DMUL" in fast[0] and "DFMA" not in fast[0]
    assert "DFMA" in ctrl[0]  # the same compiler contracts a plain a * b + c: the probe can see a DFMA
