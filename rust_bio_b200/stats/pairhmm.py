"""Mirror of `bio::stats::pairhmm::PairHMM` (reference src/stats/pairhmm) on the H100 engine.

    hmm = PairHMM.new(GapParams(prob_gap_x, prob_gap_y, prob_gap_x_extend, prob_gap_y_extend))   natural logs
    hmm.prob_related(emission, mode, max_edit_dist=None) -> float       LogProb: ln P(x and y are related)
    hmm.prob_related_batch(emissions, mode, max_edit_dist=None) -> numpy float64 array, one per emission

`mode` is a StartEndGapParams (free_start_gap_x, free_end_gap_x; GLOBAL and SEMIGLOBAL are the usual two) and
prob_start_gap_x is the trait's default.  `emission` must be a ClassEmission: the reference takes any
EmissionParameters, the engine takes per-base emission classes (for example base qualities), which cover its tests,
its doctest and its bench.  Any other emission object raises TypeError.  Where the reference asserts (PairHMM::new's
ln_one_minus_exp of a gap probability above ln_one, a NaN result) this mirror raises AssertionError.  `engine=` takes
an Engine or a MultiEngine (default: the process-wide engine on device 0).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional, Sequence

import numpy as np

from ..engine import default_engine

__all__ = ["GapParams", "StartEndGapParams", "GLOBAL", "SEMIGLOBAL", "ClassEmission", "PairHMM"]


class GapParams(NamedTuple):
    """GapParameters: natural-log probabilities to open and to extend a gap in x and in y (-inf: never)."""
    prob_gap_x: float
    prob_gap_y: float
    prob_gap_x_extend: float
    prob_gap_y_extend: float


class StartEndGapParams(NamedTuple):
    """StartEndGapParameters: free start / end gaps in x."""
    free_start_gap_x: bool
    free_end_gap_x: bool


GLOBAL = StartEndGapParams(False, False)
SEMIGLOBAL = StartEndGapParams(True, True)


class ClassEmission:
    """EmissionParameters in per-base classes.  tables: (emit_match, emit_mismatch, emit_x, emit_y), each one natural-
    log value per class (1 to 256 classes).  x_classes / y_classes: one class byte per base, or None for class 0.
    prob_emit_xy(i, j) is emit_match[y_classes[j]] when x[i] == y[j], else emit_mismatch[y_classes[j]];
    prob_emit_x(i) = emit_x[x_classes[i]]; prob_emit_y(j) = emit_y[y_classes[j]]."""

    def __init__(self, x: bytes, y: bytes, tables, x_classes: Optional[bytes] = None,
                 y_classes: Optional[bytes] = None):
        self.x, self.y = bytes(x), bytes(y)
        t = np.asarray(tables, dtype=np.float64)
        if t.ndim != 2 or t.shape[0] != 4 or not 1 <= t.shape[1] <= 256:
            raise ValueError("tables must be (emit_match, emit_mismatch, emit_x, emit_y) of 1 .. 256 classes each")
        self.tables = t
        self.x_classes = None if x_classes is None else bytes(x_classes)
        self.y_classes = None if y_classes is None else bytes(y_classes)
        for seq, cls, side in ((self.x, self.x_classes, "x"), (self.y, self.y_classes, "y")):
            if cls is not None:
                if len(cls) != len(seq):
                    raise ValueError(f"{side}_classes must have one class per base of {side}")
                if cls and max(cls) >= t.shape[1]:
                    raise ValueError(f"a class of {side} has no table entry")

    def len_x(self) -> int:
        return len(self.x)

    def len_y(self) -> int:
        return len(self.y)


def _fastexp(v: float) -> float:
    """FastExp::fastexp (utils/fastexp.rs:33-58) for a non-positive argument"""
    if not v > -500.0:
        return 0.0
    x = 1.442695041 * v
    bits = int(x)
    x -= float(bits)
    f2 = ((x * 0.006935931 + 0.019890581) * x + 0.143440676) * ((x + 4.831794110) * x) + 1.0
    return math.ldexp(1.0, bits) * f2


def _ln_add_exp(a: float, b: float) -> float:
    if b == -math.inf:
        return a
    p0, p1 = (b, a) if b > a else (a, b)
    if p0 == -math.inf:
        return -math.inf
    if p0 == math.inf:
        return math.inf
    return p0 + math.log1p(_fastexp(p1 - p0))


class PairHMM:
    """PairHMM (pairhmm.rs): the gap parameters are fixed at construction; prob_related runs on the GPU."""

    def __init__(self, gap_params: GapParams, engine=None):
        self.gap_params = GapParams(*[float(v) for v in gap_params])
        g = self.gap_params
        # PairHMM::new: ln_one_minus_exp of the open (either side) and of each extension asserts p <= 0.0
        for p in (_ln_add_exp(g.prob_gap_x, g.prob_gap_y), g.prob_gap_x_extend, g.prob_gap_y_extend):
            assert p <= 0.0, "assertion failed: p <= 0.0"
        self._engine = engine

    @classmethod
    def new(cls, gap_params: GapParams, engine=None) -> "PairHMM":
        return cls(gap_params, engine)

    def prob_related(self, emission: ClassEmission, alignment_mode: StartEndGapParams,
                     max_edit_dist: Optional[int] = None) -> float:
        return float(self.prob_related_batch([emission], alignment_mode, max_edit_dist)[0])

    def prob_related_batch(self, emissions: Sequence[ClassEmission], alignment_mode: StartEndGapParams,
                           max_edit_dist: Optional[int] = None) -> np.ndarray:
        """prob_related of every emission, which must all share one set of tables; equal x (with equal classes) are
        stored once."""
        if max_edit_dist is not None and not 0 <= int(max_edit_dist) < 1 << 64:
            raise OverflowError("max_edit_dist is a usize")
        tables = None
        for e in emissions:
            if not isinstance(e, ClassEmission):
                raise TypeError("the engine takes emissions as ClassEmission (per-base emission classes)")
            if tables is None:
                tables = e.tables
            elif e.tables.shape != tables.shape or not np.array_equal(e.tables.view(np.uint64),
                                                                       tables.view(np.uint64)):
                raise ValueError("every emission of a batch must share one set of tables")
        n = len(emissions)
        if n == 0:
            return np.zeros(0, dtype=np.float64)
        with_classes = any(e.x_classes is not None or e.y_classes is not None for e in emissions)
        parts, cparts, xo, yo, seen, pos = [], [], [], [], {}, 0
        for e in emissions:
            cx = e.x_classes if e.x_classes is not None else bytes(len(e.x))
            cy = e.y_classes if e.y_classes is not None else bytes(len(e.y))
            if (e.x, cx) not in seen:
                seen[(e.x, cx)] = pos
                parts.append(e.x)
                cparts.append(cx)
                pos += len(e.x)
            xo.append(seen[(e.x, cx)])
            yo.append(pos)
            parts.append(e.y)
            cparts.append(cy)
            pos += len(e.y)
        blob = np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8).copy()
        batch = (blob, np.array(xo, dtype=np.uint64), np.array([len(e.x) for e in emissions], dtype=np.uint32),
                 np.array(yo, dtype=np.uint64), np.array([len(e.y) for e in emissions], dtype=np.uint32))
        classes = np.frombuffer(b"".join(cparts) + b"\0", dtype=np.uint8).copy() if with_classes else None
        eng = self._engine if self._engine is not None else default_engine()
        med = None if max_edit_dist is None else int(max_edit_dist)  # (Some(usize::MAX) skips nothing, as None)
        prob, status = eng.pairhmm_batch(batch, self.gap_params, tables, bool(alignment_mode.free_start_gap_x),
                                         bool(alignment_mode.free_end_gap_x), med, classes)
        bad = np.nonzero(status)[0]
        if len(bad):
            raise AssertionError(f"emission {int(bad[0])}: assertion failed: !p.is_nan()")
        return prob
