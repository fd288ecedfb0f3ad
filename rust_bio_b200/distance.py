"""Mirror of `bio::alignment::distance` (reference src/alignment/distance.rs) on the H100 engine.

    hamming(x, y) -> int                     distance.rs:25-40
    levenshtein(x, y) -> int                 distance.rs:59-61
    simd.hamming / simd.levenshtein          distance.rs:101-138 (same values; simd.hamming's own panic message)
    simd.bounded_levenshtein(x, y, k)        distance.rs:165-172: the distance if it is <= min(k, max(|x|, |y|)),
                                             else None

Every per-pair function is a batch of one; the `*_batch` forms take [(x, y), ...] and are the form the GPU is built
for.  `engine=` takes an Engine or a MultiEngine (default: the process-wide engine on device 0).  Where the reference
panics (hamming over unequal lengths) this mirror raises AssertionError with the reference's message.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

from ._lib import DIST_NONE
from .engine import default_engine, pack_pairs

__all__ = ["hamming", "levenshtein", "hamming_batch", "levenshtein_batch", "bounded_levenshtein_batch", "simd"]

_U32_MAX = 0xFFFFFFFF
_HAMMING_MSG = "hamming distance cannot be calculated for texts of different length ({}!={})"
_SIMD_HAMMING_MSG = "simd " + _HAMMING_MSG

Pairs = Sequence[Tuple[bytes, bytes]]


def _engine(engine):
    return engine if engine is not None else default_engine()


def _hamming(pairs: Pairs, on_panic: str, msg: str, engine) -> List[Optional[int]]:
    if on_panic not in ("raise", "none"):
        raise ValueError('on_panic must be "raise" or "none"')
    if on_panic == "raise":
        for x, y in pairs:
            assert len(x) == len(y), msg.format(len(x), len(y))
    if not pairs:
        return []
    dist, status = _engine(engine).hamming_batch(pack_pairs(pairs), pair_status=True)
    return [None if s else int(d) for d, s in zip(dist, status)]


def hamming_batch(pairs: Pairs, on_panic: str = "raise", engine=None) -> List[Optional[int]]:
    """hamming over a batch.  on_panic="raise": a pair of unequal lengths raises the reference's AssertionError;
    "none": that pair's result is None and the others are computed."""
    return _hamming(pairs, on_panic, _HAMMING_MSG, engine)


def _levenshtein(pairs: Pairs, k: Optional[int], engine) -> List[Optional[int]]:
    if not pairs:
        return []
    dist = _engine(engine).levenshtein_batch(pack_pairs(pairs), k)
    if k is None:
        return [int(d) for d in dist]
    return [None if d == DIST_NONE else int(d) for d in dist]


def levenshtein_batch(pairs: Pairs, engine=None) -> List[int]:
    """levenshtein (== simd.levenshtein) over a batch: unit-cost edit distance over bytes."""
    return _levenshtein(pairs, None, engine)


def bounded_levenshtein_batch(pairs: Pairs, k: int, engine=None) -> List[Optional[int]]:
    """simd.bounded_levenshtein over a batch: per pair the distance if it is <= min(k, max(|x|, |y|)), else None."""
    k = int(k)
    if not 0 <= k <= _U32_MAX:
        raise OverflowError("k must fit in u32")
    return _levenshtein(pairs, k, engine)


def hamming(alpha: bytes, beta: bytes, engine=None) -> int:
    return hamming_batch([(alpha, beta)], engine=engine)[0]


def levenshtein(alpha: bytes, beta: bytes, engine=None) -> int:
    return levenshtein_batch([(alpha, beta)], engine=engine)[0]


class simd:  # noqa: N801  (the reference's module name)
    """bio::alignment::distance::simd: the same values as the scalar functions (distance.rs:63-173)."""

    @staticmethod
    def hamming(alpha: bytes, beta: bytes, engine=None) -> int:
        return _hamming([(alpha, beta)], "raise", _SIMD_HAMMING_MSG, engine)[0]

    @staticmethod
    def levenshtein(alpha: bytes, beta: bytes, engine=None) -> int:
        return levenshtein_batch([(alpha, beta)], engine=engine)[0]

    @staticmethod
    def bounded_levenshtein(alpha: bytes, beta: bytes, k: int, engine=None) -> Optional[int]:
        return bounded_levenshtein_batch([(alpha, beta)], k, engine=engine)[0]

    @staticmethod
    def hamming_batch(pairs: Pairs, on_panic: str = "raise", engine=None) -> List[Optional[int]]:
        return _hamming(pairs, on_panic, _SIMD_HAMMING_MSG, engine)
