"""Mirror of `bio::pattern_matching::myers` (reference src/pattern_matching/myers) on the H100 engine.

    Myers(pattern, bits=64 | 128)            simple.rs: patterns of at most 64 / 128 symbols, distances as u8
    long.Myers(pattern, bits=64 | 128)       long.rs: patterns of any length, distances as usize
    MyersBuilder().ambig(b, eqs).text_wildcard(b).build_64 / build_128 / build_long_64 / build_long_128   builder.rs

    m.distance(text) -> int                  the least distance of the pattern to any substring of the text
    m.find_all_end(text, max_dist) -> list   every (end, dist) with dist <= max_dist, ends 0-based and ascending
    m.find_best_end(text) -> (end, dist)     the first end of the least distance
    and *_batch forms over many texts, which store the pattern once.

Every per-text method is a batch of one.  `engine=` takes an Engine or a MultiEngine (default: the process-wide
engine on device 0).  Where the reference panics this mirror raises AssertionError with its message; on an empty text
`distance` returns the reference's initial max_dist (u8::MAX for the simple variants, usize::MAX - w for the long
ones), `find_all_end` is empty and `find_best_end` raises as the reference's unwrap does.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from ..engine import default_engine

__all__ = ["Myers", "long", "MyersBuilder"]

_USIZE_MAX = (1 << 64) - 1
_UNWRAP_NONE = "called `Option::unwrap()` on a `None` value"


def _blob(pattern: bytes, texts: Sequence[bytes]):
    """one pattern stored once, every text after it: (blob, x_off, x_len, y_off, y_len)"""
    n = len(texts)
    y_len = np.fromiter((len(t) for t in texts), dtype=np.uint32, count=n)
    y_off = (len(pattern) + np.concatenate([[0], np.cumsum(y_len, dtype=np.uint64)[:-1]])).astype(np.uint64) \
        if n else np.zeros(0, dtype=np.uint64)
    blob = np.frombuffer(pattern + b"".join(bytes(t) for t in texts) + b"\0", dtype=np.uint8).copy()
    return (blob, np.zeros(n, dtype=np.uint64), np.full(n, len(pattern), dtype=np.uint32), y_off, y_len)


class Myers:
    """simple.rs: Myers<u64> (bits=64) or Myers<u128> (bits=128)."""
    _long = False

    def __init__(self, pattern: bytes, bits: int = 64, engine=None, _ambig=None, _wildcards=None):
        if bits not in (64, 128):
            raise ValueError("bits must be 64 or 128")
        self.pattern = bytes(pattern)
        self.bits = bits
        self._check_pattern()
        self._engine = engine
        self._ambig: Optional[Dict[int, bytes]] = _ambig
        self._wildcards: Optional[bytes] = _wildcards

    def _check_pattern(self):
        assert len(self.pattern) <= self.bits, "Pattern too long"  # simple.rs:52-53
        assert len(self.pattern) > 0, "Pattern is empty"

    # the max_dist the reference starts from and the most find_all_end takes
    def _max_dist(self) -> int:
        return 255  # T::DistType::max_value(): u8 (simple.rs:319-325)

    def _k(self, max_dist: int) -> int:
        max_dist = int(max_dist)
        if not 0 <= max_dist <= 255:
            raise OverflowError("max_dist is a u8 for Myers<u64> / Myers<u128>")
        return max_dist

    def _run(self, texts: Sequence[bytes], k: Optional[int]):
        eng = self._engine if self._engine is not None else default_engine()
        return eng.myers_batch(_blob(self.pattern, texts), k, ambig=self._ambig, wildcards=self._wildcards)

    def distance_batch(self, texts: Sequence[bytes]) -> List[int]:
        out = [self._max_dist()] * len(texts)  # an empty text keeps the initial max_dist (myers_impl.rs:168-180)
        idx = [i for i, t in enumerate(texts) if len(t)]
        if idx:
            r = self._run([texts[i] for i in idx], None)
            for i, d in zip(idx, r["best_dist"].tolist()):
                out[i] = d
        return out

    def find_all_end_batch(self, texts: Sequence[bytes], max_dist: int) -> List[List[Tuple[int, int]]]:
        k = self._k(max_dist)
        out: List[List[Tuple[int, int]]] = [[] for _ in texts]
        idx = [i for i, t in enumerate(texts) if len(t)]
        if idx:
            r = self._run([texts[i] for i in idx], k)
            off, he, hd = r["hit_off"].tolist(), r["hit_end"].tolist(), r["hit_dist"].tolist()
            for q, i in enumerate(idx):
                out[i] = list(zip(he[off[q]:off[q + 1]], hd[off[q]:off[q + 1]]))
        return out

    def find_best_end_batch(self, texts: Sequence[bytes]) -> List[Tuple[int, int]]:
        for t in texts:
            assert len(t) > 0, _UNWRAP_NONE  # myers_impl.rs:204-206: min_by_key over no hits, then unwrap
        if not texts:
            return []
        r = self._run(texts, None)
        return [(int(e), int(d)) for e, d in zip(r["best_end"], r["best_dist"])]

    def distance(self, text: bytes) -> int:
        return self.distance_batch([bytes(text)])[0]

    def find_all_end(self, text: bytes, max_dist: int) -> List[Tuple[int, int]]:
        return self.find_all_end_batch([bytes(text)], max_dist)[0]

    def find_best_end(self, text: bytes) -> Tuple[int, int]:
        return self.find_best_end_batch([bytes(text)])[0]


class _LongMyers(Myers):
    """long.rs: long::Myers<u64> (bits=64) or long::Myers<u128> (bits=128), patterns of any length."""
    _long = True

    def _check_pattern(self):
        assert len(self.pattern) > 0, "Pattern is empty"  # long.rs:83-84
        assert len(self.pattern) <= _USIZE_MAX // 2, "Pattern too long"

    def _max_dist(self) -> int:
        return _USIZE_MAX - self.bits  # usize::MAX - word_size (long.rs:583-590)

    def _k(self, max_dist: int) -> int:
        max_dist = int(max_dist)
        if not 0 <= max_dist <= _USIZE_MAX:
            raise OverflowError("max_dist is a usize")
        return min(max_dist, self._max_dist())  # myers_impl.rs:194: max_dist.min(usize::MAX - w)


class long:  # noqa: N801  (the reference's module name)
    """bio::pattern_matching::myers::long"""
    Myers = _LongMyers


class MyersBuilder:
    """builder.rs: pattern-side ambiguities and text wildcards."""

    def __init__(self):
        self._ambigs: Dict[int, bytes] = {}
        self._wildcards = bytearray()

    def ambig(self, byte: int, equivalents: Iterable[int]) -> "MyersBuilder":
        b = byte if isinstance(byte, int) else bytes(byte)[0]
        self._ambigs[b] = self._ambigs.get(b, b"") + bytes(equivalents)
        return self

    def text_wildcard(self, wildcard: int) -> "MyersBuilder":
        self._wildcards.append(wildcard if isinstance(wildcard, int) else bytes(wildcard)[0])
        return self

    def _build(self, cls, pattern, bits, engine):
        return cls(pattern, bits, engine, dict(self._ambigs) or None, bytes(self._wildcards) or None)

    def build_64(self, pattern: bytes, engine=None) -> Myers:
        return self._build(Myers, pattern, 64, engine)

    def build_128(self, pattern: bytes, engine=None) -> Myers:
        return self._build(Myers, pattern, 128, engine)

    def build_long_64(self, pattern: bytes, engine=None) -> Myers:
        return self._build(_LongMyers, pattern, 64, engine)

    def build_long_128(self, pattern: bytes, engine=None) -> Myers:
        return self._build(_LongMyers, pattern, 128, engine)
