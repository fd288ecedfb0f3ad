"""Mirror of `bio::alignment::pairwise::banded` (reference src/alignment/pairwise/banded.rs:122-1004).

`Aligner::{new, with_capacity, with_capacity_and_scoring, with_scoring}` take the k-mer length `k`
and the band half-width `w` like the reference (banded.rs:150-267); `custom / global_ / semiglobal /
local` (banded.rs:282, 872, 901, 975) and their `*_batch` forms run K4 (k-mer matches -> SDPk++ chain
-> Band) and K3 (banded fill + walk) on the GPU.  A band with more than MAX_CELLS = 5,000,000 cells
returns the reference's empty alignment (score MIN_SCORE, no operations, xlen = ylen = 0; banded.rs:407-420).

The entry points that take the band's inputs from the caller (banded.rs:294-401, 938-975) are here too:
`custom_with_prehash / semiglobal_with_prehash` (the prehash of y only accelerates the reference's match search;
results are those of `custom / semiglobal`), `custom_with_matches`, `custom_with_expanded_matches`,
`custom_with_match_path`, each with a `*_batch` form.  `hash_kmers` / `find_kmer_matches` mirror sparse.rs:337-358
for callers that want to build those inputs the way the reference's doctests do.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

from ._lib import MIN_SCORE, MODE_CUSTOM, MODE_GLOBAL, MODE_LOCAL, MODE_SEMIGLOBAL
from .alignment import Alignment, AlignmentMode, AlignmentOperation
from .engine import Engine, Results, default_engine, pack_pairs
from .pairwise import (DEFAULT_ALIGNER_CAPACITY, AlignmentScore, MatchFunc, Scoring, _alignment_scores, _alignments,
                       _check_scoring)

MAX_CELLS = 5_000_000          # banded.rs:104
DEFAULT_MATCH_SCORE = 2        # banded.rs:105


class Aligner:
    def __init__(self, scoring: Scoring, k: int, w: int, engine: Optional[Engine] = None):
        self.scoring, self.k, self.w, self._engine = scoring, int(k), int(w), engine

    @staticmethod
    def new(gap_open: int, gap_extend: int, match_fn: MatchFunc, k: int, w: int, engine=None) -> "Aligner":
        return Aligner.with_capacity(DEFAULT_ALIGNER_CAPACITY, DEFAULT_ALIGNER_CAPACITY, gap_open, gap_extend,
                                     match_fn, k, w, engine)

    @staticmethod
    def with_capacity(m: int, n: int, gap_open: int, gap_extend: int, match_fn: MatchFunc, k: int, w: int,
                      engine=None) -> "Aligner":
        return Aligner(Scoring.new(gap_open, gap_extend, match_fn), k, w, engine)

    @staticmethod
    def with_capacity_and_scoring(m: int, n: int, scoring: Scoring, k: int, w: int, engine=None) -> "Aligner":
        _check_scoring(scoring)
        return Aligner(scoring, k, w, engine)

    @staticmethod
    def with_scoring(scoring: Scoring, k: int, w: int, engine=None) -> "Aligner":
        return Aligner.with_capacity_and_scoring(DEFAULT_ALIGNER_CAPACITY, DEFAULT_ALIGNER_CAPACITY, scoring, k, w,
                                                 engine)

    def get_mut_scoring(self) -> Scoring:
        return self.scoring

    @property
    def engine(self) -> Engine:
        if self._engine is None:
            self._engine = default_engine(0)
        return self._engine

    def _batch(self, mode: int, pairs: Sequence[Tuple[bytes, bytes]], on_panic: str = "raise") -> List[Alignment]:
        batch = pack_pairs(pairs)
        cs, keep = self.scoring.to_c(batch)
        res = Results(len(pairs), Engine.default_ops_capacity(batch), pair_status=True)
        self.engine.align_batch_banded(mode, cs, self.k, self.w, batch, results=res)
        # global/semiglobal/local overwrite .mode after custom() returns, refused or not (banded.rs:889-890)
        return _alignments(res, pairs, mode, on_panic, banded=True)

    def _batch_hinted(self, pairs, matches, paths=None, allowed_mismatches=None, use_lcskpp_union=False,
                      on_panic: str = "raise"):
        batch = pack_pairs(pairs)
        cs, keep = self.scoring.to_c(batch)
        res = Results(len(pairs), Engine.default_ops_capacity(batch), pair_status=True)
        self.engine.align_batch_banded_hinted(MODE_CUSTOM, cs, self.k, self.w, batch, matches, paths,
                                              allowed_mismatches, use_lcskpp_union, results=res)
        return _alignments(res, pairs, MODE_CUSTOM, on_panic, banded=True, result_mode=AlignmentMode.Custom)

    def _scores_batch(self, mode: int, pairs, on_panic: str = "raise") -> List[Optional[AlignmentScore]]:
        """Alignment.score / xend / yend of each pair without the traceback (b2a_align_batch_banded_scores): what the
        `*_batch` form returns in those fields; a band above MAX_CELLS gives (MIN_SCORE, 0, 0).  on_panic as in
        _batch; a panic only the traceback's interior would meet cannot be seen here, and such a pair reports its
        score (include/b200align.h)."""
        batch = pack_pairs(pairs)
        cs, keep = self.scoring.to_c(batch)
        res = self.engine.align_batch_banded_scores(mode, cs, self.k, self.w, batch)
        return _alignment_scores(res, len(pairs), on_panic)

    def custom_scores_batch(self, pairs, on_panic: str = "raise") -> List[Optional[AlignmentScore]]:
        return self._scores_batch(MODE_CUSTOM, pairs, on_panic)

    def global_scores_batch(self, pairs, on_panic: str = "raise") -> List[Optional[AlignmentScore]]:
        return self._scores_batch(MODE_GLOBAL, pairs, on_panic)

    def semiglobal_scores_batch(self, pairs, on_panic: str = "raise") -> List[Optional[AlignmentScore]]:
        return self._scores_batch(MODE_SEMIGLOBAL, pairs, on_panic)

    def local_scores_batch(self, pairs, on_panic: str = "raise") -> List[Optional[AlignmentScore]]:
        return self._scores_batch(MODE_LOCAL, pairs, on_panic)

    def visualize(self, alignment: Alignment, file=None) -> str:
        """banded.rs:1007-1030: the band of the LAST single-pair alignment ('x'), the alignment's path ('\\'), one
        text row per x position (rows = xlen + 1, columns = ylen + 1).  Prints it like the reference and returns it."""
        rows, cols = alignment.xlen + 1, alignment.ylen + 1
        ranges = self.engine.banded_band_ranges(0, alignment.ylen)
        view = [["."] * cols for _ in range(rows)]
        for j in range(cols):
            for i in range(int(ranges[j, 0]), min(int(ranges[j, 1]), rows)):
                view[i][j] = "x"
        for p in alignment.path():
            view[p[0]][p[1]] = "\\"
        text = "\n".join("".join(r) for r in view)
        print(text, file=file)
        return text

    # ---- banded.rs:294-401: the band's inputs come from the caller
    def custom_with_prehash(self, x: bytes, y: bytes, y_kmer_hash) -> Alignment:
        """banded.rs:294-302.  `y_kmer_hash` (see hash_kmers) only spares the reference the hashing of y; the
        matches it yields are find_kmer_matches(x, y, k), so this is `custom`."""
        return self.custom(x, y)

    def custom_with_prehash_batch(self, pairs, y_kmer_hashes=None):
        return self.custom_batch(pairs)

    def semiglobal_with_prehash(self, x: bytes, y: bytes, y_kmer_hash) -> Alignment:
        """banded.rs:938-975 (same clip presets and clip filtering as semiglobal)."""
        return self.semiglobal(x, y)

    def semiglobal_with_prehash_batch(self, pairs, y_kmer_hashes=None):
        return self.semiglobal_batch(pairs)

    def custom_with_matches(self, x: bytes, y: bytes, matches) -> Alignment:
        """banded.rs:313-321: `matches` = sorted [(xpos, ypos), ...]."""
        return self._batch_hinted([(x, y)], [list(matches)])[0]

    def custom_with_matches_batch(self, pairs, matches, on_panic: str = "raise"):
        return self._batch_hinted(pairs, [list(m) for m in matches], on_panic=on_panic)

    def custom_with_expanded_matches(self, x: bytes, y: bytes, matches, allowed_mismatches: Optional[int],
                                     use_lcskpp_union: bool) -> Alignment:
        """banded.rs:338-375: sparse::expand_kmer_matches when allowed_mismatches is not None, then the band
        along sdpkpp's path or along sdpkpp_union_lcskpp_path."""
        return self._batch_hinted([(x, y)], [list(matches)], None, allowed_mismatches, use_lcskpp_union)[0]

    def custom_with_expanded_matches_batch(self, pairs, matches, allowed_mismatches: Optional[int],
                                           use_lcskpp_union: bool, on_panic: str = "raise"):
        return self._batch_hinted(pairs, [list(m) for m in matches], None, allowed_mismatches, use_lcskpp_union,
                                  on_panic=on_panic)

    def custom_with_match_path(self, x: bytes, y: bytes, matches, path) -> Alignment:
        """banded.rs:391-401: the band follows matches[path[0]], matches[path[1]], ... as given."""
        return self._batch_hinted([(x, y)], [list(matches)], [list(path)])[0]

    def custom_with_match_path_batch(self, pairs, matches, paths, on_panic: str = "raise"):
        return self._batch_hinted(pairs, [list(m) for m in matches], [list(p) for p in paths], on_panic=on_panic)

    def custom_batch(self, pairs, on_panic: str = "raise"):
        return self._batch(MODE_CUSTOM, pairs, on_panic)

    def global_batch(self, pairs, on_panic: str = "raise"):
        return self._batch(MODE_GLOBAL, pairs, on_panic)

    def semiglobal_batch(self, pairs, on_panic: str = "raise"):
        return self._batch(MODE_SEMIGLOBAL, pairs, on_panic)

    def local_batch(self, pairs, on_panic: str = "raise"):
        return self._batch(MODE_LOCAL, pairs, on_panic)

    def custom(self, x: bytes, y: bytes) -> Alignment:
        return self._batch(MODE_CUSTOM, [(x, y)])[0]

    def global_(self, x: bytes, y: bytes) -> Alignment:
        return self._batch(MODE_GLOBAL, [(x, y)])[0]

    def semiglobal(self, x: bytes, y: bytes) -> Alignment:
        return self._batch(MODE_SEMIGLOBAL, [(x, y)])[0]

    def local(self, x: bytes, y: bytes) -> Alignment:
        return self._batch(MODE_LOCAL, [(x, y)])[0]


setattr(Aligner, "global", Aligner.global_)


def hash_kmers(seq: bytes, k: int):
    """sparse::hash_kmers (sparse.rs:350-358): k-mer -> list of start positions."""
    out = {}
    for i in range(max(0, len(seq) + 1 - k)):
        out.setdefault(bytes(seq[i:i + k]), []).append(i)
    return out


def find_kmer_matches(seq1: bytes, seq2: bytes, k: int):
    """sparse::find_kmer_matches (sparse.rs:337-347): all (i, j) with seq1[i..i+k] == seq2[j..j+k], sorted.
    Host-side convenience for building `custom_with_matches` inputs; the aligner itself finds matches on the GPU."""
    h = hash_kmers(seq2, k)
    out = [(i, j) for i in range(max(0, len(seq1) + 1 - k)) for j in h.get(bytes(seq1[i:i + k]), ())]
    out.sort()
    return out
