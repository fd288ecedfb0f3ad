"""Engine: one CUDA device, batches in / Alignment fields out (thin wrapper over the C ABI)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np

from . import _lib
from ._lib import B2AError, CMyersMatch, CPairHmmParams, CPairs, CResults, CScoring, CStats

Batch = Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]


def pack_pairs(pairs) -> Batch:
    """[(x_bytes, y_bytes), ...] -> (blob, x_off, x_len, y_off, y_len), 16-byte aligned sequences."""
    n = len(pairs)
    x_len = np.fromiter((len(p[0]) for p in pairs), dtype=np.uint32, count=n)
    y_len = np.fromiter((len(p[1]) for p in pairs), dtype=np.uint32, count=n)
    pad = lambda v: (v.astype(np.uint64) + np.uint64(15)) // np.uint64(16) * np.uint64(16)
    sizes = np.stack([pad(x_len), pad(y_len)], axis=1).reshape(-1)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    blob = np.zeros(int(offs[-1]) + 16, dtype=np.uint8)
    x_off, y_off = offs[0:-1:2].copy(), offs[1::2].copy()
    for i, (x, y) in enumerate(pairs):
        blob[int(x_off[i]):int(x_off[i]) + len(x)] = np.frombuffer(bytes(x), dtype=np.uint8)
        blob[int(y_off[i]):int(y_off[i]) + len(y)] = np.frombuffer(bytes(y), dtype=np.uint8)
    return blob, x_off, x_len, y_off, y_len


class Results:
    """Host outputs of one batch (numpy arrays; pass pinned arrays via `out=` for speed)."""

    def __init__(self, n_pairs: int, ops_capacity: int, out: Optional[Dict[str, np.ndarray]] = None,
                 pair_status: bool = False):
        mk = lambda name, shape, dt: (out[name] if out and name in out else np.zeros(shape, dtype=dt))
        self.n_pairs = n_pairs
        self.score = mk("score", n_pairs, np.int32)
        self.xstart = mk("xstart", n_pairs, np.uint32)
        self.xend = mk("xend", n_pairs, np.uint32)
        self.ystart = mk("ystart", n_pairs, np.uint32)
        self.yend = mk("yend", n_pairs, np.uint32)
        self.ops_off = mk("ops_off", n_pairs + 1, np.uint64)
        self.ops = mk("ops", max(1, ops_capacity), np.uint8)
        self.clip_len = mk("clip_len", 4 * max(1, n_pairs), np.uint32)
        # per-pair B2A_PAIR_* codes: requested with pair_status=True (else a pair on which the reference would
        # panic fails the whole batch, include/b200align.h)
        self.status = mk("status", max(1, n_pairs), np.uint32) if pair_status else None
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        self.c = CResults(p(self.score), p(self.xstart), p(self.xend), p(self.ystart), p(self.yend),
                          p(self.ops_off), p(self.ops), len(self.ops), p(self.clip_len),
                          p(self.status) if pair_status else None)

    def ops_of(self, i: int):
        """[(code, clip_len)] of pair i in alignment order."""
        lo, hi = int(self.ops_off[i]), int(self.ops_off[i + 1])
        res, k = [], 0
        for c in self.ops[lo:hi]:
            c = int(c)
            if c >= 4:
                res.append((c, int(self.clip_len[4 * i + k])))
                k += 1
            else:
                res.append((c, 0))
        return res

    def as_dict(self):
        return {k: getattr(self, k) for k in ("score", "xstart", "xend", "ystart", "yend")}


class ScoreResults:
    """Host outputs of a score-only batch: score, xend, yend and the per-pair B2A_PAIR_* status (numpy arrays in the
    caller's pair order); the other b2a_results fields stay NULL."""

    def __init__(self, n_pairs: int):
        self.n_pairs = n_pairs
        self.score = np.zeros(max(1, n_pairs), dtype=np.int32)
        self.xend = np.zeros(max(1, n_pairs), dtype=np.uint32)
        self.yend = np.zeros(max(1, n_pairs), dtype=np.uint32)
        self.status = np.zeros(max(1, n_pairs), dtype=np.uint32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        self.c = CResults(p(self.score), None, p(self.xend), None, p(self.yend), None, None, 0, None, p(self.status))

    def as_dict(self):
        return {k: getattr(self, k)[:self.n_pairs] for k in ("score", "xend", "yend", "status")}


class _BatchCalls:
    """The batch methods Engine and MultiEngine share: host arrays in, host results out.  A subclass binds the C entry
    points (_c_align, _c_scores, _c_banded, _c_banded_scores, _c_levenshtein, _c_hamming, _c_myers, _c_myers_fetch, _c_pairhmm: the handle's calls, each returning the rc) and _check."""

    @staticmethod
    def _cpairs(batch: Batch):
        blob, x_off, x_len, y_off, y_len = batch
        assert blob.dtype == np.uint8 and x_off.dtype == np.uint64 and y_off.dtype == np.uint64
        assert x_len.dtype == np.uint32 and y_len.dtype == np.uint32
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        return CPairs(p(blob), p(x_off), p(x_len), p(y_off), p(y_len), blob.nbytes, len(x_len))

    @staticmethod
    def default_ops_capacity(batch: Batch) -> int:
        return int(batch[2].astype(np.uint64).sum() + batch[4].astype(np.uint64).sum() + 4 * len(batch[2]))

    @staticmethod
    def _band_hints(n: int, matches, paths, allowed_mismatches, use_lcskpp_union):
        """b2a_band_hints of per-pair match lists (and paths) -> (CBandHints, the arrays it points into)"""
        from ._lib import CBandHints
        if len(matches) != n or (paths is not None and len(paths) != n):
            raise ValueError("one match list (and path) per pair")
        moff = np.zeros(n + 1, dtype=np.uint64)
        moff[1:] = np.cumsum([len(m) for m in matches])
        mxy = np.array([v for m in matches for mt in m for v in mt], dtype=np.uint32).reshape(-1)
        if mxy.size == 0:
            mxy = np.zeros(2, dtype=np.uint32)
        h = CBandHints(moff.ctypes.data, mxy.ctypes.data, None, None,
                       -1 if allowed_mismatches is None else int(allowed_mismatches), 1 if use_lcskpp_union else 0)
        keep = [moff, mxy]
        if paths is not None:
            poff = np.zeros(n + 1, dtype=np.uint64)
            poff[1:] = np.cumsum([len(p) for p in paths])
            pidx = np.array([v for p in paths for v in p] or [0], dtype=np.uint32)
            h.path_off, h.path_idx = poff.ctypes.data, pidx.ctypes.data
            keep += [poff, pidx]
        return h, keep

    def align_batch(self, mode: int, cscoring: CScoring, batch: Batch, results: Optional[Results] = None,
                    ops_capacity: Optional[int] = None) -> Results:
        """b2a_align_batch (b2a_multi_align_batch): host buffers in, host buffers out."""
        if results is None:
            results = Results(len(batch[2]), ops_capacity if ops_capacity is not None
                              else self.default_ops_capacity(batch))
        cp = self._cpairs(batch)
        self._check(self._c_align(int(mode), C.byref(cscoring), C.byref(cp), C.byref(results.c)))
        return results

    def align_batch_scores(self, mode: int, cscoring: CScoring, batch: Batch) -> Dict[str, np.ndarray]:
        """b2a_align_batch_scores: Alignment.score / xend / yend without the traceback -> {score, xend, yend, status}
        (numpy, caller's pair order; a pair the reference panics on has status B2A_PAIR_PANIC)."""
        res = ScoreResults(len(batch[2]))
        cp = self._cpairs(batch)
        self._check(self._c_scores(int(mode), C.byref(cscoring), C.byref(cp), C.byref(res.c)))
        return res.as_dict()

    def align_batch_banded(self, mode: int, cscoring: CScoring, k: int, w: int, batch: Batch,
                           results: Optional[Results] = None) -> Results:
        if results is None:
            results = Results(len(batch[2]), self.default_ops_capacity(batch))
        cp = self._cpairs(batch)
        self._check(self._c_banded(int(mode), C.byref(cscoring), int(k), int(w), C.byref(cp), None, C.byref(results.c)))
        return results

    def align_batch_banded_hinted(self, mode: int, cscoring: CScoring, k: int, w: int, batch: Batch,
                                  matches, paths=None, allowed_mismatches: Optional[int] = None,
                                  use_lcskpp_union: bool = False, results: Optional[Results] = None) -> Results:
        """banded::Aligner::custom_with_{matches, expanded_matches, match_path} over a batch
        (b2a_align_batch_banded_hinted): matches[p] = [(xpos, ypos), ...] per pair, paths[p] = [index, ...]."""
        n = len(batch[2])
        h, keep = self._band_hints(n, matches, paths, allowed_mismatches, use_lcskpp_union)
        if results is None:
            results = Results(n, self.default_ops_capacity(batch))
        cp = self._cpairs(batch)
        self._check(self._c_banded(int(mode), C.byref(cscoring), int(k), int(w), C.byref(cp), C.byref(h),
                                   C.byref(results.c)))
        return results

    def align_batch_banded_scores(self, mode: int, cscoring: CScoring, k: int, w: int, batch: Batch, matches=None,
                                  paths=None, allowed_mismatches: Optional[int] = None,
                                  use_lcskpp_union: bool = False) -> Dict[str, np.ndarray]:
        """b2a_align_batch_banded_scores: the banded aligner's Alignment.score / xend / yend without the traceback ->
        {score, xend, yend, status} (numpy, caller's pair order).  matches (and paths, allowed_mismatches,
        use_lcskpp_union) as in align_batch_banded_hinted; matches=None finds them on the device."""
        n = len(batch[2])
        h = keep = None
        if matches is not None:
            h, keep = self._band_hints(n, matches, paths, allowed_mismatches, use_lcskpp_union)
        res = ScoreResults(n)
        cp = self._cpairs(batch)
        self._check(self._c_banded_scores(int(mode), C.byref(cscoring), int(k), int(w), C.byref(cp),
                                          C.byref(h) if h is not None else None, C.byref(res.c)))
        return res.as_dict()

    def levenshtein_batch(self, batch: Batch, k: Optional[int] = None) -> np.ndarray:
        """b2a_levenshtein_batch: per pair, levenshtein(x, y) (k=None), or simd::bounded_levenshtein(x, y, k) with
        None as DIST_NONE -> uint32 numpy array in the caller's pair order."""
        kk = _lib.DIST_NONE if k is None else int(k)
        if not 0 <= kk <= _lib.DIST_NONE:
            raise ValueError("k must fit in u32")
        out = np.zeros(max(1, len(batch[2])), dtype=np.uint32)
        cp = self._cpairs(batch)
        self._check(self._c_levenshtein(kk, C.byref(cp), out.ctypes.data_as(C.c_void_p)))
        return out[:len(batch[2])]

    def hamming_batch(self, batch: Batch, pair_status: bool = True):
        """b2a_hamming_batch: per pair, hamming(x, y) -> (uint32 distances, uint32 B2A_PAIR_* statuses); a pair of
        unequal lengths is B2A_PAIR_PANIC with distance DIST_NONE.  pair_status=False: such a pair fails the call
        (B2AError) and only the distances are returned."""
        n = len(batch[2])
        out = np.zeros(max(1, n), dtype=np.uint32)
        st = np.zeros(max(1, n), dtype=np.uint32) if pair_status else None
        cp = self._cpairs(batch)
        self._check(self._c_hamming(C.byref(cp), out.ctypes.data_as(C.c_void_p),
                                    st.ctypes.data_as(C.c_void_p) if pair_status else None))
        return (out[:n], st[:n]) if pair_status else out[:n]

    def myers_batch(self, batch: Batch, k: Optional[int] = None, ambig=None, wildcards=None,
                    pair_status: bool = True) -> Dict[str, np.ndarray]:
        """b2a_myers_batch: per pair, the semi-global search of the pattern x in the text y (bio::pattern_matching::
        myers) -> {"best_end", "best_dist"} (uint32, DIST_NONE for an empty text or pattern), "status" (B2A_PAIR_*:
        an empty pattern is B2A_PAIR_PANIC) with pair_status, and with k every end whose distance is <= k as CSR:
        "hit_off" (uint64, n + 1), "hit_end", "hit_dist" (uint32).  k above u32 is clamped: a distance is at most the
        pattern length.  ambig: {pattern byte: text bytes it also matches}; wildcards: text bytes every pattern byte
        matches (MyersBuilder.ambig / text_wildcard).  pair_status=False: an empty pattern fails the call."""
        if k is not None and int(k) < 0:
            raise ValueError("k must be >= 0")
        n = len(batch[2])
        best_end = np.zeros(max(1, n), dtype=np.uint32)
        best_dist = np.zeros(max(1, n), dtype=np.uint32)
        st = np.zeros(max(1, n), dtype=np.uint32) if pair_status else None
        cm, keep = myers_match(ambig, wildcards)
        cp = self._cpairs(batch)
        hits = C.c_uint64(0)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        self._check(self._c_myers(C.byref(cm) if cm is not None else None,
                                  0 if k is None else min(int(k), _lib.DIST_NONE), C.byref(cp), p(best_end),
                                  p(best_dist), C.byref(hits) if k is not None else None,
                                  p(st) if pair_status else None))
        del keep
        out = {"best_end": best_end[:n], "best_dist": best_dist[:n]}
        if pair_status:
            out["status"] = st[:n]
        if k is not None:
            h = int(hits.value)
            off = np.zeros(n + 1, dtype=np.uint64)
            he = np.zeros(max(1, h), dtype=np.uint32)
            hd = np.zeros(max(1, h), dtype=np.uint32)
            self._check(self._c_myers_fetch(p(off), p(he), p(hd)))
            out.update(hit_off=off, hit_end=he[:h], hit_dist=hd[:h])
        return out

    def pairhmm_batch(self, batch: Batch, gap, emit, free_start_gap_x: bool, free_end_gap_x: bool,
                      max_edit_dist: Optional[int] = None, classes: Optional[np.ndarray] = None,
                      pair_status: bool = True):
        """b2a_pairhmm_batch: per pair, PairHMM::prob_related (bio::stats::pairhmm) of x and y -> float64 natural-log
        probabilities in the caller's pair order, and with pair_status the B2A_PAIR_* statuses (a NaN result, the
        reference's assert, is B2A_PAIR_PANIC).  gap: (prob_gap_x, prob_gap_y, prob_gap_x_extend, prob_gap_y_extend)
        as natural logs.  emit: four sequences (match, mismatch, x, y) of one natural-log value per class.  classes:
        None (every class 0) or uint8 class bytes laid out like the batch's blob.  max_edit_dist None: no band.
        pair_status=False: a NaN result fails the call (B2AError) and only the probabilities are returned."""
        tab = np.ascontiguousarray(np.asarray(emit, dtype=np.float64))
        if tab.ndim != 2 or tab.shape[0] != 4 or not 1 <= tab.shape[1] <= 256:
            raise ValueError("emit must be 4 tables of 1 .. 256 classes")
        med = _lib.PAIRHMM_NO_BAND if max_edit_dist is None else int(max_edit_dist)
        if not 0 <= med <= _lib.PAIRHMM_NO_BAND:
            raise ValueError("max_edit_dist must fit in u64")
        if classes is not None:
            classes = np.ascontiguousarray(classes, dtype=np.uint8)
            if classes.nbytes < batch[0].nbytes:
                raise ValueError("classes must hold one byte per blob byte")
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        ncls = tab.shape[1]
        prm = CPairHmmParams(*[float(v) for v in gap], 1 if free_start_gap_x else 0, 1 if free_end_gap_x else 0, med,
                             ncls, p(tab[0]), p(tab[1]), p(tab[2]), p(tab[3]),
                             p(classes) if classes is not None else None)
        n = len(batch[2])
        out = np.zeros(max(1, n), dtype=np.float64)
        st = np.zeros(max(1, n), dtype=np.uint32) if pair_status else None
        cp = self._cpairs(batch)
        self._check(self._c_pairhmm(C.byref(prm), C.byref(cp), p(out), p(st) if pair_status else None))
        return (out[:n], st[:n]) if pair_status else out[:n]


def myers_match(ambig=None, wildcards=None):
    """(CMyersMatch or None, the arrays it points to): the bit tables of b2a_myers_match from {pattern byte:
    equivalent text bytes} and an iterable of wildcard text bytes"""
    if not ambig and not wildcards:
        return None, None
    amb = np.zeros((256, 32), dtype=np.uint8) if ambig else None
    for p, eqs in (ambig or {}).items():
        for t in bytes(eqs):
            amb[int(p), t >> 3] |= np.uint8(1 << (t & 7))
    wild = np.zeros(32, dtype=np.uint8) if wildcards else None
    for t in (wildcards or ()):
        wild[int(t) >> 3] |= np.uint8(1 << (int(t) & 7))
    cm = CMyersMatch(amb.ctypes.data_as(C.c_void_p) if amb is not None else None,
                     wild.ctypes.data_as(C.c_void_p) if wild is not None else None)
    return cm, (amb, wild)


class Engine(_BatchCalls):
    def __init__(self, device: int = 0):
        self._L = _lib.load()
        h = C.c_void_p()
        rc = self._L.b2a_engine_create(C.byref(h), int(device))
        if rc != 0:
            raise B2AError(rc, f"cannot create engine on cuda:{device} (no CPU fallback exists)")
        self._h = h
        self.device = device
        self.stats = CStats()
        self._keep = None

    def close(self):
        if getattr(self, "_h", None):
            self._L.b2a_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise B2AError(rc, self._L.b2a_last_error(self._h).decode())

    def set_stream(self, cuda_stream: int):
        self._check(self._L.b2a_engine_set_stream(self._h, C.c_void_p(cuda_stream)))

    def set_tuning(self, lanes_per_pair: int, rows_per_lane: int):
        self._check(self._L.b2a_engine_set_tuning(self._h, lanes_per_pair, rows_per_lane))

    def last_alphabet(self) -> np.ndarray:
        """The alphabet the last stage used (given by the caller or found in the batch), ascending byte values."""
        buf = np.zeros(256, dtype=np.uint8)
        n = C.c_uint32()
        self._check(self._L.b2a_engine_last_alphabet(self._h, buf.ctypes.data_as(C.c_void_p), C.byref(n)))
        return buf[:n.value].copy()

    def set_walk(self, mode: int):
        """K2 shape: 0 automatic, 1 one lane per pair, 2 one warp per pair (b2a_engine_set_walk)."""
        self._check(self._L.b2a_engine_set_walk(self._h, int(mode)))

    def set_pipeline(self, chunks: int):
        self._check(self._L.b2a_engine_set_pipeline(self._h, int(chunks)))

    def set_traceback_budget(self, nbytes: int):
        self._check(self._L.b2a_engine_set_traceback_budget(self._h, int(nbytes)))

    def set_traceback_recompute(self, on: bool):
        """Align a pair whose traceback is above the budget by refilling it one window of strips at a time
        (b2a_engine_set_traceback_recompute); off by default: such a pair is refused."""
        self._check(self._L.b2a_engine_set_traceback_recompute(self._h, 1 if on else 0))

    def last_recompute(self) -> dict:
        """Of the last full call: pairs whose traceback was recomputed, their windows, and the windows refilled
        (b2a_engine_last_recompute)."""
        p, w, f = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.b2a_engine_last_recompute(self._h, C.byref(p), C.byref(w), C.byref(f)))
        return {"pairs": int(p.value), "windows": int(w.value), "windows_filled": int(f.value)}

    def myers_tier_pairs(self) -> list:
        """Pairs of the last myers_batch per tier: [host-answered, register tier with 1..4 words (4 entries), warp,
        pairs rerun by pass 2 to write their hits] (b2a_myers_tier_pairs; a measurement aid)."""
        buf = np.zeros(7, dtype=np.uint64)
        self._check(self._L.b2a_myers_tier_pairs(self._h, buf.ctypes.data_as(C.c_void_p), 7))
        return [int(v) for v in buf]

    def pairhmm_tier_pairs(self) -> list:
        """Pairs of the last pairhmm_batch per tier: [host-answered, one strip with 1, 2, 4, 5, 8 columns per lane (5
        entries), strips of 256 columns] (b2a_pairhmm_tier_pairs; a measurement aid)."""
        buf = np.zeros(7, dtype=np.uint64)
        self._check(self._L.b2a_pairhmm_tier_pairs(self._h, buf.ctypes.data_as(C.c_void_p), 7))
        return [int(v) for v in buf]

    def distance_tier_pairs(self) -> list:
        """Pairs of the last levenshtein_batch per tier: [host-answered, register tier with 1..4 words (4 entries),
        4-word band, 8-word band, warp] (b2a_distance_tier_pairs; a measurement aid)."""
        buf = np.zeros(8, dtype=np.uint64)
        self._check(self._L.b2a_distance_tier_pairs(self._h, buf.ctypes.data_as(C.c_void_p), 8))
        return [int(v) for v in buf]

    # the C entry points of the shared batch methods (_BatchCalls)
    def _c_align(self, mode, cs, cp, res):
        return self._L.b2a_align_batch(self._h, mode, cs, cp, res, C.byref(self.stats))

    def _c_scores(self, mode, cs, cp, res):
        return self._L.b2a_align_batch_scores(self._h, mode, cs, cp, res, C.byref(self.stats))

    def _c_banded(self, mode, cs, k, w, cp, hints, res):
        if hints is None:
            return self._L.b2a_align_batch_banded(self._h, mode, cs, k, w, cp, res, C.byref(self.stats))
        return self._L.b2a_align_batch_banded_hinted(self._h, mode, cs, k, w, cp, hints, res, C.byref(self.stats))

    def _c_levenshtein(self, k, cp, out):
        return self._L.b2a_levenshtein_batch(self._h, k, cp, out, C.byref(self.stats))

    def _c_hamming(self, cp, out, status):
        return self._L.b2a_hamming_batch(self._h, cp, out, status, C.byref(self.stats))

    def _c_myers(self, cm, k, cp, best_end, best_dist, n_hits, status):
        return self._L.b2a_myers_batch(self._h, cm, k, cp, best_end, best_dist, n_hits, status, C.byref(self.stats))

    def _c_myers_fetch(self, off, hit_end, hit_dist):
        return self._L.b2a_myers_hits_fetch(self._h, off, hit_end, hit_dist)

    def _c_pairhmm(self, prm, cp, out, status):
        return self._L.b2a_pairhmm_batch(self._h, prm, cp, out, status, C.byref(self.stats))

    def _c_banded_scores(self, mode, cs, k, w, cp, hints, res):
        return self._L.b2a_align_batch_banded_scores(self._h, mode, cs, k, w, cp, hints, res, C.byref(self.stats))

    def stage_scores(self, mode: int, cscoring: CScoring, batch: Batch):
        """b2a_batch_stage_scores: stage a score-only batch (then run(), fetch_scores())."""
        self._keep = (batch, cscoring)
        cp = self._cpairs(batch)
        self._check(self._L.b2a_batch_stage_scores(self._h, int(mode), C.byref(cscoring), C.byref(cp)))

    def fetch_scores(self) -> Dict[str, np.ndarray]:
        """b2a_batch_fetch of a score-only batch -> {score, xend, yend, status}."""
        res = ScoreResults(len(self._keep[0][2]))
        self._check(self._L.b2a_batch_fetch(self._h, C.byref(res.c), C.byref(self.stats)))
        return res.as_dict()

    @staticmethod
    def pack_bitenc_pairs(pairs):
        """[(BitEnc x, BitEnc y), ...] -> (blocks, x_block, x_len, y_block, y_len, width): the storages of all
        sequences concatenated (what b2a_packed_pairs points at)."""
        width = pairs[0][0].width if pairs else 2
        chunks, xb, xl, yb, yl, pos = [], [], [], [], [], 0
        for x, y in pairs:
            assert x.width == width and y.width == width, "one width per batch"
            xb.append(pos)
            xl.append(x.nr_symbols())
            chunks.append(x.storage)
            pos += x.nr_blocks()
            yb.append(pos)
            yl.append(y.nr_symbols())
            chunks.append(y.storage)
            pos += y.nr_blocks()
        blocks = np.concatenate(chunks + [np.zeros(4, dtype=np.uint32)]).astype(np.uint32)
        return (blocks, np.array(xb, dtype=np.uint64), np.array(xl, dtype=np.uint32), np.array(yb, dtype=np.uint64),
                np.array(yl, dtype=np.uint32), width)

    def align_batch_packed(self, mode: int, cscoring: CScoring, packed, results: Optional[Results] = None,
                           banded=None) -> Results:
        """b2a_align_batch_packed / b2a_align_batch_banded_packed: `packed` = pack_bitenc_pairs(...) (numpy arrays;
        pinned arrays give the fastest copies).  `banded` = (k, w) for the banded aligner."""
        from ._lib import CPackedPairs
        blocks, xb, xl, yb, yl, width = packed
        n = len(xl)
        if results is None:
            results = Results(n, int(xl.astype(np.uint64).sum() + yl.astype(np.uint64).sum() + 4 * n))
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        pp = CPackedPairs(p(blocks), p(xb), p(xl), p(yb), p(yl), len(blocks), n, int(width))
        if banded is None:
            self._check(self._L.b2a_align_batch_packed(self._h, int(mode), C.byref(cscoring), C.byref(pp),
                                                       C.byref(results.c), C.byref(self.stats)))
        else:
            self._check(self._L.b2a_align_batch_banded_packed(self._h, int(mode), C.byref(cscoring), int(banded[0]),
                                                              int(banded[1]), C.byref(pp), C.byref(results.c),
                                                              C.byref(self.stats)))
        return results

    def banded_band_ranges(self, pair: int, y_len: int) -> np.ndarray:
        """Band::ranges of `pair` of the last banded call: array [y_len + 1, 2] of (start, end) row ranges."""
        out = np.zeros((int(y_len) + 1, 2), dtype=np.uint32)
        self._check(self._L.b2a_banded_band_ranges(self._h, int(pair), out.ctypes.data_as(C.c_void_p), int(y_len) + 1))
        return out

    # staged form

    def banded_strip_pairs(self) -> int:
        """Pairs of the last banded call that ran the strip-wavefront fill (b2a_banded_strip_pairs)."""
        v = C.c_uint64(0)
        self._check(self._L.b2a_banded_strip_pairs(self._h, C.byref(v)))
        return int(v.value)

    def stage(self, mode: int, cscoring: CScoring, batch: Batch):
        self._keep = (batch, cscoring)
        cp = self._cpairs(batch)
        self._check(self._L.b2a_batch_stage(self._h, int(mode), C.byref(cscoring), C.byref(cp)))

    def run(self):
        self._check(self._L.b2a_batch_run(self._h))

    def fetch(self, results: Optional[Results]) -> Optional[Results]:
        self._check(self._L.b2a_batch_fetch(self._h, C.byref(results.c) if results else None,
                                            C.byref(self.stats)))
        return results

    def records_into(self, dev_ptr: int, nbytes: int) -> int:
        stride = C.c_uint32()
        self._check(self._L.b2a_batch_records_into(self._h, C.c_void_p(dev_ptr), int(nbytes), C.byref(stride)))
        return stride.value

    def compact_bytes(self) -> int:
        """Size of this batch's compact result segment (waits for the batch; see include/b200align.h)."""
        nb = C.c_uint64()
        self._check(self._L.b2a_batch_compact_bytes(self._h, C.byref(nb)))
        return int(nb.value)

    def compact_into(self, dev_ptr: int, nbytes: int) -> None:
        self._check(self._L.b2a_batch_compact_into(self._h, C.c_void_p(dev_ptr), int(nbytes)))

    def compact_fixed(self, dev_ptr: int, capacity_bytes: int) -> None:
        """b2a_batch_compact_fixed: the segment with a caller-fixed capacity; no wait, no size read-back."""
        self._check(self._L.b2a_batch_compact_fixed(self._h, C.c_void_p(dev_ptr), int(capacity_bytes)))

    def gathered_fetch(self, dev_ptr: int, segment_bytes: int, n_segments: int, results: Results):
        """b2a_gathered_fetch: gathered device segments -> host `results`; returns (pairs, d2h bytes)."""
        n, b = C.c_uint64(), C.c_uint64()
        self._check(self._L.b2a_gathered_fetch(self._h, C.c_void_p(dev_ptr), int(segment_bytes), int(n_segments),
                                               C.byref(results.c), C.byref(n), C.byref(b)))
        return int(n.value), int(b.value)

    def decode_compact(self, host_segments: np.ndarray, segment_bytes: int, n_segments: int, n_total: int,
                       ops_capacity: int) -> Results:
        """Decode `n_segments` gathered compact segments (each padded to segment_bytes) in rank order."""
        res = Results(n_total, ops_capacity)
        pair_base = ops_base = 0
        for r in range(n_segments):
            seg = host_segments[r * segment_bytes:(r + 1) * segment_bytes]
            n, nb = C.c_uint64(), C.c_uint64()
            rc = self._L.b2a_compact_decode(seg.ctypes.data_as(C.c_void_p), segment_bytes, pair_base, ops_base,
                                            C.byref(res.c), C.byref(n), C.byref(nb))
            if rc != 0:
                raise B2AError(rc, "b2a_compact_decode")
            pair_base += n.value
            ops_base += nb.value
        if pair_base != n_total:
            raise B2AError(-2, "compact segments hold %d pairs, expected %d" % (pair_base, n_total))
        res.ops_off[n_total] = ops_base
        return res

    def record_stride(self, max_m: int, max_n: int) -> int:
        return int(self._L.b2a_record_stride(max_m, max_n))

    def decode_records(self, host_records: np.ndarray, stride: int, n: int, ops_capacity: int) -> Results:
        res = Results(n, ops_capacity)
        rc = self._L.b2a_records_decode(host_records.ctypes.data_as(C.c_void_p), stride, n, C.byref(res.c))
        if rc != 0:
            raise B2AError(rc, "b2a_records_decode")
        return res


_default: Dict[int, Engine] = {}


def default_engine(device: int = 0) -> Engine:
    if device not in _default:
        _default[device] = Engine(device)
    return _default[device]


class MultiEngine(_BatchCalls):
    """Every visible GPU from one process (b2a_multi_*): the batch is split over the devices, one ncclAllGather
    reassembles the results, device 0's copy is returned.  Same results as the Engine methods of the same names, so
    pairwise.Aligner and banded.Aligner take one as their `engine`.  device_ids may repeat a device (one engine per
    entry, peer copies instead of NCCL)."""

    def __init__(self, device_ids=None):
        self._L = _lib.load()
        h = C.c_void_p()
        if device_ids is None:
            rc = self._L.b2a_multi_create(C.byref(h), None, 0)
        else:
            ids = (C.c_int32 * len(device_ids))(*device_ids)
            rc = self._L.b2a_multi_create(C.byref(h), ids, len(device_ids))
        if rc != 0:
            raise B2AError(rc, "cannot create the multi-GPU engine (no CPU fallback exists)")
        self._h = h
        self.stats = CStats()

    @property
    def n_devices(self) -> int:
        return int(self._L.b2a_multi_device_count(self._h))

    @property
    def exchange_kind(self) -> str:
        return self._L.b2a_multi_exchange_kind(self._h).decode()

    def _check(self, rc):
        if rc != 0:
            raise B2AError(rc, self._L.b2a_multi_last_error(self._h).decode())

    # the C entry points of the shared batch methods (_BatchCalls): the b2a_multi_* forms
    def _c_align(self, mode, cs, cp, res):
        return self._L.b2a_multi_align_batch(self._h, mode, cs, cp, res, C.byref(self.stats))

    def _c_scores(self, mode, cs, cp, res):
        return self._L.b2a_multi_align_batch_scores(self._h, mode, cs, cp, res, C.byref(self.stats))

    def _c_banded(self, mode, cs, k, w, cp, hints, res):
        return self._L.b2a_multi_align_batch_banded(self._h, mode, cs, k, w, cp, hints, res, C.byref(self.stats))

    def _c_levenshtein(self, k, cp, out):
        return self._L.b2a_multi_levenshtein_batch(self._h, k, cp, out, C.byref(self.stats))

    def _c_hamming(self, cp, out, status):
        return self._L.b2a_multi_hamming_batch(self._h, cp, out, status, C.byref(self.stats))

    def _c_myers(self, cm, k, cp, best_end, best_dist, n_hits, status):
        return self._L.b2a_multi_myers_batch(self._h, cm, k, cp, best_end, best_dist, n_hits, status,
                                             C.byref(self.stats))

    def _c_myers_fetch(self, off, hit_end, hit_dist):
        return self._L.b2a_multi_myers_hits_fetch(self._h, off, hit_end, hit_dist)

    def _c_pairhmm(self, prm, cp, out, status):
        return self._L.b2a_multi_pairhmm_batch(self._h, prm, cp, out, status, C.byref(self.stats))

    def _c_banded_scores(self, mode, cs, k, w, cp, hints, res):
        return self._L.b2a_multi_align_batch_banded_scores(self._h, mode, cs, k, w, cp, hints, res, C.byref(self.stats))

    def banded_band_ranges(self, pair: int, y_len: int) -> np.ndarray:
        """Band ranges stay on the engine of the device that aligned the pair: not available here (so
        banded.Aligner.visualize needs an Engine)."""
        raise NotImplementedError("band ranges are kept per device engine: banded.Aligner.visualize needs an Engine, "
                                  "not a MultiEngine")

    def close(self):
        if getattr(self, "_h", None):
            self._L.b2a_multi_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
