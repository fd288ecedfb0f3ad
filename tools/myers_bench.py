"""Myers pattern matching (b2a_myers_batch) against the semi-global aligner computing the same best distances, run on
the GPU.

Myers::distance(x, y) == -(semiglobal score) under gap_open = -1, gap_extend = -1, match 0, mismatch -1 (x aligned end
to end, y free at both ends), so b2a_align_batch_scores in semiglobal mode with that scoring answers the best-distance
question; the pattern-matching path earns its place by being faster on it, and by what the aligner cannot give: every
end within k.  For each workload three calls alternate, `--runs` times each after one warm-up call: the search
without a listing (best ends only: pass 1), with a listing at the workload's k (pass 1, the offsets and pass 2), and
the aligner.  A call's kernel time is the engine's own event-timed kernels (stats: pack + fill + walk ms); GCUPS is
sum(m * n) over the median kernel time.  Before timing, best_dist == -score is checked on every pair, and best ends
and hit lists on a sample of pairs against the oracle (tests/sim/myers_oracle.cpp).  The card's name, power limit and
maximum SM clock are read in the same call.

  python tools/myers_bench.py [--workloads adapter,window150,long1000,bytes64] [--runs 3] [--out DIR]

Workloads (synthetic, seeded):
  adapter    1,000,000 x 150-nt reads against one shared 33-nt adapter, ~10 % of reads holding a copy with ~10 %
             substitutions, k = 3 (the register tier, 1 word; the pattern is stored once)
  window150  100,000 x 150-nt patterns against 1,000-nt windows holding a copy with ~5 % substitutions, k = 10
             (the register tier, 3 words)
  long1000   1,250 x 1,000-nt patterns against 10,000-nt texts holding a copy with ~5 % substitutions, k = 50 (the warp
             tier)
  bytes64    100,000 x 64-byte random patterns against 1,000-byte random texts, sigma = 256, k = 40
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rust_bio_b200._lib import MIN_SCORE, MODE_SEMIGLOBAL, CScoring  # noqa: E402
from rust_bio_b200.engine import Engine  # noqa: E402

DNA = np.frombuffer(b"ACGT", dtype=np.uint8)


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"


def planted(rng, pats, n_text, frac, sub, alpha):
    """texts of n_text symbols, a fraction `frac` of them holding their pattern with `sub` substitutions per symbol"""
    n, P = pats.shape
    texts = alpha[rng.integers(0, len(alpha), (n, n_text))]
    rows = np.nonzero(rng.random(n) < frac)[0]
    pos = rng.integers(0, n_text - P + 1, len(rows))
    copy = pats[rows].copy()
    s = rng.random(copy.shape) < sub
    copy[s] = alpha[rng.integers(0, len(alpha), int(s.sum()))]
    texts[rows[:, None], pos[:, None] + np.arange(P)] = copy
    return texts


def batch_of(pats, texts, shared):
    """(blob, x_off, x_len, y_off, y_len): the patterns (one copy when shared), then the texts"""
    n, N = texts.shape
    P = pats.shape[1]
    head = pats[:1].tobytes() if shared else pats.tobytes()
    blob = np.frombuffer(head + texts.tobytes() + b"\0" * 16, dtype=np.uint8).copy()
    x_off = np.zeros(n, dtype=np.uint64) if shared else np.arange(n, dtype=np.uint64) * np.uint64(P)
    y_off = np.uint64(len(head)) + np.arange(n, dtype=np.uint64) * np.uint64(N)
    return blob, x_off, np.full(n, P, dtype=np.uint32), y_off, np.full(n, N, dtype=np.uint32)


def workload(name, seed=11):
    """-> (batch, k)"""
    rng = np.random.default_rng(seed)
    if name == "adapter":
        adapter = DNA[rng.integers(0, 4, (1, 33))]
        pats = np.repeat(adapter, 1_000_000, axis=0)
        return batch_of(adapter, planted(rng, pats, 150, 0.1, 0.1, DNA), True), 3
    if name == "window150":
        pats = DNA[rng.integers(0, 4, (100_000, 150))]
        return batch_of(pats, planted(rng, pats, 1000, 1.0, 0.05, DNA), False), 10
    if name == "long1000":
        pats = DNA[rng.integers(0, 4, (1250, 1000))]
        return batch_of(pats, planted(rng, pats, 10_000, 1.0, 0.05, DNA), False), 50
    if name == "bytes64":
        allb = np.arange(256, dtype=np.uint8)
        pats = rng.integers(0, 256, (100_000, 64)).astype(np.uint8)
        return batch_of(pats, allb[rng.integers(0, 256, (100_000, 1000))], False), 40
    raise ValueError(name)


def kernel_ms(st):
    return st.pack_ms + st.fill_ms + st.walk_ms + st.band_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="adapter,window150,long1000,bytes64")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--sample", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import myers_util as mu
    print(json.dumps({"card": card()}), flush=True)
    unit = CScoring(-1, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 0, -1, 1, None, None, 0)
    eng = Engine(0)
    lines = []
    for name in a.workloads.split(","):
        batch, k = workload(name)
        blob, xo, xl, yo, yl = batch
        n = len(xl)
        cells = int((xl.astype(np.uint64) * yl.astype(np.uint64)).sum())
        calls = {"best": lambda: eng.myers_batch(batch),
                 "listing": lambda: eng.myers_batch(batch, k),
                 "aligner": lambda: eng.align_batch_scores(MODE_SEMIGLOBAL, unit, batch)}
        best = calls["best"]()
        listed = calls["listing"]()
        tiers = eng.myers_tier_pairs()
        s = calls["aligner"]()
        equal = bool(np.array_equal(best["best_dist"].astype(np.int64), -s["score"].astype(np.int64)))
        equal = equal and bool(np.array_equal(best["best_dist"], listed["best_dist"]))
        rng = np.random.default_rng(5)
        sample_ok = True
        for p in rng.integers(0, n, a.sample):
            x = blob[int(xo[p]):int(xo[p]) + int(xl[p])].tobytes()
            y = blob[int(yo[p]):int(yo[p]) + int(yl[p])].tobytes()
            be, bd, hits = mu.orc_search(x, y, k)
            lo, hi = int(listed["hit_off"][p]), int(listed["hit_off"][p + 1])
            got = list(zip(listed["hit_end"][lo:hi].tolist(), listed["hit_dist"][lo:hi].tolist()))
            sample_ok = sample_ok and (int(best["best_end"][p]), int(best["best_dist"][p])) == (be, bd) and got == hits
        rows = {c: [] for c in calls}
        for r in range(a.runs):
            for path, fn in calls.items():
                t0 = time.perf_counter()
                fn()
                wall = (time.perf_counter() - t0) * 1e3
                st = eng.stats
                rows[path].append({"kernel_ms": kernel_ms(st), "pass2_ms": st.walk_ms if path == "listing" else 0.0,
                                   "call_ms": wall, "launches": st.kernel_launches})
                print(json.dumps({"workload": name, "path": path, "run": r, **rows[path][-1]}), flush=True)
        summ = {"workload": name, "pairs": n, "cells": cells, "k": k, "hits": int(listed["hit_off"][-1]),
                "pairs_with_hits": tiers[6], "tiers": tiers[:6], "best_dist_equals_aligner": equal,
                "oracle_sample_equal": sample_ok}
        for path in rows:
            km = statistics.median(x["kernel_ms"] for x in rows[path])
            summ[f"{path}_kernel_ms"] = round(km, 3)
            summ[f"{path}_call_ms"] = round(statistics.median(x["call_ms"] for x in rows[path]), 3)
            summ[f"{path}_gcups"] = round(cells / (km * 1e6), 1) if km > 0 else None
        summ["listing_pass2_ms"] = round(statistics.median(x["pass2_ms"] for x in rows["listing"]), 3)
        summ["speedup_kernel"] = round(summ["aligner_kernel_ms"] / summ["best_kernel_ms"], 2)
        print(json.dumps(summ), flush=True)
        lines.append(summ)
    eng.close()
    print(json.dumps({"card": card()}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "myers_bench.json"), "w") as f:
            json.dump({"card": card(), "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
