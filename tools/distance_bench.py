"""Edit distance (b2a_levenshtein_batch) against the aligner computing the same numbers, run on the GPU.

levenshtein(x, y) == -(global score) under gap_open = -1, gap_extend = -1, match 0, mismatch -1, so
b2a_align_batch_scores in global mode with that scoring answers the same question; the distance path earns its place
only by being faster on the same pairs.  For each workload the two are called in alternation, `--runs` times each
after one warm-up call; a call's kernel time is the engine's own event-timed kernels (stats: pack + fill + walk ms:
the distance path's blob rewrite into alphabet codes and its distance kernels; the aligner's K0, K1 and K2).  GCUPS
is sum(m * n) over the median kernel time.  Before timing, the outputs are checked equal (bounded: the distance when
-score <= k, else None).  The card's name, power limit and maximum SM clock are read in the same call.

  python tools/distance_bench.py [--workloads dna150,dna1000,prot10k,similar10k,bytes150,bytes1000] [--runs 3] [--out DIR]

Workloads (synthetic, rust_bio_b200/synth.py):
  dna150      1,000,000 x 150 x 150 DNA, levenshtein (the register tier)
  dna1000     100,000 x 1000 x 1000 DNA, levenshtein (the warp tier)
  prot10k     1,250 x 10,000 x 10,000 protein, levenshtein (the warp tier, sigma = 20)
  bytes150    100,000 x 150 x 150 uniform random bytes (sigma = 256: the register tier's largest match-mask tables)
  bytes1000   10,000 x 1000 x 1000 uniform random bytes (sigma = 256, the warp tier)
  similar10k  1,250 x ~10,000 DNA pairs, y a copy of x with ~1 % substitutions and a few indels,
              bounded_levenshtein with k = 100 (the band tier)
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

from rust_bio_b200 import synth  # noqa: E402
from rust_bio_b200._lib import DIST_NONE, MIN_SCORE, MODE_GLOBAL, CScoring  # noqa: E402
from rust_bio_b200.engine import Engine  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"


def similar_pairs(n_pairs, L, seed=3):
    """x uniform DNA of length L; y = x with 1 % substitutions, then 4 single-base insertions and 4 deletions"""
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(synth.DNA, dtype=np.uint8)
    xs = alpha[rng.integers(0, 4, (n_pairs, L))]
    ys = xs.copy()
    sub = rng.random((n_pairs, L)) < 0.01
    ys[sub] = alpha[rng.integers(0, 4, int(sub.sum()))]
    pairs = []
    for p in range(n_pairs):
        y = ys[p]
        for pos in rng.integers(0, L - 8, 4):
            y = np.insert(y, pos, alpha[rng.integers(0, 4)])
        for pos in rng.integers(0, L - 8, 4):
            y = np.delete(y, pos)
        pairs.append((xs[p].tobytes(), y.tobytes()))
    from rust_bio_b200.engine import pack_pairs
    return pack_pairs(pairs)


def workload(name):
    """-> (batch, k or None)"""
    if name == "dna150":
        return synth.uniform_pairs(synth.BASES["C2"], 0, 1_000_000, 150, 150), None
    if name == "dna1000":
        return synth.uniform_pairs(synth.BASES["C3"], 0, 100_000, 1000, 1000), None
    if name == "prot10k":
        return synth.uniform_pairs(synth.BASES["C5"], 0, 1250, 10000, 10000, alphabet=synth.PROTEIN), None
    if name == "bytes150":
        return synth.uniform_pairs(synth.BASES["C2"], 0, 100_000, 150, 150, alphabet=bytes(range(256))), None
    if name == "bytes1000":
        return synth.uniform_pairs(synth.BASES["C3"], 0, 10_000, 1000, 1000, alphabet=bytes(range(256))), None
    if name == "similar10k":
        return similar_pairs(1250, 10000), 100
    raise ValueError(name)


def kernel_ms(st):
    return st.pack_ms + st.fill_ms + st.walk_ms + st.band_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="dna150,dna1000,prot10k,similar10k,bytes150,bytes1000")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    unit = CScoring(-1, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 0, -1, 1, None, None, 0)
    eng = Engine(0)
    lines = []
    for name in a.workloads.split(","):
        batch, k = workload(name)
        n = len(batch[2])
        cells = int((batch[2].astype(np.uint64) * batch[4].astype(np.uint64)).sum())

        def dist_call():
            return eng.levenshtein_batch(batch, k)

        def align_call():
            return eng.align_batch_scores(MODE_GLOBAL, unit, batch)

        d = dist_call()
        s = align_call()
        assert not s["status"].any()
        ref = -s["score"].astype(np.int64)
        if k is not None:
            ref = np.where(ref <= k, ref, DIST_NONE)
        equal = bool(np.array_equal(d.astype(np.int64), ref))
        rows = {"distance": [], "aligner": []}
        for r in range(a.runs):
            for path, fn in (("distance", dist_call), ("aligner", align_call)):
                t0 = time.perf_counter()
                fn()
                wall = (time.perf_counter() - t0) * 1e3
                rows[path].append({"kernel_ms": kernel_ms(eng.stats), "call_ms": wall,
                                   "launches": eng.stats.kernel_launches})
                print(json.dumps({"workload": name, "path": path, "run": r, **rows[path][-1]}), flush=True)
        summ = {"workload": name, "pairs": n, "cells": cells, "k": k, "outputs_equal": equal,
                "none": int((d == DIST_NONE).sum()) if k is not None else 0}
        for path in rows:
            km = statistics.median(x["kernel_ms"] for x in rows[path])
            summ[f"{path}_kernel_ms"] = round(km, 3)
            summ[f"{path}_call_ms"] = round(statistics.median(x["call_ms"] for x in rows[path]), 3)
            summ[f"{path}_gcups"] = round(cells / (km * 1e6), 1) if km > 0 else None
        summ["speedup_kernel"] = round(summ["aligner_kernel_ms"] / summ["distance_kernel_ms"], 2)
        print(json.dumps(summ), flush=True)
        lines.append(summ)
    eng.close()
    print(json.dumps({"card": card()}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "distance_bench.json"), "w") as f:
            json.dump({"card": card(), "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
