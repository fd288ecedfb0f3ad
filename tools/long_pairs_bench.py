"""Long pairs on one GPU: the call time and the engine's per-kernel events of full and score-only calls.

  python tools/long_pairs_bench.py [--steps 3] [--out FILE]

Inputs (random DNA, y a mutated copy of x where the lengths allow, linear match 1 / mismatch -1, gap -5 / -1):
  (i)   4 pairs of 100,000 x 100,000, global;
  (ii)  1,024 reads of 150 against 200,000-long references, semiglobal -- the automatic choice falls back to the
        warp-per-pair shape 32x8 (8x20 would stage 4 whole pairs per warp), whose one 256-row strip covers the read's
        149 fill rows (the rest of the strip is padding);
  (iii) 1 pair of 200,000 x 200,000, global.
Each call runs once to warm up and then --steps times; the median wall time, the K0 / K1 / K2 event times of the last
step, the fill shape and the waves are printed as one JSON line per (input, form), after a line with the card's name,
power limit and clocks read in the same run.  GCUPS = m * n summed over the pairs / wall time.  A single long pair keeps
only about nstrips warps busy, so it runs well below the rate of a batch of many pairs.
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


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def related(rng, m, n, rate=0.08):
    alpha = np.frombuffer(b"ACGT", np.uint8)
    x = alpha[rng.integers(0, 4, m)]
    y = alpha[rng.integers(0, 4, n)]
    k = min(m, n)
    src = x[:k].copy()
    mut = rng.random(k) < rate
    src[mut] = alpha[rng.integers(0, 4, int(mut.sum()))]
    off = (n - k) // 2
    y[off:off + k] = src
    return bytes(x), bytes(y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    from rust_bio_b200._lib import CScoring
    from rust_bio_b200.engine import Engine, pack_pairs
    rng = np.random.default_rng(1)
    cases = [
        ("4x100k^2 global", 1, [related(rng, 100000, 100000) for _ in range(4)]),
        ("1024 reads 150x200k semiglobal", 2, None),
        ("1x200k^2 global", 1, [related(rng, 200000, 200000)]),
    ]
    ref = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 200000)]
    reads = []
    for q in range(1024):  # reads from the reference, 5 % mutated, aligned against the whole of it
        off = int(rng.integers(0, 200000 - 150))
        r = ref[off:off + 150].copy()
        mut = rng.random(150) < 0.05
        r[mut] = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(mut.sum()))]
        reads.append((bytes(r), bytes(ref)))
    cases[1] = (cases[1][0], cases[1][1], reads)
    MIN = -858993459
    cs = CScoring(-5, -1, MIN, MIN, MIN, MIN, 1, -1, 0, None, None, 0)
    eng = Engine(0)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    for name, mode, pairs in cases:
        batch = pack_pairs(pairs)
        cells = int((batch[2].astype(np.uint64) * batch[4].astype(np.uint64)).sum())
        for form in ("full", "score-only"):
            call = (lambda: eng.align_batch(mode, cs, batch)) if form == "full" else \
                (lambda: eng.align_batch_scores(mode, cs, batch))
            call()
            ts = []
            for _ in range(args.steps):
                t0 = time.perf_counter()
                call()
                ts.append(time.perf_counter() - t0)
            st = eng.stats
            med = statistics.median(ts)
            rec = {"input": name, "form": form, "pairs": len(pairs), "cells": cells, "call_s_median": round(med, 4),
                   "call_s_min": round(min(ts), 4), "call_s_max": round(max(ts), 4), "gcups": round(cells / med / 1e9, 1),
                   "pack_ms": round(st.pack_ms, 2), "fill_ms": round(st.fill_ms, 2), "walk_ms": round(st.walk_ms, 2),
                   "shape": f"{st.fill_lanes_per_pair}x{st.fill_rows_per_lane}", "waves": st.waves,
                   "traceback_bytes": st.traceback_bytes}
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
