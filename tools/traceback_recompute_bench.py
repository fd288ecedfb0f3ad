"""Recomputed traceback on one GPU: call time, pass-1 time, refill + walk time and windows of full calls on pairs whose
traceback is refilled one window of strips at a time (b2a_engine_set_traceback_recompute).

  python tools/traceback_recompute_bench.py [--steps 3] [--out FILE]

Inputs (random DNA, y a mutated copy of x, linear match 1 / mismatch -1, gap -5 / -1):
  (i)   1 pair of 100,000 x 100,000 global at the default budget (one window: today's path), and under budgets giving
        about 4 and about 16 windows;
  (ii)  1 pair of 100,000 x 100,000 local whose only hit lies in the last fifth of x, about 16 windows;
  (iii) 1 pair of 330,000 x 330,000 global at the default budget (its traceback is above it), and its score-only call.
Each call runs once to warm up and then --steps times; the median wall time, the last step's engine events (fill_ms:
pass 1 of a recomputed pair, else the fill; walk_ms: the refills and the walk segments, else K2) and the windows are
printed as one JSON line per case, after a line with the card's name, power limit and clocks read in the same run.
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
    y[(n - k) // 2:(n - k) // 2 + k] = src
    return bytes(x), bytes(y)


def strip_bytes(n, R=16):
    return (n + 32 - 1 + 7) // 8 * ((R + 3) // 4) * 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    from rust_bio_b200._lib import CScoring
    from rust_bio_b200.engine import Engine, pack_pairs
    MIN = -858993459
    rng = np.random.default_rng(1)
    g100 = pack_pairs([related(rng, 100000, 100000)])
    alpha = np.frombuffer(b"ACGT", np.uint8)
    x = alpha[rng.integers(0, 4, 100000)]
    y = alpha[rng.integers(0, 4, 100000)]
    y[40000:52000] = x[85000:97000]  # the hit: rows 85,000..97,000
    l100 = pack_pairs([(bytes(x), bytes(y))])
    g330 = pack_pairs([related(rng, 330000, 330000)])
    nst = (100000 - 1 + 511) // 512
    sb = strip_bytes(100000)
    per = lambda nw: ((nst + nw - 1) // nw) * sb + sb // 3
    cases = [
        ("1x100k^2 global, default budget", 1, g100, 0, "full"),
        ("1x100k^2 global, ~4 windows", 1, g100, per(4), "full"),
        ("1x100k^2 global, ~16 windows", 1, g100, per(16), "full"),
        ("1x100k^2 local, hit in the last fifth, ~16 windows", 3, l100, per(16), "full"),
        ("1x330k^2 global, default budget", 1, g330, 0, "full"),
        ("1x330k^2 global", 1, g330, 0, "score-only"),
    ]
    eng = Engine(0)
    eng.set_traceback_recompute(True)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    for name, mode, batch, budget, form in cases:
        cs = CScoring(-5, -1, MIN, MIN, MIN, MIN, 1, -1, 0, None, None, 0)
        eng.set_traceback_budget(budget)
        call = (lambda: eng.align_batch(mode, cs, batch)) if form == "full" else \
            (lambda: eng.align_batch_scores(mode, cs, batch))
        call()
        ts = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            call()
            ts.append(time.perf_counter() - t0)
        st = eng.stats
        rc = eng.last_recompute() if form == "full" else {}
        rec = {"input": name, "form": form, "budget": budget, "call_s_median": round(statistics.median(ts), 4),
               "call_s_min": round(min(ts), 4), "call_s_max": round(max(ts), 4), "fill_ms": round(st.fill_ms, 2),
               "walk_ms": round(st.walk_ms, 2), "shape": f"{st.fill_lanes_per_pair}x{st.fill_rows_per_lane}", **rc}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    eng.set_traceback_budget(0)
    eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
