"""Full vs score-only banded batches on one GPU (b2a_align_batch_banded vs b2a_align_batch_banded_scores), run on the GPU.

Each configuration is run on one engine, the two calls alternating: 2 warm-up calls of each, then `--runs` runs of each,
a run being the median of `--calls` calls.  A call is timed on the host around the whole call (it ends in a stream
synchronise: the uploads, K4, K3 and, for the full call, the ops compaction and the ops copy back).  band_ms (K4),
fill_ms (K3 / K3s, the walk included) and walk_ms (the ops compaction after K3) are the engine's stats of the run's
last call.  Before any timing the score-only outputs (score, xend, yend, status) are checked against the full call's,
and the strip-path pair counts of both calls are compared.  The card's name, power limit and maximum SM clock are read
in the same call.

  python tools/banded_score_only_bench.py [--configs C4,C4_short] [--runs 3] [--calls 5] [--out DIR]

Configurations (synthetic, rust_bio_b200/synth.py mutated_window_pairs, semiglobal, MatchParams(1, -1), gap -5 / -1):
  C4        200,000 reads of 500 against 10,000-long references, k = 32, w = 32 (the banded flagship)
  C4_short  400,000 reads of 150 against 600-long references, k = 16, w = 16: bands of a few dozen rows, nearly every
            pair on the strip path, so the K3 share of the call is larger than at C4
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
from rust_bio_b200._lib import MIN_SCORE, MODE_SEMIGLOBAL, CScoring  # noqa: E402
from rust_bio_b200.engine import Engine, Results  # noqa: E402

WARM = 2
CONFIGS = {"C4": (200_000, 500, 10_000, 32, 32), "C4_short": (400_000, 150, 600, 16, 16)}


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C4,C4_short")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
    lines = []
    eng = Engine(0)
    for name in a.configs.split(","):
        n, xl, yl, k, w = CONFIGS[name]
        batch = synth.mutated_window_pairs(synth.BASES["C4"], 0, n, xl, yl)
        res = Results(n, Engine.default_ops_capacity(batch), pair_status=True)

        def full():
            eng.align_batch_banded(MODE_SEMIGLOBAL, cs, k, w, batch, results=res)

        def scores():
            return eng.align_batch_banded_scores(MODE_SEMIGLOBAL, cs, k, w, batch)

        calls = {"full": full, "scores": scores}
        full()
        strip_full = eng.banded_strip_pairs()
        got = scores()
        strip_scores = eng.banded_strip_pairs()
        same = {f: bool(np.array_equal(getattr(res, f)[:n], got[f])) for f in ("score", "xend", "yend", "status")}
        for _ in range(WARM - 1):
            for fn in calls.values():
                fn()
        rows = {"full": [], "scores": []}
        for r in range(a.runs):
            for path, fn in calls.items():
                ts = []
                for _ in range(a.calls):
                    t0 = time.perf_counter()
                    fn()
                    ts.append((time.perf_counter() - t0) * 1e3)
                st = eng.stats
                rows[path].append({"call_ms": round(statistics.median(ts), 3), "band_ms": round(st.band_ms, 3),
                                   "fill_ms": round(st.fill_ms, 3), "walk_ms": round(st.walk_ms, 3)})
                print(json.dumps({"config": name, "path": path, "run": r, **rows[path][-1]}), flush=True)
        summ = {"config": name, "pairs": n, "outputs_equal": same, "strip_pairs": [strip_full, strip_scores]}
        for path in rows:
            for f in ("call_ms", "band_ms", "fill_ms", "walk_ms"):
                v = [x[f] for x in rows[path]]
                summ[f"{path}_{f}"] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
        summ["speedup_call"] = round(summ["full_call_ms"]["median"] / summ["scores_call_ms"]["median"], 3)
        print(json.dumps(summ), flush=True)
        lines.append(summ)
        del batch, res
    eng.close()
    print(json.dumps({"card": card()}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "banded_score_only_bench.json"), "w") as f:
            json.dump({"card": card(), "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
