"""Dev tool (run on the GPU): the 10k-read step by kernel, for pair counts around the task-round boundaries of
the 8x20 fill (1,184 resident warps x 4 pairs) -- min of `reps` runs of the engine's own CUDA-event timings."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rust_bio_b200 import synth
from rust_bio_b200._lib import CScoring, MIN_SCORE
from rust_bio_b200.engine import Engine, Results

ap = argparse.ArgumentParser()
ap.add_argument("--pairs", default="9472,10000")
ap.add_argument("--shapes", default="8x20")
ap.add_argument("--reps", type=int, default=7)
a = ap.parse_args()
eng = Engine(0)
cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
for n in map(int, a.pairs.split(",")):
    batch = synth.uniform_pairs(0xB2000002, 0, n, 150, 150)
    res = Results(n, Engine.default_ops_capacity(batch))
    for sh in a.shapes.split(","):
        g, r = map(int, sh.split("x"))
        eng.set_tuning(g, r)
        eng.stage(3, cs, batch)
        best = None
        for _ in range(a.reps):
            eng.run(); eng.fetch(res)
            st = eng.stats
            t = (st.pack_ms + st.fill_ms + st.walk_ms, st.pack_ms, st.fill_ms, st.walk_ms)
            if best is None or t[0] < best[0]:
                best = t
        print(json.dumps({"variant": os.environ.get("B2A_LIB_VARIANT", ""), "pairs": n, "shape": sh, "step_ms": round(best[0], 4),
                          "pack_ms": round(best[1], 4), "fill_ms": round(best[2], 4), "walk_compact_ms": round(best[3], 4),
                          "gcups": round(n * 22500 / best[0] / 1e6, 1), "score_sum": int(res.score.astype("int64").sum())}), flush=True)
