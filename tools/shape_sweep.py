"""Dev tool: time the K1 fill kernel for every built (G, R) shape on one workload (run on the GPU)."""
import argparse, json, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from rust_bio_b200 import synth
from rust_bio_b200._lib import CScoring, MIN_SCORE
from rust_bio_b200.engine import Engine, Results

ap = argparse.ArgumentParser()
ap.add_argument("--pairs", type=int, default=200000)
ap.add_argument("--m", type=int, default=150)
ap.add_argument("--n", type=int, default=150)
ap.add_argument("--mode", type=int, default=3)
ap.add_argument("--shapes", default="1x16,1x8,4x16,8x16,32x8,32x16")
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--walk", type=int, default=0)
a = ap.parse_args()
eng = Engine(0)
eng.set_walk(a.walk)
batch = synth.uniform_pairs(0xB2000002, 0, a.pairs, a.m, a.n)
cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
res = Results(a.pairs, Engine.default_ops_capacity(batch))
for sh in a.shapes.split(","):
    g, r = map(int, sh.split("x"))
    eng.set_tuning(g, r)
    try:
        eng.stage(a.mode, cs, batch)
        best = None
        for _ in range(a.reps):
            eng.run(); eng.fetch(res)
            st = eng.stats
            if best is None or st.fill_ms < best[0]:
                best = (st.fill_ms, st.walk_ms, st.pack_ms)
        gc = st.cells / best[0] / 1e6
        print(json.dumps({"pairs": a.pairs, "walk": a.walk, "shape": sh, "fill_ms": round(best[0], 3), "walk_ms": round(best[1], 3), "pack_ms": round(best[2], 3),
                          "fill_gcups": round(gc, 1), "total_gcups": round(st.cells / sum(best) / 1e6, 1), "tb_MB": st.traceback_bytes >> 20}), flush=True)
    except Exception as ex:
        print(json.dumps({"pairs": a.pairs, "walk": a.walk, "shape": sh, "error": str(ex)}), flush=True)
