"""Dev/measurement tool: run BASELINE configs C2..C5 (or a scaled-down number of pairs) on one GPU and
report kernel times / GCUPS per config (run on the GPU; prints one JSON line per config)."""
import argparse, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
from rust_bio_b200 import synth, scores
from rust_bio_b200._lib import CScoring, MIN_SCORE
from rust_bio_b200.engine import Engine, Results

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="C3,C4,C5")
ap.add_argument("--c3-pairs", type=int, default=20000)
ap.add_argument("--c4-pairs", type=int, default=20000)
ap.add_argument("--c5-pairs", type=int, default=64)
ap.add_argument("--shapes", default="")
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--walk", type=int, default=0)
a = ap.parse_args()
eng = Engine(0)
eng.set_walk(a.walk)
import ctypes as C


def run_full(name, mode, cs, batch, keep=None):
    res = Results(len(batch[2]), 16)  # ops not fetched (capacity checked only when ops are requested)
    res.c.ops = None
    shapes = [tuple(map(int, s.split("x"))) for s in a.shapes.split(",") if s] or [(0, 0)]
    for g, r in shapes:
        eng.set_tuning(g, r)
        try:
            t0 = time.perf_counter()
            eng.stage(mode, cs, batch)
            best = None
            for _ in range(a.reps):
                eng.run(); eng.fetch(res)
                st = eng.stats
                if best is None or st.fill_ms < best["fill_ms"]:
                    best = dict(fill_ms=st.fill_ms, walk_ms=st.walk_ms, pack_ms=st.pack_ms)
            tot = best["fill_ms"] + best["walk_ms"] + best["pack_ms"]
            print(json.dumps({"config": name, "walk": a.walk, "pairs": len(batch[2]), "G": st.fill_lanes_per_pair, "R": st.fill_rows_per_lane,
                              "waves": st.waves, **{k: round(v, 3) for k, v in best.items()},
                              "fill_gcups": round(st.cells / best["fill_ms"] / 1e6, 1),
                              "step_gcups": round(st.cells / tot / 1e6, 1), "tb_GB": round(st.traceback_bytes / 2**30, 2),
                              "wall_s": round(time.perf_counter() - t0, 2)}), flush=True)
        except Exception as ex:
            print(json.dumps({"config": name, "G": g, "R": r, "error": str(ex)}), flush=True)
    eng.set_tuning(0, 0)


for cfg in a.configs.split(","):
    if cfg == "C3":
        batch = synth.uniform_pairs(synth.BASES["C3"], 0, a.c3_pairs, 1000, 1000)
        cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
        run_full("C3 global 1000x1000", 1, cs, batch)
    elif cfg == "C5":
        batch = synth.uniform_pairs(synth.BASES["C5"], 0, a.c5_pairs, 10000, 10000, alphabet=synth.PROTEIN)
        table = np.ascontiguousarray(scores.matrix_table256("blosum62"))
        alpha = np.frombuffer(bytes(range(65, 91)) + b"*", dtype=np.uint8).copy()
        cs = CScoring(-10, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 0, 0, 0, table.ctypes.data_as(C.c_void_p),
                      alpha.ctypes.data_as(C.c_void_p), len(alpha))
        run_full("C5 local protein 10000x10000 blosum62", 3, cs, batch)
    elif cfg == "C4":
        batch = synth.mutated_window_pairs(synth.BASES["C4"], 0, a.c4_pairs, 500, 10000)  # the named generator
        cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
        res = Results(len(batch[2]), 16); res.c.ops = None
        for _ in range(a.reps):
            t1 = time.perf_counter()
            eng.align_batch_banded(2, cs, 32, 32, batch, results=res)
            wall = time.perf_counter() - t1
            st = eng.stats
        print(json.dumps({"config": "C4 banded semiglobal 500x10000 k=32 w=32", "pairs": len(batch[2]), "band_cells": int(st.cells),
                          "band_ms": round(st.band_ms, 2), "fill_ms": round(st.fill_ms, 2), "wall_s": round(wall, 3),
                          "band_gcups": round(st.cells / (st.band_ms + st.fill_ms) / 1e6, 2),
                          "mn_equiv_gcups": round(len(batch[2]) * 500 * 10000 / (st.band_ms + st.fill_ms) / 1e6, 1)}), flush=True)
