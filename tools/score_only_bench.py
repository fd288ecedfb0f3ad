"""Full vs score-only batches on one GPU (b2a_batch_stage vs b2a_batch_stage_scores), run on the GPU.

Each configuration is staged once per path (two engines, inputs resident in HBM); then the two paths are timed in
alternation, `--runs` times each: 3 warm-up steps of b2a_batch_run, then 10 timed steps, each between two CUDA
events on the engine's stream; a run reports the median step.  fill_ms, walk_ms (K2 + ops compaction) and waves are
the engine's stats of the run's last step.  Before any timing the score-only outputs (score, xend, yend, status) are
checked against the full path's.  The card's name, power limit and maximum SM clock are read in the same call.

  python tools/score_only_bench.py [--configs C2,C2_10k,C3,C5] [--runs 3] [--out DIR]

Configurations (synthetic, rust_bio_b200/synth.py):
  C2      1,000,000 x 150 x 150 DNA, local, MatchParams(1, -1), gap -5 / -1 (bench.py's flagship)
  C2_10k  10,000 pairs of the same
  C3      100,000 x 1000 x 1000 DNA, global, same scoring
  C5      1,250 x 10,000 x 10,000 protein, local, BLOSUM62, gap -11 / -1 (C5's shape)
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rust_bio_b200 import scores, synth  # noqa: E402
from rust_bio_b200._lib import MIN_SCORE, MODE_GLOBAL, MODE_LOCAL, CScoring  # noqa: E402
from rust_bio_b200.engine import Engine, ScoreResults  # noqa: E402

WARM, STEPS = 3, 10


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"


def config(name):
    """-> (batch, mode, CScoring, keepalive)"""
    dna = lambda: CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
    if name == "C2":
        return synth.uniform_pairs(synth.BASES["C2"], 0, 1_000_000, 150, 150), MODE_LOCAL, dna(), None
    if name == "C2_10k":
        return synth.uniform_pairs(synth.BASES["C2"], 0, 10_000, 150, 150), MODE_LOCAL, dna(), None
    if name == "C3":
        return synth.uniform_pairs(synth.BASES["C3"], 0, 100_000, 1000, 1000), MODE_GLOBAL, dna(), None
    if name == "C5":
        table = np.ascontiguousarray(scores.matrix_table256("blosum62"), dtype=np.int32)
        alpha = np.frombuffer(bytes(range(65, 91)) + b"*", dtype=np.uint8).copy()
        cs = CScoring(-11, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 0, 0, 0, None, None, 0)
        cs.table, cs.alphabet, cs.alphabet_len = table.ctypes.data, alpha.ctypes.data, len(alpha)
        batch = synth.uniform_pairs(synth.BASES["C5"], 0, 1250, 10000, 10000, alphabet=synth.PROTEIN)
        return batch, MODE_LOCAL, cs, (table, alpha)
    raise ValueError(name)


def fetch(eng, n):
    res = ScoreResults(n)  # (the full path's fetch takes the same NULL fields: no ops are copied back)
    eng._check(eng._L.b2a_batch_fetch(eng._h, C.byref(res.c), C.byref(eng.stats)))
    return res.as_dict()


def timed_run(torch, eng, stream):
    for _ in range(WARM):
        eng.run()
    times = []
    for _ in range(STEPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        eng.run()
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C2_10k,C3,C5")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    print(json.dumps({"card": card()}), flush=True)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    lines = []
    for name in a.configs.split(","):
        batch, mode, cs, keep = config(name)
        n = len(batch[2])
        engs = {}
        for path in ("full", "scores"):
            e = Engine(0)
            e.set_stream(stream.cuda_stream)
            (e.stage if path == "full" else e.stage_scores)(mode, cs, batch)
            engs[path] = e
        out = {}
        for path, e in engs.items():  # outputs first
            e.run()
            out[path] = fetch(e, n)
        same = {f: bool(np.array_equal(out["full"][f], out["scores"][f])) for f in ("score", "xend", "yend", "status")}
        rows = {"full": [], "scores": []}
        for k in range(a.runs):
            for path, e in engs.items():
                ms = timed_run(torch, e, stream)
                fetch(e, n)
                st = e.stats
                rows[path].append({"step_ms": round(ms, 3), "fill_ms": round(st.fill_ms, 3), "walk_ms": round(st.walk_ms, 3),
                                   "waves": st.waves, "traceback_bytes": st.traceback_bytes,
                                   "shape": f"{st.fill_lanes_per_pair}x{st.fill_rows_per_lane}"})
                print(json.dumps({"config": name, "path": path, "run": k, **rows[path][-1]}), flush=True)
        summ = {"config": name, "pairs": n, "outputs_equal": same}
        for path in rows:
            for f in ("step_ms", "fill_ms", "walk_ms"):
                v = [r[f] for r in rows[path]]
                summ[f"{path}_{f}"] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
            summ[f"{path}_waves"] = rows[path][-1]["waves"]
        summ["speedup_step"] = round(summ["full_step_ms"]["median"] / summ["scores_step_ms"]["median"], 3)
        print(json.dumps(summ), flush=True)
        lines.append(summ)
        for e in engs.values():
            e.close()
    print(json.dumps({"card": card()}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "score_only_bench.json"), "w") as f:
            json.dump({"card": card(), "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
