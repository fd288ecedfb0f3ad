"""C4 (BASELINE: banded semiglobal, 500 x 10,000 windows, k = 32, w = 32) through MultiEngine.align_batch_banded and
align_batch_banded_scores, weak scaling: 25,000 pairs per device at every device count in {1, 2, 4, 8} that is
visible.  With one visible GPU it also runs the list [0, 0]: two engines on one card, which measures the split and
exchange overhead of the multi-device path, not scaling.

Each point: 3 warm-up calls, then 5 calls timed with a host clock (the call returns host results, so it ends
synchronised); the median and every call are reported, with the per-device kernel times from the stats, GCUPS on band
cells (Band::num_cells) and the scaling efficiency against one device.  100 pairs are checked against the oracle.
Two parts of the call are also timed on their own, on device 0 with one share: the host-to-device copy of the share's
sequence bytes (from the same pageable numpy array the call reads) and the decode of one share's compact segment
into host arrays (b2a_gathered_fetch, what device 0 does once per share after the exchange).
The card and its power limit come from a read-only nvidia-smi query in the same run.

usage: python tools/multi_banded_bench.py [--per-device 25000] [--out FILE.json]
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
from rust_bio_b200._lib import MIN_SCORE, CScoring  # noqa: E402
from rust_bio_b200.engine import MultiEngine  # noqa: E402

K, W, M, N = 32, 32, 500, 10000
WARMUP, STEPS = 3, 5


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out
    except Exception as e:  # the numbers stand without it, but say so
        return [f"nvidia-smi unavailable: {e}"]


def n_visible():
    import torch
    return torch.cuda.device_count()


def run_point(ids, batch, cs, score_only):
    me = MultiEngine(ids)
    try:
        call = ((lambda: me.align_batch_banded_scores(2, cs, K, W, batch)) if score_only
                else (lambda: me.align_batch_banded(2, cs, K, W, batch)))
        for _ in range(WARMUP):
            call()
        times, stats = [], []
        for _ in range(STEPS):
            t0 = time.perf_counter()
            res = call()
            times.append((time.perf_counter() - t0) * 1e3)
            stats.append(me.stats.as_dict())
        return res, times, stats, me.exchange_kind
    finally:
        me.close()


def parts(batch, cs):
    """-> host ms of (the H2D of the share's sequence blob, the decode of one share's segment), medians of 5"""
    import torch
    from rust_bio_b200.engine import Engine, Results
    blob = batch[0]
    h2d = []
    for _ in range(WARMUP + STEPS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch.from_numpy(blob).to("cuda:0")
        torch.cuda.synchronize()
        h2d.append((time.perf_counter() - t0) * 1e3)
    eng = Engine(0)
    try:
        eng.align_batch_banded(2, cs, K, W, batch)
        nb = eng.compact_bytes()
        seg = torch.empty(nb + 256, dtype=torch.uint8, device="cuda:0")
        eng.compact_into(seg.data_ptr(), nb + 256)
        torch.cuda.synchronize()
        res = Results(len(batch[2]), Engine.default_ops_capacity(batch))
        dec = []
        for _ in range(WARMUP + STEPS):
            t0 = time.perf_counter()
            eng.gathered_fetch(seg.data_ptr(), nb + 256, 1, res)
            dec.append((time.perf_counter() - t0) * 1e3)
    finally:
        eng.close()
    return {"h2d_ms": round(statistics.median(h2d[WARMUP:]), 2), "h2d_mb": round(blob.nbytes / 1e6, 1),
            "decode_one_segment_ms": round(statistics.median(dec[WARMUP:]), 2), "segment_mb": round(nb / 1e6, 1)}


def oracle_check(batch, res, score_only, n_check=100):
    from oracle import oracle as orc
    n = len(batch[2])
    idx = np.linspace(0, n - 1, n_check).astype(int)
    blob = batch[0]
    sub = [np.ascontiguousarray(a) for a in (blob, batch[1][idx], batch[2][idx], batch[3][idx], batch[4][idx])]
    s, _ = orc.make_scoring(-5, -1, 1, -1, has_match_scores=1)
    ref = orc.banded_align_batch("semiglobal", s, K, W, *sub, threads=16, want_ops=False)[0]
    bad = 0
    for i, p in enumerate(idx):
        for f in (("score", "xend", "yend") if score_only else ("score", "xstart", "xend", "ystart", "yend")):
            got = res[f][p] if score_only else getattr(res, f)[p]
            bad += int(got) != int(ref[f][i])
    return {"pairs": n_check, "mismatched_fields": bad}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-device", type=int, default=25000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
    vis = n_visible()
    lists = [list(range(d)) for d in (1, 2, 4, 8) if d <= vis]
    if vis == 1:
        lists.append([0, 0])
    report = {"card": card(), "visible_gpus": vis, "workload": f"C4 semiglobal {M}x{N} k={K} w={W}, "
              f"{a.per_device} pairs per device entry", "points": [],
              "not_measured": [d for d in (2, 4, 8) if d > vis]}
    base = {}
    report["parts_one_share"] = parts(synth.mutated_window_pairs(synth.BASES["C4"], 0, a.per_device, M, N), cs)
    print(json.dumps({"parts_one_share": report["parts_one_share"]}), flush=True)
    for score_only in (False, True):
        for ids in lists:
            n = a.per_device * len(ids)
            batch = synth.mutated_window_pairs(synth.BASES["C4"], 0, n, M, N)
            res, times, stats, kind = run_point(ids, batch, cs, score_only)
            med = statistics.median(times)
            cells = int(stats[-1]["cells"])
            label = ("split and exchange overhead on one card, not scaling" if len(set(ids)) < len(ids)
                     else f"{len(ids)} GPU(s)")
            pt = {"devices": ids, "label": label, "score_only": score_only, "pairs": n, "exchange": kind,
                  "median_ms": round(med, 2), "calls_ms": [round(t, 2) for t in times],
                  "band_cells": cells, "gcups": round(cells / (med * 1e-3) / 1e9, 2),
                  "kernel_ms_slowest_device": {k: round(float(stats[-1][k]), 2)
                                               for k in ("band_ms", "fill_ms", "walk_ms")},
                  "h2d_mb": round(stats[-1]["h2d_bytes"] / 1e6, 1), "d2h_mb": round(stats[-1]["d2h_bytes"] / 1e6, 1),
                  "oracle": oracle_check(batch, res, score_only)}
            if ids == [0]:
                base[score_only] = med
            if score_only in base:
                pt["efficiency_vs_1"] = round(base[score_only] / med, 3)  # weak scaling: same time per call is 1.0
            report["points"].append(pt)
            print(json.dumps(pt), flush=True)
    print(json.dumps({"card": report["card"], "not_measured": report["not_measured"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
