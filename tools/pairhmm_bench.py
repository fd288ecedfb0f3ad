"""Pair-HMM likelihoods (b2a_pairhmm_batch, PairHMM::prob_related) on the GPU, against the oracle on the host.

For each workload, one warm-up call and then `--runs` calls.  Kernel ms is the engine's event-timed kernels
(stats.fill_ms), whole-call ms a host clock around the call (upload, kernels, copy back, statuses); GCUPS is
sum(len_x * len_y) over the median kernel time.  The oracle (tests/sim/pairhmm_oracle.cpp, the literal restatement of
the reference) runs a seeded subsample on every host thread the process may use (affinity mask capped by the cgroup
quota, as bench.py counts them); its rate and its results on the subsample are reported beside the GPU's: the largest
|gpu - oracle|, the share of bit-identical results, and the pairs where exactly one side is -inf (expected: none).  The
card's name, power limit and maximum SM clock are read in the same call.  There is no other GPU number for this DP to
compare with: the reference is CPU-only.

  python tools/pairhmm_bench.py [--workloads reads200,reads200_band4,quality400,long10k] [--runs 3] [--out DIR]

Workloads (synthetic, seeded; x is the window, y the read, as in the reference's bench):
  reads200        1,000,000 x 150-nt reads in 200-nt windows (5,000 windows), 1 % substitutions, semiglobal, the
                  Illumina constants of the reference's bench (benches/pairhmm.rs:15-19), max_edit_dist None
  reads200_band4  the same with max_edit_dist Some(4), the reference bench's band
  quality400      100,000 x 150-nt reads in 400-nt windows, per-base Phred classes 2..41 on the reads, gap opens
                  1e-3 / 2e-3 and extensions 0.1 / 0.2, semiglobal, None
  long10k         200 x 10,000 x 10,000 global pairs, 1 % substitutions, Illumina constants, None
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rust_bio_b200.engine import Engine  # noqa: E402

DNA = np.frombuffer(b"ACGT", dtype=np.uint8)


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"


def windows_and_reads(rng, n_reads, n_win, win_len, read_len, sub):
    """(blob, x_off, x_len, y_off, y_len): the windows stored once, then every read (a substituted copy of a random
    stretch of its window)"""
    wins = DNA[rng.integers(0, 4, (n_win, win_len))]
    w = rng.integers(0, n_win, n_reads)
    st = rng.integers(0, win_len - read_len + 1, n_reads)
    reads = wins[w[:, None], st[:, None] + np.arange(read_len)]
    s = rng.random(reads.shape) < sub
    reads[s] = DNA[rng.integers(0, 4, int(s.sum()))]
    blob = np.concatenate([wins.reshape(-1), reads.reshape(-1), np.zeros(16, np.uint8)])
    x_off = (w * win_len).astype(np.uint64)
    y_off = (n_win * win_len + np.arange(n_reads, dtype=np.uint64) * read_len).astype(np.uint64)
    return (blob, x_off, np.full(n_reads, win_len, np.uint32), y_off, np.full(n_reads, read_len, np.uint32))


def long_pairs(rng, n, length, sub):
    xs = DNA[rng.integers(0, 4, (n, length))]
    ys = xs.copy()
    s = rng.random(ys.shape) < sub
    ys[s] = DNA[rng.integers(0, 4, int(s.sum()))]
    blob = np.concatenate([xs.reshape(-1), ys.reshape(-1), np.zeros(16, np.uint8)])
    off = np.arange(n, dtype=np.uint64) * length
    ln = np.full(n, length, np.uint32)
    return blob, off, ln, off + np.uint64(n * length), ln


def illumina():
    ins, dele, subst = 2.8e-6, 5.1e-6, 0.0021
    gap = (math.log(ins), math.log(dele), -math.inf, -math.inf)
    emit = [[math.log(1 - subst)], [math.log(subst / 3)], [math.log(1 - subst)], [math.log(1 - subst)]]
    return gap, emit


def workload(name, rng):
    """-> (batch, classes or None, gap, emit, free_start, free_end, max_edit_dist, oracle sample size)"""
    if name in ("reads200", "reads200_band4"):
        gap, emit = illumina()
        b = windows_and_reads(rng, 1_000_000, 5000, 200, 150, 0.01)
        return b, None, gap, emit, True, True, (4 if name.endswith("band4") else None), 4000
    if name == "quality400":
        b = windows_and_reads(rng, 100_000, 1000, 400, 150, 0.01)
        cls = np.full(b[0].nbytes, 40, np.uint8)
        nw = 1000 * 400
        cls[nw:nw + 100_000 * 150] = rng.integers(2, 42, 100_000 * 150)
        emit = [[], [], [], []]
        for q in range(42):
            e = 10 ** (-max(q, 2) / 10)
            for k, v in enumerate((math.log(1 - e), math.log(e / 3), math.log(1 - e), math.log(1 - e))):
                emit[k].append(v)
        gap = (math.log(1e-3), math.log(2e-3), math.log(0.1), math.log(0.2))
        return b, cls, gap, emit, True, True, None, 2000
    if name == "long10k":
        gap, emit = illumina()
        return long_pairs(rng, 200, 10_000, 0.01), None, gap, emit, False, False, None, 0
    raise SystemExit(f"unknown workload {name}")


def oracle_sample(batch, cls, gap, emit, fs, fe, med, idx, threads):
    import pairhmm_util as pu
    blob, xo, xl, yo, yl = batch
    sub = (blob, cls, xo[idx], xl[idx], yo[idx], yl[idx])
    t = time.perf_counter()
    out = pu.orc_batch(gap, (int(fs), int(fe)), med, emit, sub, threads=threads)
    return out, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="reads200,reads200_band4,quality400,long10k")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    from oracle import oracle as orc
    threads = orc.hardware_threads()
    print(json.dumps({"card": card(), "host_threads": threads}), flush=True)
    eng = Engine(0)
    lines = []
    for name in args.workloads.split(","):
        rng = np.random.default_rng(args.seed)
        batch, cls, gap, emit, fs, fe, med, n_sample = workload(name, rng)
        cells = int((batch[2].astype(np.uint64) * batch[4].astype(np.uint64)).sum())
        kern, wall = [], []
        for r in range(args.runs + 1):
            t = time.perf_counter()
            prob, st = eng.pairhmm_batch(batch, gap, emit, fs, fe, med, cls)
            dt = time.perf_counter() - t
            if r:
                kern.append(eng.stats.fill_ms)
                wall.append(dt * 1e3)
        tiers = eng.pairhmm_tier_pairs()
        n = len(batch[2])
        if n_sample == 0:  # the long pairs: one per thread
            n_sample = min(n, threads)
        idx = np.sort(np.random.default_rng(args.seed + 1).choice(n, min(n, n_sample), replace=False))
        want, t_orc = oracle_sample(batch, cls, gap, emit, fs, fe, med, idx, threads)
        got = prob[idx]
        both = np.isfinite(got) & np.isfinite(want)
        one_inf = int(np.sum(np.isinf(got) != np.isinf(want)))
        same = float(np.mean(got.view(np.uint64) == want.view(np.uint64)))
        dmax = float(np.max(np.abs(got[both] - want[both]))) if both.any() else 0.0
        s_cells = int((batch[2][idx].astype(np.uint64) * batch[4][idx].astype(np.uint64)).sum())
        km = statistics.median(kern)
        row = {"workload": name, "pairs": n, "cells": cells, "kernel_ms": round(km, 3),
               "kernel_ms_runs": [round(v, 3) for v in kern], "gcups": round(cells / (km * 1e-3) / 1e9, 2),
               "call_ms": round(statistics.median(wall), 2), "tiers": tiers, "panics": int(np.count_nonzero(st)),
               "oracle": {"pairs": len(idx), "threads": threads, "gcups": round(s_cells / t_orc / 1e9, 4)},
               "sample": {"max_abs_diff": dmax, "bit_identical": round(same, 5), "inf_mismatch": one_inf}}
        lines.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": card()}), flush=True)
    eng.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pairhmm_bench.json"), "w") as f:
            json.dump({"card": card(), "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
