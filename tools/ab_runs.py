"""Dev tool: A/B runs of two library builds on one GPU, alternated run by run (run on the GPU).

The libraries are told apart by B2A_LIB_VARIANT (rust_bio_b200/_lib.py): "" is the default build,
"<name>" is csrc/libb200align_<name>.so (python -m rust_bio_b200.build with B2A_VARIANT=<name>).

  python tools/ab_runs.py sweep --variants parent, --out DIR   # tools/shape_sweep.py per variant
  python tools/ab_runs.py bench --variants parent, --runs 3 --out DIR [--dump]

`bench` runs `bench.py --gpus 1 --no-cpu-baseline` (A B A B ...), keeps every JSON line and prints the
median / min / max of the flagship value and of the C2 kernel times per variant; with --dump the last run of
each variant also writes its outputs (bench.py --dump-outputs) and the .npy files are compared one by one.
The card name, power limit and clocks are read in the same command and printed first.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def run(variant, args, log):
    env = dict(os.environ, B2A_LIB_VARIANT=variant)
    r = subprocess.run([sys.executable, *args], cwd=ROOT, env=env, capture_output=True, text=True)
    tag = variant or "default"
    with open(log, "a") as f:
        f.write(f"### {tag}: {' '.join(args)} (rc {r.returncode})\n{r.stdout}\n{r.stderr[-4000:]}\n")
    if r.returncode != 0:
        print(f"[{tag}] rc {r.returncode}\n{r.stderr[-2000:]}", flush=True)
    return [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{")]


def spread(vals):
    return {"median": round(statistics.median(vals), 4), "min": round(min(vals), 4), "max": round(max(vals), 4),
            "n": len(vals)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["sweep", "bench"])
    ap.add_argument("--variants", default="parent,", help="comma separated B2A_LIB_VARIANT values ('' = default)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--shapes", default="1x16,2x16,1x20")
    ap.add_argument("--dump", action="store_true")
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    log = os.path.join(a.out, f"{a.what}.log")
    variants = a.variants.split(",")
    print("card:", card(), flush=True)
    res = {v: [] for v in variants}
    for k in range(a.runs):
        for v in variants:
            if a.what == "sweep":
                lines = run(v, ["tools/shape_sweep.py", "--pairs", str(a.pairs), "--shapes", a.shapes], log)
            else:
                args = ["bench.py", "--gpus", "1", "--no-cpu-baseline"]
                if a.dump and k == a.runs - 1:
                    args += ["--dump-outputs", os.path.join(a.out, "dump_" + (v or "default"))]
                lines = run(v, args, log)
            for l in lines:
                print(json.dumps({"variant": v or "default", "run": k, **l}), flush=True)
            res[v].extend((k, l) for l in lines)
    print("card:", card(), flush=True)
    summary = {}
    for v in variants:
        if a.what == "sweep":
            for sh in a.shapes.split(","):
                rows = [l for _, l in res[v] if l.get("shape") == sh and "fill_ms" in l]
                if rows:
                    summary[f"{v or 'default'} {sh}"] = {"fill_ms": spread([r["fill_ms"] for r in rows]),
                                                        "walk_ms": spread([r["walk_ms"] for r in rows])}
        else:
            rows = [l for _, l in res[v] if "kernel_ms" in l and "value" in l and isinstance(l["kernel_ms"], dict)
                    and "fill" in l["kernel_ms"]]
            if rows:
                s = {"value": spread([r["value"] for r in rows]),
                     "fill_ms": spread([r["kernel_ms"]["fill"] for r in rows]),
                     "walk_and_compact_ms": spread([r["kernel_ms"]["walk_and_compact"] for r in rows])}
                for name in sorted({c["name"] for r in rows for c in r.get("configs", [])}):
                    cs = [c for r in rows for c in r.get("configs", []) if c["name"] == name and "ms_per_step" in c]
                    s[name + "_ms_per_step"] = spread([c["ms_per_step"] for c in cs])
                    s[name + "_parity_ok"] = all((c.get("parity_sample") or {}).get("ok", False) for c in cs)
                summary[v or "default"] = s
    print(json.dumps({"summary": summary}), flush=True)
    if a.what == "bench" and a.dump and len(variants) == 2:
        import numpy as np
        d0, d1 = (os.path.join(a.out, "dump_" + (v or "default")) for v in variants)
        names = sorted(set(os.listdir(d0)) | set(os.listdir(d1))) if os.path.isdir(d0) and os.path.isdir(d1) else []
        diff = [n for n in names if not (os.path.exists(os.path.join(d0, n)) and os.path.exists(os.path.join(d1, n))
                                         and np.array_equal(np.load(os.path.join(d0, n)), np.load(os.path.join(d1, n))))]
        print(json.dumps({"dump_files": len(names), "dump_differ": diff}), flush=True)


if __name__ == "__main__":
    main()
