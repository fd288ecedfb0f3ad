"""Builds rust_bio_b200/csrc/libb200align.so in-tree with nvcc for sm_90a (H100).

Usage: python -m rust_bio_b200.build [--force]
The K1 fill kernel is instantiated once per (lanes-per-pair, rows-per-lane) shape in its own
translation unit so the shapes compile in parallel; everything is linked into one shared library
that exports the C ABI of include/b200align.h.  cudart is linked statically so the library loads
(and reports B2A_E_NO_DEVICE) on a machine without a GPU driver.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
VARIANT = os.environ.get("B2A_VARIANT", "")  # dev knob: a differently configured build beside the default one
OBJ = os.path.join(CSRC, "build" + (("_" + VARIANT) if VARIANT else ""))
SO = os.path.join(CSRC, "libb200align%s.so" % (("_" + VARIANT) if VARIANT else ""))
SHAPES = [(1, 16), (1, 8), (1, 20), (2, 16), (2, 20), (4, 16), (8, 16), (8, 20), (32, 8), (32, 16)]
# the shapes the engine's automatic choice picks also get the score-only (F_NOTB) fill, in translation units of their own
NOTB_SHAPES = [(1, 16), (8, 16), (8, 20), (32, 8), (32, 16)]
# the warp-per-pair shapes also get the recomputed-traceback fills (a pair above the traceback budget), in their own units
RECOMPUTE_SHAPES = [(32, 8), (32, 16)]
# minimum resident CTAs per SM asked of ptxas per shape (__launch_bounds__): measured choice, see DESIGN.md
MIN_BLOCKS = {(1, 16): int(os.environ.get("B2A_MINB_1_16", "3")), (8, 16): int(os.environ.get("B2A_MINB_8_16", "3")),
              (8, 20): int(os.environ.get("B2A_MINB_8_20", "1"))}  # 8x20 at 3 CTAs/SM (168 registers) was slower
KS_DEFS = [f"-D{k}={os.environ[k]}" for k in ("B2A_KS_R", "B2A_KS_MINB") if os.environ.get(k)]  # strip-fill geometry knobs
W_8_20 = os.environ.get("B2A_W_8_20")  # warps per CTA of the 8x20 fill (default in b2a_common.cuh)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fwrapv", "--expt-relaxed-constexpr"] + ([f"-DB2A_W_8_20={W_8_20}"] if W_8_20 else []) + KS_DEFS
HEADERS = ["b2a_common.cuh", "b2a_coop.cuh", "b2a_fill.cuh", "b2a_walk.cuh", "b2a_kernels.cuh", "b2a_plan.h", "b2a_banded.cuh", "b2a_banded_strip.cuh",
           "b2a_fill_launch.h", os.path.join("..", "..", "include", "b200align.h")]


def _stale(target: str, sources) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "flags.txt")  # objects built with other flags (another architecture) are rebuilt
    want = " ".join([NVCC, *FLAGS]) + "\n"
    if not os.path.exists(stamp):
        force = True
    else:
        with open(stamp) as f:
            force = force or f.read() != want
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    objs = []
    src = os.path.join(CSRC, "b2a_fill_inst.cu")
    for kind, shapes in (("", SHAPES), ("notb_", NOTB_SHAPES), ("recompute_", RECOMPUTE_SHAPES)):
        for g, r in shapes:
            o = os.path.join(OBJ, f"fill_{kind}{g}_{r}.o")
            objs.append(o)
            if force or _stale(o, hdrs + [src]):
                defs = {"": [], "notb_": ["-DB2A_NOTB"], "recompute_": ["-DB2A_RECOMPUTE"]}[kind]
                jobs.append([NVCC, *FLAGS, f"-DB2A_G={g}", f"-DB2A_R={r}", f"-DB2A_MINB={MIN_BLOCKS.get((g, r), 1)}",
                             *defs, "-c", src, "-o", o])
    eo = os.path.join(OBJ, "engine.o")
    objs.append(eo)
    esrc = os.path.join(CSRC, "b2a_engine.cu")
    dist_h = os.path.join(CSRC, "b2a_distance.cuh")  # engine.o, distance.o and myers.o only
    myers_h = os.path.join(CSRC, "b2a_myers.cuh")  # engine.o and myers.o only
    phmm_h = os.path.join(CSRC, "b2a_pairhmm.cuh")  # engine.o and pairhmm.o only
    if force or _stale(eo, hdrs + [esrc, dist_h, myers_h, phmm_h]):
        jobs.append([NVCC, *FLAGS, "-c", esrc, "-o", eo])
    so = os.path.join(OBJ, "banded_strip_notb.o")  # the strip fill's score-only twins, beside engine.o
    objs.append(so)
    ssrc = os.path.join(CSRC, "b2a_banded_strip_notb.cu")
    if force or _stale(so, hdrs + [ssrc]):
        jobs.append([NVCC, *FLAGS, "-c", ssrc, "-o", so])
    do = os.path.join(OBJ, "distance.o")  # the edit-distance kernels (b2a_distance.cuh: their lane logic)
    objs.append(do)
    dsrc = os.path.join(CSRC, "b2a_distance.cu")
    if force or _stale(do, hdrs + [dsrc, dist_h]):
        jobs.append([NVCC, *FLAGS, "-c", dsrc, "-o", do])
    yo = os.path.join(OBJ, "myers.o")  # the pattern-matching kernels (b2a_myers.cuh: their lane logic)
    objs.append(yo)
    ysrc = os.path.join(CSRC, "b2a_myers.cu")
    if force or _stale(yo, hdrs + [ysrc, dist_h, myers_h]):
        jobs.append([NVCC, *FLAGS, "-c", ysrc, "-o", yo])
    ho = os.path.join(OBJ, "pairhmm.o")  # the pair-HMM kernels (b2a_pairhmm.cuh: their lane logic)
    objs.append(ho)
    hsrc = os.path.join(CSRC, "b2a_pairhmm.cu")
    if force or _stale(ho, hdrs + [hsrc, phmm_h]):
        jobs.append([NVCC, *FLAGS, "-c", hsrc, "-o", ho])
    mo = os.path.join(OBJ, "multi.o")
    objs.append(mo)
    msrc = os.path.join(CSRC, "b2a_multi.cu")
    if force or _stale(mo, [msrc, os.path.join(CSRC, "..", "..", "include", "b200align.h")]):
        jobs.append([NVCC, *FLAGS, "-c", msrc, "-o", mo])
    po = os.path.join(OBJ, "peak.o")
    objs.append(po)
    psrc = os.path.join(CSRC, "b2a_peak.cu")
    if force or _stale(po, [psrc]):
        jobs.append([NVCC, *FLAGS, "-c", psrc, "-o", po])
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for log in ex.map(_run, jobs):
                if verbose and log:
                    print(log, file=sys.stderr)
    if jobs or force or _stale(SO, objs):
        _run([NVCC, "-shared", "-o", SO, *objs, *ARCH, "-ldl"])
        with open(stamp, "w") as f:
            f.write(want)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
