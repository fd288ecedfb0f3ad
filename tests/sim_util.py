"""ctypes driver for tests/sim/libb2asim.so: the GPU kernels' per-lane logic compiled for the host
(thread-per-pair shape lane after lane; the G > 1 fill shapes and the W = 32 banded kernels on 32 cooperatively
scheduled contexts standing in for a warp).  A test tool for the not-gpu suite; the product never loads it."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "sim", "b2a_sim.cpp")
_KS_R = os.environ.get("B2A_SIM_KS_R", "")  # dev knob: the strip fill's rows per lane in the host build
_KREL = os.environ.get("B2A_SIM_KREL_BITS", "")  # test knob: column-chunk length (log2) of the relative packed trackers
SO = os.path.join(HERE, "sim", "libb2asim%s%s.so" % ((("_r" + _KS_R) if _KS_R else ""), (("_k" + _KREL) if _KREL else "")))
DEPS = [SRC] + [os.path.join(ROOT, "rust_bio_b200", "csrc", f)
                for f in ("b2a_common.cuh", "b2a_coop.cuh", "b2a_fill.cuh", "b2a_walk.cuh", "b2a_plan.h", "b2a_banded.cuh", "b2a_banded_strip.cuh")]


class SimScoring(C.Structure):
    _fields_ = [("gap_open", C.c_int32), ("gap_extend", C.c_int32), ("xclip_prefix", C.c_int32),
                ("xclip_suffix", C.c_int32), ("yclip_prefix", C.c_int32), ("yclip_suffix", C.c_int32),
                ("match_score", C.c_int32), ("mismatch_score", C.c_int32),
                ("has_match_scores", C.c_int32), ("table", C.POINTER(C.c_int32)),
                ("alphabet", C.c_void_p), ("alphabet_len", C.c_uint32)]


def build():
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in DEPS):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fwrapv", "-fPIC", "-shared",
                               "-Wno-unknown-pragmas"] + ([f"-DB2A_KS_R={_KS_R}"] if _KS_R else []) +
                              ([f"-DB2A_KREL_BITS={_KREL}"] if _KREL else []) + ["-o", SO, SRC])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.sim_align_batch.restype = C.c_int
    return _lib


def align_batch(mode, orc_scoring, blob, x_off, x_len, y_off, y_len, R=16, force_general=0, garbage=None, no_pack=0, no_lut=0, G=1, warp_walk=0, rel_pack=0):
    """Takes an oracle.OrcScoring (same layout). Returns dict of arrays + list of op lists."""
    s = SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    x_off = np.ascontiguousarray(x_off, dtype=np.uint64)
    y_off = np.ascontiguousarray(y_off, dtype=np.uint64)
    x_len = np.ascontiguousarray(x_len, dtype=np.uint32)
    y_len = np.ascontiguousarray(y_len, dtype=np.uint32)
    n = len(x_len)
    cap = x_len.astype(np.uint64) + y_len.astype(np.uint64) + np.uint64(4)
    ops_off = np.concatenate([[0], np.cumsum(cap)]).astype(np.uint64)
    ops = np.zeros(int(ops_off[-1]), dtype=np.uint8)
    out = {k: np.zeros(n, dtype=np.uint32) for k in ("xstart", "xend", "ystart", "yend", "n_ops", "status")}
    out["score"] = np.zeros(n, dtype=np.int32)
    out["clip_len"] = np.zeros(4 * n, dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    if garbage is None:  # run with two different scratch fills and insist on identical results
        a = align_batch(mode, orc_scoring, blob, x_off, x_len, y_off, y_len, R, force_general, 0x00, no_pack, no_lut, G, warp_walk, rel_pack)
        b = align_batch(mode, orc_scoring, blob, x_off, x_len, y_off, y_len, R, force_general, 0x7F, no_pack, no_lut, G, warp_walk, rel_pack)
        for k in a[0]:
            assert np.array_equal(a[0][k], b[0][k]), ("scratch-dependent result", k)
        assert a[1] == b[1], "scratch-dependent ops"
        return a
    rc = lib().sim_align_batch_g(int(mode), C.byref(s), p(blob), p(x_off), p(x_len), p(y_off), p(y_len),
                               C.c_uint64(n), int(G), int(R), int(force_general) | (2 if no_pack else 0) | (4 if no_lut else 0) | (8 if warp_walk else 0) | (16 if rel_pack else 0), int(garbage), p(out["score"]),
                               p(out["xstart"]), p(out["xend"]), p(out["ystart"]), p(out["yend"]),
                               p(out["n_ops"]), p(out["clip_len"]), p(out["status"]), p(ops), p(ops_off))
    assert rc == 0
    oplists = []
    for i in range(n):
        codes = ops[int(ops_off[i]):int(ops_off[i]) + int(out["n_ops"][i])]
        oplists.append(decode_ops(codes, out["clip_len"][4 * i:4 * i + 4]))
    return out, oplists


def decode_ops(codes, clips):
    """uint8 op codes + clip_len[4] -> [(code, len)] like the oracle wrapper returns."""
    res, k = [], 0
    for c in codes:
        c = int(c)
        if c >= 4:
            res.append((c, int(clips[k])))
            k += 1
        else:
            res.append((c, 0))
    return res


def banded_batch(mode, orc_scoring, k, w, blob, x_off, x_len, y_off, y_len, cap_matches=4096, want_ranges=False):
    """K4 + K3 device functions (b2a_banded.cuh) compiled for the host; two scratch fills must agree."""
    s = SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    x_off = np.ascontiguousarray(x_off, dtype=np.uint64)
    y_off = np.ascontiguousarray(y_off, dtype=np.uint64)
    x_len = np.ascontiguousarray(x_len, dtype=np.uint32)
    y_len = np.ascontiguousarray(y_len, dtype=np.uint32)
    n = len(x_len)
    cap = x_len.astype(np.uint64) + y_len.astype(np.uint64) + np.uint64(8)
    ops_off = np.concatenate([[0], np.cumsum(cap)]).astype(np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    results = []
    for garbage in (0x00, 0x7F):
        ops = np.zeros(int(ops_off[-1]), dtype=np.uint8)
        out = {k_: np.zeros(n, dtype=np.uint32) for k_ in ("xstart", "xend", "ystart", "yend", "n_ops", "status")}
        out["score"] = np.zeros(n, dtype=np.int32)
        out["clip_len"] = np.zeros(4 * n, dtype=np.uint32)
        out["num_cells"] = np.zeros(n, dtype=np.uint64)
        rng = np.zeros(int(2 * (y_len.astype(np.uint64) + 1).sum()), dtype=np.uint64) if want_ranges else None
        L = lib()
        L.sim_banded_batch.restype = C.c_int
        rc = L.sim_banded_batch(int(mode), C.byref(s), C.c_uint32(k), C.c_uint32(w), p(blob), p(x_off), p(x_len),
                                p(y_off), p(y_len), C.c_uint64(n), C.c_uint32(cap_matches), int(garbage),
                                p(out["score"]), p(out["xstart"]), p(out["xend"]), p(out["ystart"]), p(out["yend"]),
                                p(out["n_ops"]), p(out["clip_len"]), p(out["status"]), p(out["num_cells"]),
                                p(rng) if want_ranges else None, p(ops), p(ops_off))
        assert rc == 0
        oplists = [decode_ops(ops[int(ops_off[i]):int(ops_off[i]) + int(out["n_ops"][i])],
                              out["clip_len"][4 * i:4 * i + 4]) if out["status"][i] == 0 else None
                   for i in range(n)]
        results.append((out, oplists, rng))
    a, b = results
    for k_ in a[0]:
        assert np.array_equal(a[0][k_], b[0][k_]), ("scratch-dependent result", k_)
    assert a[1] == b[1]
    return a


def banded_hinted_one(orc_scoring, k, w, x: bytes, y: bytes, matches, path=None, allowed_mismatches=None,
                      use_lcskpp_union=False, cap_matches=4096):
    """K4 with caller-supplied band inputs + K3 (host build of b2a_banded.cuh), custom mode.
    -> (fields, ops, cells) or None when the device code flags a reference panic; two scratch fills must agree."""
    s = SimScoring.from_buffer_copy(bytes(orc_scoring))
    res = []
    for garbage in (0x00, 0x7F):
        xy = np.array([v for mt in matches for v in mt], dtype=np.uint32) if matches else np.zeros(2, np.uint32)
        pi = np.array(path if path else [0], dtype=np.uint32)
        score = C.c_int32(0)
        coords = (C.c_uint32 * 4)()
        clip = (C.c_uint32 * 4)()
        n_ops, status, cells = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        ops = (C.c_uint8 * (len(x) + len(y) + 16))()
        rc = lib().sim_banded_hinted_one(
            C.byref(s), C.c_uint32(k), C.c_uint32(w), x, C.c_uint32(len(x)), y, C.c_uint32(len(y)),
            xy.ctypes.data_as(C.c_void_p), C.c_uint64(len(matches)), pi.ctypes.data_as(C.c_void_p),
            C.c_uint64(len(path) if path is not None else 0), C.c_int(1 if path is not None else 0),
            C.c_int(-1 if allowed_mismatches is None else int(allowed_mismatches)),
            C.c_int(1 if use_lcskpp_union else 0), C.c_uint32(cap_matches), C.c_int(garbage), C.byref(score),
            coords, C.byref(n_ops), clip, C.byref(status), C.byref(cells), ops)
        assert rc == 0
        if status.value != 0:
            res.append(("status", status.value))
            continue
        fields = {"score": score.value, "xstart": coords[0], "xend": coords[1], "ystart": coords[2],
                  "yend": coords[3]}
        res.append((fields, decode_ops(bytes(ops[:n_ops.value]), list(clip)), int(cells.value)))
    assert res[0] == res[1], "scratch contents leak into the result"
    return None if res[0][0] == "status" else res[0]


def banded_warp32_one(mode, orc_scoring, k, w, x: bytes, y: bytes, matches=None, path=None, allowed_mismatches=None,
                      use_lcskpp_union=False, cap_matches=4096, want_ranges=False):
    """K4 + K3 as the GPU runs them (W = 32), with 32 host threads as the lanes of one warp.
    -> (fields, ops, cells[, ranges]) or None when the device code flags a reference panic."""
    s = SimScoring.from_buffer_copy(bytes(orc_scoring))
    res = []
    for garbage in (0x00, 0x7F):
        xy = np.array([v for mt in (matches or []) for v in mt], dtype=np.uint32) if matches else np.zeros(2, np.uint32)
        pi = np.array(path if path else [0], dtype=np.uint32)
        score = C.c_int32(0)
        coords = (C.c_uint32 * 4)()
        clip = (C.c_uint32 * 4)()
        n_ops, status, cells = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        ops = (C.c_uint8 * (len(x) + len(y) + 16))()
        rng = np.zeros(2 * (len(y) + 1), dtype=np.uint64)
        rc = lib().sim_banded_warp32_one(
            C.c_int(int(mode)), C.byref(s), C.c_uint32(k), C.c_uint32(w), x, C.c_uint32(len(x)), y, C.c_uint32(len(y)),
            C.c_int(1 if matches is not None else 0), xy.ctypes.data_as(C.c_void_p),
            C.c_uint64(len(matches) if matches is not None else 0), pi.ctypes.data_as(C.c_void_p),
            C.c_uint64(len(path) if path is not None else 0), C.c_int(1 if path is not None else 0),
            C.c_int(-1 if allowed_mismatches is None else int(allowed_mismatches)),
            C.c_int(1 if use_lcskpp_union else 0), C.c_uint32(cap_matches), C.c_int(garbage), C.byref(score),
            coords, C.byref(n_ops), clip, C.byref(status), C.byref(cells),
            rng.ctypes.data_as(C.c_void_p) if want_ranges else None, ops)
        assert rc == 0, "the 32 lanes disagreed on K4's result"
        if status.value != 0:
            res.append(("status", status.value))
            continue
        fields = {"score": score.value, "xstart": coords[0], "xend": coords[1], "ystart": coords[2],
                  "yend": coords[3]}
        out = (fields, decode_ops(bytes(ops[:n_ops.value]), list(clip)), int(cells.value))
        if want_ranges:
            out = out + ([(int(rng[2 * j]), int(rng[2 * j + 1])) for j in range(len(y) + 1)],)
        res.append(out)
    assert res[0] == res[1], "scratch contents leak into the result"
    return None if res[0][0] == "status" else res[0]


def banded_strip_task(mode, orc_scoring, k, w, pairs, cap_matches=4096):
    """Up to four pairs through K4 (W = 32), ONE warp-task of the strip-wavefront fill (b2a_banded_strip.cuh, 8 emulated
    lanes per pair) and its finish pass.  -> list of (fields, ops) or None per pair (None: the pair is not eligible
    for the strip path or was handed back); two scratch fills must agree."""
    from rust_bio_b200.engine import pack_pairs
    s = SimScoring.from_buffer_copy(bytes(orc_scoring))
    blob, x_off, x_len, y_off, y_len = pack_pairs(pairs)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    x_off = np.ascontiguousarray(x_off, dtype=np.uint64)
    y_off = np.ascontiguousarray(y_off, dtype=np.uint64)
    x_len = np.ascontiguousarray(x_len, dtype=np.uint32)
    y_len = np.ascontiguousarray(y_len, dtype=np.uint32)
    n = len(pairs)
    cap = x_len.astype(np.uint64) + y_len.astype(np.uint64) + np.uint64(8)
    ops_off = np.concatenate([[0], np.cumsum(cap)]).astype(np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    res = []
    for garbage in (0x00, 0x7F):
        ops = np.zeros(int(ops_off[-1]), dtype=np.uint8)
        score = np.zeros(n, dtype=np.int32)
        coords = np.zeros(4 * n, dtype=np.uint32)
        n_ops = np.zeros(n, dtype=np.uint32)
        clip = np.zeros(4 * n, dtype=np.uint32)
        status = np.zeros(n, dtype=np.uint32)
        path = np.zeros(n, dtype=np.uint32)
        L = lib()
        L.sim_banded_strip_task.restype = C.c_int
        rc = L.sim_banded_strip_task(int(mode), C.byref(s), C.c_uint32(k), C.c_uint32(w), p(blob),
                                     C.c_uint64(len(blob)), p(x_off), p(x_len),
                                     p(y_off), p(y_len), C.c_uint32(n), C.c_uint32(cap_matches), int(garbage), p(score),
                                     p(coords), p(n_ops), p(clip), p(status), p(path), p(ops), p(ops_off))
        assert rc == 0, rc
        out = []
        for i in range(n):
            if not path[i]:
                out.append(None)
                continue
            fields = {"score": int(score[i]), "xstart": int(coords[4 * i]), "xend": int(coords[4 * i + 1]),
                      "ystart": int(coords[4 * i + 2]), "yend": int(coords[4 * i + 3])}
            out.append((fields, decode_ops(ops[int(ops_off[i]):int(ops_off[i]) + int(n_ops[i])], clip[4 * i:4 * i + 4])))
        res.append(out)
    assert res[0] == res[1], "scratch contents leak into the result"
    return res[0]
