"""The C-ABI library loads without a GPU and exports every symbol include/b200align.h declares."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b200align.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2a_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_list_agree():
    from rust_bio_b200 import _lib
    assert _declared() == sorted(_lib.ABI_SYMBOLS)


def test_library_exports_every_declared_symbol():
    from rust_bio_b200 import _lib, build
    if not os.path.exists(_lib.SO_PATH):
        build.build()
    L = C.CDLL(_lib.SO_PATH)
    for name in _declared():
        assert hasattr(L, name), name


def test_no_cpu_fallback_without_device():
    """On a machine without a usable sm_90 (H100) device the engine refuses to exist (no CPU path)."""
    import torch
    from rust_bio_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.load()
    h = C.c_void_p()
    assert L.b2a_engine_create(C.byref(h), 0) == -2  # B2A_E_NO_DEVICE
    from rust_bio_b200.engine import Engine
    with pytest.raises(_lib.B2AError):
        Engine(0)


def test_mirror_asserts_like_the_reference():
    """Constructor panics of the reference (mod.rs:199-200, 292-293, 322, 517-518) surface as AssertionError."""
    from rust_bio_b200.pairwise import Aligner, MatchParams, Scoring
    with pytest.raises(AssertionError, match="gap_open can't be positive"):
        Aligner.with_capacity(10, 10, 1, -1, MatchParams.new(1, -1))
    with pytest.raises(AssertionError, match="gap_extend can't be positive"):
        Scoring.new(-1, 1, MatchParams.new(1, -1))
    with pytest.raises(AssertionError, match="match_score can't be negative"):
        MatchParams.new(-1, -1)
    with pytest.raises(AssertionError, match="mismatch_score can't be positive"):
        MatchParams.new(1, 1)
    with pytest.raises(AssertionError, match="Clipping penalty can't be positive"):
        Scoring.from_scores(-5, -1, 1, -1).xclip(5)
    s = Scoring.from_scores(-5, -1, 1, -1).xclip(-5)
    assert s.xclip_prefix == -5 and s.xclip_suffix == -5 and s.yclip_prefix == -858993459
    assert s.match_scores == (1, -1)
    assert Scoring.new(-5, -1, lambda a, b: 1).match_scores is None


def test_traceback_cell_mirror():
    """pairwise::TracebackCell (mod.rs:1026-1114): 4 bits each for I (0-3), D (4-7), S (8-11)."""
    from rust_bio_b200.pairwise import TracebackCell as T
    c = T.new()
    assert (c.get_i_bits(), c.get_d_bits(), c.get_s_bits()) == (T.TB_START,) * 3 and c == T()
    c.set_s_bits(T.TB_YCLIP_SUFFIX)
    c.set_i_bits(T.TB_INS)
    c.set_d_bits(T.TB_XCLIP_PREFIX)
    assert c.v == (8 << 8) | (5 << 4) | 1
    c.set_s_bits(T.TB_MATCH)  # overwrites only its own nibble
    assert (c.get_i_bits(), c.get_d_bits(), c.get_s_bits()) == (1, 5, 4)
    c.set_all(T.TB_SUBST)
    assert c.v == 0x333
    with pytest.raises(AssertionError, match="TB_MAX"):
        c.set_i_bits(9)
