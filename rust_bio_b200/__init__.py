"""rust_bio_b200: H100-native batched drop-in for rust-bio's `bio::alignment::pairwise` hot path.

Layout: csrc/ (CUDA kernels + C ABI, include/b200align.h), pairwise.py / alignment.py / scores.py
(host-side mirror of the reference interface), engine.py (ctypes over the C ABI), synth.py
(deterministic benchmark inputs), dist.py (pair-list sharding + the single all-gather).
"""
from . import alignment, scores  # noqa: F401

__version__ = "0.1.0"
